"""Loader of the STAGED, UNMODIFIED reference modules (TEST INFRASTRUCTURE — see oracle/__init__.py, oracle/stage_ref.py).

``load()`` imports ``models.dit_crossattn.DiT``, ``models.vae3d_dib.VAE`` and ``models.diffusion.create_diffusion`` from
``oracle/_ref/`` (byte-identical copies of the reference's files) and returns them in a namespace.  The reference's
top-level package names (``models``, ``utils``) are generic, so they are imported with ``oracle/_ref`` first on
``sys.path`` and then taken out of ``sys.modules`` again: the classes keep working (their relative imports were
resolved at import time) and nothing else in the process — e.g. ``tpxl_b200.install()``'s aliases — is disturbed.

The un-vendored ``xformers.ops`` (models/attention.py:17) is restated, not copied:
    memory_efficient_attention(q, k, v, attn_bias=None, p=0.0, scale=None) on [B, N, H, Dh] tensors
        = softmax(q k^T * (scale or Dh^-1/2)) v      -> torch SDPA on the [B, H, N, Dh] views
    unbind = torch.unbind
This is the same shim tests/golden/make_golden.py uses to generate the fp32 fixtures.
"""
from __future__ import annotations

import os
import sys
import types
from types import SimpleNamespace

import torch

from . import stage_ref

_cache = None


def available() -> bool:
    return stage_ref.staged()


def _xformers_shim():
    import torch.nn.functional as F

    def memory_efficient_attention(q, k, v, attn_bias=None, p=0.0, scale=None):
        assert attn_bias is None and p == 0.0
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), scale=scale)
        return o.transpose(1, 2)

    xf, ops = types.ModuleType("xformers"), types.ModuleType("xformers.ops")
    ops.memory_efficient_attention = memory_efficient_attention
    ops.unbind = torch.unbind
    xf.ops = ops
    return xf, ops


def load() -> SimpleNamespace:
    """-> namespace(DiT, VAE, create_diffusion, root).  Raises FileNotFoundError when oracle/_ref is not staged."""
    global _cache
    if _cache is not None:
        return _cache
    if not available():
        raise FileNotFoundError("oracle/_ref is not staged: run `python oracle/stage_ref.py` where a reference checkout exists")
    taken = ("models", "utils", "xformers")
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in taken}
    for k in saved:
        del sys.modules[k]
    xf, ops = _xformers_shim()
    sys.modules["xformers"], sys.modules["xformers.ops"] = xf, ops
    sys.path.insert(0, stage_ref.DEST)
    try:
        from models.dit_crossattn import DiT
        from models.vae3d_dib import VAE
        from models.diffusion import create_diffusion
    finally:
        sys.path.remove(stage_ref.DEST)
        for k in [k for k in sys.modules if k.split(".")[0] in taken]:
            del sys.modules[k]
        sys.modules.update(saved)
    _cache = SimpleNamespace(DiT=DiT, VAE=VAE, create_diffusion=create_diffusion, root=stage_ref.DEST)
    return _cache


def raymarcher_available() -> bool:
    return stage_ref.raymarcher_staged()


_rm_cache = None


def load_raymarcher():
    """-> the reference's ``dva.ray_marcher.RayMarcher`` over its own CUDA extensions (mvpraymarchlib, utilslib) built by
    oracle/stage_ref.py.  ``dva`` is a generic top-level name, so it is imported with ``oracle/_ref`` first on ``sys.path`` and taken
    out of ``sys.modules`` again, as ``load()`` does.  Raises FileNotFoundError when the extensions were not built."""
    global _rm_cache
    if _rm_cache is not None:
        return _rm_cache
    if not raymarcher_available():
        raise FileNotFoundError("the reference's ray marcher is not built: run `python oracle/stage_ref.py` where a reference checkout exists")
    taken = ("dva", "mvpraymarchlib", "utilslib")
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in taken}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, stage_ref.DEST)
    try:
        from dva.ray_marcher import RayMarcher
    finally:
        sys.path.remove(stage_ref.DEST)
        for k in [k for k in sys.modules if k.split(".")[0] in taken]:
            del sys.modules[k]
        sys.modules.update(saved)
    _rm_cache = RayMarcher
    return _rm_cache


def build_dit(cfg: dict, state_dict: dict, device="cpu"):
    """Reference DiT with the given (reference-keyed) parameters, fp32 modules as inference.py:254-265 builds them."""
    ref = load()
    with torch.device("meta"):
        m = ref.DiT(**cfg)
    m = m.to_empty(device=device)
    m.load_state_dict({k: v.to(device=device, dtype=torch.float32) for k, v in state_dict.items()}, strict=True)
    return m.eval()


def build_vae(cfg: dict, decoder_state_dict: dict, device="cpu"):
    """Reference VAE; only decoder.* / post_quant_conv.* are needed by decode(), the encoder keeps its default init."""
    ref = load()
    m = ref.VAE(**cfg)
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in decoder_state_dict.items()}, strict=False)
    assert not unexpected, unexpected
    assert all(k.startswith(("encoder.", "quant_conv.")) for k in missing), [k for k in missing if not k.startswith(("encoder.", "quant_conv."))][:5]
    return m.to(device).eval()
