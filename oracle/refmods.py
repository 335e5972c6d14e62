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

``build_dinov2`` and ``build_primsdf`` build the image conditioner and PrimSDF from the same staged tree, with the same ``sys.modules``
discipline, inside the import window (the conditioner resolves its hub and ViT modules by relative import when it is built).
"""
from __future__ import annotations

import contextlib
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


@contextlib.contextmanager
def _staged_import(taken, modules=None):
    """Import from oracle/_ref with the top-level names in taken set aside, and the stand-in modules {name: module} installed, for the
    duration of the block; afterwards sys.modules is as it was."""
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in taken}
    for k in saved:
        del sys.modules[k]
    sys.modules.update(modules or {})
    sys.path.insert(0, stage_ref.DEST)
    try:
        yield
    finally:
        sys.path.remove(stage_ref.DEST)
        for k in [k for k in sys.modules if k.split(".")[0] in taken]:
            del sys.modules[k]
        sys.modules.update(saved)


def load() -> SimpleNamespace:
    """-> namespace(DiT, VAE, create_diffusion, root).  Raises FileNotFoundError when oracle/_ref is not staged."""
    global _cache
    if _cache is not None:
        return _cache
    if not available():
        raise FileNotFoundError("oracle/_ref is not staged: run `python oracle/stage_ref.py` where a reference checkout exists")
    xf, ops = _xformers_shim()
    with _staged_import(("models", "utils", "xformers"), {"xformers": xf, "xformers.ops": ops}):
        from models.dit_crossattn import DiT
        from models.vae3d_dib import VAE
        from models.diffusion import create_diffusion
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
    with _staged_import(("dva", "mvpraymarchlib", "utilslib")):
        from dva.ray_marcher import RayMarcher
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


def conditioner_available() -> bool:
    return stage_ref.conditioner_staged()


def primsdf_available() -> bool:
    return stage_ref.primsdf_staged()


def build_dinov2(state_dict: dict, device="cpu"):
    """The reference's ``Dinov2Wrapper("dinov2_vitb14_reg")`` (freeze=True, as configs/inference_dit.yml builds it) with the given
    parameters, fp32, in eval mode.  ``_build_dinov2`` is bound to ``pretrained=False`` (no hub download), as tests/golden/make_golden.py
    does.  The ViT is imported with the xformers stand-in installed, so ``MemEffAttention`` takes its xformers branch
    (``memory_efficient_attention`` on [B, N, H, Dh]), as it does where xformers is installed; ``layers/block.py`` asks xformers for
    the nested-tensor helpers (``fmha``, ``scaled_index_add``, ``index_select_cat``) only, which a batched tensor input never reaches,
    and takes its plain branch."""
    if not conditioner_available():
        raise FileNotFoundError("the reference's conditioner is not staged: run `python oracle/stage_ref.py` where a reference checkout exists")
    xf, ops = _xformers_shim()
    with _staged_import(("models", "utils", "xformers"), {"xformers": xf, "xformers.ops": ops}):
        from models.conditioner.image_dinov2 import Dinov2Wrapper
        import models.conditioner.dinov2.hub.backbones as bb
        import models.conditioner.dinov2.layers.attention as attention
        import models.conditioner.dinov2.layers.block as block
        assert attention.XFORMERS_AVAILABLE and attention.memory_efficient_attention is ops.memory_efficient_attention, \
            "layers/attention.py did not take its xformers branch"
        assert not block.XFORMERS_AVAILABLE, "layers/block.py took its xformers branch"
        Dinov2Wrapper._build_dinov2 = staticmethod(lambda model_name, modulation_dim=None, pretrained=True:
                                                   getattr(bb, model_name)(modulation_dim=modulation_dim, pretrained=False))
        m = Dinov2Wrapper("dinov2_vitb14_reg", freeze=True)
    m.load_state_dict({k: v.to(dtype=torch.float32) for k, v in state_dict.items()}, strict=True)
    return m.to(device).eval()


def build_primsdf(srt: torch.Tensor, feat: torch.Tensor, device="cpu"):
    """The reference's ``PrimSDF`` over srt [K, 4] and feat [K, 6 S^3] (fp32), in eval mode.  ``trimesh`` (imported, unused on the query
    path) is stubbed only while models/primsdf.py is imported, as tests/golden/make_golden.py does."""
    if not primsdf_available():
        raise FileNotFoundError("the reference's PrimSDF is not staged: run `python oracle/stage_ref.py` where a reference checkout exists")
    with _staged_import(("models", "utils", "trimesh"), {"trimesh": types.ModuleType("trimesh")}):
        from models.primsdf import PrimSDF
    K = srt.shape[0]
    S = round((feat.shape[1] // 6) ** (1 / 3))
    assert feat.shape == (K, 6 * S ** 3), tuple(feat.shape)
    m = PrimSDF(num_prims=K, dim_feat=6, prim_shape=S)
    m.srt_param.data = torch.as_tensor(srt).to(torch.float32).clone()
    m.feat_param.data = torch.as_tensor(feat).to(torch.float32).clone()
    return m.to(device).eval()


def build_vae(cfg: dict, decoder_state_dict: dict, device="cpu"):
    """Reference VAE; only decoder.* / post_quant_conv.* are needed by decode(), the encoder keeps its default init."""
    ref = load()
    m = ref.VAE(**cfg)
    missing, unexpected = m.load_state_dict({k: v.float() for k, v in decoder_state_dict.items()}, strict=False)
    assert not unexpected, unexpected
    assert all(k.startswith(("encoder.", "quant_conv.")) for k in missing), [k for k in missing if not k.startswith(("encoder.", "quant_conv."))][:5]
    return m.to(device).eval()
