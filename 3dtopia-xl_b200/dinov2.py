"""Host-side mirror of the reference's image encoder (SURVEY.md §8f-2), built from the DiT kernels.  Parity: its oracle
(oracle/dinov2.py) is pinned to the reference's own output (tests/golden/dinov2.npz); on the GPU, tests/test_gpu_dinov2_stages.py
checks every stage of every block against that oracle in fp64 (DESIGN.md §2) and tests/test_gpu_zz_extra.py the output against the
fixture.  ``install()`` does not alias it.

Drop-in for ``models.conditioner.image_dinov2.Dinov2Wrapper('dinov2_vitb14_reg', freeze=True)``
(/root/reference/models/conditioner/image_dinov2.py:10-61): same state_dict keys (``model.cls_token`` ...), same
``forward(image[N,H,W,3] in 0..255) -> [N, 1370, 768]``.  Compute contract: the reference runs this encoder in fp32 (TF32 when
inference.py:379 enabled it); here the residual stream and LayerNorm are fp32 and every Linear takes fp16 inputs with fp32
accumulation, like the DiT (10-bit-mantissa inputs, as TF32).  Launch plan per image batch, all through the C ABI:

    patch embedding   tpx_linear_gated   (pixels / 255 as fp16 [N*1369, 588->640] x W'; Normalize folded into W', b'; accumulates
                                          onto the position embedding already sitting in the token buffer)
    12 x block        tpx_ln_modulate (LayerNorm affine as shift = beta, scale = gamma - 1) -> tpx_linear_heads (qkv, 12 heads x 64,
                      padded to 80, V transposed) -> tpx_attention_tc (wgmma) -> tpx_linear_gated (proj, LayerScale as the gate, fp32 residual)
                      -> tpx_ln_modulate -> tpx_linear (fc1) -> tpx_gelu_erf -> tpx_linear_gated (fc2, LayerScale)
    final norm        tpx_ln_modulate with zero shift / scale (plain LN to fp16), then class token + patch tokens are gathered
                      (register tokens dropped) and the LayerNorm affine applied in fp32
"""
from __future__ import annotations

import contextlib
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib

IMG, PATCH, DIM, DEPTH, HEADS, N_REG, DH, DHP = 518, 14, 768, 12, 12, 4, 64, 80
KPATCH, KPAD = PATCH * PATCH * 3, 640                       # 588 patch values, padded to a multiple of the 64-wide K tile
MEAN = (0.48145466, 0.4578275, 0.40821073)                   # image_dinov2.py:21
STD = (0.26862954, 0.26130258, 0.27577711)


def _shapes() -> "OrderedDict[str, tuple]":
    s: "OrderedDict[str, tuple]" = OrderedDict()
    m = "model."
    s[m + "cls_token"], s[m + "pos_embed"], s[m + "register_tokens"] = (1, 1, DIM), (1, (IMG // PATCH) ** 2 + 1, DIM), (1, N_REG, DIM)
    s[m + "patch_embed.proj.weight"], s[m + "patch_embed.proj.bias"] = (DIM, 3, PATCH, PATCH), (DIM,)
    for i in range(DEPTH):
        b = f"{m}blocks.{i}."
        for nm, shp in (("norm1.weight", (DIM,)), ("norm1.bias", (DIM,)), ("attn.qkv.weight", (3 * DIM, DIM)), ("attn.qkv.bias", (3 * DIM,)),
                        ("attn.proj.weight", (DIM, DIM)), ("attn.proj.bias", (DIM,)), ("ls1.gamma", (DIM,)), ("norm2.weight", (DIM,)),
                        ("norm2.bias", (DIM,)), ("mlp.fc1.weight", (4 * DIM, DIM)), ("mlp.fc1.bias", (4 * DIM,)),
                        ("mlp.fc2.weight", (DIM, 4 * DIM)), ("mlp.fc2.bias", (DIM,)), ("ls2.gamma", (DIM,))):
            s[b + nm] = shp
    s[m + "norm.weight"], s[m + "norm.bias"] = (DIM,), (DIM,)
    return s


class _Stop(Exception):
    """Raised by a tap at the requested stop of Dinov2Wrapper._forward."""


@contextlib.contextmanager
def _stopped():
    try:
        yield
    except _Stop:
        pass


class Dinov2Wrapper(nn.Module):
    def __init__(self, model_name: str = "dinov2_vitb14_reg", modulation_dim: Optional[int] = None, freeze: bool = True):
        super().__init__()
        if model_name != "dinov2_vitb14_reg" or modulation_dim is not None:
            raise NotImplementedError(f"only the released encoder (dinov2_vitb14_reg, no modulation) is built; got {model_name!r}, "
                                      f"modulation_dim={modulation_dim}")
        self.modulation_dim = None
        self._shapes = _shapes()
        self._anchor = nn.Parameter(torch.zeros(1), requires_grad=False)     # so .to(device) / .parameters() behave
        self._sd: Optional["OrderedDict[str, torch.Tensor]"] = None
        self._dev_w = None                                                   # device-side fp16 operands, built lazily
        self._dev = None

    # ---- parameters under the reference's key names ---------------------------------------------------------------------------
    def state_dict(self, *args, **kwargs):
        if self._sd is None:
            self._sd = OrderedDict((k, torch.zeros(shp)) for k, shp in self._shapes.items())
        return OrderedDict(self._sd)

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        state_dict = {k: v for k, v in state_dict.items() if "mask_token" not in k}      # dropped by the reference too (hub/backbones.py)
        if state_dict and not any(k.startswith("model.") for k in state_dict):           # a hub checkpoint of the bare ViT (no wrapper prefix)
            state_dict = {"model." + k: v for k, v in state_dict.items()}
        missing, unexpected = _lib.check_state_dict("Dinov2Wrapper", self._shapes, state_dict, strict)
        cur = self.state_dict()
        self._sd = OrderedDict((k, state_dict[k].detach() if k in state_dict else cur[k]) for k in self._shapes)
        self._dev_w = None
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        self._dev_w = None
        return out

    # ---- device operands ------------------------------------------------------------------------------------------------------
    def _operands(self, dev: torch.device):
        if self._dev_w is not None and self._dev == dev:
            return self._dev_w
        # folded in fp64, so every fp16 / fp32 operand is one rounding of its exact value
        sd = {k: v.detach().to(dev, torch.float64) for k, v in self.state_dict().items()}
        m = "model."
        w = {}
        # Normalize((x - mean) / std) folded into the patch embedding: conv(W, (p - mean)/std) + b = conv(W/std, p) + (b - sum W*mean/std);
        # the patch vector is laid out (i, j, c) — the order of a [14,14,3] window of the NHWC picture — and zero padded to KPAD
        W = sd[m + "patch_embed.proj.weight"]
        std = torch.tensor(STD, dtype=torch.float64, device=dev).view(1, 3, 1, 1)
        mean = torch.tensor(MEAN, dtype=torch.float64, device=dev).view(1, 3, 1, 1)
        Wn = W / std
        wp = torch.zeros(DIM, KPAD, dtype=torch.float64, device=dev)
        wp[:, :KPATCH] = Wn.permute(0, 2, 3, 1).reshape(DIM, KPATCH)
        w["patch_w"] = wp.half().contiguous()
        w["patch_b"] = (sd[m + "patch_embed.proj.bias"] - (Wn * mean).sum(dim=(1, 2, 3))).half().contiguous()
        pos = sd[m + "pos_embed"][0]
        w["row0"] = (sd[m + "cls_token"][0, 0] + pos[0]).float().contiguous()                 # class token + its position, fp32
        w["regs"] = sd[m + "register_tokens"][0].float().contiguous()                          # registers carry no position (vision_transformer.py:222-231)
        w["pos_patches"] = pos[1:].float().contiguous()
        w["ones"] = torch.ones(1, DIM, device=dev, dtype=torch.float16)
        for i in range(DEPTH):
            b = f"{m}blocks.{i}."
            for nm in ("attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight",
                       "mlp.fc2.bias"):
                w[f"{i}.{nm}"] = sd[b + nm].half().contiguous()
            for n in ("1", "2"):
                w[f"{i}.ln{n}.scale"] = (sd[b + f"norm{n}.weight"] - 1.0).half().view(1, DIM).contiguous()     # LN * h(1 + scale) + shift
                w[f"{i}.ln{n}.shift"] = sd[b + f"norm{n}.bias"].half().view(1, DIM).contiguous()
                w[f"{i}.ls{n}"] = sd[b + f"ls{n}.gamma"].half().view(1, DIM).contiguous()
        # final norm: plain LN to fp16 (zero shift and scale), then the affine in fp32 on the host side, so that a gain far below 1 keeps
        # its relative precision (as modulation h(1 + h(g - 1)) its absolute error of ~2^-12 would be a large fraction of such a gain)
        w["zeros"] = torch.zeros(1, DIM, device=dev, dtype=torch.float16)
        w["norm.weight"] = sd[m + "norm.weight"].float().contiguous()
        w["norm.bias"] = sd[m + "norm.bias"].float().contiguous()
        self._dev_w, self._dev = w, dev
        return w

    # ---- forward ----------------------------------------------------------------------------------------------------------------
    def forward(self, image: torch.Tensor, mod: torch.Tensor = None) -> torch.Tensor:
        assert image.shape[-1] == 3, "image: [N, H, W, C] (image_dinov2.py:46-47)"
        assert mod is None, "Unexpected modulation input in dinov2 forward."
        return self._forward(image)

    def _forward(self, image: torch.Tensor, taps: Optional[dict] = None, stop: Optional[tuple] = None) -> Optional[torch.Tensor]:
        """The launch plan.  taps (parity tests): a dict that receives clones of the buffers as the launches leave them — "embed" (the
        fp32 token block after the patch embedding), per block i (i, "ln1"), (i, "q"), (i, "k"), (i, "vT"), (i, "att"), (i, "res1")
        (residual after proj), (i, "ln2"), (i, "fc1"), (i, "hid") (after the GELU), (i, "res2") (residual after fc2), then "out16" (the
        normalised tokens before the affine).  stop = one of those keys ends the run after that tap and returns None.  Without taps
        the launches are the same."""
        if not image.is_cuda:
            raise _lib.TpxError("Dinov2Wrapper runs on CUDA only (no CPU path): move the module and the image to the GPU")
        if image.shape[1] != image.shape[2]:
            raise ValueError("square images only (the released pipeline feeds 518 x 518)")
        lib = _lib.lib()
        dev = image.device
        w = self._operands(dev)
        x = image.float()
        if x.shape[1] != IMG:                       # Resize(518, bicubic) of the reference's Compose, on the host side of the boundary
            x = F.interpolate(x.permute(0, 3, 1, 2), size=(IMG, IMG), mode="bicubic", align_corners=False, antialias=True).permute(0, 2, 3, 1)
        n, g = x.shape[0], IMG // PATCH
        np_, nt = g * g, g * g + 1 + N_REG                                    # 1369 patches, 1374 tokens
        patches = torch.zeros(n * np_, KPAD, dtype=torch.float16, device=dev)
        patches[:, :KPATCH] = (x / 255.0).reshape(n, g, PATCH, g, PATCH, 3).permute(0, 1, 3, 2, 4, 5).reshape(n * np_, KPATCH).half()
        tok = torch.empty(n, nt, DIM, dtype=torch.float32, device=dev)        # fp32 residual stream
        tok[:, 0] = w["row0"]
        tok[:, 1:1 + N_REG] = w["regs"]
        tok[:, 1 + N_REG:] = w["pos_patches"]
        rows = n * nt
        ln = torch.empty(rows, DIM, dtype=torch.float16, device=dev)
        q = torch.empty(n, HEADS, nt, DHP, dtype=torch.float16, device=dev)
        k = torch.empty_like(q)
        ntp = (nt + 7) // 8 * 8
        vT = torch.zeros(n, HEADS, DHP, ntp, dtype=torch.float16, device=dev)   # V transposed (keys contiguous) for the attention kernel's P V operand
        att = torch.empty(rows, DIM, dtype=torch.float16, device=dev)
        hid = torch.empty(rows, 4 * DIM, dtype=torch.float16, device=dev)
        out16 = torch.empty(rows, DIM, dtype=torch.float16, device=dev)

        def tap(key, buf):
            if taps is not None:
                taps[key] = buf.clone()
            if key == stop:
                raise _Stop

        with torch.cuda.device(dev), _stopped():
            st = _lib.stream_ptr()
            for b in range(n):                      # patch tokens of picture b: rows 5.. of its token block, added onto the position embedding
                _lib.check(lib.tpx_linear_gated(patches[b * np_:].data_ptr(), KPAD, w["patch_w"].data_ptr(), w["patch_b"].data_ptr(),
                                                w["ones"].data_ptr(), DIM, 1, np_, tok[b, 1 + N_REG:].data_ptr(), DIM, np_, DIM, KPAD, 0, st),
                           "patch embedding")
            xr = tok.view(rows, DIM)
            tap("embed", tok)
            for i in range(DEPTH):
                _lib.check(lib.tpx_ln_modulate(xr.data_ptr(), rows, DIM, 1e-6, w[f"{i}.ln1.shift"].data_ptr(), w[f"{i}.ln1.scale"].data_ptr(), DIM, rows, 1,
                                               ln.data_ptr(), None, None, 0, st), "norm1")
                tap((i, "ln1"), ln)
                _lib.check(lib.tpx_linear_heads(ln.data_ptr(), DIM, w[f"{i}.attn.qkv.weight"].data_ptr(), w[f"{i}.attn.qkv.bias"].data_ptr(), q.data_ptr(),
                                                k.data_ptr(), vT.data_ptr(), rows, 3 * DIM, DIM, DIM, HEADS, DH, DHP, nt, 1.0, 0, 2, ntp, st), "qkv")
                tap((i, "q"), q)
                tap((i, "k"), k)
                tap((i, "vT"), vT)
                _lib.check(lib.tpx_attention_tc(q.data_ptr(), k.data_ptr(), vT.data_ptr(), att.data_ptr(), n, HEADS, nt, nt, ntp, DH, DH ** -0.5, st), "attention")
                tap((i, "att"), att)
                _lib.check(lib.tpx_linear_gated(att.data_ptr(), DIM, w[f"{i}.attn.proj.weight"].data_ptr(), w[f"{i}.attn.proj.bias"].data_ptr(),
                                                w[f"{i}.ls1"].data_ptr(), DIM, 1, rows, xr.data_ptr(), DIM, rows, DIM, DIM, 0, st), "proj")
                tap((i, "res1"), tok)
                _lib.check(lib.tpx_ln_modulate(xr.data_ptr(), rows, DIM, 1e-6, w[f"{i}.ln2.shift"].data_ptr(), w[f"{i}.ln2.scale"].data_ptr(), DIM, rows, 1,
                                               ln.data_ptr(), None, None, 0, st), "norm2")
                tap((i, "ln2"), ln)
                _lib.check(lib.tpx_linear(ln.data_ptr(), DIM, w[f"{i}.mlp.fc1.weight"].data_ptr(), w[f"{i}.mlp.fc1.bias"].data_ptr(), hid.data_ptr(), 4 * DIM,
                                          rows, 4 * DIM, DIM, 0, 1.0, 0, st), "fc1")
                tap((i, "fc1"), hid)
                _lib.check(lib.tpx_gelu_erf(hid.data_ptr(), rows * 4 * DIM, st), "gelu")
                tap((i, "hid"), hid)
                _lib.check(lib.tpx_linear_gated(hid.data_ptr(), 4 * DIM, w[f"{i}.mlp.fc2.weight"].data_ptr(), w[f"{i}.mlp.fc2.bias"].data_ptr(),
                                                w[f"{i}.ls2"].data_ptr(), DIM, 1, rows, xr.data_ptr(), DIM, rows, DIM, 4 * DIM, 0, st), "fc2")
                tap((i, "res2"), tok)
            _lib.check(lib.tpx_ln_modulate(xr.data_ptr(), rows, DIM, 1e-6, w["zeros"].data_ptr(), w["zeros"].data_ptr(), DIM, rows, 1,
                                           out16.data_ptr(), None, None, 0, st), "final norm")
            tap("out16", out16)
        if stop is not None:
            return None
        o = out16.view(n, nt, DIM)
        o = torch.cat([o[:, :1], o[:, 1 + N_REG:]], dim=1).float()          # [N, 1370, 768], class token first (image_dinov2.py:56-60)
        return o * w["norm.weight"] + w["norm.bias"]                         # the final norm's affine in fp32
