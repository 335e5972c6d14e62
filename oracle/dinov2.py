"""Oracle restatement of the image conditioner's encoder (TEST INFRASTRUCTURE — see oracle/__init__.py): SURVEY §8f-2, the next
row after the PrimSDF query.  This module and its fixture are the parity anchor of the CUDA encoder (tpxl_b200.dinov2).

Restates, for the released configuration (configs/inference_dit.yml:48-51: ``dinov2_vitb14_reg``, frozen, no modulation):
  * Dinov2Wrapper.forward            models/conditioner/image_dinov2.py:44-61   ([N,H,W,3] in 0..255 -> /255 -> Resize(518, bicubic)
                                                                                 -> Normalize -> ViT -> cat[cls, patch tokens])
  * DinoVisionTransformer            models/conditioner/dinov2/models/vision_transformer.py:208-265 (prepare_tokens_with_masks,
                                      forward_features; 4 register tokens inserted after the class token, LayerNorm eps 1e-6)
  * Block / Attention / Mlp / LayerScale   dinov2/layers/block.py:87-93, attention.py:56-69, mlp.py:33-39, layer_scale.py:26-27
                                      (pre-norm; 12 heads x 64; GELU (erf); per-channel LayerScale on both branches)
  * PatchEmbed                       dinov2/layers/patch_embed.py:66-80 (14x14 stride-14 convolution, no norm)
Square 518 x 518 inputs only (what inference.py feeds, configs/inference_dit.yml:18-19): then the position embedding is used
as stored (vision_transformer.py:191-192) and the Resize is the identity.  Other square sizes go through the same bicubic
antialiased resize torchvision applies to tensors.  The arithmetic is fp32 like the reference (it runs outside autocast,
inference.py:317).

Branch functions (patch_embed, attn_branch, mlp_branch, final_norm) take a ``Policy`` (oracle.dit):
  ``Policy("fp32")``  no rounding point: the reference's arithmetic, in the dtype of the weights and the image (fp64 for the
                      stage tests: the exact encoder);
  ``Policy("fp16")``  the CUDA encoder's documented compute contract (3dtopia-xl_b200/dinov2.py): pixels h(x / 255); the Normalize
                      folded into the patch weights, both rounded to fp16; LayerNorm affine as modulation, h(LN(x) h(1 + h(g - 1)) + h(beta));
                      fp16 weights and bias in every Linear with one rounding h(acc + b); q, k, v in fp16 and the attention output
                      rounded; h(gelu(.)); the residual update xres += h(h(gamma) h(acc + b)) in fp32 (residual_add); the final norm
                      as h(LN(x)) * g + b, its affine in fp32 after the fp16 boundary.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .dit import Policy, r16

IMG, PATCH, DIM, DEPTH, HEADS, N_REG = 518, 14, 768, 12, 12, 4
MEAN = (0.48145466, 0.4578275, 0.40821073)          # image_dinov2.py:21 (the CLIP statistics, as the reference uses them)
STD = (0.26862954, 0.26130258, 0.27577711)


def shapes(depth: int = DEPTH, dim: int = DIM) -> "OrderedDict[str, Tuple[int, ...]]":
    """state_dict keys / shapes of Dinov2Wrapper('dinov2_vitb14_reg') in the reference's order."""
    s: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    m = "model."
    s[m + "cls_token"] = (1, 1, dim)
    s[m + "pos_embed"] = (1, (IMG // PATCH) ** 2 + 1, dim)
    s[m + "register_tokens"] = (1, N_REG, dim)
    s[m + "patch_embed.proj.weight"], s[m + "patch_embed.proj.bias"] = (dim, 3, PATCH, PATCH), (dim,)
    for i in range(depth):
        b = f"{m}blocks.{i}."
        s[b + "norm1.weight"], s[b + "norm1.bias"] = (dim,), (dim,)
        s[b + "attn.qkv.weight"], s[b + "attn.qkv.bias"] = (3 * dim, dim), (3 * dim,)
        s[b + "attn.proj.weight"], s[b + "attn.proj.bias"] = (dim, dim), (dim,)
        s[b + "ls1.gamma"] = (dim,)
        s[b + "norm2.weight"], s[b + "norm2.bias"] = (dim,), (dim,)
        s[b + "mlp.fc1.weight"], s[b + "mlp.fc1.bias"] = (4 * dim, dim), (4 * dim,)
        s[b + "mlp.fc2.weight"], s[b + "mlp.fc2.bias"] = (dim, 4 * dim), (dim,)
        s[b + "ls2.gamma"] = (dim,)
    s[m + "norm.weight"], s[m + "norm.bias"] = (dim,), (dim,)
    return s


def synth_weights(seed: int, depth: int = DEPTH, dim: int = DIM) -> "OrderedDict[str, torch.Tensor]":
    """Random weights with the magnitudes of a trained ViT (LayerScale ~0.3, LayerNorm gains ~1, Glorot-scaled matrices), from
    one numpy RandomState so the fixture generator and the tests rebuild the same tensors."""
    rs = np.random.RandomState(seed)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shp in shapes(depth, dim).items():
        a = rs.standard_normal(size=shp).astype(np.float32)
        if name.endswith("gamma"):
            a = 0.3 + 0.1 * a
        elif "norm" in name and name.endswith("weight"):
            a = 1.0 + 0.1 * a
        elif name.endswith("bias"):
            a = 0.02 * a
        elif len(shp) >= 2 and "token" not in name and "pos_embed" not in name:
            fan_in, fan_out = int(np.prod(shp[1:])), shp[0]
            a = a * np.float32(np.sqrt(2.0 / (fan_in + fan_out)))
        else:
            a = 0.2 * a                                   # class / register tokens, position embedding
        sd[name] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return sd


def preprocess(image: torch.Tensor) -> torch.Tensor:
    """[N,H,W,3] in 0..255 -> normalised [N,3,518,518]   (image_dinov2.py:48-50 with the Compose of :19-22)."""
    assert image.shape[-1] == 3 and image.shape[1] == image.shape[2], "square RGB images"
    x = image.permute(0, 3, 1, 2) / 255.0
    if x.shape[-1] != IMG:
        x = F.interpolate(x, size=(IMG, IMG), mode="bicubic", align_corners=False, antialias=True)   # torchvision Resize on tensors
    mean = torch.tensor(MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (x - mean) / std


def _ln(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, pol: Policy) -> torch.Tensor:
    """LayerNorm(eps 1e-6) with affine (w, b); under the policy the affine is the modulation h(LN(x) h(1 + h(w - 1)) + h(b))."""
    if not pol.amp:
        return F.layer_norm(x, (x.shape[-1],), w, b, 1e-6)
    return r16(F.layer_norm(x, (x.shape[-1],), None, None, 1e-6) * r16(1 + r16(w - 1)) + r16(b))


def patch_embed(sd: Dict[str, torch.Tensor], image: torch.Tensor, pol: Policy) -> torch.Tensor:
    """[N,H,W,3] in 0..255 -> the token block [N, 1 + N_REG + 1369, 768]: class token + its position, the register tokens (no
    position), then the patch embedding + positions."""
    m = "model."
    W, b = sd[m + "patch_embed.proj.weight"], sd[m + "patch_embed.proj.bias"]
    if not pol.amp:
        x = F.conv2d(preprocess(image), W, b, stride=PATCH)
    else:
        x = image.permute(0, 3, 1, 2)
        if x.shape[-1] != IMG:          # the CUDA encoder resizes the 0..255 picture, then scales
            x = F.interpolate(x, size=(IMG, IMG), mode="bicubic", align_corners=False, antialias=True)
        mean = torch.tensor(MEAN, dtype=W.dtype, device=W.device).view(1, 3, 1, 1)
        std = torch.tensor(STD, dtype=W.dtype, device=W.device).view(1, 3, 1, 1)
        Wn = W / std
        x = r16(F.conv2d(r16(x / 255.0), r16(Wn), r16(b - (Wn * mean).sum(dim=(1, 2, 3))), stride=PATCH))
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat((sd[m + "cls_token"].expand(x.shape[0], -1, -1), x), dim=1) + sd[m + "pos_embed"]
    return torch.cat((x[:, :1], sd[m + "register_tokens"].expand(x.shape[0], -1, -1), x[:, 1:]), dim=1)


def _gate(gamma: torch.Tensor, y: torch.Tensor, pol: Policy) -> torch.Tensor:
    return r16(r16(gamma) * y) if pol.amp else y * gamma


def attn_branch(sd: Dict[str, torch.Tensor], i: int, x: torch.Tensor, pol: Policy, taps: dict | None = None, heads: int = HEADS) -> torch.Tensor:
    """The LayerScale'd attention increment of block i (block.py:87-93, attention.py:56-69).  taps (optional) receives "ln" (norm1
    output), "q" / "k" / "v" [B, heads, N, 64] and "ao" (the attention output before proj, [B, N, C])."""
    p = f"model.blocks.{i}."
    B, N, C = x.shape
    h = _ln(x, sd[p + "norm1.weight"], sd[p + "norm1.bias"], pol)
    qkv = pol.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    a = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2])                    # softmax(q k^T / sqrt(64)) v
    a = pol.rnd(a.transpose(1, 2).reshape(B, N, C))
    if taps is not None:
        taps.update(ln=h, q=qkv[0], k=qkv[1], v=qkv[2], ao=a)
    return _gate(sd[p + "ls1.gamma"], pol.linear(a, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"]), pol)


def mlp_branch(sd: Dict[str, torch.Tensor], i: int, x: torch.Tensor, pol: Policy, taps: dict | None = None) -> torch.Tensor:
    """The LayerScale'd MLP increment of block i (mlp.py:33-39, GELU erf form).  taps receives "ln" (norm2 output) and "hid" (after
    the GELU)."""
    p = f"model.blocks.{i}."
    h = _ln(x, sd[p + "norm2.weight"], sd[p + "norm2.bias"], pol)
    hid = pol.rnd(F.gelu(pol.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])))
    if taps is not None:
        taps.update(ln=h, hid=hid)
    return _gate(sd[p + "ls2.gamma"], pol.linear(hid, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"]), pol)


def residual_add(x: torch.Tensor, inc: torch.Tensor, pol: Policy) -> torch.Tensor:
    """x + inc; under the policy the residual stream is fp32, so the sum is rounded to fp32 (and comes back in x's dtype)."""
    return (x.float() + inc.float()).to(x.dtype) if pol.amp else x + inc


def final_norm(sd: Dict[str, torch.Tensor], x: torch.Tensor, pol: Policy) -> torch.Tensor:
    """The final LayerNorm over all tokens (register rows included); under the policy h(LN(x)) * g + b: the normalised value crosses
    the fp16 boundary, the affine does not (a gain far below 1 would otherwise turn the fixed absolute error of the modulation form
    into a large relative one)."""
    w, b = sd["model.norm.weight"], sd["model.norm.bias"]
    if not pol.amp:
        return F.layer_norm(x, (x.shape[-1],), w, b, 1e-6)
    return r16(F.layer_norm(x, (x.shape[-1],), None, None, 1e-6)) * w + b


def block(sd: Dict[str, torch.Tensor], i: int, x: torch.Tensor, pol: Policy = Policy("fp32")) -> torch.Tensor:
    x = residual_add(x, attn_branch(sd, i, x, pol), pol)
    return residual_add(x, mlp_branch(sd, i, x, pol), pol)


def forward(sd: Dict[str, torch.Tensor], image: torch.Tensor, depth: int = DEPTH, return_blocks: bool = False, pol: Policy = Policy("fp32")):
    """Dinov2Wrapper.forward: [N,518,518,3] -> [N, 1 + 37*37, 768] = cat[class token, patch tokens] after the final LayerNorm.  The
    arithmetic runs in the image's dtype (fp32 as the reference; fp64 with fp64 weights for the exact encoder)."""
    x = patch_embed(sd, image if image.is_floating_point() else image.float(), pol)
    outs = []
    for i in range(depth):
        x = block(sd, i, x, pol)
        if return_blocks:
            outs.append(x)
    x = final_norm(sd, x, pol)
    ret = torch.cat((x[:, :1], x[:, 1 + N_REG:]), dim=1)
    return (ret, outs) if return_blocks else ret
