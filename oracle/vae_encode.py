"""Oracle restatement of the 3D-conv VAE encoder (TEST INFRASTRUCTURE — see oracle/__init__.py), beside oracle/vae.py's decoder.

Restates, over a reference-keyed ``state_dict`` (encoder.* / quant_conv.* keys):
  * VAE.encode              /root/reference/models/vae3d_dib.py:431-435   (the posterior's parameters: quant_conv(encoder(x)))
  * Encoder.forward         vae3d_dib.py:310-327
  * DownBlock._forward      vae3d_dib.py:178-184   (downsample = Conv3d(k3, s2, p1))
with oracle/vae.py's ResnetBlock / VolumeAttention / convolution restatements and precision policies, and the space-to-depth form of
the stride-2 convolution the GPU encoder runs.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from .dit import Policy
from .vae import _conv, _gn, resnet_block, volume_attention

Tensor = torch.Tensor


ENCODE_STAGES = ("conv_in", "down0_res0", "down0_res1", "downsample", "down1_res0", "down1_res1", "mid_res0", "mid_attn", "mid_res1",
                 "norm_out")


def encode_stage(k: int, sd, x: Tensor, pol: Policy) -> Tensor:
    """Encoder stage k (0..9 as ENCODE_STAGES, 10 = conv_out + quant_conv) on NCDHW input x."""
    e = "encoder."
    res = {1: "down_blocks.0.nets.0.", 2: "down_blocks.0.nets.1.", 4: "down_blocks.1.nets.0.", 5: "down_blocks.1.nets.1.",
           6: "mid_block.nets.0.", 8: "mid_block.nets.1."}
    if k == 0:
        return _conv(pol, x, sd[e + "conv_in.weight"], sd[e + "conv_in.bias"], padding=1)
    if k in res:
        return resnet_block(sd, e + res[k], x, pol)
    if k == 3:
        return _conv(pol, x, sd[e + "down_blocks.0.downsample.weight"], sd[e + "down_blocks.0.downsample.bias"], stride=2, padding=1)
    if k == 7:
        return volume_attention(sd, e + "mid_block.attns.0.", x, pol)
    if k == 9:
        return pol.rnd(F.silu(_gn(sd, e + "norm_out.", x)))      # conv_out's input: rounded to fp16 under autocast
    assert k == 10
    h = _conv(pol, x, sd[e + "conv_out.weight"], sd[e + "conv_out.bias"], padding=1)
    return _conv(pol, h, sd["quant_conv.weight"], sd["quant_conv.bias"])


def encode(sd: Dict[str, Tensor], x: Tensor, precision: str = "fp32", stages: dict | None = None) -> Tensor:
    """VAE.encode up to the posterior: x [P,6,8,8,8] -> parameters [P,2,4,4,4].  ``stages`` (optional dict) receives the ten
    intermediates of ENCODE_STAGES (NCDHW)."""
    pol = Policy(precision)
    sd = {k: v.float() if v.dtype in (torch.float16, torch.bfloat16) else v for k, v in sd.items()}
    h = x if x.dtype == torch.float64 else x.float()
    for k in range(11):
        h = encode_stage(k, sd, h, pol)
        if stages is not None and k < 10:
            stages[ENCODE_STAGES[k]] = h
    return h


def space_to_depth(x: Tensor) -> Tensor:
    """NCDHW [P, C, 2S, 2S, 2S] -> [P, 8C, S, S, S], channel ((az*2 + ay)*2 + ax)*C + c holds x[..., 2z+az, 2y+ay, 2x+ax]."""
    P, C, D = x.shape[:3]
    S = D // 2
    return x.reshape(P, C, S, 2, S, 2, S, 2).permute(0, 3, 5, 7, 1, 2, 4, 6).reshape(P, 8 * C, S, S, S)


def space_to_depth_weight(w: Tensor) -> Tensor:
    """Conv3d(k3, s2, p1) weight [Cout, Cin, 3, 3, 3] -> the stride-1 / pad-1 weight [Cout, 8 Cin, 3, 3, 3] over space_to_depth(x):
    per axis, block offset k' and phase a take original tap (k', a) = (0, 1) -> 0, (1, 0) -> 1, (1, 1) -> 2; all else is zero.
    The index map the encoder's repack kernel (launch_pack_conv3_s2d) implements."""
    Cout, Cin = w.shape[:2]
    out = w.new_zeros(Cout, 2, 2, 2, Cin, 3, 3, 3)
    pick = {(0, 1): 0, (1, 0): 1, (1, 1): 2}
    for (kz, az), tz in pick.items():
        for (ky, ay), ty in pick.items():
            for (kx, ax), tx in pick.items():
                out[:, az, ay, ax, :, kz, ky, kx] = w[:, :, tz, ty, tx]
    return out.reshape(Cout, 8 * Cin, 3, 3, 3)
