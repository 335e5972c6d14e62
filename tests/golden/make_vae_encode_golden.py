#!/usr/bin/env python
"""Regenerate tests/golden/vae_encode.npz: the reference's own VAE (oracle/_ref, staged by oracle/stage_ref.py; xformers restated by
oracle/refmods.py) run in fp32 on the CPU over seeded full-VAE weights (synth seed 2027) and eight PrimX cells:

    0-2  analytic SDF cells: a sphere inside the cell, a plane crossing it, a sphere off-centre (channel 0 = 5 * signed distance in
         cell units, channels 1-5 smooth colour / material ramps in [-1, 1]);
    3-4  constant fields;
    5-7  the reference decoder's output for seeded random latents (what VAE.forward round trips).

Stored: ``x`` [8,6,8,8,8] fp32; ``stage_<name>`` for the ten encoder stages of oracle.vae_encode.ENCODE_STAGES, every primitive and
every voxel (NCDHW) but only the channels listed in ``channels_<name>`` (every 4th of a 32-channel stage, every 8th of a 256-channel
one: each convolution mixes all channels, so any of them carries a wrong stage) and rounded to fp16, which keeps the file near 0.5 MB;
``parameters`` [8,2,4,4,4], ``mode``, ``kl`` (against N(0,1)), ``kl_other`` (against the posterior of the cells rolled by one), ``nll``
(of ``nll_sample``) and ``forward_mode`` (= VAE.forward(x, sample=False)[0]) in fp32.

    python tests/golden/make_vae_encode_golden.py
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refmods, vae_encode as ove  # noqa: E402
from tpxl_b200 import synth  # noqa: E402

SEED = 2027


def cells() -> torch.Tensor:
    g = torch.Generator().manual_seed(SEED + 1)
    c = (torch.arange(8, dtype=torch.float64) + 0.5) / 8 * 2 - 1          # voxel centres in [-1, 1]
    z, y, x = torch.meshgrid(c, c, c, indexing="ij")
    ramps = torch.stack([x, y, z, x * y, 0.5 * (x + z)])                  # 5 smooth channels in [-1, 1]
    out = []
    for sdf in ((x ** 2 + y ** 2 + z ** 2).sqrt() - 0.6, 0.3 * x + 0.5 * y - 0.8 * z + 0.1, ((x - 0.4) ** 2 + (y + 0.3) ** 2 + z ** 2).sqrt() - 0.9):
        out.append(torch.cat([5 * sdf[None], ramps.roll(len(out), 0)]))
    for v in (0.7, -0.4):
        out.append(torch.full((6, 8, 8, 8), v, dtype=torch.float64))
    x6 = torch.stack(out).float()
    return x6, g


def main():
    ref = refmods.load()
    sd = synth.synth_state_dict(synth.vae_encoder_shapes(**synth.FULL_VAE), SEED)
    sd.update(synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), SEED + 2))
    m = ref.VAE(**synth.FULL_VAE)
    m.load_state_dict(sd, strict=True)
    m = m.eval()
    x, g = cells()
    with torch.no_grad():
        z = torch.randn(3, 1, 4, 4, 4, generator=g) * 0.8
        x = torch.cat([x, m.decode(z)]).contiguous()
        taps = {}
        enc = m.encoder
        hooks = [(enc.conv_in, "conv_in"), (enc.down_blocks[0].nets[0], "down0_res0"), (enc.down_blocks[0].nets[1], "down0_res1"),
                 (enc.down_blocks[0].downsample, "downsample"), (enc.down_blocks[1].nets[0], "down1_res0"), (enc.down_blocks[1].nets[1], "down1_res1"),
                 (enc.mid_block.nets[0], "mid_res0"), (enc.mid_block.attns[0], "mid_attn"), (enc.mid_block.nets[1], "mid_res1"),
                 (enc.norm_out, "norm_out")]
        handles = [mod.register_forward_hook(lambda _m, _i, o, n=name: taps.__setitem__(n, o.detach().clone())) for mod, name in hooks]
        post = m.encode(x)
        for h in handles:
            h.remove()
        taps["norm_out"] = F.silu(taps["norm_out"])
        other = type(post)(post.parameters.roll(1, 0))
        nll_sample = post.mode() + 0.25 * torch.randn(post.mean.shape, generator=g)
        fwd, _ = m(x, sample=False)
    assert set(taps) == set(ove.ENCODE_STAGES)
    out = dict(x=x.numpy(), parameters=post.parameters.numpy(), mode=post.mode().numpy(), kl=post.kl().numpy(), kl_other=post.kl(other).numpy(),
               nll_sample=nll_sample.numpy(), nll=post.nll(nll_sample).numpy(), forward_mode=fwd.numpy(), seed=np.int64(SEED))
    for name in ove.ENCODE_STAGES:
        t = taps[name]
        ch = np.arange(0, t.shape[1], 4 if t.shape[1] <= 32 else 8)
        out["channels_" + name] = ch
        out["stage_" + name] = t[:, ch].numpy().astype(np.float16)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "vae_encode.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
