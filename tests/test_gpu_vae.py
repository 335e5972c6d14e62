"""GPU: implicit-GEMM 3-D convolutions and VAE.decode against F.conv3d, the oracle and the reference fixture.

Tolerance: the decoder computes with fp16 tensor-core inputs and fp32 accumulation / statistics; against the fp32
reference (as inference.py:339 invokes it) relative L2 <= 1e-2, the distance at which the reference's own
autocast(fp16) run sits (oracle fp16 policy, printed)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle
import tpxl_b200
from tpxl_b200 import _lib, synth
from gpu_util import rel_l2, st
import parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pack(w):   # [Cout,Cin,3,3,3] -> [Cout, 27*Cin], k = tap*Cin + ci
    return w.permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1).contiguous()


@pytest.mark.parametrize("P,S,Cc,Cout,resid", [(6, 4, 256, 256, False), (5, 4, 256, 256, True), (3, 8, 256, 32, False), (3, 8, 32, 32, True), (2, 8, 32, 32, False)])
def test_conv3d_k3_implicit_gemm(P, S, Cc, Cout, resid):
    g = torch.Generator(device=DEV).manual_seed(P * S + Cc)
    x = torch.randn(P, S, S, S, Cc, generator=g, device=DEV).half()
    w = (torch.randn(Cout, Cc, 3, 3, 3, generator=g, device=DEV) * (27 * Cc) ** -0.5).half()
    b = torch.randn(Cout, generator=g, device=DEV).half()
    r = torch.randn(P, S, S, S, Cout, generator=g, device=DEV).half() if resid else None
    alpha = 0.5 ** 0.5 if resid else 1.0
    out = torch.empty(P, S, S, S, Cout, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().tpx_conv3d_k3(x.data_ptr(), _pack(w).data_ptr(), b.data_ptr(), _lib.ptr(r), alpha, out.data_ptr(), P, S, Cc, Cout, st()))
    ref = F.conv3d(x.float().permute(0, 4, 1, 2, 3), w.float(), b.float(), padding=1).permute(0, 2, 3, 4, 1)
    if resid:
        ref = (ref + r.float()) * alpha
    torch.cuda.synchronize()
    assert rel_l2(out.float(), ref) < 2e-3


def test_decode_against_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "vae_decode.npz"))
    sd = synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 103)
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    vae.load_state_dict(sd)
    vae = vae.to(DEV)
    z = torch.from_numpy(g["z"]).to(DEV)
    with torch.no_grad():
        out = vae.decode(z)
        out16 = vae.decode(z.half())
        o16 = oracle.vae.decode({k: v.to(DEV) for k, v in sd.items()}, z, "fp16")
    ref = torch.from_numpy(g["out"]).to(DEV)
    r = dict(ours_vs_ref32=rel_l2(out, ref), oracle16_vs_ref32=rel_l2(o16, ref), half_io=rel_l2(out16.float(), ref))
    print(r)
    assert out.dtype == torch.float32 and out16.dtype == torch.float16 and out.shape == (4, 6, 8, 8, 8) and out.is_contiguous()
    assert r["ours_vs_ref32"] < 1e-2 and r["half_io"] < 1e-2
    assert r["ours_vs_ref32"] < parity.bound(r["oracle16_vs_ref32"])
    out.mul_(2)   # caller mutates the result in place (inference.py:345-346): must be a fresh, writable tensor


def test_decode_full_batch_properties():
    """2048 primitives (config #4): finite, deterministic, and primitive-wise independent (any sub-batch decodes identically)."""
    sd = synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 71)
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    vae.load_state_dict(sd)
    vae = vae.to(DEV)
    rs = np.random.RandomState(72)
    z = torch.from_numpy((rs.standard_normal(size=(2048, 64)) * np.array(synth.LATENT_STD[4:]) + np.array(synth.LATENT_MEAN[4:])).astype(np.float32)).reshape(2048, 1, 4, 4, 4).to(DEV)
    with torch.no_grad():
        full = vae.decode(z)
        again = vae.decode(z)
        part = vae.decode(z[1000:1007].contiguous())
        sub = z[3::8].contiguous()                          # 256 primitives strided over the whole batch, against the oracle
        ref = oracle.vae.decode({k: v.to(DEV) for k, v in sd.items()}, sub, "fp32")
    assert torch.isfinite(full).all() and torch.equal(full, again)
    assert torch.equal(part, full[1000:1007])
    got = full[3::8]
    per_prim = (got - ref).flatten(1).norm(dim=1) / ref.flatten(1).norm(dim=1).clamp_min(1e-20)
    print("256 strided primitives vs oracle fp32: rel-L2", rel_l2(got, ref), "worst primitive", float(per_prim.max()))
    assert rel_l2(got, ref) < 1e-2 and float(per_prim.max()) < 3e-2


def test_error_paths():
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    with pytest.raises(_lib.TpxError):
        vae.decode(torch.zeros(1, 1, 4, 4, 4))
    vae.load_state_dict(synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 73))
    vae = vae.to(DEV)
    with pytest.raises(ValueError):
        vae.decode(torch.zeros(1, 1, 8, 8, 8, device=DEV))
    assert vae.decode(torch.zeros(0, 1, 4, 4, 4, device=DEV)).shape == (0, 6, 8, 8, 8)
