"""GPU: VAE.encode / VAE.forward, the encoder stage by stage and the kernels it adds (conv_in 6 -> 32, the stride-2 downsample through
its space-to-depth pack, conv_out + quant_conv).

* Stage-local parity, as for the decoder (test_gpu_vae_stages.py): oracle stage k (oracle.vae.encode_stage) runs on the kernel's stage
  k-1 tap, in fp64 exactly and with the fp16 policy's rounding points; ours <= 2.5 x policy + 1e-4 (relative L2 against fp64) per
  primitive, per channel and per voxel class, where the classes separate voxels on the low faces (coordinate 0: the zero padding the
  stride-2 layer reads) from those on the high faces only and from the interior.
* One-hot weights, bit-exact: conv_in's taps, the downsample's taps (low-side padding included) and conv_out + quant_conv (channel 0
  mean, 1 log-variance, NCDHW).
* End to end against the reference's own encoder (tests/golden/vae_encode.npz) and, when oracle/_ref is staged, against the reference
  under autocast on 2048 primitives.
* Invariance (calls, batchings, input dtype, decode untouched), the posterior, and the launch count.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tpxl_b200
from oracle import refmods, vae as ov, vae_encode as ove
from oracle.dit import Policy
from tpxl_b200 import _lib, synth
from gpu_util import rel_l2
import parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 2027
N_STAGES = 10
# launches tpx_vae_encode makes through each stage (conv_in 1, 8^3 blocks 4 + 4, downsample 2, 32 -> 256 block 5, 256 blocks and the
# attention 4 each, norm_out 1) and in all (conv_out + quant_conv 1)
LAUNCHES_THROUGH = [1, 5, 9, 11, 16, 20, 24, 28, 32, 33]
ENCODE_LAUNCHES = 34


def _check_against_bound(name, ours, pol, ref):
    """ours / pol / ref: [P, S^3, C] fp64.  The bound (tests/parity.py) per primitive, per channel and per voxel class (low faces,
    high faces, both, interior)."""
    cls = parity.face_class(round(ref.shape[1] ** (1 / 3)))
    return parity.check(name, ours, pol, ref, {"primitive": parity.sequence, "channel": parity.channel, "class": parity.pooled(cls)})


def _full_sd(seed=SEED):
    sd = synth.synth_state_dict(synth.vae_encoder_shapes(**synth.FULL_VAE), seed)
    sd.update(synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), seed + 2))
    return sd


def _vae(sd):
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    vae.load_state_dict(sd)
    return vae.to(DEV)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "vae_encode.npz")))


@pytest.fixture(scope="module")
def encoder(fx):
    """The fixture's weights, and 2048 PrimX cells: the fixture's eight, then decoder outputs of seeded latents scaled per primitive."""
    sd = _full_sd()
    vae = _vae(sd)
    g = torch.Generator().manual_seed(72)
    z = (torch.randn(2040, 1, 4, 4, 4, generator=g) * torch.exp(torch.randn(2040, 1, 1, 1, 1, generator=g) * 0.3)).to(DEV)
    with torch.no_grad():
        x = torch.cat([torch.from_numpy(fx["x"]).to(DEV), vae.decode(z)]).contiguous()
    return vae, {k: v.to(DEV, torch.float64) for k, v in sd.items()}, x


@pytest.mark.parametrize("xdt", [torch.float32, torch.float16], ids=["x32", "x16"])
@pytest.mark.parametrize("P", [1, 3, 129, 2048])
def test_stage_local_parity(encoder, P, xdt):
    vae, sd, x_all = encoder
    x = x_all[:P].to(xdt).contiguous()
    idx = torch.arange(0, P, 89, device=DEV) if P > 64 else torch.arange(P, device=DEV)
    if int(idx[-1]) != P - 1:
        idx = torch.cat([idx, torch.tensor([P - 1], device=DEV)])
    f64, f16 = Policy("fp32"), Policy("fp16")
    prev = x[idx].double()
    worst = {}
    with torch.no_grad():
        for k in range(N_STAGES + 1):
            if k < N_STAGES:
                tap = vae.debug_encode_stage(x, k)
                assert tap.dtype == torch.float16 and tap.shape == (P, *vae.ENC_STAGE_SHAPES[k])
                got = tap[idx].double()
                if P > 64:
                    assert torch.equal(vae.debug_encode_stage(x[idx].contiguous(), k), tap[idx]), k
            ref = parity.to_cl(ove.encode_stage(k, sd, prev, f64))
            pol = parity.to_cl(ove.encode_stage(k, sd, prev, f16))
            if k < N_STAGES:
                worst[k] = _check_against_bound(f"stage {k}", got, pol, ref)
                prev = parity.to_ncdhw(got)
            else:
                out = vae.encode(x).parameters
                assert out.dtype == xdt and out.shape == (P, 2, 4, 4, 4)
                worst["moments"] = _check_against_bound("moments", parity.to_cl(out[idx].double()), pol, ref)
    print({k: {h: round(v, 3) for h, v in w.items()} for k, w in worst.items()})


def test_encode_launches_match_the_stage_taps(encoder):
    vae, _, x_all = encoder
    lib = _lib.lib()
    x = x_all[:5].contiguous()
    with torch.no_grad():
        vae.encode(x)
        n0 = lib.tpx_launch_count()
        out = vae.encode(x).parameters
        assert lib.tpx_launch_count() - n0 == ENCODE_LAUNCHES
        for k in range(N_STAGES):
            n0 = lib.tpx_launch_count()
            vae.debug_encode_stage(x, k)
            assert lib.tpx_launch_count() - n0 == LAUNCHES_THROUGH[k], k
        assert torch.equal(vae.encode(x).parameters, out)
    with pytest.raises(ValueError):
        vae.debug_encode_stage(x, N_STAGES)
    with pytest.raises(ValueError):
        vae.encode(x[:, :5])


def _one_hot(sd, key, index, extra=None):
    sd = dict(sd)
    w = torch.zeros_like(sd[key])
    w[index] = 1.0
    sd[key] = w
    sd[key.replace(".weight", ".bias")] = torch.zeros_like(sd[key.replace(".weight", ".bias")])
    sd.update(extra or {})
    return _vae(sd)


@pytest.mark.parametrize("xdt", [torch.float32, torch.float16], ids=["x32", "x16"])
@pytest.mark.parametrize("co,ci,tap", [(0, 0, (0, 0, 0)), (17, 3, (2, 1, 0)), (31, 5, (1, 1, 1))])
def test_conv_in_one_hot_is_a_shift(encoder, co, ci, tap, xdt):
    """conv_in with one 1.0 at (co, ci, kz, ky, kx): channel co at (z, y, x) is the fp16-rounded input channel ci at
    (z + kz - 1, y + ky - 1, x + kx - 1), 0 outside the volume; every other channel is 0."""
    _, _, x_all = encoder
    x = (x_all[:3] * 3).to(xdt).contiguous()
    vae = _one_hot(_full_sd(91), "encoder.conv_in.weight", (co, ci, *tap))
    with torch.no_grad():
        got = parity.to_ncdhw(vae.debug_encode_stage(x, 0))
    want = torch.zeros_like(got)
    kz, ky, kx = tap
    src = F.pad(x[:, ci].half(), (1, 1, 1, 1, 1, 1))
    want[:, co] = src[:, kz:kz + 8, ky:ky + 8, kx:kx + 8]
    assert bool((want != 0).any())
    assert torch.equal(got, want)


@pytest.mark.parametrize("co,ci,tap", [(0, 0, (0, 0, 0)), (5, 30, (2, 2, 2)), (31, 7, (0, 2, 1)), (12, 12, (1, 1, 1)), (3, 9, (1, 0, 2))])
def test_downsample_one_hot_is_a_strided_shift(encoder, co, ci, tap):
    """Conv3d(k3, s2, p1) with one 1.0 at (co, ci, kz, ky, kx): output channel co at (z, y, x) is input channel ci at
    (2z + kz - 1, 2y + ky - 1, 2x + kx - 1) — the low side's zero padding for k = 0 at 0 — and every other output is 0."""
    _, _, x_all = encoder
    x = x_all[:3].contiguous()
    vae = _one_hot(_full_sd(92), "encoder.down_blocks.0.downsample.weight", (co, ci, *tap))
    with torch.no_grad():
        a = parity.to_ncdhw(vae.debug_encode_stage(x, 2))
        got = parity.to_ncdhw(vae.debug_encode_stage(x, 3))
    want = torch.zeros_like(got)
    kz, ky, kx = tap
    src = F.pad(a[:, ci], (1, 1, 1, 1, 1, 1))       # src[i + 1] = a[i]
    want[:, co] = src[:, kz:kz + 8:2, ky:ky + 8:2, kx:kx + 8:2]
    assert bool((want != 0).any())
    assert torch.equal(got, want)


@pytest.mark.parametrize("odt", [torch.float32, torch.float16], ids=["out32", "out16"])
@pytest.mark.parametrize("ci,co,tap,swap", [(0, 0, (0, 0, 0), False), (255, 1, (2, 1, 0), False), (100, 0, (1, 1, 1), True)])
def test_conv_out_one_hot_through_quant_conv(encoder, ci, co, tap, swap, odt):
    """conv_out with one 1.0 at (co, ci, kz, ky, kx) and quant_conv the identity (or the channel swap): moment channel co (or 1 - co)
    at (z, y, x) is the norm_out activation ci at (z + kz - 1, ...), 0 outside; the other moment channel is 0.  NCDHW [P, 2, 4, 4, 4]."""
    _, _, x_all = encoder
    x = x_all[:3].to(odt).contiguous()
    qw = torch.tensor([[0.0, 1.0], [1.0, 0.0]] if swap else [[1.0, 0.0], [0.0, 1.0]]).reshape(2, 2, 1, 1, 1)
    vae = _one_hot(_full_sd(93), "encoder.conv_out.weight", (co, ci, *tap), {"quant_conv.weight": qw, "quant_conv.bias": torch.zeros(2)})
    with torch.no_grad():
        a = parity.to_ncdhw(vae.debug_encode_stage(x, 9)).float()
        got = vae.encode(x).parameters.float()
    want = torch.zeros_like(got)
    kz, ky, kx = tap
    src = F.pad(a[:, ci], (1, 1, 1, 1, 1, 1))
    want[:, (1 - co) if swap else co] = src[:, kz:kz + 4, ky:ky + 4, kx:kx + 4]
    assert bool((want != 0).any())
    assert torch.equal(got, want)


def test_encode_matches_the_reference_fixture(encoder, fx):
    """The fixture's eight cells (analytic SDFs, constant fields, decoder outputs) against the reference's fp32 encoder: ours is within
    2.5 x the fp16 policy's own distance + 1e-4, on the parameters and on forward(x, sample=False)."""
    vae, sd, _ = encoder
    x = torch.from_numpy(fx["x"]).to(DEV)
    ref = torch.from_numpy(fx["parameters"]).to(DEV).double()
    with torch.no_grad():
        out, post = vae(x, sample=False)
        pol = ove.encode(sd, x.double(), "fp16")
        pol_dec = ov.decode(sd, pol[:, :1], "fp16")
    got = post.parameters.double()
    for i in range(8):
        a, b = rel_l2(got[i], ref[i]), rel_l2(pol[i], ref[i])
        print(f"cell {i}: ours {a:.2e} policy {b:.2e}")
        assert a <= parity.bound(b), i
    fr = torch.from_numpy(fx["forward_mode"]).to(DEV).double()
    assert out.dtype == torch.float32 and out.shape == (8, 6, 8, 8, 8)
    assert rel_l2(out, fr) <= parity.bound(rel_l2(pol_dec, fr))
    assert torch.equal(post.mode(), post.parameters[:, :1])


def test_encode_2048_primitives_against_the_reference_under_autocast(encoder):
    if not refmods.available():
        pytest.skip("oracle/_ref is not staged")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    vae, sd, x = encoder
    ref = refmods.load().VAE(**synth.FULL_VAE)
    ref.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    ref = ref.to(DEV).eval()
    with torch.no_grad():
        r32 = torch.cat([ref.encode(x[i:i + 256]).parameters for i in range(0, 2048, 256)])
        with torch.autocast("cuda", dtype=torch.float16):
            r16 = torch.cat([ref.encode(x[i:i + 256]).parameters for i in range(0, 2048, 256)]).float()
        o = vae.encode(x).parameters
        o16 = vae.encode(x.half()).parameters.float()
    ours_vs_ref16, ref16_vs_ref32, ours_vs_ref32 = rel_l2(o, r16), rel_l2(r16, r32), rel_l2(o, r32)
    per_prim = (o - r32).flatten(1).norm(dim=1) / r32.flatten(1).norm(dim=1).clamp_min(1e-20)
    print(f"encode 2048: ours_vs_ref16 {ours_vs_ref16:.3e} ref16_vs_ref32 {ref16_vs_ref32:.3e} ours_vs_ref32 {ours_vs_ref32:.3e} "
          f"per-primitive max {float(per_prim.max()):.3e}")
    assert torch.equal(o16, o)
    assert ours_vs_ref32 < max(1e-3, 1.5 * ref16_vs_ref32) and ours_vs_ref32 < 5e-3
    assert ours_vs_ref16 < max(1e-3, 1.5 * ref16_vs_ref32)
    assert float(per_prim.max()) < 2e-2


def test_encode_is_invariant_to_calls_batching_and_input_dtype(encoder):
    vae, _, x = encoder
    with torch.no_grad():
        full = vae.encode(x).parameters
        assert torch.equal(vae.encode(x).parameters, full)
        for P in (1, 3, 129):
            assert torch.equal(vae.encode(x[:P]).parameters, full[:P]), P
        chunks = torch.cat([vae.encode(x[i:i + n]).parameters for i, n in ((0, 1), (1, 3), (4, 129), (133, 2048 - 133))])
        assert torch.equal(chunks, full)
        half = vae.encode(x.half()).parameters
        assert half.dtype == torch.float16 and torch.equal(half.float(), full)
        empty = vae.encode(x[:0])
        assert empty.parameters.shape == (0, 2, 4, 4, 4) and empty.mean.shape == (0, 1, 4, 4, 4)


def test_decode_is_untouched_by_encode(encoder):
    vae, _, x = encoder
    z = torch.randn(37, 1, 4, 4, 4, generator=torch.Generator().manual_seed(5)).to(DEV)
    with torch.no_grad():
        before = vae.decode(z)
        vae.encode(x[:300])
        assert torch.equal(vae.decode(z), before)


def test_posterior_sample_and_logvar_clamp(encoder):
    vae, _, x = encoder
    with torch.no_grad():
        post = vae.encode(x[:9])
        torch.manual_seed(123)
        s = post.sample()
        torch.manual_seed(123)
        want = post.mean + post.std * torch.randn(post.mean.shape, device=DEV, dtype=post.parameters.dtype)
        assert torch.equal(s, want)
        torch.manual_seed(124)
        dec, p2 = vae(x[:9], sample=True)
        torch.manual_seed(124)
        assert torch.equal(dec, vae.decode(p2.mean + p2.std * torch.randn(p2.mean.shape, device=DEV)))
    for bias, bound in ((100.0, 20.0), (-100.0, -30.0)):
        sd = _full_sd()
        sd["quant_conv.bias"] = torch.tensor([0.0, bias])
        v = _vae(sd)
        with torch.no_grad():
            p = v.encode(x[:4])
        assert bool((p.parameters[:, 1] != bound).all()) and bool((p.logvar == bound).all())
        assert torch.equal(p.std, torch.exp(0.5 * p.logvar)) and torch.isfinite(p.var).all()


def test_missing_encoder_tensors_are_named(encoder):
    sd = _full_sd()
    del sd["encoder.mid_block.attns.0.attn.qkv.weight"]
    sd["quant_conv.bias"] = torch.zeros(3)
    v = _vae(sd)
    z = torch.zeros(2, 1, 4, 4, 4, device=DEV)
    with torch.no_grad():
        v.decode(z)                                 # the decode path never looks at the encoder tensors
        with pytest.raises(RuntimeError, match="attns.0.attn.qkv.weight.*quant_conv.bias"):
            v.encode(torch.zeros(2, 6, 8, 8, 8, device=DEV))
    bad = tpxl_b200.VAE(**{**synth.FULL_VAE, "down_channels": [16, 256]}).to(DEV)
    with pytest.raises(NotImplementedError):
        bad.encode(torch.zeros(2, 6, 8, 8, 8, device=DEV))


def test_encode_primvolume_inverts_the_sampling_glue(encoder):
    """PrimXPipeline.encode_primvolume(decode_latents(sample)): srt comes back to within fp32 rounding, the 64 feature channels are the
    posterior mode of the unpacked volumes, merged into the normalised latent space."""
    vae, _, _ = encoder
    pipe = tpxl_b200.PrimXPipeline(None, vae, latent_mean=synth.LATENT_MEAN, latent_std=synth.LATENT_STD, num_prims=5)
    lat = torch.randn(2, 5, 68, generator=torch.Generator().manual_seed(21)).to(DEV)
    with torch.no_grad():
        rp = pipe.decode_latents(lat)
        back = pipe.encode_primvolume(rp)
        srt, feats = pipe.codec.unpack(rp)
        want = pipe.codec.merge(srt, vae.encode(feats).mode())
    assert back.shape == (2, 5, 68) and back.dtype == torch.float32
    assert torch.equal(back, want)
    assert float((back[..., :4] - lat[..., :4]).abs().max()) < 1e-5
