"""GPU: the VAE decoder stage by stage, and the kernels it is built from at the decoder's own shapes.

* Stage-local parity.  ``VAE.debug_stage`` (tpx_vae_debug_stage) returns the activation after each of the decoder's ten stages.
  Stage k of the oracle (oracle/vae.py) runs on the kernel's own stage k-1 tap, so errors do not compound, twice in fp64: exactly
  ("fp64") and with the fp16 policy's rounding points ("policy", the reference under autocast).  Bound, as relative L2 against fp64:
  ours <= 2.5 x policy + 1e-4, for every primitive, for every voxel class (corner / edge / face / interior of the 4^3 or 8^3
  volume: halo and zero-padding errors land on the boundary classes) and for every channel (tile errors land on channels).
* Exact one-hot weight checks of the convolutions' index maps (k2 upsample sub-lattice, conv_in and conv_out taps with the
  ConvTranspose flip): a single 1.0 weight copies activations, so the result must match bit for bit.
* tpx_linear_heads / tpx_attention at the decoder's attention shape, and the online-softmax rescale of the mma.sync attention kernel.
* GroupNorm on every dispatch path with inputs whose mean is large against their spread, constant groups, and mixed groups.
"""
import pytest
import torch
import torch.nn.functional as F

import oracle
import tpxl_b200
from oracle import vae as ov
from oracle.dit import Policy
from tpxl_b200 import _lib, synth
from gpu_util import rel_l2, st
import parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N_STAGES = 10
# the oracle's stage functions: stage -> resnet block prefix
RES_PREFIX = {1: "mid_block.nets.0.", 3: "mid_block.nets.1.", 4: "up_blocks.0.nets.0.", 5: "up_blocks.0.nets.1.", 7: "up_blocks.1.nets.0.",
              8: "up_blocks.1.nets.1."}
# kernel launches tpx_vae_decode makes up to the end of each stage (conv_in 1, resnet block at 4^3 4, attention 4, upsample 8,
# resnet block with shortcut 5, resnet block at 8^3 4, norm_out 1) and in all (conv_out 1)
LAUNCHES_THROUGH = [1, 5, 9, 13, 17, 21, 29, 34, 38, 39]
DECODE_LAUNCHES = 40


def _stage(k: int, sd, x, pol: Policy):
    """Decoder stage k (0..9, 10 = conv_out) of oracle.vae.decode on NCDHW input x."""
    d = "decoder."
    if k == 0:
        x = ov._conv(pol, x, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
        return ov._conv(pol, x, sd[d + "conv_in.weight"], sd[d + "conv_in.bias"], padding=1)
    if k in RES_PREFIX:
        return ov.resnet_block(sd, d + RES_PREFIX[k], x, pol)
    if k == 2:
        return ov.volume_attention(sd, d + "mid_block.attns.0.", x, pol)
    if k == 6:
        return ov._convT(pol, x, sd[d + "up_blocks.0.upsample.weight"], sd[d + "up_blocks.0.upsample.bias"], stride=2)
    if k == 9:
        return pol.rnd(F.silu(ov._gn(sd, d + "norm_out.", x)))    # conv_out's input: rounded to fp16 under autocast
    assert k == 10
    return ov._convT(pol, x, sd[d + "conv_out.weight"], sd[d + "conv_out.bias"], stride=1, padding=1)


def _check_against_bound(name, ours, pol, ref):
    """ours / pol / ref: [P, S^3, C] fp64.  The bound (tests/parity.py) per primitive, per channel and per voxel class (how many
    coordinates lie on the volume's boundary)."""
    cls = parity.boundary_count(round(ref.shape[1] ** (1 / 3)))
    return parity.check(name, ours, pol, ref, {"primitive": parity.sequence, "channel": parity.channel, "class": parity.pooled(cls)})


@pytest.fixture(scope="module")
def decoder():
    sd = synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 71)
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    vae.load_state_dict(sd)
    vae = vae.to(DEV)
    g = torch.Generator().manual_seed(72)       # latents as VAE.decode sees them: the denormalised feature channels
    z = torch.randn(2048, 64, generator=g, dtype=torch.float64) * torch.tensor(synth.LATENT_STD[4:], dtype=torch.float64) \
        + torch.tensor(synth.LATENT_MEAN[4:], dtype=torch.float64)
    return vae, {k: v.to(DEV, torch.float64) for k, v in sd.items()}, z.float().reshape(2048, 1, 4, 4, 4).to(DEV)


def _decode_raw(vae, z, out_dtype):
    out = torch.empty(z.shape[0], 6, 8, 8, 8, dtype=out_dtype, device=DEV)
    base, nbytes = vae._workspace(_lib.lib(), z.shape[0])
    _lib.check(_lib.lib().tpx_vae_decode(vae._handle, z.data_ptr(), _lib.dtype_tag(z), out.data_ptr(), _lib.dtype_tag(out), z.shape[0], base, nbytes, st()))
    return out


# P = 1, 3: a half 128-row tile at 4^3; 33 / 34: the halo kernel's persistent CTAs take a second tile from 34 on (132 SMs); 2048: the
# released batch, checked on a strided subset that holds the first and the last primitive
@pytest.mark.parametrize("zdt", [torch.float32, torch.float16], ids=["z32", "z16"])
@pytest.mark.parametrize("P", [1, 3, 33, 34, 2048])
def test_stage_local_parity(decoder, P, zdt):
    vae, sd, z_all = decoder
    z = z_all[:P].to(zdt).contiguous()
    idx = torch.arange(0, P, 89, device=DEV) if P > 64 else torch.arange(P, device=DEV)
    assert int(idx[0]) == 0 and int(idx[-1]) == P - 1
    f64, f16 = Policy("fp32"), Policy("fp16")    # "fp32" = no rounding: on fp64 tensors it is the exact fp64 reference
    prev = z[idx].double()
    worst = {}
    with torch.no_grad():
        for k in range(N_STAGES + 1):
            if k < N_STAGES:
                tap = vae.debug_stage(z, k)
                assert tap.dtype == torch.float16 and tap.shape == (P, *vae.STAGE_SHAPES[k])
                got = tap[idx].double()
                if P > 64:      # a primitive's result does not depend on the batch it is decoded in
                    assert torch.equal(vae.debug_stage(z[idx].contiguous(), k), tap[idx]), k
            else:
                outs = {dt: _decode_raw(vae, z, dt) for dt in (torch.float32, torch.float16)}
            ref = parity.to_cl(_stage(k, sd, prev, f64))
            pol = parity.to_cl(_stage(k, sd, prev, f16))
            if k < N_STAGES:
                print(f"stage {k}: activation rms {float(got.pow(2).mean().sqrt()):.3f}")
                worst[k] = _check_against_bound(f"stage {k}", got, pol, ref)
                prev = parity.to_ncdhw(got)
            else:
                for dt, o in outs.items():
                    worst[f"out {dt}"] = _check_against_bound(f"decode output {dt}", parity.to_cl(o[idx].double()), pol, ref)
    print({k: {h: round(v, 3) for h, v in w.items()} for k, w in worst.items()})


def test_decode_launches_match_the_stage_taps(decoder):
    """decode launches exactly its schedule; each stage tap runs that schedule's prefix."""
    vae, _, z_all = decoder
    lib = _lib.lib()
    z = z_all[:5].contiguous()
    with torch.no_grad():
        vae.decode(z)                       # workspace allocation, first-launch attributes
        n0 = lib.tpx_launch_count()
        out = vae.decode(z)
        assert lib.tpx_launch_count() - n0 == DECODE_LAUNCHES
        for k in range(N_STAGES):
            n0 = lib.tpx_launch_count()
            vae.debug_stage(z, k)
            assert lib.tpx_launch_count() - n0 == LAUNCHES_THROUGH[k], k
        assert torch.equal(vae.decode(z), out)
    with pytest.raises(ValueError):
        vae.debug_stage(z, N_STAGES)
    base, nbytes = vae._workspace(lib, 5)
    tap = torch.empty(5, 64, 256, dtype=torch.float16, device=DEV)
    assert lib.tpx_vae_debug_stage(vae._handle, z.data_ptr(), 0, 5, N_STAGES, tap.data_ptr(), base, nbytes, st()) == -1     # TPX_ERR_ARG
    assert b"bad stage" in lib.tpx_last_error()


def _one_hot_decoder(sd, key, index):
    """A decoder whose weight `key` is zero except for a single 1.0 at `index`, with that layer's bias zero."""
    sd = dict(sd)
    w = torch.zeros_like(sd[key])
    w[index] = 1.0
    sd[key] = w
    sd[key.replace(".weight", ".bias")] = torch.zeros_like(sd[key.replace(".weight", ".bias")])
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    vae.load_state_dict(sd)
    return vae.to(DEV)


@pytest.fixture(scope="module")
def synth_sd():
    return synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 91)


@pytest.mark.parametrize("ci,co,abc", [(37, 201, (1, 0, 1)), (0, 255, (0, 0, 0)), (255, 0, (1, 1, 1))])
def test_upsample_one_hot_fills_its_sub_lattice(decoder, synth_sd, ci, co, abc):
    """ConvTranspose3d(k2, s2) weight [Cin, Cout, 2, 2, 2] with one 1.0 at (ci, co, a, b, c): output channel co at (2z+a, 2y+b, 2x+c)
    is input channel ci at (z, y, x); every other output is 0."""
    _, _, z_all = decoder
    z = z_all[:3].contiguous()
    vae = _one_hot_decoder(synth_sd, "decoder.up_blocks.0.upsample.weight", (ci, co, *abc))
    with torch.no_grad():
        x = parity.to_ncdhw(vae.debug_stage(z, 5))
        u = parity.to_ncdhw(vae.debug_stage(z, 6))
    want = torch.zeros_like(u)
    a, b, c = abc
    want[:, co, a::2, b::2, c::2] = x[:, ci]
    assert bool((x[:, ci] != 0).any())
    assert torch.equal(u, want)


@pytest.mark.parametrize("odt", [torch.float32, torch.float16], ids=["out32", "out16"])
@pytest.mark.parametrize("ci,co,tap", [(5, 2, (0, 1, 2)), (31, 0, (2, 2, 0)), (0, 5, (1, 1, 1))])
def test_conv_out_one_hot_is_a_flipped_shift(decoder, synth_sd, ci, co, tap, odt):
    """conv_out is ConvTranspose3d(k3, s1, p1) with weight [Cin, Cout, 3, 3, 3]: one 1.0 at (ci, co, kz, ky, kx) gives output channel co
    at (z, y, x) = input channel ci at (z + 1 - kz, y + 1 - ky, x + 1 - kx), 0 where that is outside the volume, 0 on other channels."""
    _, _, z_all = decoder
    z = z_all[:3].contiguous()
    vae = _one_hot_decoder(synth_sd, "decoder.conv_out.weight", (ci, co, *tap))
    with torch.no_grad():
        x = parity.to_ncdhw(vae.debug_stage(z, 9)).float()
        out = _decode_raw(vae, z, odt).float()
    want = torch.zeros_like(out)
    kz, ky, kx = tap
    src = F.pad(x[:, ci], (1, 1, 1, 1, 1, 1))       # src[i + 1] = x[i]
    want[:, co] = src[:, 2 - kz:10 - kz, 2 - ky:10 - ky, 2 - kx:10 - kx]
    assert bool((want != 0).any())
    assert torch.equal(out, want)


@pytest.mark.parametrize("zdt", [torch.float32, torch.float16], ids=["z32", "z16"])
@pytest.mark.parametrize("co,tap", [(0, (0, 0, 0)), (129, (2, 1, 0)), (255, (1, 1, 1))])
def test_conv_in_one_hot_is_a_shift(decoder, synth_sd, co, tap, zdt):
    """post_quant_conv = identity and conv_in (Conv3d k3, p1, weight [C, 1, 3, 3, 3]) with one 1.0 at (co, 0, kz, ky, kx): channel co at
    (z, y, x) is the fp16-rounded latent at (z + kz - 1, y + ky - 1, x + kx - 1), 0 outside; every other channel is 0."""
    _, _, z_all = decoder
    z = (z_all[:4] * 3).to(zdt).contiguous()
    sd = dict(synth_sd)
    sd["post_quant_conv.weight"], sd["post_quant_conv.bias"] = torch.ones(1, 1, 1, 1, 1), torch.zeros(1)
    vae = _one_hot_decoder(sd, "decoder.conv_in.weight", (co, 0, *tap))
    with torch.no_grad():
        got = parity.to_ncdhw(vae.debug_stage(z, 0))
    want = torch.zeros_like(got)
    kz, ky, kx = tap
    src = F.pad(z[:, 0].half(), (1, 1, 1, 1, 1, 1))
    want[:, co] = src[:, kz:kz + 4, ky:ky + 4, kx:kx + 4]
    assert bool((want != 0).any())
    assert torch.equal(got, want)


def test_linear_heads_at_the_decoder_attention_shape():
    """The decoder's qkv projection: 8 heads x Dh = DhP = 32, 64 tokens per primitive, 256-wide tiles, no bias.  33 primitives (M = 2112,
    a half 128-row tile at the end); every element of the three outputs is written, in [b, head, token, d] order."""
    P, H, Dh, N, K = 33, 8, 32, 64, 256
    g = torch.Generator(device=DEV).manual_seed(5)
    A = torch.randn(P * N, K, generator=g, device=DEV).half()
    W = (torch.randn(3 * H * Dh, K, generator=g, device=DEV) / 16).half()
    outs = [torch.full((P, H, N, Dh), 7.0, dtype=torch.float16, device=DEV) for _ in range(3)]
    _lib.check(_lib.lib().tpx_linear_heads(A.data_ptr(), K, W.data_ptr(), None, outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(),
                                           P * N, 3 * H * Dh, K, H * Dh, H, Dh, Dh, N, 1.0, 256, -1, 0, st()), "tpx_linear_heads")
    ref = (A.double() @ W.double().t()).reshape(P, N, 3, H, Dh).permute(2, 0, 3, 1, 4)
    torch.cuda.synchronize()
    for w in range(3):
        err = (outs[w].double() - ref[w]).abs()
        assert float((err - ref[w].abs() * 2 ** -11).max()) < 1e-4, (w, float(err.max()))


def _attention_ref(q, k, v, Dh, scale):
    s = torch.matmul(q[..., :Dh].double(), k[..., :Dh].double().transpose(-1, -2)) * scale
    B, H, Nq = q.shape[:3]
    return torch.matmul(torch.softmax(s, -1), v[..., :Dh].double()).permute(0, 2, 1, 3).reshape(B, Nq, H * Dh), s


def test_attention_at_the_decoder_shape():
    """2048 primitives x 8 heads of 64-token self-attention at DhP = 32 (grid.z = 2048), against fp64."""
    B, H, Nt, Dh = 2048, 8, 64, 32
    g = torch.Generator(device=DEV).manual_seed(6)
    q, k, v = (torch.randn(B, H, Nt, Dh, generator=g, device=DEV).half() for _ in range(3))
    out = torch.full((B, Nt, H * Dh), 9.0, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().tpx_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, Nt, Nt, Dh, Dh, Dh ** -0.5, st()))
    ref, _ = _attention_ref(q, k, v, Dh, Dh ** -0.5)
    torch.cuda.synchronize()
    err = (out.double() - ref).abs()
    per_batch = err.flatten(1).amax(1)
    print("max |err|", float(err.max()), "rel-L2", rel_l2(out, ref), "worst primitive", int(per_batch.argmax()))
    assert rel_l2(out, ref) < 1e-3 and float((err - 1e-3 * ref.abs()).max()) < 2e-3


@pytest.mark.parametrize("Dh,DhP", [(32, 32), (72, 80), (80, 80)])
def test_attention_mma_sync_rescale(Dh, DhP):
    """Logits with a standard deviation of ~8 and key norms that grow from one 64-key tile to the next, so the running row maximum
    of the mma.sync kernel jumps by far more than 2^8 between tiles: the rescale of O and of the row sums.  Nk = 1000 is ragged."""
    B, H, Nq, Nk = 1, 2, 256, 1000
    g = torch.Generator(device=DEV).manual_seed(Dh * 13 + DhP)
    q = torch.zeros(B, H, Nq, DhP, dtype=torch.float16, device=DEV)
    k = torch.zeros(B, H, Nk, DhP, dtype=torch.float16, device=DEV)
    v = torch.zeros(B, H, Nk, DhP, dtype=torch.float16, device=DEV)
    q[..., :Dh] = (torch.randn(B, H, Nq, Dh, generator=g, device=DEV) * 8).half()
    kscale = 0.3 + 0.15 * (torch.arange(Nk, device=DEV) // 64).float()
    k[..., :Dh] = (torch.randn(B, H, Nk, Dh, generator=g, device=DEV) * kscale[None, None, :, None]).half()
    v[..., :Dh] = torch.randn(B, H, Nk, Dh, generator=g, device=DEV).half()
    out = torch.full((B, Nq, H * Dh), 9.0, dtype=torch.float16, device=DEV)
    scale = Dh ** -0.5
    _lib.check(_lib.lib().tpx_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, H, Nq, Nk, Dh, DhP, scale, st()))
    ref, s = _attention_ref(q, k, v, Dh, scale)
    tiles = s[..., : (Nk // 64) * 64].reshape(B, H, Nq, -1, 64).amax(-1)
    assert bool((tiles.diff(dim=-1) * 1.4427 > 8).any()), "the inputs were meant to force a rescale"
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert rel_l2(out, ref) < 2e-3


# (S^3, C, groups) -> dispatch path of launch_groupnorm_silu
GN_PATHS = {"stream256_4cube": (64, 256, 32), "stream256_8cube": (512, 32, 32), "stream512": (512, 256, 32), "res8": (64, 256, 16),
            "res0": (96, 64, 32)}


def _gn_input(S3, C, groups, case, P, g):
    """fp16 [P, S3, C]: per (primitive, group) spread sigma and mean mu = ratio * sigma; 'constant': every group one value;
    'mixed': groups cycle through mean/spread 1000, centred, and constant within each primitive."""
    cpg = C // groups
    sigma = torch.exp(torch.randn(P, 1, groups, 1, generator=g, device=DEV, dtype=torch.float64) * 0.5)
    sign = torch.where(torch.rand(P, 1, groups, 1, generator=g, device=DEV) < 0.5, -1.0, 1.0).double()
    n = torch.randn(P, S3, groups, cpg, generator=g, device=DEV, dtype=torch.float64)
    const = (torch.randn(P, 1, groups, 1, generator=g, device=DEV, dtype=torch.float64) * 300).expand(P, S3, groups, cpg)
    if case == "constant":
        x = const
    elif case == "mixed":
        kind = torch.arange(groups, device=DEV)[None, None, :, None] % 3
        x = torch.where(kind == 0, sign * 1000 * sigma + sigma * n, torch.where(kind == 1, sigma * n, const))
    else:
        x = sign * float(case) * sigma + sigma * n
    return x.reshape(P, S3, C).half()


@pytest.mark.parametrize("case", ["0", "30", "300", "1000", "constant", "mixed"])
@pytest.mark.parametrize("path", list(GN_PATHS))
def test_groupnorm_statistics_robust_to_offsets(path, case):
    """GroupNorm(+SiLU) against fp64 on the same fp16 input, with group means up to 1000 standard deviations away from 0: max |error|
    <= 4e-3 (about two fp16 ulps) on outputs of magnitude <= 4, relative 1e-3 above."""
    S3, C, groups = GN_PATHS[path]
    P = 3
    g = torch.Generator(device=DEV).manual_seed(S3 * 7 + C + groups)
    x = _gn_input(S3, C, groups, case, P, g)
    gamma = (torch.randn(C, generator=g, device=DEV) * 0.1 + 1).half()
    beta = (torch.randn(C, generator=g, device=DEV) * 0.1).half()
    ref_n = F.group_norm(x.double().permute(0, 2, 1), groups, gamma.double(), beta.double(), eps=1e-5).permute(0, 2, 1)
    for silu in (0, 1):
        out = torch.empty_like(x)
        _lib.check(_lib.lib().tpx_groupnorm_silu(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), P, S3, C, groups, 1e-5, silu, out.data_ptr(), st()))
        ref = F.silu(ref_n) if silu else ref_n
        torch.cuda.synchronize()
        err = (out.double() - ref).abs()
        small = ref.abs() <= 4
        worst_small = float(err[small].max()) if bool(small.any()) else 0.0
        worst_large = float((err[~small] / ref[~small].abs()).max()) if bool((~small).any()) else 0.0
        print(f"{path} mean/std {case} silu {silu}: max |err| {worst_small:.2e} (|out| <= 4), max rel err {worst_large:.2e} (|out| > 4)")
        assert torch.isfinite(out).all()
        assert worst_small <= 4e-3 and worst_large <= 1e-3, (silu, worst_small, worst_large)
