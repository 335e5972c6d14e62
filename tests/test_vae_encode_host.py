"""CPU: the VAE encoder's host side — the oracle restatement against the reference's own encoder (tests/golden/vae_encode.npz), the
posterior mirror, the encoder's state_dict contract and checkpoint loading, the space-to-depth route of the stride-2 convolution,
the PrimX -> latent codec inverses, and the refusals without a GPU."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tpxl_b200
from oracle import vae as ov, vae_encode as ove
from tpxl_b200 import _lib, synth
from tpxl_b200.vae import DiagonalGaussianDistribution

SEED = 2027


@pytest.fixture(scope="module")
def fx(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "vae_encode.npz")))


@pytest.fixture(scope="module")
def full_sd():
    sd = synth.synth_state_dict(synth.vae_encoder_shapes(**synth.FULL_VAE), SEED)
    sd.update(synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), SEED + 2))
    return sd


def _rel(a, b):
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).norm() / torch.as_tensor(b).double().norm())


def test_oracle_encode_matches_the_reference_fixture(fx, full_sd):
    """oracle.vae_encode.encode at the fp32 policy reproduces the reference's stages (stored on a channel subset, rounded to fp16) and its
    parameters."""
    stages = {}
    with torch.no_grad():
        params = ove.encode(full_sd, torch.from_numpy(fx["x"]), "fp32", stages=stages)
    for name in ove.ENCODE_STAGES:
        ch = torch.from_numpy(fx["channels_" + name])
        assert len(ch) >= 8 and int(ch[0]) == 0
        assert _rel(stages[name][:, ch], fx["stage_" + name].astype(np.float32)) < 1e-3, name
    assert _rel(params, fx["parameters"]) < 1e-5
    assert params.shape == (8, 2, 4, 4, 4)


def test_posterior_mirror_matches_the_reference_posterior(fx):
    p = torch.from_numpy(fx["parameters"])
    post = DiagonalGaussianDistribution(p)
    assert torch.equal(post.mode(), torch.from_numpy(fx["mode"]))
    other = DiagonalGaussianDistribution(p.roll(1, 0))
    np.testing.assert_allclose(post.kl().numpy(), fx["kl"], rtol=1e-6)
    np.testing.assert_allclose(post.kl(other).numpy(), fx["kl_other"], rtol=1e-6)
    np.testing.assert_allclose(post.nll(torch.from_numpy(fx["nll_sample"])).numpy(), fx["nll"], rtol=1e-6)
    assert post.mean.shape == (8, 1, 4, 4, 4) and post.logvar.shape == (8, 1, 4, 4, 4)
    # the clamp, exp and deterministic branches
    q = torch.zeros(2, 2, 4, 4, 4)
    q[:, 1] = torch.tensor([-100.0, 100.0])[:, None, None, None]
    d = DiagonalGaussianDistribution(q)
    assert torch.equal(d.logvar[:, 0, 0, 0, 0], torch.tensor([-30.0, 20.0]))
    assert torch.equal(d.std, torch.exp(0.5 * d.logvar)) and torch.equal(d.var, torch.exp(d.logvar))
    det = DiagonalGaussianDistribution(q, deterministic=True)
    assert not det.std.any() and float(det.kl()) == 0.0 and float(det.nll(q[:, :1])) == 0.0
    torch.manual_seed(11)
    s = post.sample()
    torch.manual_seed(11)
    assert torch.equal(s, post.mean + post.std * torch.randn(post.mean.shape, dtype=p.dtype))


def test_encoder_shape_contract(golden_dir):
    keys = json.load(open(os.path.join(golden_dir, "state_dict_keys.json")))["vae"]
    want = {k: v for k, v in keys.items() if k.startswith(("encoder.", "quant_conv."))}
    assert {k: list(v) for k, v in synth.vae_encoder_shapes(**synth.FULL_VAE).items()} == want
    dec = {k: v for k, v in keys.items() if not k.startswith(("encoder.", "quant_conv."))}
    assert {k: list(v) for k, v in synth.vae_decoder_shapes(**synth.FULL_VAE).items()} == dec


def test_space_to_depth_route_is_the_stride_2_convolution():
    """Stride-2 / pad-1 Conv3d 8^3 -> 4^3 == stride-1 / pad-1 Conv3d at 4^3 over the space-to-depth input with the repacked weight, in
    fp64; the repacked weight is zero on every +1 block tap and on the phase-0 half of every -1 tap."""
    g = torch.Generator().manual_seed(4)
    x = torch.randn(3, 32, 8, 8, 8, generator=g, dtype=torch.float64)
    w = torch.randn(32, 32, 3, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(32, generator=g, dtype=torch.float64)
    want = F.conv3d(x, w, b, stride=2, padding=1)
    ws = ove.space_to_depth_weight(w)
    got = F.conv3d(ove.space_to_depth(x), ws, b, padding=1)
    assert float((got - want).abs().max()) < 1e-12
    assert not ws[..., 2, :, :].any() and not ws[..., :, 2, :].any() and not ws[..., :, :, 2].any()
    assert not ws.reshape(32, 2, 2, 2, 32, 3, 3, 3)[:, 0, :, :, :, 0].any()
    assert int((ws != 0).sum()) == w.numel()


def test_encode_needs_cuda_and_checks_its_inputs_in_order(full_sd):
    v = tpxl_b200.VAE(**synth.FULL_VAE)
    v.load_state_dict(full_sd)
    for bad in (torch.zeros(1), torch.zeros(2, 6, 8, 8, 8)):
        with pytest.raises(NotImplementedError, match="CUDA only"):
            v.encode(bad)
        with pytest.raises(NotImplementedError, match="CUDA only"):
            v(bad, sample=False)
        with pytest.raises(NotImplementedError, match="CUDA only"):
            v.debug_encode_stage(bad, 0)
    with pytest.raises(ValueError):
        v.debug_encode_stage(torch.zeros(1, 6, 8, 8, 8), 10)
    assert set(v.state_dict()) == set(full_sd)


def test_load_checkpoint_reads_the_encoder_only_when_asked(tmp_path, full_sd):
    path = os.path.join(tmp_path, "vae.pt")
    torch.save({"model_state_dict": full_sd}, path)
    v = tpxl_b200.VAE(**synth.FULL_VAE)
    v.load_checkpoint(path)
    assert not v._extra
    v.load_checkpoint(path, encoder=True)
    assert list(v._extra) == [k for k in full_sd if k.startswith(("encoder.", "quant_conv."))]
    assert torch.equal(v._extra["quant_conv.weight"], full_sd["quant_conv.weight"])
    assert set(v.state_dict()) == set(full_sd)


def test_codec_inverses_on_the_host():
    """unpack inverts pack (inference.py:343-346) and merge inverts split (inference.py:330, :335), with and without per-channel
    statistics, to within a few fp32 ulps."""
    g = torch.Generator().manual_seed(8)
    B, P = 2, 5
    srt = torch.rand(B, P, 4, generator=g)
    dec = torch.randn(B * P, 6, 8, 8, 8, generator=g)
    sample = torch.randn(B, P, 68, generator=g)
    for codec in (tpxl_b200.LatentCodec(synth.LATENT_MEAN, synth.LATENT_STD, 1.0), tpxl_b200.LatentCodec(None, None, 0.5)):
        packed = ov.pack_decoded(dec, B, P)
        s2 = srt.clone()
        if not codec.perchannel_norm:
            s2[..., 0:1] = s2[..., 0:1] / 10 + 0.05
        rs, rf = codec.unpack(torch.cat([s2, packed], -1))
        assert float((rf - dec).abs().max()) <= 4 * 2 ** -23 * (1 + float(dec.abs().max()))
        assert float((rs - srt).abs().max()) <= 16 * 2 ** -23
        if codec.perchannel_norm:
            srt_p, feat_p = ov.denormalise_latents(sample, torch.tensor(synth.LATENT_MEAN), torch.tensor(synth.LATENT_STD))
        else:
            srt_p, feat_p = sample[..., :4], sample[..., 4:] / 0.5
        back = codec.merge(srt_p, feat_p.reshape(B * P, 1, 4, 4, 4))
        assert back.shape == (B, P, 68)
        assert float((back - sample).abs().max()) <= 8 * 2 ** -23 * (1 + float(sample.abs().max()) * 8)
    with pytest.raises(ValueError):
        codec.unpack(torch.zeros(1, 2, 3))


def test_posterior_resolves_under_the_reference_path():
    tpxl_b200.install()
    from models.vae3d_dib import DiagonalGaussianDistribution as D, VAE
    assert D is DiagonalGaussianDistribution and VAE is tpxl_b200.VAE


def test_encoder_entries_check_arguments_before_the_device():
    """The encoder handle's entries refuse bad arguments without touching a device; creation stops at the device guard."""
    if torch.cuda.is_available():
        pytest.skip("checks the no-device path")
    lib = _lib.load_library()
    cfg = _lib.VaeConfig(1, 6, 256, 32, 8)
    h = ctypes.c_void_p()
    assert lib.tpx_vae_encoder_create(ctypes.byref(cfg), ctypes.byref(h)) == -2 and b"cudaGetDevice" in lib.tpx_last_error()
    bad = _lib.VaeConfig(1, 6, 128, 32, 8)
    assert lib.tpx_vae_encoder_create(ctypes.byref(bad), ctypes.byref(h)) < 0 and b"down_channels" in lib.tpx_last_error()
    P = 1 << 20
    assert lib.tpx_vae_encoder_workspace_bytes(None, 4) == 0
    assert lib.tpx_vae_encode(None, P, 0, P, 0, 1, P, 1 << 30, None) == -1 and b"null" in lib.tpx_last_error()
    assert lib.tpx_vae_encode_debug_stage(None, P, 0, 1, 0, P, P, 1 << 30, None) == -1
    assert lib.tpx_vae_encoder_finalize(None, None) == -1
