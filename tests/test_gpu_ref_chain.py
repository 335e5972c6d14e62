"""GPU: the first and last stages of the image-to-SDF path against THE REFERENCE'S OWN MODULES on the same H100 — the DINOv2 image
conditioner, the chain image -> y -> DDIM-25 -> glue -> VAE.decode -> recon_param at the shipped architecture, and the PrimSDF query on
the primitives that chain produces.  The modules are the byte-identical staged copies under oracle/_ref (oracle/stage_ref.py; loaders
oracle/refmods.py build_dinov2 / build_primsdf / build_dit / build_vae).  Weights are synthetic.

Precision settings of the reference runs:
    ref32      fp32, TF32 off for matmul and cuDNN                                  the exact-fp32 yardstick
    ref_tf32   fp32, TF32 on for matmul and cuDNN and cuDNN autotuning on, as inference.py:377-380 sets them (not torch's defaults)
    ref16      torch.autocast('cuda', fp16)                                         the reference's own fp16 path

a. Encoder.  ours, ref16 and ref_tf32 against ref32 on the fixture's 518 x 518 picture, the same picture as inference.py:306-311 builds
   it (uint8 RGB times an int64 mask: int64, background zero), a 224 x 224 picture (the Resize path) and a batch of three, for
   synth_weights(105) and the stage suite's hard draw.  Asserted: the stage suites' rule (tests/parity.py) with ref16 as the policy and
   ref32 as exact, per image, per (image, 128-token block) and on the class-token row, and the worst output channel <= 6e-3 of ref32.
   The same rule per channel does not hold: the encoder's documented fp16 policy is itself further from fp32 than autocast on a few
   channels (DESIGN.md section 2), so that partition alone is a strict xfail until the contract is decided.  Every reference block is
   hooked and set against our (i, "res2") tap, so a message names the first block whose residual leaves the rule.  The rule rejects 1 %
   errors on one channel, one block of the second image or the class token of the reference's TF32 run.
b. Chain.  The masked int64 picture -> y -> DDIM-25 (v, squaredcos_cap_v2, CFG 6, clip_denoised=False) from a seeded x_T -> the released
   glue (per-channel statistics, latent_nf 1.0) -> VAE.decode -> recon_param at the steps inference.py decodes (0, 10, 20, 24):
       R     reference conditioner ref_tf32, reference DiT under autocast, reference VAE ref_tf32     (as inference.py)
       R32   reference conditioner ref32, DiT fp32, VAE fp32, TF32 off everywhere
       Rc16  reference conditioner under autocast, DiT under autocast, VAE fp32 (TF32 off)
       O     ours throughout (Dinov2Wrapper, DiT, sampler, PrimXPipeline.decode_latents)
       O_y   R's y, then ours (separates the conditioner's share from the DiT's)
   Rules: rel(X, R32) <= 1.25 x rel(Rc16, R32) and rel(X, R) <= 1.5 x max(rel(R, R32), rel(Rc16, R32)) (two independent fp16
   perturbations: sqrt 2 expected).  Asserted: both for O and O_y at all 25 samples, the final sample within 1e-2 of R, every tensor
   finite and every recon_param's shape, both for O_y on recon_param's srt part at every decoded step and for O where it was measured
   within them, and the feature part against the decoder's own contract at R32's latents (VAE.decode as tests/test_gpu_ref_fp16.py holds
   it).  Strict xfails, one per (part, step) measured outside: O's srt part at steps 10, 20 and 24 (the encoder's policy; O_y is within) and O's
   feature part at every step (our decoder is fp16 by contract, Rc16's fp32).
c. PrimSDF.  Our query against the reference module on R's recon_param (K = 2048) and test_gpu_primsdf_grad's _random scene: on
   inference.py:107-116's grid at resolution 128 in its 8192-point chunks and on random points inside and outside the primitives, eval and
   train, and PrimSDF.sdf_grid(128).  Values within 2e-5 (rtol and atol); at most 1 % of sdf values may differ, each at an fp32 tie.
   The backward (differentiable=True) against the reference's CUDA autograd for grad_x, grad_srt, grad_feat: relative L2 <= 1e-4 and
   cosine >= 1 - 1e-6; uncovered tied points get no upstream gradient.
"""
import contextlib
import importlib
import time

import numpy as np
import pytest
import torch

import parity
import tpxl_b200
from gpu_util import rel_l2
from oracle import dinov2 as odn
from oracle import refmods
from oracle import vae as ovae
from oracle.dit import Policy
from pictures import golden_picture, masked_picture, small_picture
from test_gpu_dinov2_stages import _hard_weights
from test_gpu_primsdf_grad import _random
from tpxl_b200 import synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (refmods.available() and refmods.conditioner_available() and refmods.primsdf_available()),
                                                  reason="the reference's modules are not staged (python oracle/stage_ref.py where the reference checkout exists)")]
DEV = torch.device("cuda:0")
dn = importlib.import_module("tpxl_b200.dinov2")
CHANNEL_BOUND = 6e-3                   # worst output channel against exact fp32 (the stage suite's end-to-end bound)
NTOK = 1370
PARTS = {"image": parity.sequence, "block": parity.block(128), "channel": parity.channel,
         "class": parity.tokens(torch.tensor([0] + [-1] * (NTOK - 1)))}
BLOCK_PARTS = {h: PARTS[h] for h in ("image", "block", "channel")}      # a block's residual also holds the four register rows
KW16 = dict(precision_dtype=torch.float16, enable_amp=True)
DIFF = dict(noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
DECODED = (0, 10, 20, 24)              # the steps inference.py:326-328 decodes and renders for 25 steps
PRIM_TOL = dict(rtol=2e-5, atol=2e-5)


@contextlib.contextmanager
def _precision(tf32, benchmark=False):
    """TF32 for matmul and cuDNN, and cuDNN autotuning, for the duration of the block; inference.py:377-380 sets all three."""
    b = torch.backends
    old = b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32, b.cudnn.benchmark
    b.cuda.matmul.allow_tf32 = b.cudnn.allow_tf32 = tf32
    b.cudnn.benchmark = benchmark
    try:
        yield
    finally:
        b.cuda.matmul.allow_tf32, b.cudnn.allow_tf32, b.cudnn.benchmark = old


# ---- a. the encoder ---------------------------------------------------------------------------------------------------------------
def _pictures():
    img = golden_picture(1105)
    masked = masked_picture(img)
    return {"fixture fp32": torch.from_numpy(img), "masked int64": torch.from_numpy(masked), "224 resize": torch.from_numpy(small_picture(img)),
            "batch of three": torch.from_numpy(np.concatenate([img, masked.astype(np.float32), np.ascontiguousarray(img[:, :, ::-1])], 0))}


_ENC = {}


def _encoders(weights):
    """(reference Dinov2Wrapper, ours, fp64 state dict) on the GPU."""
    if weights not in _ENC:
        sd = odn.synth_weights(105) if weights == "synth" else _hard_weights()
        ours = dn.Dinov2Wrapper()
        ours.load_state_dict(sd)
        _ENC[weights] = (refmods.build_dinov2(sd, DEV), ours.to(DEV).eval(), {k: v.to(DEV, torch.float64) for k, v in sd.items()})
    return _ENC[weights]


def run_reference(enc, img, how, blocks=None):
    """The reference conditioner on img under how = "32" / "tf32" / "16" -> fp32 [n, 1370, 768]; blocks (a list) receives every block's
    output [n, 1374, 768] when given."""
    hooks = [] if blocks is None else [b.register_forward_hook(lambda m, i, o: blocks.append(o.float().clone())) for b in enc.model.blocks]
    try:
        with torch.no_grad(), _precision(how == "tf32", benchmark=how == "tf32"):
            if how == "16":
                with torch.autocast("cuda", dtype=torch.float16):
                    return enc(img).float()
            return enc(img).float()
    finally:
        for h in hooks:
            h.remove()


def _encoder_runs(weights, name):
    ref, ours, sd64 = _encoders(weights)
    img = _pictures()[name].to(DEV)
    b32, b16 = [], []
    r32, r16, rtf = run_reference(ref, img, "32", b32), run_reference(ref, img, "16", b16), run_reference(ref, img, "tf32")
    taps = {}
    with torch.no_grad():
        o = ours._forward(img, taps)
        o16 = odn.forward(sd64, img.double(), pol=Policy("fp16"))
    return dict(ours=o.double(), ref16=r16.double(), ref32=r32.double(), ref_tf32=rtf.double(), oracle16=o16,
                blocks=[(taps[(i, "res2")].double(), b16[i].double(), b32[i].double()) for i in range(12)])


PICTURES = ["fixture fp32", "masked int64", "224 resize", "batch of three"]
ASSERTED_PARTS = {h: PARTS[h] for h in ("image", "block", "class")}


@pytest.mark.parametrize("name", PICTURES)
@pytest.mark.parametrize("weights", ["synth", "hard"])
def test_encoder_against_the_reference(weights, name):
    """The four figures and every block against ref32; the rule against autocast per image, (image, 128-token block) and on the class
    token; the worst output channel within 6e-3 of ref32."""
    r = _encoder_runs(weights, name)
    o, r16, r32 = r["ours"], r["ref16"], r["ref32"]
    assert o.shape == r32.shape == (len(r32), NTOK, 768)
    assert all(bool(torch.isfinite(t).all()) for t in (o, r16, r32, r["ref_tf32"]))
    tag = f"[ref-chain] encoder {weights:5s} {name:14s}"
    print(f"{tag}: ours_vs_ref16={rel_l2(o, r16):.3e} oracle16_vs_ref16={rel_l2(r['oracle16'], r16):.3e} ref16_vs_ref32={rel_l2(r16, r32):.3e} "
          f"ours_vs_ref32={rel_l2(o, r32):.3e} ref_tf32_vs_ref32={rel_l2(r['ref_tf32'], r32):.3e}")
    for i, (ob, pb, eb) in enumerate(r["blocks"]):
        o_i, p_i = parity.ratios(ob, pb, eb, parity.channel)
        print(f"{tag} block {i:2d}: ours_vs_ref32 {rel_l2(ob, eb):.3e}  ref16_vs_ref32 {rel_l2(pb, eb):.3e}  worst channel ours {float(o_i.max()):.2e} "
              f"ref16 {float(p_i.max()):.2e}{'' if not parity.rejects(ob, pb, eb, BLOCK_PARTS) else '  outside the rule'}")
    oo, pp = parity.ratios(o, r16, r32, PARTS["channel"])
    print(f"{tag}: rule against ref16, channel (not asserted here): worst ours / bound {float((oo / parity.bound(pp)).max()):.2f}")
    first = next((i for i, (ob, pb, eb) in enumerate(r["blocks"]) if parity.rejects(ob, pb, eb, {"image": PARTS["image"], "block": PARTS["block"]})), None)
    worst = parity.check(f"{tag} (first block outside the image / block rule: {first})", o, r16, r32, ASSERTED_PARTS)
    print(f"{tag}: rule against ref16: worst ours / bound " + ", ".join(f"{h} {v:.2f}" for h, v in worst.items()))
    per_ch = (o - r32).norm(dim=(0, 1)) / r32.norm(dim=(0, 1))
    per_ch16 = (r16 - r32).norm(dim=(0, 1)) / r32.norm(dim=(0, 1))
    print(f"{tag}: worst channel {float(per_ch.max()):.2e} (ref16 {float(per_ch16.max()):.2e}), bound {CHANNEL_BOUND:.0e}")
    assert float(per_ch.max()) <= CHANNEL_BOUND, (int(per_ch.argmax()), float(per_ch.max()))


@pytest.mark.xfail(strict=True, reason="the encoder's fp16 policy (oracle.dinov2 Policy('fp16'), which the kernels follow: oracle16_vs_ref16 "
                                       "equals ours_vs_ref16) is further from fp32 than autocast on a few output channels, from block 0 on "
                                       "(DESIGN.md section 2); whether to change that contract is a separate decision")
@pytest.mark.parametrize("name", PICTURES)
@pytest.mark.parametrize("weights", ["synth", "hard"])
def test_encoder_channel_rule_against_autocast(weights, name):
    """The rule against autocast per channel alone; the message names the first block whose residual leaves it."""
    r = _encoder_runs(weights, name)
    first = next((i for i, (ob, pb, eb) in enumerate(r["blocks"]) if parity.rejects(ob, pb, eb, {"channel": PARTS["channel"]})), None)
    parity.check(f"encoder {weights} {name} (first block outside the channel rule: {first})", r["ours"], r["ref16"], r["ref32"],
                 {"channel": PARTS["channel"]})


def test_encoder_rule_rejects_one_percent_errors():
    """On the batch of three (synth weights), the reference's TF32 run passes the rule against autocast, and a 1 % error in it on one
    channel, on one 128-token block of the second image or on the class token fails it."""
    r = _encoder_runs("synth", "batch of three")
    o, r16, r32 = r["ref_tf32"], r["ref16"], r["ref32"]
    assert not parity.rejects(o, r16, r32, PARTS)
    for what, how, region in (("channel 517", "channel", (slice(None), slice(None), 517)), ("tokens 640-767 of image 1", "block", (1, slice(640, 768))),
                              ("class token", "class", (slice(None), 0))):
        bad = o.clone()
        bad[region] *= 1.01
        oo, pp = parity.ratios(bad, r16, r32, PARTS[how])
        print(f"[ref-chain] 1 % on {what}: worst {how} partition at {float((oo / parity.bound(pp)).max()):.1f} x the bound")
        assert parity.rejects(bad, r16, r32, {how: PARTS[how]}), what


# ---- b. the chain -----------------------------------------------------------------------------------------------------------------
def _loop(diff, fwd, x_T, y, kw):
    mk = dict(y=y, cfg_scale=6.0, **kw)
    return [s["sample"].clone() for s in diff.ddim_sample_loop_progressive(fwd, x_T.shape, x_T, clip_denoised=False, model_kwargs=mk,
                                                                          progress=False, device=DEV)]


@pytest.fixture(scope="module")
def chain():
    """{"y", "samples", "recon"} per chain name; recon maps each decoded step to recon_param [1, 2048, 3076]."""
    t0 = time.time()
    img = _pictures()["masked int64"].to(DEV)
    esd = odn.synth_weights(105)
    ref_enc = refmods.build_dinov2(esd, DEV)
    our_enc = dn.Dinov2Wrapper()
    our_enc.load_state_dict(esd)
    our_enc = our_enc.to(DEV).eval()
    y = {"R": run_reference(ref_enc, img, "tf32"), "R32": run_reference(ref_enc, img, "32"), "Rc16": run_reference(ref_enc, img, "16")}
    with torch.no_grad():
        y["O"] = our_enc(img)
    y["O_y"] = y["R"]
    del ref_enc, our_enc

    dsd = synth.device_state_dict(synth.dit_shapes(**synth.FULL_DIT), 241, DEV, torch.float16)
    ref_dit = refmods.build_dit(synth.FULL_DIT, dsd, DEV)
    our_dit = tpxl_b200.DiT(**{k: v for k, v in synth.FULL_DIT.items() if k != "gradient_checkpointing"})
    our_dit.load_state_dict(dsd)
    our_dit = our_dit.to(DEV).eval()
    del dsd
    vsd = synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 242)
    ref_vae = refmods.build_vae(synth.FULL_VAE, vsd, DEV)
    our_vae = tpxl_b200.VAE(**synth.FULL_VAE)
    our_vae.load_state_dict(vsd)
    our_vae = our_vae.to(DEV)
    pipe = tpxl_b200.PrimXPipeline(our_dit, our_vae, latent_mean=synth.LATENT_MEAN, latent_std=synth.LATENT_STD, latent_nf=1.0)
    mean = torch.Tensor(synth.LATENT_MEAN)[None, None, :].to(DEV)           # inference.py:291-293
    std = torch.Tensor(synth.LATENT_STD)[None, None, :].to(DEV)
    x_T = torch.randn(1, 2048, 68, generator=torch.Generator(device=DEV).manual_seed(243), device=DEV)

    rdiff = refmods.load().create_diffusion("ddim25", **DIFF)
    odiff = tpxl_b200.create_diffusion("ddim25", **DIFF)
    samples, recon = {}, {}
    with torch.no_grad():
        for name, tf32, kw in (("R", True, KW16), ("R32", False, dict(precision_dtype=torch.float32, enable_amp=False)), ("Rc16", False, KW16)):
            with _precision(tf32, benchmark=tf32):
                samples[name] = _loop(rdiff, ref_dit.forward_with_cfg, x_T, y[name], kw)
                recon[name] = {k: ovae.inference_glue(samples[name][k], ref_vae.decode, mean, std, 1.0, True) for k in DECODED}
        for name in ("O", "O_y"):
            samples[name] = _loop(odiff, our_dit.forward_with_cfg, x_T, y[name], KW16)
            recon[name] = {k: pipe.decode_latents(samples[name][k]) for k in DECODED}
        # the decoder alone on R32's latents: ours, and the reference's under autocast (its fp32 decode is recon["R32"])
        with _precision(False):
            decoder = {"ours": {k: pipe.decode_latents(samples["R32"][k]) for k in DECODED}}
            def decode16(z):                                                   # the decoder under autocast, the glue in fp32
                with torch.autocast("cuda", dtype=torch.float16):
                    out = ref_vae.decode(z)
                return out.float()
            decoder["ref16"] = {k: ovae.inference_glue(samples["R32"][k], decode16, mean, std, 1.0, True) for k in DECODED}
    torch.cuda.synchronize()
    print(f"[ref-chain] five chains in {time.time() - t0:.0f} s")
    del ref_dit, our_dit, ref_vae, our_vae, pipe
    torch.cuda.empty_cache()
    return {"y": y, "samples": samples, "recon": recon, "decoder": decoder}


CHAINS = ("R", "R32", "Rc16", "O", "O_y")
# (part, decoded step) where O was measured outside the chain rules (DESIGN.md section 2): the srt part at steps 10, 20 and 24 (the encoder's policy:
# O_y meets both rules there), the feature part at every step (our decoder computes in fp16 by contract, Rc16's in fp32)
O_OUTSIDE = (("srt", 10), ("srt", 20), ("srt", 24), ("feat", 0), ("feat", 10), ("feat", 20), ("feat", 24))


def _rules(tag, get):
    """get(chain name) -> tensor.  All five finite; prints the figures.  -> {who: (rel(who, R32) / (1.25 rel(Rc16, R32)),
    rel(who, R) / (1.5 max(rel(R, R32), rel(Rc16, R32))))} for who in O, O_y: both rules hold where both are <= 1."""
    t = {n: get(n).double() for n in CHAINS}
    for n in CHAINS:
        assert bool(torch.isfinite(t[n]).all()), (tag, n)
    f = {f"{a}_{b}": rel_l2(t[a], t[b]) for a, b in (("O", "R32"), ("Rc16", "R32"), ("R", "R32"), ("O", "R"), ("O_y", "R"), ("O_y", "R32"))}
    b1, b2 = 1.25 * f["Rc16_R32"], 1.5 * max(f["R_R32"], f["Rc16_R32"])
    used = {w: (f[f"{w}_R32"] / b1, f[f"{w}_R"] / b2) for w in ("O", "O_y")}
    print(f"[ref-chain] {tag:16s} " + "  ".join(f"{k}={v:.3e}" for k, v in f.items()) +
          "   used " + ", ".join(f"{w} {a:.2f} / {b:.2f}" for w, (a, b) in used.items()) + " of the bounds")
    return used, f


def test_conditioning_tokens(chain):
    """y itself: the encoder figures on the picture the chain feeds (its rule is asserted per partition in a.)."""
    y = chain["y"]
    print("[ref-chain] y: " + "  ".join(f"{n}_vs_R32={rel_l2(y[n].double(), y['R32'].double()):.3e}" for n in ("R", "Rc16", "O")))
    assert all(bool(torch.isfinite(t).all()) for t in y.values())


def test_chain_samples_every_step(chain):
    """Both rules for O and for O_y at every one of the 25 samples; the final sample of O within 1e-2 of R."""
    s = chain["samples"]
    assert all(len(v) == 25 for v in s.values())
    for k in range(25):
        used, f = _rules(f"sample step {k:2d}", lambda n: s[n][k])
        assert max(used["O"]) <= 1 and max(used["O_y"]) <= 1, (k, used, f)
    assert f["O_R"] < 1e-2, f


def test_chain_recon_param(chain):
    """Every recon_param of every chain (and of the decoder runs) has its shape and is finite; at every decoded step both rules hold for
    O_y on the srt part, and for O on the srt part wherever O_OUTSIDE does not list the step.  The feature part (our decoder is fp16 by
    contract) is held to the decoder's contract at the chain's own latents, R32's: ours against the reference's fp32 and autocast decodes
    as tests/test_gpu_ref_fp16.py holds VAE.decode."""
    rc, dec = chain["recon"], chain["decoder"]
    for runs in (rc, dec):
        for n, steps in runs.items():
            assert set(steps) == set(DECODED), n
            for k, t in steps.items():
                assert t.shape == (1, 2048, 4 + 6 * 512) and t.dtype == torch.float32, (n, k, tuple(t.shape), t.dtype)
                assert bool(torch.isfinite(t).all()), (n, k)
    failed = []                                     # every step is measured and printed before any verdict
    for k in DECODED:
        used, f = _rules(f"recon {k:2d} srt", lambda n: rc[n][k][..., :4])
        if max(used["O_y"]) > 1:
            failed.append((k, "O_y srt", used))
        if ("srt", k) not in O_OUTSIDE and max(used["O"]) > 1:
            failed.append((k, "O srt", used))
        _rules(f"recon {k:2d} feat", lambda n: rc[n][k][..., 4:])
        o, r32, r16 = dec["ours"][k][..., 4:].double(), rc["R32"][k][..., 4:].double(), dec["ref16"][k][..., 4:].double()
        d = dict(ours_vs_ref32=rel_l2(o, r32), ours_vs_ref16=rel_l2(o, r16), ref16_vs_ref32=rel_l2(r16, r32))
        print(f"[ref-chain] decoder {k:2d} feat  " + "  ".join(f"{a}={v:.3e}" for a, v in d.items()))
        if not (d["ours_vs_ref32"] < max(1e-3, 1.5 * d["ref16_vs_ref32"]) and d["ours_vs_ref32"] < 5e-3
                and d["ours_vs_ref16"] < max(1e-3, 1.5 * d["ref16_vs_ref32"])):
            failed.append((k, "decoder feat", d))
        if not rel_l2(dec["ours"][k][..., :4], rc["R32"][k][..., :4]) < 1e-6:      # the same latents: the srt glue alone
            failed.append((k, "decoder srt", rel_l2(dec["ours"][k][..., :4], rc["R32"][k][..., :4])))
    srt = rc["R"][24][0, :, :4]
    print(f"[ref-chain] R's final primitives: scale in [{float(srt[:, 0].min()):.3f}, {float(srt[:, 0].max()):.3f}], "
          f"{int((srt[:, 0] <= 0).sum())} not positive; centres in [{float(srt[:, 1:].min()):.2f}, {float(srt[:, 1:].max()):.2f}]")
    assert not failed, failed


@pytest.mark.xfail(strict=True, reason="measured outside the rules (DESIGN.md section 2): the srt part at steps 10, 20 and 24 through the encoder's fp16 "
                                       "policy, the feature part because our VAE.decode computes in fp16 by contract and Rc16's in fp32")
@pytest.mark.parametrize("part,step", O_OUTSIDE)
def test_chain_recon_param_outside_the_rules(chain, part, step):
    rc = chain["recon"]
    sl = slice(0, 4) if part == "srt" else slice(4, None)
    used, f = _rules(f"recon {step:2d} {part}", lambda n: rc[n][step][..., sl])
    assert max(used["O"]) <= 1, (step, part, used, f)


# ---- c. PrimSDF ---------------------------------------------------------------------------------------------------------------------
def _scene(name, chain):
    if name == "recon R":
        rp = chain["recon"]["R"][24][0].float()
        srt, feat = rp[:, :4], rp[:, 4:]
    else:
        srt, feat, _, _ = _random(2048, 8, 8, 51)
    return srt.contiguous().to(DEV), feat.contiguous().to(DEV)


def _points(srt, n, seed):
    """Half inside a primitive's box (its centre + |scale| x uniform(-1, 1)^3), half uniform in [-1.3, 1.3]^3."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    k = torch.randint(0, srt.shape[0], (n // 2,), generator=g, device=DEV)
    inside = srt[k, 1:4] + srt[k, :1].abs() * (torch.rand(n // 2, 3, generator=g, device=DEV) * 2 - 1)
    return torch.cat([inside, torch.rand(n - n // 2, 3, generator=g, device=DEV) * 2.6 - 1.3])


def _grid_points(R=128):
    xx = torch.linspace(-1, 1, R, device=DEV)                                # inference.py:108-109
    return torch.stack(torch.meshgrid(xx, xx, xx, indexing="ij"), dim=-1).reshape(-1, 3)


def _ours(srt, feat, train, **kw):
    m = tpxl_b200.PrimSDF(num_prims=srt.shape[0], dim_feat=6, prim_shape=8, **kw).train(train)
    m.srt_param.data = srt.clone()
    m.feat_param.data = feat.clone()
    m.srt_param.requires_grad_(True)
    m.feat_param.requires_grad_(True)
    return m.to(DEV)


def _query(m, pts, chunk=8192):
    with torch.no_grad():
        outs = [m(c) for c in torch.split(pts, chunk)]                       # inference.py:110-114
    return {k: torch.cat([o[k] for o in outs]) for k in ("sdf", "tex", "mat")}


def _same_query(tag, x, ours, ref, srt):
    """tex / mat within PRIM_TOL; sdf within it except at <= 1 % of the points, each an fp32 tie."""
    for k in ("tex", "mat"):
        torch.testing.assert_close(ours[k], ref[k], **PRIM_TOL, msg=lambda m: f"{tag} {k}: {m}")
    bad = ~torch.isclose(ours["sdf"], ref["sdf"], **PRIM_TOL)[:, 0]
    nbad = int(bad.sum())
    ties = parity.fp32_ties(x[bad].double(), srt.double(), 8)
    err = float((ours["sdf"] - ref["sdf"]).abs().max())
    print(f"[ref-chain] {tag}: {x.shape[0]} points, sdf max |diff| {err:.2e}, {nbad} off (all fp32 ties: {bool(ties.all())}), "
          f"tex {float((ours['tex'] - ref['tex']).abs().max()):.2e}, mat {float((ours['mat'] - ref['mat']).abs().max()):.2e}")
    assert nbad <= 0.01 * x.shape[0], (tag, nbad)
    assert bool(ties.all()), (tag, x[bad][~ties][:4].tolist(), ours["sdf"][bad][~ties][:4].tolist(), ref["sdf"][bad][~ties][:4].tolist())


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("scene", ["recon R", "random"])
def test_primsdf_forward_against_the_reference(chain, scene, mode):
    srt, feat = _scene(scene, chain)
    train = mode == "train"
    ref = refmods.build_primsdf(srt, feat, DEV).train(train)
    m = _ours(srt, feat, train)
    grid = _grid_points()
    ours_g, ref_g = _query(m, grid), _query(ref, grid)
    _same_query(f"{scene} {mode} grid 128^3", grid, ours_g, ref_g, srt)
    with torch.no_grad():
        sg = m.sdf_grid(128)
    assert sg.shape == (128, 128, 128) and torch.equal(sg.reshape(-1, 1), ours_g["sdf"]), "sdf_grid differs from forward over the grid"
    x = _points(srt, 200000, 52 + train)
    _same_query(f"{scene} {mode} random points", x, _query(m, x), _query(ref, x), srt)


GRADS = ("grad_x", "grad_srt", "grad_feat")


@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("scene", ["recon R", "random"])
def test_primsdf_backward_against_the_reference_autograd(chain, scene, mode):
    """n = 32768 points: the reference's dense [n, K, 3] intermediates are 0.8 GB each under its autograd."""
    srt, feat = _scene(scene, chain)
    train = mode == "train"
    n = 32768
    x = _points(srt, n, 61 + train)
    G = torch.randn(n, 6, generator=torch.Generator(device=DEV).manual_seed(62), device=DEV)
    if not train:
        xd, sd = x.double(), srt.double()
        covered = ((1 - ((xd[:, None] - sd[None, :, 1:4]) / sd[None, :, :1]).abs().amax(-1)) > 0).any(1)
        tie = torch.zeros(n, dtype=torch.bool, device=DEV)
        tie[~covered] = parity.fp32_ties(xd[~covered], sd, 8)
        G[tie] = 0
        print(f"[ref-chain] {scene} eval backward: {int((~covered).sum())} uncovered points, {int(tie.sum())} fp32 ties without upstream gradient")
    got, want = {}, {}
    for who, m in (("ours", _ours(srt, feat, train, differentiable=True)), ("ref", refmods.build_primsdf(srt, feat, DEV).train(train))):
        xx = x.clone().requires_grad_(True)
        o = m(xx)
        torch.cat([o["sdf"], o["tex"], o["mat"]], 1).backward(G)
        (got if who == "ours" else want).update(zip(GRADS, (xx.grad, m.srt_param.grad, m.feat_param.grad)))
    for k in GRADS:
        a, b = got[k].double().flatten(), want[k].double().flatten()
        rel, cos = float((a - b).norm() / b.norm()), float(a @ b / (a.norm() * b.norm()))
        print(f"[ref-chain] {scene} {mode} {k}: rel-L2 {rel:.2e}  1-cos {1 - cos:.2e}")
        assert rel <= 1e-4 and cos >= 1 - 1e-6, (scene, mode, k, rel, cos)
