"""GPU: the sampling loop through the reference-facing generator API against the oracle loop, and size-independent
properties at the shipped size."""
import pytest
import torch

import oracle
import tpxl_b200
from tpxl_b200 import synth
from gpu_util import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CFG = dict(seq_length=256, in_channels=68, condition_channels=768, hidden_size=384, depth=2, num_heads=16, attn_proj_bias=True, cond_drop_prob=0.1)


def _setup(seed=51):
    sd = synth.synth_state_dict(synth.dit_shapes(**CFG), seed)
    m = tpxl_b200.DiT(**CFG)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    x, y = synth.synth_inputs(2, 256, 68, 64, 768, seed + 1)
    return sd, m, x.to(DEV), y.to(DEV)


@pytest.mark.parametrize("ddim", [True, False])
def test_sampling_loop_matches_oracle(ddim):
    sd, m, x, y = _setup()
    respacing = "ddim25" if ddim else "10"
    d = tpxl_b200.create_diffusion(respacing, noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
    kw = dict(y=y, cfg_scale=6.0, precision_dtype=torch.float16, enable_amp=True)
    fn = d.ddim_sample_loop_progressive if ddim else d.p_sample_loop_progressive
    torch.manual_seed(3)
    ours = [o for o in fn(m.forward_with_cfg, x.shape, x, clip_denoised=False, model_kwargs=kw, progress=False, device=DEV)]
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    s = oracle.diffusion.Schedule(respacing)
    torch.manual_seed(3)
    ref = list(oracle.diffusion.sample_loop(s, lambda xx, tt: oracle.dit.forward_with_cfg(sdd, xx, tt, y, 6.0, 16, "fp16"), x, ddim=ddim,
                                            step_noise=torch.randn_like))
    assert len(ours) == len(ref) == d.num_timesteps
    assert set(ours[0]) == {"sample", "pred_xstart"} and ours[0]["sample"].dtype == torch.float32
    errs = [rel_l2(a["sample"], b["sample"]) for a, b in zip(ours, ref)]
    print("per-step rel-L2:", ["%.1e" % e for e in errs])
    assert max(errs) < 5e-3 and rel_l2(ours[-1]["pred_xstart"], ref[-1]["pred_xstart"]) < 5e-3


def test_reference_style_sampler_can_drive_the_model():
    """The DiT also has to work under a sampler that maps timesteps itself and passes device tensors (respace.py:124-129)."""
    sd, m, x, y = _setup(53)
    d = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v")
    tmap = torch.tensor(d.timestep_map, device=DEV)
    ts = torch.tensor([24, 24], device=DEV)
    with torch.no_grad():
        a = m.forward_with_cfg(x, tmap[ts], y, cfg_scale=6.0, enable_amp=True)
        b = m.forward_with_cfg(x, torch.tensor([960, 960], device=DEV), y, cfg_scale=6.0, enable_amp=True)
    assert torch.equal(a, b)


def test_conditioning_cache_tracks_tensor_identity_and_version():
    sd, m, x, y = _setup(55)
    t = torch.tensor([480, 480], device=DEV)
    with torch.no_grad():
        a = m.forward_with_cfg(x, t, y, cfg_scale=3.0, enable_amp=True).clone()
        y2 = y.clone()
        b = m.forward_with_cfg(x, t, y2, cfg_scale=3.0, enable_amp=True).clone()
        y2.mul_(0.5)                                     # in-place edit bumps the version counter -> K/V recomputed
        c = m.forward_with_cfg(x, t, y2, cfg_scale=3.0, enable_amp=True).clone()
        e = m.forward_with_cfg(x, t, y, cfg_scale=0.0, enable_amp=True)      # cfg_scale 0 -> pure unconditional branch
        f = m.forward_with_cfg(x, t, y2, cfg_scale=0.0, enable_amp=True)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert torch.equal(e, f)


def test_conditioning_cache_survives_address_reuse_between_requests():
    """app.py:108-131: every request builds a fresh function-local y against a module-level model.  After request 1's y is
    freed the caching allocator hands the SAME address to request 2's y (same shape, version 0) — the hoisted K/V must still be
    recomputed.  The cache holds a strong reference to the tensor it was computed from, so the address cannot be recycled."""
    sd, m, x, _ = _setup(57)
    t = torch.tensor([480, 480], device=DEV)
    g = torch.Generator(device=DEV).manual_seed(58)
    with torch.no_grad():
        y1 = torch.randn(2, 77, 768, generator=g, device=DEV)
        vals2 = torch.randn(2, 77, 768, generator=g, device=DEV).cpu()
        m.forward_with_cfg(x, t, y1, cfg_scale=3.0, enable_amp=True)
        p1 = y1.data_ptr()
        del y1                                             # request 1 returns: its y dies
        y2 = torch.empty(2, 77, 768, device=DEV)           # request 2: the allocator would reuse the freed block if nothing held it
        y2.copy_(vals2)
        reused = y2.data_ptr() == p1
        got = m.forward_with_cfg(x, t, y2, cfg_scale=3.0, enable_amp=True).clone()
        fresh = tpxl_b200.DiT(**CFG)
        fresh.load_state_dict(sd)
        fresh = fresh.to(DEV).eval()
        want = fresh.forward_with_cfg(x, t, y2, cfg_scale=3.0, enable_amp=True)
    print("address reused by the allocator:", reused)
    assert not reused                                      # the cached tensor is held alive, so its block was not handed out again
    assert torch.equal(got, want)
    # and the situation the bug needs — same address, same shape, version 0, different values — as a direct check
    with torch.no_grad():
        m._cond_ref = None                                 # drop the strong reference (what round 1 effectively did) ...
        y3 = torch.empty(2, 77, 768, device=DEV)
        y3.copy_(vals2 * 0.5)
        got3 = m.forward_with_cfg(x, t, y3, cfg_scale=3.0, enable_amp=True)     # ... a cache without a live reference never hits
        want3 = fresh.forward_with_cfg(x, t, y3, cfg_scale=3.0, enable_amp=True)
    assert torch.equal(got3, want3)


def test_model_without_null_embedding_runs_plain_forward():
    """cond_drop_prob = 0 (the constructor default, as in the reference): no null_cond_embedding exists; forward() works,
    forward_with_cfg raises like the reference's attribute lookup would (dit_crossattn.py:208)."""
    import oracle
    cfg = dict(CFG, cond_drop_prob=0.0)
    sd = synth.synth_state_dict(synth.dit_shapes(**cfg), 59)
    assert "null_cond_embedding" not in sd
    m = tpxl_b200.DiT(**cfg)
    m.load_state_dict(sd)
    m = m.to(DEV).eval()
    x, y = synth.synth_inputs(1, cfg["seq_length"], cfg["in_channels"], 77, cfg["condition_channels"], 60)
    t = torch.tensor([200], device=DEV)
    with torch.no_grad():
        out = m.forward(x.to(DEV), t, y.to(DEV), torch.float16, True)
        ref = oracle.dit.forward({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV), t, y.to(DEV), cfg["num_heads"], "fp16")
    assert rel_l2(out.float(), ref) < 3e-3
    with pytest.raises(AttributeError):
        m.forward_with_cfg(x.to(DEV), t, y.to(DEV), cfg_scale=2.0, enable_amp=True)


def test_full_size_ddim_properties():
    """Shipped size, full depth: determinism, finite outputs, and sample-index independence (one sample alone ==
    the same sample inside a batch of two) — the property the one-sample-per-GPU sharding rests on."""
    sd = synth.device_state_dict(synth.dit_shapes(**synth.FULL_DIT), 61, DEV, torch.float16)
    m = tpxl_b200.DiT(**synth.FULL_DIT)
    m.load_state_dict(sd)
    m = m.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(62)
    x = torch.randn(2, 2048, 68, generator=g, device=DEV)
    y = torch.randn(2, 1370, 768, generator=g, device=DEV)
    d = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v")
    kw = dict(y=y, cfg_scale=6.0, precision_dtype=torch.float16, enable_amp=True)
    steps = []
    for i, o in enumerate(d.ddim_sample_loop_progressive(m.forward_with_cfg, x.shape, x, clip_denoised=False, model_kwargs=kw, device=DEV)):
        steps.append(o["sample"])
        if i == 2:
            break
    again = next(iter(d.ddim_sample_loop_progressive(m.forward_with_cfg, x.shape, x, clip_denoised=False, model_kwargs=kw, device=DEV)))["sample"]
    kw1 = dict(kw, y=y[1:2].contiguous())
    solo = next(iter(d.ddim_sample_loop_progressive(m.forward_with_cfg, (1, 2048, 68), x[1:2].contiguous(), clip_denoised=False, model_kwargs=kw1, device=DEV)))["sample"]
    assert all(torch.isfinite(s).all() for s in steps)
    assert torch.equal(again, steps[0])
    assert rel_l2(solo, steps[0][1:2]) < 1e-3


# ---- timestep table (DiT.set_timesteps / tpx_dit_forward_step): the hoisted timestep MLP + adaLN rows must change nothing -----------------
def test_timestep_table_rows_are_bit_identical_to_the_per_step_computation():
    sd, m, x, y = _setup(57)
    d = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v")
    tmap = list(d.timestep_map)                    # 25 timesteps -> 4 table passes (8 + 8 + 8 + 1): first / middle / lone-last rows below
    with torch.no_grad():
        plain = {t: m.forward_with_cfg(x, torch.tensor([t, t], device=DEV), y, cfg_scale=6.0, enable_amp=True).clone() for t in (0, 280, 320, 600, 960)}
        plain_fwd = m.forward(x, torch.tensor([600, 600], device=DEV), y, torch.float16, True).clone()
        m.set_timesteps(tmap)
        for t, ref in plain.items():
            got = m.forward_with_cfg(x, torch.tensor([t, t], device=DEV), y, cfg_scale=6.0, enable_amp=True, t_host=t)
            assert torch.equal(got, ref), t
        assert torch.equal(m.forward(x, torch.tensor([600, 600], device=DEV), y, torch.float16, True, t_host=600), plain_fwd)
        # one sample per batch (B = 1) reads the same row
        one = m.forward_with_cfg(x[:1], torch.tensor([320], device=DEV), y[:1].contiguous(), cfg_scale=6.0, enable_amp=True).clone()
        assert torch.equal(m.forward_with_cfg(x[:1], torch.tensor([320], device=DEV), y[:1].contiguous(), cfg_scale=6.0, enable_amp=True, t_host=320), one)
        # a timestep that is not in the table: the call computes it per step as before
        off = m.forward_with_cfg(x, torch.tensor([333, 333], device=DEV), y, cfg_scale=6.0, enable_amp=True).clone()
        assert torch.equal(m.forward_with_cfg(x, torch.tensor([333, 333], device=DEV), y, cfg_scale=6.0, enable_amp=True, t_host=333), off)
        assert not torch.equal(off, plain[320])


def test_timestep_table_is_dropped_when_weights_change():
    sd, m, x, y = _setup(59)
    t = torch.tensor([480, 480], device=DEV)
    with torch.no_grad():
        m.set_timesteps([480, 520])
        a = m.forward_with_cfg(x, t, y, cfg_scale=6.0, enable_amp=True, t_host=480).clone()
        sd2 = synth.synth_state_dict(synth.dit_shapes(**CFG), 60)
        m.load_state_dict(sd2)                       # re-ingests: a table derived from the old adaLN weights must not be used
        assert m._ts_key is None
        b = m.forward_with_cfg(x, t, y, cfg_scale=6.0, enable_amp=True, t_host=480).clone()
        fresh = tpxl_b200.DiT(**CFG)
        fresh.load_state_dict(sd2)
        fresh = fresh.to(DEV).eval()
        c = fresh.forward_with_cfg(x, t, y, cfg_scale=6.0, enable_amp=True)
        m.set_timesteps([480, 520])
        e = m.forward_with_cfg(x, t, y, cfg_scale=6.0, enable_amp=True, t_host=480)
    assert not torch.equal(a, b) and torch.equal(b, c) and torch.equal(e, c)
    with pytest.raises(tpxl_b200._lib.TpxError):     # straight at the C ABI: a timestep outside the table is an error there, not a fallback
        lib = tpxl_b200._lib.lib()
        ws, nbytes = m._workspace(4)
        out = torch.empty(2, 256, 136, dtype=torch.float16, device=DEV)
        tpxl_b200._lib.check(lib.tpx_dit_forward_step(m._handle, x.data_ptr(), 7, 2, 1, 6.0, out.data_ptr(), ws, nbytes,
                                                      tpxl_b200._lib.stream_ptr()))


@pytest.mark.parametrize("ddim", [True, False])
def test_sampling_loop_is_unchanged_by_the_timestep_hoist(ddim):
    sd, m, x, y = _setup(61)
    kw = dict(y=y, cfg_scale=6.0, precision_dtype=torch.float16, enable_amp=True)
    runs = []
    for hoist in (False, True):
        d = tpxl_b200.create_diffusion("ddim25" if ddim else "10", noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
        d.hoist_timesteps = hoist
        m._ts_key = None
        fn = d.ddim_sample_loop_progressive if ddim else d.p_sample_loop_progressive
        torch.manual_seed(5)
        runs.append([o["sample"].clone() for o in fn(m.forward_with_cfg, x.shape, x, clip_denoised=False, model_kwargs=kw, progress=False, device=DEV)])
        assert (m._ts_key is not None) == hoist
    assert len(runs[0]) == len(runs[1]) and all(torch.equal(a, b) for a, b in zip(*runs))


def test_clip_denoised_loop_reproduces_the_reference_fixture(golden_dir):
    """clip_denoised=True (the reference's default argument) through the CUDA loop: seeded model outputs replayed through the REFERENCE
    sampler on the CPU are the fixture (tests/golden/make_sampler_clip_golden.py); the same outputs replayed through this package's loop on
    the GPU must give the same 25 samples / clamped x_0 predictions (same fp32 ops in the same order: a few ulp at most)."""
    import os
    import numpy as np
    g = np.load(os.path.join(golden_dir, "sampler_clip.npz"))
    x_T = torch.from_numpy(g["x_T"]).to(DEV)
    outs = iter(torch.from_numpy(g["outs25"]).to(DEV))
    d = tpxl_b200.create_diffusion("ddim25", noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
    seen_t = []

    def replay(x, t, **kw):
        seen_t.append(t.tolist())
        return next(outs)

    traj = list(d.ddim_sample_loop_progressive(replay, tuple(x_T.shape), x_T, clip_denoised=True, model_kwargs={}, progress=False, device=DEV))
    assert len(traj) == 25 and seen_t[0] == [960, 960] and seen_t[-1] == [0, 0]
    for i, o in enumerate(traj):
        assert float(o["pred_xstart"].abs().max()) <= 1.0
        assert rel_l2(o["pred_xstart"], torch.from_numpy(g["ddim25_x0"][i]).to(DEV)) < 1e-5, i
        assert rel_l2(o["sample"], torch.from_numpy(g["ddim25_samples"][i]).to(DEV)) < 1e-5, i


@pytest.mark.parametrize("par,clip", [("eps", False), ("eps", True), ("xstart", False), ("xstart", True)])
def test_eps_and_xstart_parameterisations_reproduce_the_reference_fixture(golden_dir, par, clip):
    """create_diffusion(parameterization="eps" | "xstart") ("eps" is the reference's default argument): the same update kernel with other
    host coefficients.  Seeded model outputs replayed through the REFERENCE sampler on the CPU are the fixture
    (tests/golden/make_sampler_param_golden.py); replayed through this package's CUDA loop they must give the same 25 samples."""
    import os
    import numpy as np
    g = np.load(os.path.join(golden_dir, "sampler_param.npz"))
    x_T = torch.from_numpy(g["x_T"]).to(DEV)
    outs = iter(torch.from_numpy(g["outs25"]).to(DEV))
    d = tpxl_b200.create_diffusion("ddim25", noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization=par)
    traj = list(d.ddim_sample_loop_progressive(lambda x, t, **kw: next(outs), tuple(x_T.shape), x_T, clip_denoised=clip, model_kwargs={}, progress=False, device=DEV))
    tag = f"{par}_ddim25" + ("_clip" if clip else "")
    for i, o in enumerate(traj):
        assert rel_l2(o["pred_xstart"], torch.from_numpy(g[tag + "_x0"][i]).to(DEV)) < 1e-5, i
        assert rel_l2(o["sample"], torch.from_numpy(g[tag + "_samples"][i]).to(DEV)) < 1e-5, i
