"""CPU: the C-ABI library builds for sm_90a, loads, and exports exactly what include/tpx.h declares; host-side
logic (schedule, respacing, coefficient rounding, state_dict contract) works without a GPU; the compute path
refuses to run without one."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

import tpxl_b200
from tpxl_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__._load_build_module().build()
    return _lib.load_library()


def _header_prototypes():
    """[(name, return type, [parameter types])] of include/tpx.h, in declaration order."""
    src = open(os.path.join(ROOT, "include", "tpx.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = []
    for ret, name, params in re.findall(r"^\s*((?:const\s+)?\w+\s*\**)\s*\b(tpx_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src, flags=re.M):
        params = " ".join(params.split())
        types = [] if params in ("", "void") else [re.sub(r"\s*\w+$", "", p.strip()) for p in params.split(",")]
        protos.append((name, ret.strip(), types))
    return protos


_SCALARS = {"int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
            "double": ctypes.c_double, "uint8_t": ctypes.c_uint8}
_STRUCTS = {"tpx_dit_config": _lib.DitConfig, "tpx_vae_config": _lib.VaeConfig, "tpx_sampler_coefs": _lib.SamplerCoefs}


def _ctype_matches(c_type: str, ct) -> bool:
    """Does the ctypes type `ct` pass a value of the C type `c_type` correctly?"""
    t = " ".join(c_type.replace("const", " ").replace("*", " * ").split())
    base, stars = t.split(" ")[0], t.count("*")
    if stars == 0:
        return ct is None if base == "void" else ct is _SCALARS[base]
    if stars == 1 and base == "char":
        return ct is ctypes.c_char_p
    if stars == 1 and base in _STRUCTS:
        return ct is ctypes.POINTER(_STRUCTS[base])
    if stars == 1:      # device / host data or an opaque handle: any pointer, or a typed pointer to the same scalar
        return ct is ctypes.c_void_p or (base in _SCALARS and ct is ctypes.POINTER(_SCALARS[base]))
    return stars == 2 and ct in (ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p))


def test_library_exports_every_declared_symbol(lib):
    protos = _header_prototypes()
    names = [n for n, _, _ in protos]
    assert len(names) >= 25 and len(set(names)) == len(names)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/tpx.h but not exported"
    assert list(_lib.SIGNATURES) == names, "ctypes table and header disagree (names or order)"
    for name, ret, params in protos:
        res, args = _lib.SIGNATURES[name]
        assert _ctype_matches(ret, res), f"{name}: return type {ret} bound as {res}"
        assert len(args) == len(params), f"{name}: {len(params)} parameters declared, {len(args)} bound"
        for i, (c_type, ct) in enumerate(zip(params, args)):
            assert _ctype_matches(c_type, ct), f"{name}: parameter {i} ({c_type}) bound as {ct}"
    assert lib.tpx_version() == 100


def test_stateless_entries_check_device_first(lib):
    """Every stateless entry that enqueues device work runs the device guard (tpx_device_check) after its argument checks and before
    any other CUDA call: without a usable device, valid arguments fail there with TPX_ERR_CUDA naming cudaGetDevice."""
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses below must never reach a GPU")
    P = 1 << 20                                    # non-null, 256-B aligned, never dereferenced
    coefs = _lib.SamplerCoefs()
    grid_bytes = lib.tpx_primsdf_grid_bytes(1024)
    mc_bytes = lib.tpx_mc_workspace_bytes(2, 2, 2)
    cc_bytes, dec_bytes = lib.tpx_mesh_components_workspace_bytes(3, 1), lib.tpx_decimate_workspace_bytes(3, 1)
    calls = {
        "tpx_sampler_step": (1, P, P, 1, None, 8, 4, ctypes.byref(coefs), P, P, None),
        "tpx_latent_split": (P, None, None, 1.0, 2, 8, P, P, None),
        "tpx_primvolume_pack": (P, P, 1, 2, 8, 4, 0, P, None),
        "tpx_linear": (P, 128, P, None, P, 128, 128, 128, 128, 0, 1.0, 0, None),
        "tpx_linear_gated": (P, 128, P, None, P, 0, 1, 128, P, 128, 128, 128, 128, 0, None),
        "tpx_linear_heads": (P, 128, P, None, P, P, P, 128, 384, 128, 128, 2, 64, 64, 64, 1.0, 0, -1, 0, None),
        "tpx_ln_modulate": (P, 8, 128, 1e-6, P, P, 0, 8, 1, P, None, None, 0, None),
        "tpx_attention": (P, P, P, P, 1, 1, 8, 8, 64, 64, 0.125, None),
        "tpx_attention_tc": (P, P, P, P, 1, 1, 8, 8, 8, 72, 0.125, None),
        "tpx_cfg_combine": (P, 64, 2.0, P, None),
        "tpx_groupnorm_silu": (P, P, P, 1, 64, 256, 32, 1e-5, 1, P, None),
        "tpx_conv3d_k3": (P, P, P, None, 1.0, P, 1, 8, 32, 32, None),
        "tpx_gelu_erf": (P, 64, None),
        "tpx_primsdf_query": (P, P, P, 8, 2, 8, 6, 1, P, None),
        "tpx_primsdf_grid_build": (P, 2, P, grid_bytes, None),
        "tpx_primsdf_query_grid": (P, P, P, P, grid_bytes, 8, 2, 8, 6, 1, P, None),
        "tpx_primsdf_sdf_grid": (P, 4, P, P, None, 0, 2, 8, 6, 1, P, None),
        "tpx_raymarch_preview": (P, P, P, P, P, P, P, P, 1, 2, 8, 8, 8, 1.0, 0.01, 8.0, 8.0, P, None),
        "tpx_mc_count": (P, 2, 2, 2, 0.0, P, mc_bytes, P, None),
        "tpx_mc_emit": (P, 2, 2, 2, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0, 1.0, P, mc_bytes, P, P, None),
        "tpx_mesh_components_count": (P, 3, P, 1, 8, 0.05, P, cc_bytes, P, None),
        "tpx_mesh_components_emit": (P, 3, 1, P, cc_bytes, P, P, None),
        "tpx_decimate": (P, 3, P, 1, 0, P, dec_bytes, P, None, 0, None),
        "tpx_decimate_emit": (3, 1, P, dec_bytes, P, P, None),
        "tpx_uv_rasterize": (P, 3, P, 1, 8, 8, P, P, None),
        "tpx_rast_interpolate": (P, 3, 2, P, 1, P, 8, 8, P, None),
        "tpx_primsdf_bake": (P, 8, 8, P, 3, P, 1, P, P, None, 0, 2, 8, 6, P, P, None),
        "tpx_texture_inpaint": (P, P, 8, 8, 6, 2, P, lib.tpx_texture_inpaint_bytes(8, 8), None, None),
    }
    failed = {}
    for name, args in calls.items():
        rc = getattr(lib, name)(*args)
        msg = lib.tpx_last_error()
        if rc != -2 or b"cudaGetDevice" not in msg:
            failed[name] = (rc, msg)
    assert not failed, failed


def test_header_cites_reference_interfaces():
    src = open(os.path.join(ROOT, "include", "tpx.h")).read()
    for cite in ("dit_crossattn.py:184-202", "gaussian_diffusion.py", "vae3d_dib.py:437-440", "attention.py"):
        assert cite in src


def test_sass_contains_hopper_tensor_and_tma_ops(lib):
    """The GEMM really is wgmma + TMA (HGMMA / UTMALDG in SASS)."""
    import subprocess
    obj = os.path.join(ROOT, "3dtopia-xl_b200", "build", "gemm_tc.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    # warpgroup tensor-core MMA, TMA loads, and the bulk-store epilogues: plain tensor stores and the L2-side reduce-add that
    # carries the gated residual
    for mnem in ("HGMMA", "UTMALDG", "UTMASTG", "UTMAREDG"):
        assert mnem in sass, mnem


def test_compute_path_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.TpxError):
        _lib.lib()
    m = tpxl_b200.DiT(seq_length=8, in_channels=8, condition_channels=16, hidden_size=128, depth=1, num_heads=4, cond_drop_prob=0.1)
    with pytest.raises(_lib.TpxError):
        m.forward(torch.zeros(1, 8, 8), torch.zeros(1, dtype=torch.int64), torch.zeros(1, 3, 16))
    with pytest.raises(_lib.TpxError):
        list(tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v").ddim_sample_loop_progressive(
            lambda *a, **k: None, (1, 8, 8), noise=torch.zeros(1, 8, 8), device="cpu"))
    with pytest.raises(_lib.TpxError):
        m.set_timesteps([0, 40])                     # the timestep table lives in the C library: no handle, no table
    # argument validation of the timestep-table entries happens before any CUDA call
    raw = _lib.load_library()
    assert raw.tpx_dit_timesteps_bytes(None, 25) == 0
    arr = (ctypes.c_int64 * 2)(0, 40)
    assert raw.tpx_dit_set_timesteps(None, arr, 2, None, 0, None) == -1 and b"null" in raw.tpx_last_error()
    assert raw.tpx_dit_forward_step(None, None, 0, 1, 1, 6.0, None, None, 0, None) == -1


def test_dit_debug_entries_reject_bad_arguments(lib):
    """tpx_dit_debug_stage / tpx_dit_debug_tap check the stop point and the tap before anything else, then their pointers; none of
    these calls reaches the device.  (A block outside the model's depth needs a handle: tests/test_gpu_dit_stages.py.)"""
    P = 1 << 20
    for stage in (-1, 4):
        assert lib.tpx_dit_debug_stage(P, P, P, 1, 0, 0, stage, P, 1 << 20, None) == -1
        assert b"bad stage" in lib.tpx_last_error()
    for h, t in ((None, P), (P, None)):
        assert lib.tpx_dit_debug_stage(h, P, t, 1, 0, 0, 1, P, 1 << 20, None) == -1
        assert b"null" in lib.tpx_last_error()
    for which in (-1, 4):
        assert lib.tpx_dit_debug_tap(P, P, 2, which, 1, P, None) == -1
        assert b"bad tap" in lib.tpx_last_error()
    for n_seq, count in ((2, 0), (2, 3), (0, 0)):
        assert lib.tpx_dit_debug_tap(P, P, n_seq, 0, count, P, None) == -1
        assert b"count" in lib.tpx_last_error()
    for h, ws, dst in ((None, P, P), (P, None, P), (P, P, None)):
        assert lib.tpx_dit_debug_tap(h, ws, 2, 0, 2, dst, None) == -1
        assert b"null" in lib.tpx_last_error()


def test_schedule_matches_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "sampler.npz"))
    for k in (25, 50, 100, 200):
        d = tpxl_b200.create_diffusion(f"ddim{k}", noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
        assert np.array_equal(np.array(d.timestep_map), g[f"map_ddim{k}"])
        np.testing.assert_allclose(d.alphas_cumprod, g[f"acp_ddim{k}"], rtol=1e-13)
        assert d.num_timesteps == k
    d = tpxl_b200.create_diffusion("", noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
    np.testing.assert_allclose(d.betas, g["betas_full"], rtol=1e-12)
    assert np.array_equal(np.array(tpxl_b200.create_diffusion("10", "squaredcos_cap_v2", parameterization="v").timestep_map), g["map_sec10"])
    d25 = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v")
    for nm in ("posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2", "sqrt_recipm1_alphas_cumprod"):
        np.testing.assert_allclose(getattr(d25, nm), g[nm + "_ddim25"], rtol=1e-12)
    dl = tpxl_b200.create_diffusion("ddim50", noise_schedule="linear", diffusion_steps=1000, parameterization="v")
    assert np.array_equal(np.array(dl.timestep_map), g["map_linear_ddim50"])
    np.testing.assert_allclose(dl.alphas_cumprod, g["acp_linear_ddim50"], rtol=1e-12)
    assert tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2").parameterization == "eps"      # the reference's default argument (__init__.py:14)
    with pytest.raises(NotImplementedError):
        tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v", learn_sigma=False)   # fixed variances: C-channel model output
    with pytest.raises(NotImplementedError):
        tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="bogus")
    with pytest.raises(ValueError):
        tpxl_b200.create_diffusion("ddim600", "squaredcos_cap_v2", parameterization="v")


def test_step_coefficients_are_fp32_rounded_like_extract_into_tensor():
    import oracle
    d = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v")
    s = oracle.diffusion.Schedule("ddim25")
    for i in (0, 1, 12, 24):
        for eta in (0.0, 0.5):
            k = d.step_coefs(i, eta)
            ab, abp = torch.tensor(s.alphas_cumprod[i]).float(), torch.tensor(s.alphas_cumprod_prev[i]).float()
            sigma = eta * torch.sqrt((1 - abp) / (1 - ab)) * torch.sqrt(1 - ab / abp)
            assert k.sqrt_ab == float(torch.tensor(s.sqrt_alphas_cumprod[i]).float())
            assert k.sigma == float(sigma)
            # torch's CPU scalar sqrt is not always correctly rounded (1 ulp); numpy / CUDA sqrtf are
            assert abs(k.c_x0 - float(torch.sqrt(abp))) <= 1.2e-7 * k.c_x0
            assert k.c_eps == float(np.sqrt(np.float32(float(1 - abp - sigma ** 2))))
            assert abs(k.c_eps - float(torch.sqrt(1 - abp - sigma ** 2))) <= 1.2e-7 * k.c_eps
            assert k.nonzero == (0.0 if i == 0 else 1.0)


def test_host_coefficients_and_update_order_reproduce_the_reference_with_clip(golden_dir):
    """The DDIM update the CUDA kernel performs (ddim_step_kernel: one explicitly rounded fp32 op per reference tensor op, the clamp of
    process_xstart in between) restated in numpy float32 on the HOST coefficients of SpacedDiffusion.step_coefs — product code that runs
    without a GPU — reproduces the reference sampler's 25-step clip_denoised=True trajectory BIT FOR BIT (fixture: the reference's own
    sampler on replayed model outputs, tests/golden/make_sampler_clip_golden.py)."""
    g = np.load(os.path.join(golden_dir, "sampler_clip.npz"))
    d = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization="v")
    f = np.float32
    x = g["x_T"].copy()
    for n, i in enumerate(reversed(range(25))):
        k = d.step_coefs(i, 0.0, True)
        assert k.clip == 1 and float(k.sigma) == 0.0
        v = g["outs25"][n][..., :68]
        x0 = (f(k.sqrt_ab) * x - f(k.sqrt_1mab) * v).astype(f)
        x0 = np.minimum(np.maximum(x0, f(-1)), f(1))
        eps = ((f(k.sqrt_recip_ab) * x - x0) / f(k.sqrt_recipm1_ab)).astype(f)
        x = (x0 * f(k.c_x0) + f(k.c_eps) * eps).astype(f)
        assert np.array_equal(x0, g["ddim25_x0"][n]) and np.array_equal(x, g["ddim25_samples"][n]), n


@pytest.mark.parametrize("par", ["eps", "xstart"])
@pytest.mark.parametrize("clip", [False, True])
def test_eps_and_xstart_parameterisations_reproduce_the_reference_bit_for_bit(golden_dir, par, clip):
    """create_diffusion's other parameterisations ("eps" is the reference's default argument) reach the SAME update kernel through the
    host coefficients alone (pred_xstart = a x_t - b out with per-step (a, b), SpacedDiffusion.step_coefs).  The kernel's op order in
    numpy float32 on those coefficients reproduces the reference sampler's 25-step DDIM trajectory bit for bit (fixture: the reference's
    own sampler on replayed model outputs, tests/golden/make_sampler_param_golden.py)."""
    g = np.load(os.path.join(golden_dir, "sampler_param.npz"))
    d = tpxl_b200.create_diffusion("ddim25", "squaredcos_cap_v2", parameterization=par)
    f = np.float32
    x = g["x_T"].copy()
    tag = f"{par}_ddim25" + ("_clip" if clip else "")
    with np.errstate(over="ignore", invalid="ignore"):
        for n, i in enumerate(reversed(range(25))):
            k = d.step_coefs(i, 0.0, clip)
            v = g["outs25"][n][..., :68]
            x0 = (f(k.sqrt_ab) * x - f(k.sqrt_1mab) * v).astype(f)
            if clip:
                x0 = np.minimum(np.maximum(x0, f(-1)), f(1))
            eps = ((f(k.sqrt_recip_ab) * x - x0) / f(k.sqrt_recipm1_ab)).astype(f)
            x = (x0 * f(k.c_x0) + f(k.c_eps) * eps).astype(f)
            assert np.array_equal(x0, g[tag + "_x0"][n]) and np.array_equal(x, g[tag + "_samples"][n]), n


def test_state_dict_contract_on_host(golden_dir):
    keys = json.load(open(os.path.join(golden_dir, "state_dict_keys.json")))
    m = tpxl_b200.DiT(**{k: v for k, v in synth.FULL_DIT.items()})
    assert {k: list(v) for k, v in m._shapes.items()} == keys["dit"]
    tiny = dict(seq_length=8, in_channels=8, condition_channels=16, hidden_size=128, depth=1, num_heads=4, attn_proj_bias=True, cond_drop_prob=0.1)
    m = tpxl_b200.DiT(**tiny)
    sd = synth.synth_state_dict(synth.dit_shapes(**tiny), 5)
    m.load_state_dict(sd)
    assert list(m.state_dict().keys()) == list(sd.keys())
    bad = dict(sd)
    bad["blocks.0.attn.qkv.weight"] = torch.zeros(3, 3)
    with pytest.raises(RuntimeError, match="size mismatch"):
        m.load_state_dict(bad)
    del bad["blocks.0.attn.qkv.weight"]
    with pytest.raises(RuntimeError, match="Missing key"):
        m.load_state_dict(bad)
    assert next(m.parameters()).device.type == "cpu"
    v = tpxl_b200.VAE(**synth.FULL_VAE)
    full_keys = {k: torch.zeros(s) for k, s in keys["vae"].items()}
    res = v.load_state_dict(full_keys)          # encoder.* keys accepted, as in the released checkpoint
    assert not res.missing_keys and not res.unexpected_keys
    with pytest.raises(NotImplementedError):
        tpxl_b200.VAE(in_channels=6, latent_channels=4, out_channels=6, up_channels=[256, 32])
    with pytest.raises(NotImplementedError):
        v.encode(torch.zeros(1))


def test_install_aliases_reference_module_paths():
    tpxl_b200.install()
    import importlib
    assert importlib.import_module("models.dit_crossattn").DiT is tpxl_b200.DiT
    assert importlib.import_module("models.vae3d_dib").VAE is tpxl_b200.VAE
    from models.diffusion import create_diffusion
    assert create_diffusion is tpxl_b200.create_diffusion
    assert importlib.import_module("models.primsdf").PrimSDF is tpxl_b200.PrimSDF


def test_primsdf_host_contract():
    """models/primsdf.py:19-50: constructor kwargs of configs/inference_dit.yml:22-30, the two parameters and their slices,
    load_state_dict / .data reassignment as inference.py:90-103,369 uses them; no CPU compute path."""
    m = tpxl_b200.PrimSDF(num_prims=32, dim_feat=6, prim_shape=8, init_scale=0.05, sdf2alpha_var=0.005, auto_scale_init=True, init_sampling="uniform")
    assert list(m.state_dict().keys()) == ["srt_param", "feat_param"]
    assert tuple(m.srt_param.shape) == (32, 4) and tuple(m.feat_param.shape) == (32, 6 * 512)
    m.load_state_dict({"srt_param": torch.rand(32, 4), "feat_param": torch.randn(32, 3072)})
    assert m.feat_geo.shape == (32, 512) and m.feat_tex.shape == (32, 1536) and m.feat_mat.shape == (32, 1024)
    assert torch.equal(m.pos, m.srt_param[:, 1:4]) and torch.equal(m.scale, m.srt_param[:, 0:1])
    m.srt_param.data = m.srt_param.data[:7]              # the reference filters primitives in place
    m.feat_param.data = m.feat_param.data[:7]
    assert m.srt_param.shape[0] == 7
    np.testing.assert_allclose(m.sdf2alpha(torch.tensor([0.0, 0.005])).numpy(), [1.0, np.exp(-1.0)], rtol=1e-6)
    with pytest.raises(tpxl_b200._lib.TpxError):
        m.eval()(torch.zeros(5, 3))
    with pytest.raises(ValueError):
        m(torch.zeros(5, 2))


def test_product_and_tools_do_not_use_the_oracle():
    """oracle/ is test infrastructure: only tests/, __graft_entry__ (build + smoke) and bench.py's CPU legs may touch it."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    offenders = []
    for sub in ("3dtopia-xl_b200", "tools"):
        for dirpath, _, files in os.walk(os.path.join(root, sub)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h")):
                    src = open(os.path.join(dirpath, f), encoding="utf-8", errors="replace").read()
                    if re.search(r"^\s*(import|from)\s+oracle\b", src, re.M) or "oracle/" in src and f.endswith((".cu", ".cuh", ".h")):
                        offenders.append(os.path.join(sub, f))
    assert not offenders, offenders


def test_respacing_strings_match_reference(golden_dir):
    """respace.py:12-62 through the reference itself: 'ddimK' strides, section counts, and the specs it rejects."""
    fx = np.load(os.path.join(golden_dir, "sampler.npz"))
    cases = json.loads(str(fx["space_cases"]))
    from tpxl_b200.diffusion import space_timesteps
    assert len(cases) >= 18
    for spec, want in cases.items():
        if want == "ValueError":
            with pytest.raises(ValueError):
                space_timesteps(1000, spec)
        else:
            assert sorted(space_timesteps(1000, spec)) == want, spec


def test_timestep_hoist_is_offered_only_to_this_packages_own_dit_methods():
    """SpacedDiffusion's loops may build DiT's timestep table and pass ``t_host=`` only when the model they are handed is the package's
    un-overridden DiT.forward / forward_with_cfg (bound method or module); everything else must see the reference's call signature."""
    import tpxl_b200
    d = tpxl_b200.create_diffusion("ddim25", noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v")
    cfg = dict(seq_length=8, in_channels=8, condition_channels=16, hidden_size=128, depth=1, num_heads=8)
    m = tpxl_b200.DiT(**cfg)
    assert d.hoist_timesteps
    assert d._hoist_owner(m.forward_with_cfg, {}) is m and d._hoist_owner(m.forward, {"y": None}) is m and d._hoist_owner(m, {}) is m
    assert d._hoist_owner(lambda x, t, **kw: m.forward_with_cfg(x, t, **kw), {}) is None          # a wrapper (e.g. respace._WrappedModel)
    assert d._hoist_owner(torch.nn.Linear(2, 2), {}) is None and d._hoist_owner(torch.nn.Linear(2, 2).forward, {}) is None
    assert d._hoist_owner(m.forward_with_cfg, {"t_host": 3}) is None                                 # the caller already decides

    class Sub(tpxl_b200.DiT):
        def forward_with_cfg(self, x, t, y, **kw):      # an override need not know t_host
            return super().forward_with_cfg(x, t, y, **kw)

    s = Sub(**cfg)
    assert d._hoist_owner(s.forward_with_cfg, {}) is None and d._hoist_owner(s.forward, {}) is s and d._hoist_owner(s, {}) is s
    d.hoist_timesteps = False
    assert d._hoist_owner(m.forward_with_cfg, {}) is None
    long = tpxl_b200.create_diffusion("", noise_schedule="linear", diffusion_steps=5000, parameterization="v")   # more steps than a table holds
    assert long.num_timesteps == 5000 and long._hoist_owner(m.forward_with_cfg, {}) is None
    # the two reference signatures still bind positionally (inference.py:278-280 passes keywords; gaussian_diffusion.py:279 positionals + kwargs)
    import inspect
    for fn in (tpxl_b200.DiT.forward, tpxl_b200.DiT.forward_with_cfg):
        names = list(inspect.signature(fn).parameters)
        assert names[:4] == ["self", "x", "t", "y"] and names[-1] == "t_host" and inspect.signature(fn).parameters["t_host"].default is None
