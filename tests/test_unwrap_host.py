"""CPU: the box-projection unwrap and noise-filter oracle (oracle/unwrap.py) against the reference's own outputs
(tests/golden/unwrap.npz, tests/golden/make_unwrap_golden.py), stage by stage; the invariants of the atlas; and the new C entry points
refusing to run without a device."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import unwrap as ou
from tpxl_b200 import _lib

MESHES = ("torus", "spheres", "shell")
ROT_TOL = 2e-5


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(os.path.join(golden_dir, "unwrap.npz"))


def mesh(g, name):
    return g[f"{name}_v"], g[f"{name}_f"].astype(np.int64)


@pytest.mark.parametrize("name", MESHES)
def test_oracle_reproduces_reference_stage_by_stage(g, name):
    v, f = mesh(g, name)
    k = lambda s: g[f"{name}_{s}"]                                           # noqa: E731
    np.testing.assert_allclose(ou.vertex_normals(v, f), k("normals"), rtol=0, atol=1e-6)
    slc, fuv, margin = ou.project(v, k("normals"), f)
    assert np.array_equal(slc, k("slice")) and margin.min() > 1e-6
    np.testing.assert_allclose(fuv, k("face_uv"), rtol=0, atol=1e-6)
    # the slice means sum expected tangents up to 1e12 apart (the (-1)-norm quirk), so torch's fp32 reduction order shows at ~1e-5
    _, ruv = ou.rotate(v, k("normals"), f, k("face_uv"), k("slice"))
    np.testing.assert_allclose(ruv, k("rot_uv"), rtol=0, atol=ROT_TOL)
    asg, mk = ou.assign(v, f, k("rot_uv"), k("slice"))
    assert np.array_equal(asg, k("assign")) and not ou.ambiguous(mk).any()
    np.testing.assert_allclose(ou.place(k("rot_uv"), k("assign"), 0.02), k("placed"), rtol=0, atol=1e-6)
    uv, vidx = ou.unique(k("placed"))
    assert np.array_equal(uv, k("uv")) and np.array_equal(vidx, k("vidx"))


@pytest.mark.parametrize("name", MESHES)
def test_oracle_end_to_end_invariants(g, name):
    v, f = mesh(g, name)
    out = ou.unwrap(v, ou.vertex_normals(v, f), f, 0.02)
    np.testing.assert_allclose(out["uv"][out["vidx"]], g[f"{name}_uv"][g[f"{name}_vidx"]], rtol=0, atol=ROT_TOL)
    assert out["uv"].min() >= 0 and out["uv"].max() <= 1
    cell = ou.slot_cells(out["assign"])
    p = out["placed"]
    eps = 1e-6
    assert (p[..., 0] >= cell[:, None, 0] - eps).all() and (p[..., 0] <= cell[:, None, 2] + eps).all()
    assert (p[..., 1] >= cell[:, None, 1] - eps).all() and (p[..., 1] <= cell[:, None, 3] + eps).all()
    assert ou.residual_overlaps(out["rot_uv"], out["assign"]) == 0
    assert ou.residual_overlaps(out["rot_uv"], out["slice"]) > 0        # the assignment had work to do


def test_fixture_reaches_every_kind_of_slot(g):
    assert (g["torus_assign"] >= 6).any() and ((g["torus_assign"] >= 8) & (g["torus_assign"] <= 11)).any()
    assert (g["spheres_assign"] == 12).any()


@pytest.mark.parametrize("name", ["dense", "spread"])
def test_noise_filter_oracle_equals_reference(g, name):
    keep, nn = ou.noise_filter(g[f"noise_{name}_srt"])
    assert np.array_equal(keep, g[f"noise_{name}_keep"]) and np.array_equal(nn, g[f"noise_{name}_nn"])
    if name == "spread":
        assert (nn == np.arange(len(nn))).any()                          # the diagonal is 1, not infinity


def test_unwrap_entries_check_device_first():
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses below must never reach a GPU")
    import __graft_entry__
    __graft_entry__._load_build_module().build()
    lib = _lib.load_library()
    P = 1 << 20
    ws = lib.tpx_uv_unwrap_workspace_bytes(3, 1)
    assert ws > 0 and lib.tpx_uv_unwrap_workspace_bytes(0, 1) == 0
    taps = (ctypes.c_void_p * 6)()
    calls = {"tpx_vertex_normals": (P, 3, P, 1, P, ws, P, None), "tpx_uv_unwrap": (P, P, 3, P, 1, 0.02, P, ws, P, taps, None),
             "tpx_uv_unwrap_emit": (3, 1, P, ws, P, P, None), "tpx_prim_noise_filter": (P, 4, P, None, None)}
    for name, args in calls.items():
        rc = getattr(lib, name)(*args)
        assert rc == -2 and b"cudaGetDevice" in lib.tpx_last_error(), name
    assert lib.tpx_uv_unwrap(P, P, 3, P, 1, 0.7, P, ws, P, None, None) == -1      # argument checks come first
