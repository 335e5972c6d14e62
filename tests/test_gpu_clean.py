"""-m gpu: mesh clean-up (close-vertex merge, duplicate / null faces, non-manifold repair; csrc/mesh_simplify.cu through
tpxl_b200.mesh.clean_mesh) against the numpy oracle (oracle/clean.py), byte for byte, and PrimSDF.extract_mesh / extract_texmesh with
merge_distance and repair on the synthetic shell."""
import sys

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import clean as oc
from tpxl_b200 import mesh

from test_decimate_host import MESHES, fin_and_pinch
from test_gpu_mesh import _shell_module
from parity import same_mesh

pytestmark = pytest.mark.gpu


def _cuda(V, F):
    return torch.from_numpy(np.ascontiguousarray(V, np.float32)).cuda(), torch.from_numpy(np.ascontiguousarray(F, np.int64)).cuda()


def _clean(v, f, v_pct, repair=True):
    return mesh.clean_mesh(v, f, v_pct=v_pct, min_f=8, min_d=5, repair=repair, remesh=False)


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("v_pct", [0, 0.3, 1, 3])
def test_clean_matches_oracle(name, v_pct):
    V, F, _ = MESHES[name]()
    dv, df = _cuda(V, F)
    same_mesh(mesh._weld(dv, df, v_pct / 100), oc.weld(V, F, v_pct / 100), f"{name} weld")
    want = oc.clean_mesh(V, F, v_pct, 8, 5, True)
    got = _clean(dv, df, v_pct)
    same_mesh(got, want, f"{name} clean")
    side = torch.cuda.Stream()
    again = _clean(dv, df, v_pct)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = _clean(dv, df, v_pct)
    torch.cuda.current_stream().wait_stream(side)
    for v, f in (again, other):
        assert torch.equal(v, got[0]) and torch.equal(f, got[1]), f"{name}: repeated call differs"
    if got[1].shape[0]:
        mesh.decimate(got[0], got[1], got[1].shape[0] // 2)             # the output feeds decimate directly


def test_repair_fin_pinch_and_numpy():
    for Vm, Fm, _ in fin_and_pinch():
        same_mesh(mesh._repair(*_cuda(Vm, Fm)), oc.repair(Vm, Fm), "repair")
        same_mesh(_clean(*_cuda(Vm, Fm), 1), oc.clean_mesh(Vm, Fm, 1, 8, 5, True), "clean")
    V, F, _ = MESHES["torus"]()
    G = np.concatenate([F, F[:5, ::-1], [[F[7, 0], F[7, 0], F[7, 2]]]])  # duplicates of either winding and a repeated index
    v, f = _clean(V, G, 1)                                               # numpy in, numpy out
    want = oc.clean_mesh(V, G, 1, 8, 5, True)
    assert v.dtype == np.float64 and f.dtype == np.int64
    assert np.array_equal(v, want[0].astype(np.float64)) and np.array_equal(f, want[1])
    e = _clean(torch.zeros(0, 3, device="cuda"), torch.zeros(0, 3, dtype=torch.int64, device="cuda"), 1)
    assert e[0].shape == (0, 3) and e[1].shape == (0, 3)
    bad = torch.from_numpy(F).cuda()
    bad[2, 1] = len(V)
    with pytest.raises(ValueError):
        _clean(torch.from_numpy(V).cuda(), bad, 1)


def test_adversarial_sizes_complete():
    rng = np.random.default_rng(5)
    n = 200000
    V = rng.uniform(0, 1e-3, (n, 3)).astype(np.float32)                 # all within r of each other: one seed
    V[0] = 0
    F = np.stack([np.arange(n - 2), np.arange(1, n - 1), np.arange(2, n)], 1)
    v, f = mesh._weld(*_cuda(V, F), 1.01)
    assert v.shape[0] == 0 and f.shape[0] == 0
    Vs, Fs, _ = MESHES["sphere"]()                                      # r below every edge: no merges
    same_mesh(mesh._weld(*_cuda(Vs, Fs), 1e-7), (Vs, Fs), "no merge")


def test_shell_r128_matches_oracle():
    m = _shell_module()
    v0, f0 = m.extract_mesh(128)
    V, F = v0.cpu().numpy(), f0.cpu().numpy()
    info = {}
    w = mesh._weld(v0, f0, 0.01, info)
    want_w = oc.weld(V, F, 0.01)
    same_mesh(w, want_w, "shell weld")
    same_mesh(mesh._repair(*w), oc.repair(*want_w), "shell repair")
    print(f"R=128: F {len(F)} -> welded {len(want_w[1])} in {info['rounds']} rounds")


def test_extract_mesh_with_clean_up():
    m = _shell_module()
    R = 256
    grid = m.sdf_grid(R)
    v0, f0 = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
    v1, f1 = mesh._weld(v0, f0, 0.01)
    v2, f2 = mesh._remove_small(v1, f1, 8, 0.05)
    v3, f3 = mesh._repair(v2, f2)
    v4, f4 = mesh._decimate(v3, f3, 100000)
    ve, fe = m.extract_mesh(R, merge_distance=0.01, min_faces=8, min_diameter=0.05, repair=True, target_faces=100000)
    assert torch.equal(ve, v4) and torch.equal(fe, f4), "extract_mesh differs from the explicit chain"
    base = m.extract_mesh(R, min_faces=8, min_diameter=0.05, target_faces=100000)
    dflt = m.extract_mesh(R, min_faces=8, min_diameter=0.05, target_faces=100000, merge_distance=0.0, repair=False)
    assert torch.equal(base[0], dflt[0]) and torch.equal(base[1], dflt[1])
    vb, fb = mesh._decimate(*mesh._remove_small(v0, f0, 8, 0.05), 100000)
    assert torch.equal(base[0], vb) and torch.equal(base[1], fb)        # the defaults are today's chain
    print(f"R=256: F {f0.shape[0]} -> welded {f1.shape[0]} -> filtered {f2.shape[0]} -> repaired {f3.shape[0]} -> {f4.shape[0]}")
    out = m.extract_texmesh(R, 100000, 256, 0.02, 8, 0.05, merge_distance=0.01, repair=True)
    assert out["f"].shape[0] > 0 and int(out["f"].max()) < out["v"].shape[0]
    assert out["vt"].shape == (3 * out["f"].shape[0], 2) and float(out["vt"].min()) >= 0 and float(out["vt"].max()) <= 1
    assert out["albedo"].shape == (256, 256, 3) and torch.isfinite(out["albedo"]).all()


def test_bound_meshutils_equals_mesh_clean_mesh():
    V, F, _ = MESHES["two_spheres"]()
    try:
        tpxl_b200.install(meshutils=True)
        from utils.meshutils import clean_mesh, decimate_mesh
        got = clean_mesh(V, F, min_f=8, min_d=5, repair=True, remesh=False)
        want = mesh.clean_mesh(V, F, min_f=8, min_d=5, repair=True, remesh=False)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        d = decimate_mesh(got[0], got[1], len(got[1]) // 2)
        e = mesh.decimate(got[0], got[1], len(got[1]) // 2)
        assert np.array_equal(d[0], e[0]) and np.array_equal(d[1], e[1])
    finally:
        sys.modules.pop("utils.meshutils", None)
