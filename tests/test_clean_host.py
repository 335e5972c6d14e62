"""CPU: the clean-up oracle (oracle/clean.py) — greedy seeds, duplicate / null faces, the non-manifold repair on the fin and pinch
meshes — and the clean-up entry points without a GPU."""
import sys

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import clean as oc
from oracle import decimate as od
from tpxl_b200 import _lib

from test_decimate_host import MESHES, fin_and_pinch, sphere


def _edge_face_counts(F):
    a, b = F, np.roll(F, -1, 1)
    key = (np.minimum(a, b) << 32 | np.maximum(a, b)).ravel()
    return np.unique(key, return_counts=True)[1]


def _fans(F, v):
    """Number of fans of the faces at v (edge-connected through edges incident to v)."""
    fs = np.flatnonzero((F == v).any(1))
    parent = {int(f): int(f) for f in fs}

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for i in fs:
        for j in fs:
            if i < j and len(set(F[i]) & set(F[j])) == 2:
                parent[find(int(j))] = find(int(i))
    return len({find(int(f)) for f in fs})


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("v_pct", [0.3, 1, 3])
def test_oracle_seeds_are_r_apart_and_cover(name, v_pct):
    V, F, _ = MESHES[name]()
    used = np.zeros(len(V), bool)
    used[F.ravel()] = True
    r = oc.merge_radius(V, used, v_pct / 100)
    rep = oc.seeds(V, used, r)
    s = np.flatnonzero(used & (rep == np.arange(len(V))))
    P = V.astype(np.float64)
    d2 = ((P[s][:, None] - P[s][None]) ** 2).sum(-1)
    np.fill_diagonal(d2, np.inf)
    assert (d2 >= r * r).all()                                          # seeds pairwise >= r apart
    cap = np.flatnonzero(used & (rep != np.arange(len(V))))
    assert (rep[cap] < cap).all() and (rep[rep[cap]] == rep[cap]).all()
    assert (((P[cap] - P[rep[cap]]) ** 2).sum(1) < r * r).all()        # every vertex within r of its seed
    v, f = oc.weld(V, F, v_pct / 100)
    assert len(f) <= len(F) and len(np.unique(f)) == len(v)
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 2] != f[:, 0])).all()
    assert len(np.unique(np.sort(f, 1), axis=0)) == len(f)
    p = v[f].astype(np.float64)
    assert (np.abs(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])).sum(1) > 0).all()


def test_oracle_chain_and_single_cluster():
    # a - b - c on a line, spacing 0.6 r: b joins a, c (1.2 r from a) is a seed of its own; a far triangle fixes the box
    r_frac = 0.1
    D = 10.0 * np.sqrt(3)
    r = r_frac * D
    V = np.array([[0, 0, 0], [0.6 * r, 0, 0], [1.2 * r, 0, 0], [10, 10, 10], [10, 9, 10], [9, 10, 10]], np.float32)
    F = np.array([[0, 1, 2], [3, 4, 5]])
    used = np.ones(6, bool)
    rep = oc.seeds(V, used, oc.merge_radius(V, used, r_frac))
    assert rep[:3].tolist() == [0, 0, 2]
    # every vertex within r of every other: one seed
    rng = np.random.default_rng(0)
    Vc = rng.uniform(0, 1, (200, 3)).astype(np.float32)
    Fc = np.arange(198)[:, None] + np.arange(3)[None]
    u = np.ones(200, bool)
    assert (oc.seeds(Vc, u, oc.merge_radius(Vc, u, 1.01)) == 0).all()
    v, f = oc.weld(Vc, Fc, 1.01)
    assert len(v) == 0 and len(f) == 0
    # r below every edge: nothing merges
    Vs, Fs, _ = sphere()
    v, f = oc.weld(Vs, Fs, 1e-6)
    assert np.array_equal(v, Vs) and np.array_equal(f, Fs)


def test_oracle_duplicates_null_and_repeated_faces():
    V, F, _ = sphere()
    extra = np.array([F[3][::-1], F[0], [F[5, 0], F[5, 0], F[5, 1]]])      # opposite winding of face 3, a copy of 0, a repeated index
    v, f = oc.weld(V, np.concatenate([F, extra]), 0.0)
    assert np.array_equal(v, V) and np.array_equal(f, F)                   # the lower ids stay
    Ff = np.concatenate([F[:3][::-1], F[3:]])                              # reversed copy first: it is the lower id and stays
    G = np.concatenate([Ff, F[:1][:, ::-1]])
    v, f = oc.weld(V, G, 0.0)
    assert np.array_equal(f, Ff)
    Vn = np.concatenate([V, [[0, 0, 0], [1, 1, 1], [2, 2, 2]]]).astype(np.float32)      # a collinear (null) face is dropped
    n = len(V)
    v, f = oc.weld(Vn, np.concatenate([F, [[n, n + 1, n + 2]]]), 0.0)
    assert np.array_equal(v, V) and np.array_equal(f, F)
    v, f = oc.weld(*MESHES["integer"]()[:2], 0.0)
    p = v[f].astype(np.float64)
    assert (np.abs(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])).sum(1) > 0).all()


def test_oracle_clean_without_merge_or_repair_is_the_component_filter():
    for name in ("sphere", "torus", "two_spheres", "open_field"):
        V, F, _ = MESHES[name]()
        want = od.remove_small_components(V, F, 8, 0.05)
        got = oc.clean_mesh(V, F, v_pct=0, min_f=8, min_d=5, repair_mesh=False)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), name


def test_oracle_repair_fin_and_pinch():
    (Vf, Ff, (a, b, apex)), (Vp, Fp, (j,)) = fin_and_pinch()
    # fin: three faces on edge (a, b); the one of smallest area goes first and leaves two, so it is the only one deleted
    v, f = oc.repair(Vf, Ff)
    assert (_edge_face_counts(f) <= 2).all() and len(f) == len(Ff) - 1
    on = np.flatnonzero((Ff == a).any(1) & (Ff == b).any(1))
    p = Vf[Ff[on]].astype(np.float64)
    gone = on[np.argmin(np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=1))]
    assert len(on) == 3 and np.array_equal(f, od.compact(Vf, np.delete(Ff, gone, 0))[1])
    # pinch: j has two fans; the first sphere keeps j, the second gets one copy at the same position, last
    v, f = oc.repair(Vp, Fp)
    assert len(f) == len(Fp) and len(v) == len(np.unique(Fp)) + 1
    assert np.array_equal(v[-1].view(np.int32), Vp[j].view(np.int32))
    assert _fans(Fp, j) == 2 and _fans(f, j) == 1 and _fans(f, len(v) - 1) == 1
    half = len(Fp) // 2
    assert (f[half:] == len(v) - 1).any() and not (f[:half] == len(v) - 1).any()
    for Vm, Fm in ((Vf, Ff), (Vp, Fp)):
        v, f = oc.repair(Vm, Fm)
        assert (_edge_face_counts(f) <= 2).all()
        assert all(_fans(f, w) == 1 for w in range(len(v)))


def test_entry_points_without_gpu():
    raw = _lib.load_library()
    assert 0 < raw.tpx_mesh_weld_workspace_bytes(100, 200) and raw.tpx_mesh_weld_workspace_bytes(1 << 31, 5) == 0
    assert 0 < raw.tpx_mesh_repair_workspace_bytes(100, 200) and raw.tpx_mesh_repair_workspace_bytes(5, 1 << 30) == 0
    V, F, _ = sphere(12)
    with pytest.raises(NotImplementedError):
        tpxl_b200.mesh.clean_mesh(V, F)                                     # remesh=True, the reference's default
    with pytest.raises(NotImplementedError):
        tpxl_b200.mesh.decimate_mesh(V, F, 100, optimalplacement=False)
    with pytest.raises(NotImplementedError):
        tpxl_b200.mesh.decimate_mesh(V, F, 100, remesh=True)
    with pytest.raises(NotImplementedError):
        tpxl_b200.mesh.decimate_mesh(V, F, 100, backend="pyfqmr")
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for fn in (lambda v, f: tpxl_b200.mesh.clean_mesh(v, f, min_f=8, min_d=5, remesh=False), lambda v, f: tpxl_b200.mesh.decimate_mesh(v, f, 10)):
        with pytest.raises(_lib.TpxError):
            fn(V, F)
        with pytest.raises(_lib.TpxError):
            fn(torch.from_numpy(V), torch.from_numpy(F))
    m = tpxl_b200.PrimSDF(num_prims=4).eval()
    with pytest.raises(_lib.TpxError):
        m.extract_mesh(8, merge_distance=0.01, repair=True)


def test_install_meshutils_binding():
    sys.modules.pop("utils.meshutils", None)
    tpxl_b200.install()
    assert "utils.meshutils" not in sys.modules
    try:
        tpxl_b200.install(meshutils=True)
        m = sys.modules["utils.meshutils"]
        assert m.clean_mesh is tpxl_b200.mesh.clean_mesh and m.decimate_mesh is tpxl_b200.mesh.decimate_mesh
        from utils.meshutils import clean_mesh, decimate_mesh  # noqa: F401
    finally:
        sys.modules.pop("utils.meshutils", None)


def test_clean_entries_check_device_first():
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses below must never reach a GPU")
    lib = _lib.load_library()
    P = 1 << 20                                    # non-null, 256-B aligned, never dereferenced
    wb, rb = lib.tpx_mesh_weld_workspace_bytes(3, 1), lib.tpx_mesh_repair_workspace_bytes(3, 1)
    calls = {"tpx_mesh_weld_count": (P, 3, P, 1, 0.01, P, wb, P, None), "tpx_mesh_weld_emit": (P, 3, 1, P, wb, P, P, None),
             "tpx_mesh_repair_count": (P, 3, P, 1, P, rb, P, None), "tpx_mesh_repair_emit": (P, 3, 1, P, rb, P, P, None)}
    for name, args in calls.items():
        rc = getattr(lib, name)(*args)
        assert rc == -2 and b"cudaGetDevice" in lib.tpx_last_error(), name
    assert lib.tpx_mesh_weld_count(P, 3, P, 1, -1.0, P, wb, P, None) == -1          # argument checks come first
    assert lib.tpx_mesh_repair_count(P, 3, P, 1, P, rb - 1, P, None) == -1
