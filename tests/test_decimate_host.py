"""CPU: the decimation and component-filter oracle (oracle/decimate.py) on marching-cubes meshes — topology kept, targets met, rounds
independent, fixed vertices untouched, labels equal to scipy's — and the entry points without a GPU."""
from collections import Counter

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph
import torch

import tpxl_b200
from oracle import decimate as od
from oracle import mesh as omesh
from tpxl_b200 import _lib


def _grid(R):
    g = np.linspace(-1, 1, R)
    return np.meshgrid(g, g, g, indexing="ij")


def _world(V, R):
    return (V / (R - 1) * 2 - 1).astype(np.float32)


def sphere(R=28, r=0.6):
    x, y, z = _grid(R)
    V, F = omesh.marching_cubes(np.sqrt(x * x + y * y + z * z) - r)
    return _world(V, R), F, lambda p: p


def torus(R=32, a=0.55, b=0.22):
    x, y, z = _grid(R)
    V, F = omesh.marching_cubes(np.sqrt((np.sqrt(x * x + y * y) - a) ** 2 + z * z) - b)

    def grad(p):
        q = np.sqrt(p[:, 0] ** 2 + p[:, 1] ** 2)
        c = np.stack([p[:, 0] / q * a, p[:, 1] / q * a, np.zeros(len(p))], 1)
        return p - c
    return _world(V, R), F, grad


def two_spheres(R=30):
    x, y, z = _grid(R)
    d1 = np.sqrt((x - 0.45) ** 2 + y * y + z * z) - 0.35
    d2 = np.sqrt((x + 0.5) ** 2 + y * y + z * z) - 0.3
    V, F = omesh.marching_cubes(np.minimum(d1, d2))
    W = _world(V, R)

    def grad(p):
        c = np.where((p[:, 0] > 0)[:, None], [0.45, 0, 0], [-0.5, 0, 0])
        return p - c
    return W, F, grad


def open_field(shape=(20, 22, 18), seed=4):
    """Smooth random field whose surface runs into the volume's faces: an open mesh with boundary loops."""
    rng = np.random.default_rng(seed)
    g = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    f = np.zeros(shape)
    for _ in range(5):
        k = rng.normal(size=3) * 0.3
        f += np.sin(sum(k[d] * g[d] for d in range(3)) + rng.uniform(0, 2 * np.pi))
    V, F = omesh.marching_cubes(f.astype(np.float32))
    return V.astype(np.float32), F, None


def integer_field(shape=(12, 11, 10), seed=3):
    """Values in {-2..2} with iso 0 on lattice points: coincident vertices and zero-area faces; border outside, so closed."""
    vol = np.random.default_rng(seed).integers(-2, 3, size=shape).astype(np.float32)
    vol[[0, -1]] = 1
    vol[:, [0, -1]] = 1
    vol[:, :, [0, -1]] = 1
    V, F = omesh.marching_cubes(vol)
    return V.astype(np.float32), F, None


MESHES = {"sphere": sphere, "torus": torus, "two_spheres": two_spheres, "open_field": open_field, "integer": integer_field}


def directed_edges(F):
    d = Counter()
    for a, b, c in F.tolist():
        for u, v in ((a, b), (b, c), (c, a)):
            d[(u, v)] += 1
    return d


def is_closed_oriented(F):
    d = directed_edges(F)
    return bool(d) and all(n == 1 and d.get((v, u), 0) == 1 for (u, v), n in d.items())


def boundary_vertices(F):
    und = Counter()
    for (u, v), n in directed_edges(F).items():
        und[(min(u, v), max(u, v))] += n
    return sorted({w for e, n in und.items() if n != 2 for w in e})


def euler(V, F):
    e = {(min(u, v), max(u, v)) for (u, v) in directed_edges(F)}
    return len(np.unique(F)) - len(e) + len(F)


def n_components(F):
    return len(np.unique(od.component_labels(F)))


@pytest.mark.parametrize("name", sorted(MESHES))
def test_oracle_decimation_keeps_topology_and_meets_target(name):
    V, F, grad = MESHES[name]()
    closed = is_closed_oriented(F)
    assert closed or name == "open_field"
    bverts = boundary_vertices(F)
    assert bool(bverts) == (name == "open_field")
    chi, ncomp = euler(V, F), n_components(F)
    for frac in (0.5, 0.1):
        T = int(len(F) * frac)
        v, f, rounds = od.decimate(V, F, T, record=True)
        assert v.dtype == np.float32 and f.dtype == np.int64
        if len(f) > T:                          # boundary vertices stay fixed: a mesh with long borders can run out of collapses
            assert name == "open_field" and frac == 0.1 and rounds[-1]["F"] == len(f), (name, T, len(f))
        else:
            assert len(f) in (T - 1, T), (name, T, len(f))
        assert len(np.unique(f)) == len(v) and f.min() == 0 and f.max() == len(v) - 1
        if closed:
            assert is_closed_oriented(f)
        assert euler(v, f) == chi and n_components(f) == ncomp
        # every round's collapses have disjoint stars (no face holds vertices of two accepted edges)
        for r in rounds:
            owner = np.full(len(V), -1)
            for i, (a, b) in enumerate(r["accepted"]):
                owner[a] = owner[b] = i
            o = owner[r["faces"]]
            o = np.where(o < 0, np.iinfo(np.int64).max, o)
            mn = o.min(1)
            assert ((o == mn[:, None]) | (o == np.iinfo(np.int64).max)).all(), name
        assert [r["F"] for r in rounds] == sorted((r["F"] for r in rounds), reverse=True)
        # boundary vertices are never moved or removed
        if bverts:
            have = {tuple(p) for p in v.view(np.int32).tolist()}
            assert all(tuple(V[w].view(np.int32).tolist()) in have for w in bverts)
        if grad is not None:
            p = v[f].astype(np.float64)
            n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
            dots = np.einsum("ij,ij->i", n, grad(p.mean(1)))
            assert (dots[np.abs(n).sum(1) > 0] > 0).all(), (name, frac)


def test_oracle_unreachable_target_and_small_meshes():
    V, F, _ = sphere()
    v, f, rounds = od.decimate(V, F, 1, record=True)
    assert len(f) == 4 and is_closed_oriented(f)                      # down to a tetrahedron, which no collapse may reduce
    v2, f2 = od.decimate(V, F, len(F))
    assert np.array_equal(v2, V) and np.array_equal(f2, F)           # target >= F: the input
    tet_v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    tet_f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    assert is_closed_oriented(tet_f)
    v3, f3 = od.decimate(tet_v, tet_f, 0)
    assert np.array_equal(f3, tet_f) and np.array_equal(v3, tet_v)


def fin_and_pinch():
    """A sphere with a fin (a third face on one edge: both ends non-manifold, its apex a boundary vertex), and two spheres sharing
    one vertex (two fans at it)."""
    V, F, _ = sphere(24)
    a, b = F[0, 0], F[0, 1]
    apex = len(V)
    Vf = np.concatenate([V, (V[a] + V[b])[None] * 0.6])
    Ff = np.concatenate([F, [[a, apex, b]]])
    V2 = V + np.float32(1.3) * np.array([1, 0, 0], np.float32)
    j = int(np.argmax(V[:, 0]))                                       # rightmost vertex of the first sphere
    k = int(np.argmin(V2[:, 0]))                                      # leftmost of the second
    V2[k] = V[j]
    F2 = F + len(V)
    F2[F2 == k + len(V)] = j
    Vp = np.concatenate([V, V2])
    Fp = np.concatenate([F, F2])
    return (Vf, Ff, [a, b, apex]), (Vp, Fp, [j])


def test_oracle_fixed_vertices_are_kept_bit_for_bit():
    for Vm, Fm, fixed in fin_and_pinch():
        frozen, _ = od.vertex_state(*od._corners(Fm, len(Vm))[1:4])
        assert frozen[fixed].all()
        v, f = od.decimate(Vm, Fm, len(Fm) // 5)
        assert len(f) < len(Fm) // 4
        have = {tuple(p) for p in v.view(np.int32).tolist()}
        for w in fixed:
            assert tuple(Vm[w].view(np.int32).tolist()) in have


def test_oracle_component_labels_match_scipy():
    V1, F1, _ = two_spheres()
    V2, F2, _ = integer_field((10, 9, 11), 7)
    V3, F3, _ = open_field((14, 12, 13), 9)
    for V, F in ((V1, F1), (V2, F2), (V3, F3)):
        lab = od.component_labels(F)
        e = np.concatenate([np.minimum(F, np.roll(F, -1, 1)), np.maximum(F, np.roll(F, -1, 1))], 1)
        key = (e[:, :3] << 32 | e[:, 3:]).ravel()
        fid = np.repeat(np.arange(len(F)), 3)
        order = np.lexsort((fid, key))
        same = key[order][1:] == key[order][:-1]
        u, w = fid[order][:-1][same], fid[order][1:][same]
        g = scipy.sparse.coo_matrix((np.ones(len(u)), (u, w)), shape=(len(F), len(F)))
        n, sl = scipy.sparse.csgraph.connected_components(g, directed=False)
        assert len(np.unique(lab)) == n
        for c in range(n):                                            # same partition, labelled by the smallest face id
            members = np.flatnonzero(sl == c)
            assert (lab[members] == members.min()).all()


def test_oracle_component_filter():
    V, F, _ = two_spheres()
    lab = od.component_labels(F)
    sizes = Counter(lab.tolist())
    assert len(sizes) == 2
    small = min(sizes.values())
    v, f = od.remove_small_components(V, F, min_faces=small + 1, min_diameter=0.0)
    assert len(f) == len(F) - small and is_closed_oriented(f)
    v, f = od.remove_small_components(V, F, min_faces=0, min_diameter=0.99)
    assert len(f) == 0 and len(v) == 0
    v, f = od.remove_small_components(V, F, min_faces=8, min_diameter=0.05)
    assert np.array_equal(v, V) and np.array_equal(f, F)
    with pytest.raises(ValueError):
        od.remove_small_components(V, np.array([[0, 1, len(V)]]))
    with pytest.raises(ValueError):
        od.decimate(V, np.array([[0, 1, 1]]), 0)


def test_entry_points_without_gpu():
    raw = _lib.load_library()
    n = raw.tpx_decimate_workspace_bytes(4_100_000, 8_200_000)
    assert 100 * 8_200_000 < n < 400 * 8_200_000
    assert 0 < raw.tpx_mesh_components_workspace_bytes(100, 200) and raw.tpx_decimate_workspace_bytes(100, 1 << 31) == 0
    assert raw.tpx_mesh_components_workspace_bytes(1 << 31, 5) == 0
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    V, F, _ = sphere(12)
    for fn in (lambda v, f: tpxl_b200.mesh.decimate(v, f, 10), lambda v, f: tpxl_b200.mesh.remove_small_components(v, f)):
        with pytest.raises(_lib.TpxError):
            fn(V, F)
        with pytest.raises(_lib.TpxError):
            fn(torch.from_numpy(V), torch.from_numpy(F))
    m = tpxl_b200.PrimSDF(num_prims=4).eval()
    with pytest.raises(_lib.TpxError):
        m.extract_mesh(8, min_faces=8, min_diameter=0.05, target_faces=100)
