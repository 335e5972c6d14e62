"""CPU: the isotropic remeshing oracle (oracle/remesh.py) on marching-cubes meshes — topology kept, features untouched, vertices on
the input, valence energy falling across the flips — small hand-built cases, and the entry points without a GPU."""
from collections import Counter

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph
import torch

from oracle import decimate as od
from oracle import remesh as orm
from tpxl_b200 import _lib, mesh

from test_decimate_host import MESHES


def _mean_edge(V, F):
    e = V[F].astype(np.float64)
    return float(np.linalg.norm(e - np.roll(e, -1, 1), axis=2).mean())


def _closed_oriented(F):
    """every directed edge appears once and its reverse once"""
    d = Counter(zip(F.ravel(), np.roll(F, -1, 1).ravel()))
    return all(c == 1 and d.get((b, a), 0) == 1 for (a, b), c in d.items())


def _euler_per_component(F):
    if len(F) == 0:
        return []
    V = int(F.max()) + 1
    a, b = F.ravel(), np.roll(F, -1, 1).ravel()
    g = scipy.sparse.coo_matrix((np.ones(len(a)), (a, b)), shape=(V, V))
    _, lab = scipy.sparse.csgraph.connected_components(g, directed=False)
    used = np.unique(F)
    E = np.unique(np.minimum(a, b) << 32 | np.maximum(a, b))
    out = []
    for c in np.unique(lab[used]):
        nv = int((lab[used] == c).sum())
        ne = int((lab[E >> 32] == c).sum())
        nf = int((lab[F[:, 0]] == c).sum())
        out.append(nv - ne + nf)
    return out


def _shares(V, F, L):
    """(share of edges in [4/5 L, 4/3 L], share of valence-6 vertices)"""
    a, b = F.ravel(), np.roll(F, -1, 1).ravel()
    E = np.unique(np.minimum(a, b) << 32 | np.maximum(a, b))
    ln = np.linalg.norm(V[E >> 32].astype(np.float64) - V[E & 0xFFFFFFFF].astype(np.float64), axis=1)
    val = np.bincount(np.concatenate([E >> 32, E & 0xFFFFFFFF]), minlength=len(V))
    return round(float(((ln >= 0.8 * L) & (ln <= 4 / 3 * L)).mean()), 3), round(float((val[np.unique(F)] == 6).mean()), 3)


def _segment_d2(p, a, b):
    ab = b - a
    t = np.clip(((p - a) * ab).sum(-1) / np.maximum((ab * ab).sum(-1), 1e-300), 0.0, 1.0)
    q = a + t[..., None] * ab
    return ((p - q) ** 2).sum(-1)


def _independent_distance(pts, P0, T0):
    """Distance from each point to the input surface: the orthogonal projection onto a face's plane when its barycentric coordinates
    are all >= 0, else the nearest point of the face's three edges; minimum over the faces of non-zero area.  Not the oracle's
    Ericson region walk."""
    tri = P0[T0].astype(np.float64)
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    n = np.cross(b - a, c - a)
    nn = (n * n).sum(1)
    live = nn > 0
    a, b, c, n, nn = a[live], b[live], c[live], n[live], nn[live]
    out = []
    for p in np.asarray(pts, np.float64):
        h = ((p - a) * n).sum(1) / nn
        q = p - h[:, None] * n
        w0 = (np.cross(b - q, c - q) * n).sum(1)
        w1 = (np.cross(c - q, a - q) * n).sum(1)
        w2 = (np.cross(a - q, b - q) * n).sum(1)
        inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
        d2 = np.where(inside, ((p - q) ** 2).sum(1), np.inf)
        d2 = np.minimum(d2, np.minimum(_segment_d2(p, a, b), np.minimum(_segment_d2(p, b, c), _segment_d2(p, c, a))))
        out.append(np.sqrt(d2.min()))
    return np.array(out)


def _features(V, F, feature_deg=30.0):
    P, T = od.check_mesh(V, F)
    C = orm.initial_creases(P, T, orm.params(1.0, feature_deg)[2])
    return orm.state(P, T, C)[-1]


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("scale", [0.6, 1.8])
def test_remesh_oracle_invariants(name, scale):
    V, F, _ = MESHES[name]()
    L = scale * _mean_edge(V, F)
    P0, T0 = od.check_mesh(V, F)
    feat0 = _features(V, F)
    for it in (1, 3):
        v, f, info = orm.remesh(V, F, L, it, record=True)
        assert len(info) == it
        assert not ((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 2] == f[:, 0])).any()
        assert _closed_oriented(f) == _closed_oriented(F)
        assert sorted(_euler_per_component(f)) == sorted(_euler_per_component(F))
        have = {tuple(p) for p in v.view(np.int32)}
        assert all(tuple(p) in have for p in P0[feat0].view(np.int32)), "a feature vertex moved or vanished"
        for r in info:
            assert r["energy"][1] <= r["energy"][0]
        # the projected vertices of every iteration (none where every vertex is a feature): each lands at the distance of the input's
        # closest point to its position before the projection, recomputed with an independent routine (plane projection, else the
        # nearest of the three edges), and on the input
        before = np.concatenate([r["projected"][1] for r in info])
        after = np.concatenate([r["projected"][2] for r in info])
        if len(before):
            sel = np.arange(len(before))[:: max(1, len(before) // 120)]
            got = np.linalg.norm(after[sel].astype(np.float64) - before[sel].astype(np.float64), axis=1)
            want, on = _independent_distance(before[sel], P0, T0), _independent_distance(after[sel], P0, T0)
            scale = max(1.0, float(np.abs(P0).max()))
            assert np.abs(got - want).max() < 1e-6 * scale and on.max() < 1e-6 * scale
        print(f"\n{name} L={L:.4g} it={it}: F {len(F)} -> {len(f)}; shares before {_shares(P0, T0, L)} after {_shares(v, f, L)}")


def test_zero_iterations_and_arguments():
    V, F, _ = MESHES["sphere"]()
    v, f = orm.remesh(V, F, 0.05, 0)
    w = od.compact(*od.check_mesh(V, F))
    assert np.array_equal(v, w[0]) and np.array_equal(f, w[1])
    for bad in (dict(target_len=0.0), dict(target_len=np.inf), dict(target_len=0.1, iterations=-1), dict(target_len=0.1, feature_deg=-1)):
        with pytest.raises(ValueError):
            orm.remesh(V, F, **bad)


def test_one_long_edge_split():
    V = np.array([[0, 0, 0], [4, 0, 0], [2, 1, 0], [2, -1, 0]], np.float32)
    F = np.array([[0, 1, 2], [1, 0, 3]], np.int64)
    P, T, C, ns = orm.split(V, F, np.zeros(0, np.int64), 3.0 ** 2)
    assert ns == 1 and len(P) == 5 and np.array_equal(P[4], [2, 0, 0])
    assert np.array_equal(T, [[0, 4, 2], [4, 1, 2], [1, 4, 3], [4, 0, 3]])


def _bipyramid(n=8, h=0.1):
    """Apex 0 at height h, apex 1 at -h, rim 2..n+1 on the unit circle counter-clockwise; outward winding, top fan first."""
    ang = 2 * np.pi * np.arange(n) / n
    V = np.concatenate([[[0, 0, h], [0, 0, -h]], np.stack([np.cos(ang), np.sin(ang), np.zeros(n)], 1)]).astype(np.float32)
    top = [[0, 2 + i, 2 + (i + 1) % n] for i in range(n)]
    bot = [[1, 2 + (i + 1) % n, 2 + i] for i in range(n)]
    return V, np.array(top + bot, np.int64)


def test_one_flip_quad():
    # apexes of valence 8, rim of valence 4: every spoke flip gains 2·8 - 12 = 4.  The smallest key is spoke (0, 2); every other
    # candidate touches one of its quad's vertices {0, 2, 3, 9}, so it is the one flip of the round.  Quad: x = 0, y = 2, faces
    # (0, 2, 3) (slot 0, c = 3) and (0, 9, 2) (slot 7, d = 9) become (x, d, c) = (0, 9, 3) and (d, y, c) = (9, 2, 3).
    V, F = _bipyramid()
    assert _closed_oriented(F)
    T, k = orm.flip_round(V, F, np.zeros(0, np.int64), np.cos(np.radians(30)))
    assert k == 1
    want = F.copy()
    want[0], want[7] = [0, 9, 3], [9, 2, 3]
    assert np.array_equal(T, want)
    assert _closed_oriented(T)
    assert orm.valence_energy(T, len(V)) == orm.valence_energy(F, len(V)) - 4


def _antiprism(r=0.06):
    """Equator triangle e = 0, 1, 2 (radius r, not a face), upper triangle u = 3, 4, 5 and lower triangle l = 6, 7, 8 (radius 1, z = ±1)
    joined to it by antiprism bands: a closed surface where the equator's vertices have valence 6 and the others 4."""
    e = [[r * np.cos(a), r * np.sin(a), 0] for a in np.radians([0, 120, 240])]
    u = [[np.cos(a), np.sin(a), 1] for a in np.radians([60, 180, 300])]
    lo = [[np.cos(a), np.sin(a), -1] for a in np.radians([60, 180, 300])]
    V = np.array(e + u + lo, np.float32)
    F = [[3, 4, 5], [6, 8, 7]]
    for i in range(3):
        j = (i + 1) % 3
        F += [[i, j, 3 + i], [j, 3 + j, 3 + i], [j, i, 6 + i], [j, 6 + i, 6 + j]]
    return V, np.array(F, np.int64)


def test_collapse_blocked_by_link_condition():
    # the equator edges are the only short edges; each has the third equator vertex as a common neighbour besides the two opposite
    # vertices, while every other rule holds: not features, degrees 6 + 6 >= 7 and 4, 4 >= 4, short, star normals kept
    V, F = _antiprism()
    assert _closed_oriented(F)
    lo2, hi2 = 0.2 ** 2, 10.0 ** 2
    FACE, OUT, IN, n, frozen, deg, feat = orm.state(V, F, np.zeros(0, np.int64))
    assert not feat.any() and list(deg) == [6, 6, 6] + [4] * 6
    E = orm._edges(F)
    short = E[orm._len2(V[E >> 32], V[E & orm.M32]) < lo2]
    assert sorted(short.tolist()) == [0 << 32 | 1, 0 << 32 | 2, 1 << 32 | 2]
    a, b = np.array([0, 0, 1]), np.array([1, 2, 2])
    mid = ((V[a].astype(np.float64) + V[b]) * 0.5).astype(np.float32)
    assert od._star_ok(V, F, FACE, n, b, a, mid).all() and od._star_ok(V, F, FACE, n, a, b, mid).all()
    P, T, k = orm.collapse_round(V, F, np.zeros(0, np.int64), lo2, hi2)
    assert k == 0 and np.array_equal(T, F)
    # what fails is the link: N(0) ∩ N(1) = {2, c, d}, one more than the two vertices opposite the edge
    nb = lambda v: set(OUT[v, :n[v]].tolist())                                 # noqa: E731 (closed fans: OUT lists every neighbour)
    assert nb(0) & nb(1) == {2, 3, 6}


def test_entry_points_without_gpu():
    raw = _lib.load_library()
    assert 0 < raw.tpx_remesh_workspace_bytes(100, 200) and raw.tpx_remesh_workspace_bytes(1 << 31, 5) == 0
    assert 0 < raw.tpx_remesh_grid_bytes(200) and raw.tpx_remesh_grid_bytes(1 << 31) == 0
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    V, F, _ = MESHES["sphere"]()
    with pytest.raises(_lib.TpxError):
        mesh.remesh(V, F, 0.05)
    with pytest.raises(_lib.TpxError):
        mesh.remesh(torch.from_numpy(V), torch.from_numpy(F), 0.05)


def test_remesh_entries_check_device_first():
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses below must never reach a GPU")
    lib = _lib.load_library()
    P = 1 << 20                                    # non-null, 256-B aligned, never dereferenced
    wb, gb = lib.tpx_remesh_workspace_bytes(3, 1), lib.tpx_remesh_grid_bytes(1)
    calls = {"tpx_remesh_begin": (P, 3, P, 1, 0.5, P, gb, P, wb, P, P, None),
             "tpx_remesh_split_count": (P, 3, P, 1, P, 0, 0.1, P, wb, P, None),
             "tpx_remesh_split_emit": (P, 3, 1, P, 0, 0, P, wb, P, P, P, None),
             "tpx_remesh_relax": (P, 3, P, 1, P, 0, P, 3, 1, P, gb, 0.1, 0.5, P, wb, P, None)}
    for name, args in calls.items():
        rc = getattr(lib, name)(*args)
        assert rc == -2 and b"cudaGetDevice" in lib.tpx_last_error(), name
    assert lib.tpx_remesh_split_count(P, 3, P, 1, P, 0, -0.1, P, wb, P, None) == -1   # argument checks come first
    assert lib.tpx_remesh_begin(P, 3, P, 1, 0.5, P, gb - 1, P, wb, P, P, None) == -1
