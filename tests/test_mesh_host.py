"""CPU: the generated marching-cubes case table, the oracle mesh (tests/golden/primsdf_grid.npz, closedness, orientation, vertex
contract, exact-iso values), the mcubes binding of install(), and the mesh entry points without a GPU."""
import itertools
import os
import sys
from collections import Counter

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import mesh as omesh
from tpxl_b200 import _lib, mc_table

CORN = np.array([(n & 1, (n >> 1) & 1, (n >> 2) & 1) for n in range(8)])


def test_committed_header_is_the_generator_output():
    assert open(mc_table.HEADER).read() == mc_table.render(), "csrc/mc_tables.cuh is stale: run python 3dtopia-xl_b200/mc_table.py"
    edges, count, owner, axis = omesh.load_table()
    assert edges.shape[0] == 256 and count.shape == (256,)
    assert count[0] == 0 and count[255] == 0
    header = open(mc_table.HEADER).read()
    kernel_max = int(header.split("constexpr int kMcMaxTris = ", 1)[1].split(";")[0])
    assert int(count.max()) == kernel_max == edges.shape[1]
    for c in range(256):
        assert (edges[c, :count[c]] >= 0).all() and (edges[c, count[c]:] == -1).all()
    # edge e joins owner corner and owner | 1 << axis: all 12 distinct unit edges of the cube
    pairs = {(int(o), int(o) | (1 << int(a))) for o, a in zip(owner, axis)}
    assert len(pairs) == 12 and all(((o >> int(a)) & 1) == 0 for o, a in zip(owner, axis))


def _face_segments_from_signs(inside, face):
    """Segments a face must carry, from its 4 corner signs alone: 2 crossings -> that pair; 4 -> the two pairs around each inside corner."""
    cyc = face
    ring = [(cyc[i], cyc[(i + 1) % 4]) for i in range(4)]
    cross = [e for e in ring if inside[e[0]] != inside[e[1]]]
    key = lambda e: (min(e), max(e))  # noqa: E731
    if len(cross) == 2:
        return {frozenset(map(key, cross))}
    if len(cross) == 4:
        segs = set()
        for c in cyc:
            if inside[c]:
                segs.add(frozenset(key(e) for e in ring if c in e))
        return segs
    return set()


def test_no_triangle_chord_lies_in_a_cube_face_unless_it_is_a_face_segment():
    edges, count, owner, axis = omesh.load_table()
    corner_pair = [(int(o), int(o) | (1 << int(a))) for o, a in zip(owner, axis)]
    faces = []
    for ax in range(3):
        u, v = [a for a in range(3) if a != ax]
        for side in (0, 1):
            cs = [n for n in range(8) if CORN[n][ax] == side]
            order = [(0, 0), (1, 0), (1, 1), (0, 1)]
            faces.append(sorted(cs, key=lambda n: order.index((CORN[n][u], CORN[n][v]))))
    for c in range(256):
        inside = [(c >> n) & 1 for n in range(8)]
        for tri in edges[c, :count[c]]:
            for a, b in ((tri[0], tri[1]), (tri[1], tri[2]), (tri[2], tri[0])):
                ea, eb = corner_pair[a], corner_pair[b]
                for f in faces:
                    if set(ea) <= set(f) and set(eb) <= set(f):
                        assert frozenset((ea, eb)) in _face_segments_from_signs(inside, f), (c, ea, eb)


def _check_closed_oriented(F):
    d = Counter()
    for a, b, c in F.tolist():
        for u, v in ((a, b), (b, c), (c, a)):
            d[(u, v)] += 1
    assert d, "empty mesh"
    for (u, v), n in d.items():
        assert n == 1 and d.get((v, u), 0) == 1, (u, v, n)


def _expected_vertices(vol, iso):
    """Straight loop over the lattice: sign-changing edges in (point, axis) order and their positions."""
    X, Y, Z = vol.shape
    out = []
    for i, j, k in itertools.product(range(X), range(Y), range(Z)):
        for a in range(3):
            q = [i, j, k]
            q[a] += 1
            if q[a] >= vol.shape[a]:
                continue
            f0, f1 = float(vol[i, j, k]), float(vol[tuple(q)])
            if (f0 < iso) != (f1 < iso):
                p = [float(i), float(j), float(k)]
                p[a] += (iso - f0) / (f1 - f0)
                out.append(p)
    return np.array(out).reshape(-1, 3)


def test_oracle_random_fields_are_closed_oriented_and_cover_all_cases():
    rng = np.random.default_rng(0)
    cases = set()
    for n, (X, Y, Z) in enumerate([(10, 10, 10)] * 12 + [(7, 12, 9), (5, 5, 16)]):
        vol = rng.standard_normal((X, Y, Z)).astype(np.float32)
        vol[[0, -1]] = 1.0
        vol[:, [0, -1]] = 1.0
        vol[:, :, [0, -1]] = 1.0
        iso = 0.0 if n % 2 == 0 else 0.25
        cases |= set(omesh.cube_cases(vol, iso).ravel().tolist())
        V, F = omesh.marching_cubes(vol, iso)
        assert F.dtype == np.int64 and V.dtype == np.float64
        _check_closed_oriented(F)
        assert len(np.unique(F)) == len(V)                      # every vertex is used (border outside: no open edges)
        np.testing.assert_allclose(V, _expected_vertices(vol, iso), rtol=0, atol=1e-12)
    assert cases == set(range(256))


def test_oracle_sphere_volume_and_normals():
    R, r = 40, 0.6
    g = np.linspace(-1, 1, R)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    V, F = omesh.marching_cubes(np.sqrt(x * x + y * y + z * z) - r, 0.0)
    _check_closed_oriented(F)
    W = V / (R - 1) * 2 - 1
    a, b, c = W[F[:, 0]], W[F[:, 1]], W[F[:, 2]]
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6
    exact = 4 / 3 * np.pi * r ** 3
    assert vol > 0 and abs(vol - exact) < 0.01 * exact, (vol, exact)
    normal = np.cross(b - a, c - a)
    grad = (a + b + c) / 3
    assert (np.einsum("ij,ij->i", normal, grad) > 0).mean() >= 0.99


def test_oracle_values_equal_to_iso_are_outside():
    rng = np.random.default_rng(3)
    vol = rng.integers(-2, 3, size=(9, 8, 7)).astype(np.float32)
    V, F = omesh.marching_cubes(vol, 0.0)
    assert np.isfinite(V).all() and len(F) > 0
    np.testing.assert_allclose(V, _expected_vertices(vol, 0.0), rtol=0, atol=1e-12)
    t = V - np.floor(V)
    on_lattice = np.isclose(V, np.round(V))
    assert ((t >= 0) & (t <= 1)).all()
    # a vertex can reach a lattice point only at the end whose value equals iso (t = 0 or 1): that end is the outside one
    assert on_lattice.all(1).any()
    for v in V[on_lattice.all(1)]:
        assert vol[tuple(np.round(v).astype(int))] == 0.0


def test_oracle_reproduces_reference_grid(golden_dir):
    import oracle
    g = np.load(os.path.join(golden_dir, "primsdf_grid.npz"))
    R = g["grid"].shape[0]
    xx = torch.linspace(-1, 1, R)
    pts = torch.stack(torch.meshgrid(xx, xx, xx, indexing="ij"), -1).reshape(-1, 3)
    out = oracle.primsdf.query(pts, torch.from_numpy(g["srt"]), torch.from_numpy(g["feat"]), S=8, dim_feat=6, inference=True)
    np.testing.assert_allclose(out["sdf"].reshape(R, R, R).numpy(), g["grid"], rtol=2e-5, atol=2e-5)
    V, F = omesh.marching_cubes(g["grid"], 0.0)
    assert len(F) > 1000
    _check_closed_oriented(F)


def test_install_binds_mcubes_only_on_request():
    saved = sys.modules.pop("mcubes", None)
    try:
        tpxl_b200.install()
        assert "mcubes" not in sys.modules
        sentinel = object()
        sys.modules["mcubes"] = sentinel
        tpxl_b200.install()
        assert sys.modules["mcubes"] is sentinel
        tpxl_b200.install(mcubes=True)
        import mcubes
        assert mcubes.marching_cubes is tpxl_b200.mesh.marching_cubes
    finally:
        sys.modules.pop("mcubes", None)
        if saved is not None:
            sys.modules["mcubes"] = saved


def test_entry_points_without_gpu():
    raw = _lib.load_library()
    n = raw.tpx_mc_workspace_bytes(512, 512, 512)
    assert 6 * 512 ** 3 < n <= 8 * 512 ** 3                      # about 6 bytes per grid point: R = 512 fits in about 1 GB
    assert raw.tpx_mc_workspace_bytes(1, 5, 5) == 0 and raw.tpx_mc_workspace_bytes(1291, 1291, 1291) == 0
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.TpxError):
        tpxl_b200.mesh.marching_cubes(np.zeros((4, 4, 4), np.float32))
    with pytest.raises(_lib.TpxError):
        tpxl_b200.mesh.marching_cubes(torch.zeros(4, 4, 4))
    with pytest.raises(ValueError):
        tpxl_b200.mesh.marching_cubes(np.zeros((4, 4), np.float32))
    m = tpxl_b200.PrimSDF(num_prims=4).eval()
    with pytest.raises(_lib.TpxError):
        m.sdf_grid(8)
    with pytest.raises(_lib.TpxError):
        m.extract_mesh(8)
