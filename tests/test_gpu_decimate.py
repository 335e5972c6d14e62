"""-m gpu: mesh clean-up and decimation (csrc/mesh_simplify.cu through tpxl_b200.mesh) against the numpy oracle, byte for byte, and
PrimSDF.extract_mesh(min_faces, min_diameter, target_faces) on the synthetic shell at R = 256 -> 100 000 faces."""
import numpy as np
import pytest
import torch

from oracle import decimate as od
from tpxl_b200 import _lib, mesh

from test_decimate_host import MESHES, fin_and_pinch
from test_gpu_mesh import _shell_module
from parity import same_mesh

pytestmark = pytest.mark.gpu


def _cuda(V, F):
    return torch.from_numpy(np.ascontiguousarray(V, np.float32)).cuda(), torch.from_numpy(np.ascontiguousarray(F, np.int64)).cuda()


@pytest.mark.parametrize("name", sorted(MESHES))
def test_decimate_matches_oracle(name):
    V, F, _ = MESHES[name]()
    dv, df = _cuda(V, F)
    side = torch.cuda.Stream()
    for T in (len(F) // 2, len(F) // 10, 1):
        want = od.decimate(V, F, T)
        got = mesh.decimate(dv, df, T)
        same_mesh(got, want)
        again = mesh.decimate(dv, df, T)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            other = mesh.decimate(dv, df, T)
        torch.cuda.current_stream().wait_stream(side)
        for v, f in (again, other):
            assert torch.equal(v, got[0]) and torch.equal(f, got[1]), f"{name} T={T}: repeated call differs"


def test_fixed_vertices_and_small_cases_match_oracle():
    for Vm, Fm, _ in fin_and_pinch():
        same_mesh(mesh.decimate(*_cuda(Vm, Fm), len(Fm) // 5), od.decimate(Vm, Fm, len(Fm) // 5))
    tet_v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    tet_f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    same_mesh(mesh.decimate(*_cuda(tet_v, tet_f), 0), (tet_v, tet_f))
    V, F, _ = MESHES["sphere"]()
    same_mesh(mesh.decimate(*_cuda(V, F), len(F)), (V, F))
    v, f = mesh.decimate(V, F, len(F) // 3)                              # numpy in, numpy out
    want = od.decimate(V, F, len(F) // 3)
    assert v.dtype == np.float64 and f.dtype == np.int64
    assert np.array_equal(v, want[0].astype(np.float64)) and np.array_equal(f, want[1])
    e = mesh.decimate(torch.zeros(0, 3, device="cuda"), torch.zeros(0, 3, dtype=torch.int64, device="cuda"), 0)
    assert e[0].shape == (0, 3) and e[1].shape == (0, 3)


@pytest.mark.parametrize("name", sorted(MESHES))
def test_component_filter_matches_oracle(name):
    V, F, _ = MESHES[name]()
    dv, df = _cuda(V, F)
    lab = od.component_labels(F)
    sizes = np.bincount(lab, minlength=len(F))
    for mf, md in ((8, 0.05), (int(sizes[sizes > 0].min()) + 1, 0.0), (0, 0.4), (0, 2.0)):
        want = od.remove_small_components(V, F, mf, md)
        got = mesh.remove_small_components(dv, df, mf, md)
        same_mesh(got, want)
        assert all(torch.equal(a, b) for a, b in zip(got, mesh.remove_small_components(dv, df, mf, md)))
    # many small pieces: the two spheres plus copies of a tiny tetrahedron, interleaved in face order
    tet_v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32) * 0.01
    Vs, Fs = [V], [F]
    for i in range(20):
        Vs.append(tet_v + np.float32(0.05 * i - 0.5))
        Fs.append(np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]]) + sum(len(x) for x in Vs[:-1]))
    Vc, Fc = np.concatenate(Vs), np.concatenate(Fs)
    perm = np.random.default_rng(1).permutation(len(Fc))
    same_mesh(mesh.remove_small_components(*_cuda(Vc, Fc[perm]), 8, 0.05), od.remove_small_components(Vc, Fc[perm], 8, 0.05))


def test_invalid_input_raises():
    V, F, _ = MESHES["sphere"]()
    dv, df = _cuda(V, F)
    bad_range = df.clone()
    bad_range[5, 1] = len(V)
    bad_neg = df.clone()
    bad_neg[0, 0] = -1
    bad_rep = df.clone()
    bad_rep[3, 2] = bad_rep[3, 0]
    for fn in (lambda v, f: mesh.decimate(v, f, 10), lambda v, f: mesh.remove_small_components(v, f)):
        for f in (bad_range, bad_neg, bad_rep, df[:, :2], df.int()):
            with pytest.raises(ValueError):
                fn(dv, f)
        with pytest.raises(ValueError):
            fn(dv.double(), df)
        with pytest.raises(_lib.TpxError):
            fn(dv.cpu(), df.cpu())
    with pytest.raises(ValueError):
        mesh.decimate(dv, df, -1)
    # the C entry points check the faces themselves too
    lib = _lib.lib()
    n = int(lib.tpx_decimate_workspace_bytes(len(V), len(F)))
    ws = torch.empty(n, dtype=torch.uint8, device="cuda")
    counts = torch.empty(3, dtype=torch.int64, device="cuda")
    rc = lib.tpx_decimate(dv.data_ptr(), len(V), bad_rep.data_ptr(), len(F), 10, ws.data_ptr(), n, counts.data_ptr(), None, 0, _lib.stream_ptr())
    assert rc == -1 and b"repeated" in lib.tpx_last_error()
    n = int(lib.tpx_mesh_components_workspace_bytes(len(V), len(F)))
    ws = torch.empty(n, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tpx_mesh_components_count(dv.data_ptr(), len(V), bad_range.data_ptr(), len(F), 8, 0.05, ws.data_ptr(), n, counts.data_ptr(),
                                             _lib.stream_ptr()))
    assert counts[:2].tolist() == [-1, -1]


def _chi_per_component(F):
    """Sorted Euler characteristics V - E + F of the edge-connected components of F (numpy / scipy, for meshes of millions of faces)."""
    import scipy.sparse
    import scipy.sparse.csgraph
    e = np.stack([np.minimum(F, np.roll(F, -1, 1)), np.maximum(F, np.roll(F, -1, 1))], 2).reshape(-1, 2)
    key = e[:, 0] << 32 | e[:, 1]
    fid = np.repeat(np.arange(len(F)), 3)
    order = np.argsort(key, kind="stable")
    same = key[order][1:] == key[order][:-1]
    u, w = fid[order][:-1][same], fid[order][1:][same]
    g = scipy.sparse.coo_matrix((np.ones(len(u), np.int8), (u, w)), shape=(len(F), len(F)))
    n, lab = scipy.sparse.csgraph.connected_components(g, directed=False)
    nf = np.bincount(lab, minlength=n)
    _, first = np.unique(key, return_index=True)
    ne = np.bincount(lab[fid[first]], minlength=n)
    _, firstv = np.unique(F.ravel(), return_index=True)
    nv = np.bincount(lab[fid[firstv]], minlength=n)
    return sorted((nv - ne + nf).tolist())


def _orientation(F):
    """(every directed edge occurs once, number of directed edges whose reverse is missing) in numpy, for large meshes."""
    a, b = F.ravel(), np.roll(F, -1, 1).ravel()
    key = a << 32 | b
    u = np.unique(key)
    return len(u) == len(key), int((~np.isin(b << 32 | a, u)).sum())


def _trilinear(grid, p, R):
    """grid [R,R,R] on linspace(-1, 1, R)^3 sampled at world points p [n,3] (float64 numpy)."""
    u = np.clip((p + 1) / 2 * (R - 1), 0, R - 1 - 1e-9)
    i = np.floor(u).astype(np.int64)
    t = u - i
    out = np.zeros(len(p))
    for c in range(8):
        o = np.array([(c >> 2) & 1, (c >> 1) & 1, c & 1])
        w = np.prod(np.where(o[None] == 1, t, 1 - t), 1)
        out += w * grid[i[:, 0] + o[0], i[:, 1] + o[1], i[:, 2] + o[2]]
    return out


def _gradient(grid, p, R):
    h = 2.0 / (R - 1)
    g = np.zeros_like(p)
    for d in range(3):
        e = np.zeros(3)
        e[d] = 0.5 * h
        g[:, d] = _trilinear(grid, p + e, R) - _trilinear(grid, p - e, R)
    return g


def test_shell_r256_filtered_and_decimated_to_100k():
    m = _shell_module()
    R = 256
    grid = m.sdf_grid(R)
    v0, f0 = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
    v1, f1 = mesh.remove_small_components(v0, f0, 8, 0.05)
    trace = []
    v2, f2 = mesh._decimate(v1, f1, 100000, trace)
    ve, fe = m.extract_mesh(R, min_faces=8, min_diameter=0.05, target_faces=100000)
    assert torch.equal(ve, v2) and torch.equal(fe, f2), "extract_mesh differs from the explicit chain"
    assert torch.equal(m.extract_mesh(R)[1], f0)                           # default arguments: marching cubes only
    F = f2.shape[0]
    print(f"R=256: F {f0.shape[0]} -> filtered {f1.shape[0]} -> {F} in {len(trace)} rounds")
    # The synthetic shell is random per-voxel detail: its filtered mesh has a genus in the thousands, and collapses that keep the
    # topology cannot remove a handle, so the run stops above 100 000 when a round finds no valid collapse (measured on an H100:
    # 8 203 241 -> 203 997 faces in 377 rounds).  A reachable target ends at T - 1 or T.
    assert F in (99999, 100000) or (F > 100000 and trace[-1] == F and F <= 250000), F
    fn = f2.cpu().numpy()
    # the shell's field is negative on parts of the box faces, so the marching-cubes mesh has borders there: oriented in and out,
    # and the border (whose vertices are frozen) is kept edge for edge
    o_in, b_in = _orientation(f1.cpu().numpy())
    o_out, b_out = _orientation(fn)
    assert o_in and o_out and b_in == b_out and b_in > 0, (o_in, o_out, b_in, b_out)
    chi_in, chi_out = _chi_per_component(f1.cpu().numpy()), _chi_per_component(fn)      # one characteristic per component, unchanged
    assert chi_in == chi_out, (chi_in[:10], chi_out[:10])
    # error figures, reported rather than bounded here: the shell's sdf is not a distance (|grad| is about 36 per unit length), so
    # |sdf| / voxel overstates the distance to the surface by that factor, and its voxel-scale noise is finer than the output triangles
    g = grid.cpu().numpy().astype(np.float64)
    p = v2.cpu().numpy().astype(np.float64)
    tri = p[fn]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    agree = float((np.einsum("ij,ij->i", n, _gradient(g, tri.mean(1), R)) > 0).mean())
    err = np.abs(_trilinear(g, p, R)) / (2.0 / 255)
    print(f"normals agreeing with the grid gradient: {agree:.5f}; |sdf| at vertices: mean {err.mean():.4f} max {err.max():.3f} voxels")
    assert np.isfinite(p).all()
