"""-m gpu: isotropic remeshing (csrc/mesh_remesh.cu through tpxl_b200.mesh.remesh) against the numpy oracle (oracle/remesh.py), byte
for byte, and PrimSDF.extract_mesh(remesh_pct=) / extract_texmesh(remesh=) on the synthetic shell."""
import numpy as np
import pytest
import torch

from oracle import decimate as od
from oracle import remesh as orm
from tpxl_b200 import _lib, mesh

from test_decimate_host import MESHES
from test_gpu_mesh import _shell_module
from parity import same_mesh
from test_remesh_host import _closed_oriented, _euler_per_component, _mean_edge, _shares

pytestmark = pytest.mark.gpu


def _cuda(V, F):
    return torch.from_numpy(np.ascontiguousarray(V, np.float32)).cuda(), torch.from_numpy(np.ascontiguousarray(F, np.int64)).cuda()


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("scale", [0.6, 1.8])
@pytest.mark.parametrize("iterations", [1, 3])
def test_remesh_matches_oracle(name, scale, iterations):
    V, F, _ = MESHES[name]()
    L = scale * _mean_edge(V, F)
    want = orm.remesh(V, F, L, iterations)
    dv, df = _cuda(V, F)
    got = mesh.remesh(dv, df, L, iterations)
    same_mesh(got, want, f"{name} L={L:.4g} it={iterations}")
    side = torch.cuda.Stream()
    again = mesh.remesh(dv, df, L, iterations)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = mesh.remesh(dv, df, L, iterations)
    torch.cuda.current_stream().wait_stream(side)
    for v, f in (again, other):
        assert torch.equal(v, got[0]) and torch.equal(f, got[1]), f"{name}: repeated call differs"


def _bottom_layer_case():
    """Tiny triangles in a 100-unit box (grid cell side 100 / 160 = 0.625).  The point p = (50.1, 50.1, 0.3) is in cell (80, 80, 0), the
    grid's bottom layer.  Face 1, 0.6 above p, is registered only in cell (80, 80, 1), the column inside shell 1 directly above p's
    cell; face 0, 0.76 away, is in cell (81, 80, 0) on the rim of shell 1.  A shell walk that skips the inside column's top cell when
    its bottom one is clamped at the grid's edge returns face 0."""
    V = np.array([[50.8, 50.0, 0.0], [51.1, 50.0, 0.0], [50.8, 50.3, 0.0],          # face 0, at z = 0
                  [50.0, 50.0, 0.9], [50.3, 50.0, 0.9], [50.0, 50.3, 0.9],          # face 1, above p
                  [0.0, 0.0, 0.0], [0.3, 0.0, 0.0], [0.0, 0.3, 0.0],                 # the box's corners
                  [99.7, 99.7, 100.0], [100.0, 99.7, 100.0], [99.7, 100.0, 100.0]], np.float32)
    F = np.arange(12, dtype=np.int64).reshape(4, 3)
    return V, F, np.array([[50.1, 50.1, 0.3]], np.float32)


def test_projection_matches_brute_force():
    V, F, p = _bottom_layer_case()
    q, fid = mesh._closest(*_cuda(V, F), torch.from_numpy(p).cuda())
    wq, wf = orm.nearest(p, V, F)
    assert wf.tolist() == [1] and fid.cpu().tolist() == [1]
    assert np.array_equal(q.cpu().numpy().view(np.int32), wq.view(np.int32))
    # points all over and around the meshes' boxes (bottom and top cell layers and outside the grid included) against brute force
    rng = np.random.default_rng(1)
    for name in ("sphere", "open_field", "integer"):
        V, F, _ = MESHES[name]()
        lo, hi = V.min(0), V.max(0)
        ext = hi - lo
        pts = (lo - 0.2 * ext + rng.random((3000, 3)) * 1.4 * ext).astype(np.float32)
        pts[:500, 2] = lo[2] + rng.random(500).astype(np.float32) * 0.05 * ext[2]               # the bottom layers
        pts[500:1000] = V[rng.integers(0, len(V), 500)]                                          # on the mesh
        q, fid = mesh._closest(*_cuda(V, F), torch.from_numpy(pts).cuda())
        wq, wf = orm.nearest(pts, V, F)
        assert np.array_equal(fid.cpu().numpy(), wf), name
        assert np.array_equal(q.cpu().numpy().view(np.int32), wq.view(np.int32)), name


def test_remesh_zero_iterations_numpy_and_errors():
    V, F, _ = MESHES["sphere"]()
    v, f = mesh.remesh(V, F, 0.05, 0)
    want = od.compact(*od.check_mesh(V, F))
    assert v.dtype == np.float64 and f.dtype == np.int64
    assert np.array_equal(v.astype(np.float32), want[0]) and np.array_equal(f, want[1])
    v, f = mesh.remesh(V, F, 0.05, 1)
    wv, wf = orm.remesh(V, F, 0.05, 1)
    assert np.array_equal(v.astype(np.float32).view(np.int32), wv.view(np.int32)) and np.array_equal(f, wf)
    dv, df = _cuda(V, F)
    for bad in (dict(target_len=0.0), dict(target_len=float("nan")), dict(target_len=0.05, iterations=-1), dict(target_len=0.05, feature_deg=181.0)):
        with pytest.raises(ValueError):
            mesh.remesh(dv, df, **bad)
    bad_f = df.clone()
    bad_f[0, 1] = bad_f[0, 0]
    with pytest.raises(ValueError):
        mesh.remesh(dv, bad_f, 0.05)
    with pytest.raises(_lib.TpxError):
        mesh.remesh(dv.cpu(), df.cpu(), 0.05)
    # the C entries reject malformed input themselves
    lib = _lib.lib()
    Vn, Fn = dv.shape[0], df.shape[0]
    ws = torch.empty(int(lib.tpx_remesh_workspace_bytes(Vn, Fn)), dtype=torch.uint8, device="cuda")
    gb = int(lib.tpx_remesh_grid_bytes(Fn))
    grid = torch.empty(gb, dtype=torch.uint8, device="cuda")
    cr = torch.empty(3 * Fn, dtype=torch.int64, device="cuda")
    counts = torch.zeros(3, dtype=torch.int64, device="cuda")
    st = _lib.stream_ptr()
    assert lib.tpx_remesh_begin(dv.data_ptr(), Vn, bad_f.data_ptr(), Fn, 0.5, grid.data_ptr(), gb, ws.data_ptr(), ws.numel(), cr.data_ptr(),
                                counts.data_ptr(), st) == 0
    assert int(counts[0]) == -1
    assert lib.tpx_remesh_begin(dv.data_ptr(), Vn, df.data_ptr(), Fn, 0.5, grid.data_ptr(), gb - 1, ws.data_ptr(), ws.numel(), cr.data_ptr(),
                                counts.data_ptr(), st) < 0
    assert lib.tpx_remesh_split_count(dv.data_ptr(), Vn, df.data_ptr(), Fn, cr.data_ptr(), 0, -1.0, ws.data_ptr(), ws.numel(), counts.data_ptr(), st) < 0
    assert lib.tpx_remesh_split_count(dv.data_ptr(), Vn, bad_f.data_ptr(), Fn, cr.data_ptr(), 0, 0.05, ws.data_ptr(), ws.numel(), counts.data_ptr(), st) == 0
    assert counts.tolist() == [-1, -1, -1]
    v2 = dv.clone()
    assert lib.tpx_remesh_relax(v2.data_ptr(), Vn, bad_f.clone().data_ptr(), Fn, cr.data_ptr(), 0, dv.data_ptr(), Vn, Fn, grid.data_ptr(), gb, 0.05, 0.5,
                                ws.data_ptr(), ws.numel(), counts.data_ptr(), st) < 0


def test_shell_chain_extract_mesh_and_texmesh():
    m = _shell_module()
    R = 256
    grid = m.sdf_grid(R)
    v0, f0 = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
    v1, f1 = mesh._remove_small(v0, f0, 8, 0.05)
    vd, fd = mesh._decimate(v1, f1, 100000)
    assert f1.shape[0] > 100000
    d = vd.max(0).values.double() - vd.min(0).values.double()
    L = 0.01 * float(torch.sqrt((d * d).sum()))
    info = []
    vr, fr = mesh.remesh(vd, fd, L, 3, info=info)
    ve, fe = m.extract_mesh(R, min_faces=8, min_diameter=0.05, target_faces=100000, remesh_pct=1)
    assert torch.equal(ve, vr) and torch.equal(fe, fr)
    Vd, Fd, Vr, Fr = vd.cpu().numpy(), fd.cpu().numpy(), vr.cpu().numpy(), fr.cpu().numpy()
    assert _closed_oriented(Fd) == _closed_oriented(Fr)
    assert sorted(_euler_per_component(Fd)) == sorted(_euler_per_component(Fr))
    # frozen (border / non-manifold) vertices of the decimated mesh survive bit for bit
    FACE, OUT, IN, n, _ = od._corners(Fd, len(Vd))
    frozen, _ = od.vertex_state(OUT, IN, n)
    if frozen.any():
        have = {tuple(p) for p in Vr.view(np.int32)}
        assert all(tuple(p) in have for p in Vd[frozen].view(np.int32))
    # output vertices lie on the decimated input: spot-check the oracle's exact closest point for a sample
    idx = np.random.default_rng(0).choice(len(Vr), 200, replace=False)
    tri = Vd[Fd].astype(np.float64)
    best = np.full(len(idx), np.inf)
    for i in range(0, len(Fd), 20000):
        t = tri[i:i + 20000]
        p = np.repeat(Vr[idx].astype(np.float64), len(t), 0)
        q = orm.closest_point(p, *(np.tile(t[:, j], (len(idx), 1)) for j in range(3)))
        dd = ((q - p) ** 2).sum(1).reshape(len(idx), len(t))
        best = np.minimum(best, dd.min(1))
    assert np.sqrt(best).max() < 1e-6, np.sqrt(best).max()
    print(f"\nshell: decimated {len(Fd)} faces -> remeshed {len(Fr)} faces, L = {L:.5f}; per iteration {info}")
    print("  edge-length share in [4/5 L, 4/3 L] and valence-6 share: before", _shares(Vd, Fd, L), "after", _shares(Vr, Fr, L), flush=True)
    out = m.extract_texmesh(resolution=R, target_faces=100000, atlas=256, remesh=True)
    Fn = out["f"].shape[0]
    assert 0 < Fn and int(out["f"].max()) < out["v"].shape[0]
    assert out["vt"].shape == (3 * Fn, 2) and out["ft"].shape == (Fn, 3) and out["albedo"].shape == (256, 256, 3)
    assert out["metallicRoughness"].shape == (256, 256, 3)
    lo = m.extract_texmesh(resolution=64, target_faces=10 ** 7, atlas=64, remesh=True)
    hi = m.extract_texmesh(resolution=64, target_faces=10 ** 7, atlas=64, remesh=False)
    for k in ("v", "f", "vt", "ft", "albedo", "metallicRoughness"):
        assert torch.equal(lo[k], hi[k]), k
