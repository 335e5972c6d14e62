"""-m gpu: mesh extraction — marching cubes (tpx_mc_count / tpx_mc_emit, tpxl_b200.mesh) against the float64 oracle, and the PrimSDF
sdf grid (tpx_primsdf_sdf_grid) against PrimSDF.forward over extract_texmesh's points and the reference fixture."""
import os

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import mesh as omesh
from tpxl_b200 import _lib, mesh
from parity import is_fp32_tie

pytestmark = pytest.mark.gpu
SHAPES = [(2, 2, 2), (3, 5, 7), (17, 31, 9), (64, 64, 64), (130, 97, 66), (128, 128, 128)]


def _smooth(shape, seed):
    """Smooth random field: a few random plane waves, so surfaces are large and varied."""
    rng = np.random.default_rng(seed)
    grids = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    f = np.zeros(shape)
    for _ in range(6):
        k = rng.normal(size=3) * 0.35
        f += np.sin(sum(k[d] * grids[d] for d in range(3)) + rng.uniform(0, 2 * np.pi))
    return f.astype(np.float32)


def _fields(shape):
    n = int(np.prod(shape))
    yield "smooth", _smooth(shape, n), 0.0
    yield "smooth_iso", _smooth(shape, n + 1), 0.4
    yield "integer", np.random.default_rng(n).integers(-2, 3, size=shape).astype(np.float32), 0.0
    yield "constant", np.full(shape, 0.5, np.float32), 0.0
    yield "constant_at_iso", np.zeros(shape, np.float32), 0.0


def _check_against_oracle(vol, iso, verts, faces, atol):
    ov, of = omesh.marching_cubes(vol, float(np.float32(iso)))      # the kernel compares and interpolates against fp32(iso)
    assert verts.dtype == torch.float32 and faces.dtype == torch.int64
    assert torch.equal(faces.cpu(), torch.from_numpy(of)), "faces differ from the oracle"
    assert verts.shape == ov.shape
    if len(ov):
        err = float(np.abs(verts.cpu().double().numpy() - ov).max())
        assert err <= atol, err
    return ov, of


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_kernel_matches_oracle(shape):
    side = torch.cuda.Stream()
    for name, vol, iso in _fields(shape):
        dv = torch.from_numpy(vol).cuda()
        v1, f1 = mesh.marching_cubes(dv, iso)
        _check_against_oracle(vol, iso, v1, f1, 1e-5)
        if name.startswith("constant"):
            assert v1.shape == (0, 3) and f1.shape == (0, 3)
        v2, f2 = mesh.marching_cubes(dv, iso)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            v3, f3 = mesh.marching_cubes(dv, iso)
        torch.cuda.current_stream().wait_stream(side)
        for v, f in ((v2, f2), (v3, f3)):
            assert torch.equal(v, v1) and torch.equal(f, f1), f"{name}: repeated call differs"


def test_numpy_entry_and_errors():
    vol = _smooth((20, 24, 28), 5)
    vn, fn = mesh.marching_cubes(vol, 0.1)
    vd, fd = mesh.marching_cubes(torch.from_numpy(vol).cuda(), 0.1)
    assert vn.dtype == np.float64 and fn.dtype == np.int64 and len(fn) > 100
    assert np.array_equal(vn, vd.cpu().double().numpy()) and np.array_equal(fn, fd.cpu().numpy())
    v64, f64 = mesh.marching_cubes(vol.astype(np.float64), 0.1)      # the numpy entry converts to fp32
    assert np.array_equal(v64, vn) and np.array_equal(f64, fn)
    for shape in ((1, 5, 5), (5, 0, 5)):
        v, f = mesh.marching_cubes(torch.zeros(shape, device="cuda"))
        assert v.shape == (0, 3) and f.shape == (0, 3)
    with pytest.raises(_lib.TpxError):
        mesh.marching_cubes(torch.zeros(4, 4, 4))
    with pytest.raises(ValueError):
        mesh.marching_cubes(torch.zeros(4, 4, device="cuda"))
    with pytest.raises(ValueError):
        mesh.marching_cubes(torch.zeros(4, 4, 4, dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError):
        mesh.marching_cubes(np.zeros((4, 4)))


def _shell_module(K=2048, S=8):
    """The synthetic object of tools/primsdf_perf.py: primitives on a noisy sphere shell."""
    g = torch.Generator().manual_seed(0)
    d = torch.randn(K, 3, generator=g)
    pos = d / d.norm(dim=1, keepdim=True) * (0.55 + 0.1 * torch.rand(K, 1, generator=g))
    srt = torch.cat([0.03 + 0.05 * torch.rand(K, 1, generator=g), pos], 1)
    m = tpxl_b200.PrimSDF(num_prims=K, dim_feat=6, prim_shape=S).eval()
    m.srt_param.data = srt
    m.feat_param.data = torch.randn(K, 6 * S ** 3, generator=g)
    return m.cuda()


@pytest.mark.parametrize("R", [128, 256])
def test_sdf_grid_and_extract_mesh_match_the_chunked_reference_path(R):
    m = _shell_module()
    # inference.py:107-116 through this package's forward
    xx = torch.linspace(-1, 1, R, device="cuda")
    pts = torch.stack(torch.meshgrid(xx, xx, xx, indexing="ij"), dim=-1).reshape(-1, 3)
    with torch.no_grad():
        want = torch.cat([m(c)["sdf"] for c in torch.split(pts, 8192)], 0).reshape(R, R, R)
    grid = m.sdf_grid(R)
    assert grid.shape == (R, R, R) and grid.dtype == torch.float32
    assert torch.equal(grid, want), f"{int((grid != want).sum())} of {R ** 3} grid values differ"
    verts, faces = m.extract_mesh(R)
    g = grid.cpu().numpy()
    ov, of = omesh.marching_cubes(g, 0.0)
    assert len(of) > 1000
    assert torch.equal(faces.cpu(), torch.from_numpy(of))
    world = ov / (R - 1.0) * 2.0 - 1.0                   # inference.py:122-124
    err = float(np.abs(verts.cpu().double().numpy() - world).max())
    print(f"R={R}: V={len(ov)} F={len(of)} max |vertex - oracle| = {err:.2e}")
    assert err <= 2e-6, err


def test_sdf_grid_matches_reference_fixture(golden_dir):
    fx = np.load(os.path.join(golden_dir, "primsdf_grid.npz"))
    K, R = fx["srt"].shape[0], fx["grid"].shape[0]
    m = tpxl_b200.PrimSDF(num_prims=K, dim_feat=6, prim_shape=8).eval()
    m.srt_param.data = torch.from_numpy(fx["srt"])
    m.feat_param.data = torch.from_numpy(fx["feat"])
    m = m.cuda()
    got = m.sdf_grid(R).cpu().numpy()
    bad = ~np.isclose(got, fx["grid"], rtol=2e-5, atol=2e-5)
    assert bad.mean() <= 0.01, f"{bad.sum()} of {R ** 3} values differ"
    xx = torch.linspace(-1, 1, R).double()
    srt = torch.from_numpy(fx["srt"]).double()
    for i, j, k in zip(*np.nonzero(bad)):
        assert is_fp32_tie(torch.stack([xx[i], xx[j], xx[k]]), srt, 8), (i, j, k, got[i, j, k], fx["grid"][i, j, k])
    # the exhaustive path (no binned lists) gives the same grid
    lib = _lib.lib()
    srt_d, feat_d = m.srt_param.data.contiguous(), m.feat_param.data.contiguous()
    ex = torch.empty(R, R, R, device="cuda")
    coords = torch.linspace(-1, 1, R, device="cuda")
    _lib.check(lib.tpx_primsdf_sdf_grid(coords.data_ptr(), R, srt_d.data_ptr(), feat_d.data_ptr(), None, 0, K, 8, 6, 1, ex.data_ptr(), _lib.stream_ptr()))
    assert torch.equal(ex.cpu(), torch.from_numpy(got))
    verts, faces = m.extract_mesh(R)
    ov, of = omesh.marching_cubes(got, 0.0)
    assert torch.equal(faces.cpu(), torch.from_numpy(of)) and len(of) > 1000
