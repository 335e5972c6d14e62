"""-m gpu: PrimSDF point query (tpx_primsdf_query / tpxl_b200.PrimSDF) against the reference fixture and the oracle."""
import os

import numpy as np
import pytest
import torch

import oracle
import tpxl_b200
from tpxl_b200 import _lib
from parity import is_fp32_tie

pytestmark = pytest.mark.gpu
TOL = dict(rtol=2e-5, atol=2e-5)   # fp32 throughout; differences are summation order / fma contraction only


def _module(srt, feat, K, S=8):
    m = tpxl_b200.PrimSDF(num_prims=K, dim_feat=6, prim_shape=S).eval()
    m.srt_param.data = torch.as_tensor(srt)
    m.feat_param.data = torch.as_tensor(feat)
    return m.cuda()


def test_matches_reference_fixture(golden_dir):
    fx = np.load(os.path.join(golden_dir, "primsdf.npz"))
    m = _module(fx["srt"], fx["feat"], fx["srt"].shape[0])
    out = m(torch.from_numpy(fx["pts"]).cuda())
    for k in ("sdf", "tex", "mat"):
        np.testing.assert_allclose(out[k].cpu().numpy(), fx[k], err_msg=k, **TOL)
    cov = torch.from_numpy(fx["covered"])
    m.train()
    tr = m(torch.from_numpy(fx["pts"]).cuda())
    assert float(tr["sdf"].cpu()[~cov].abs().max()) == 0.0
    np.testing.assert_allclose(tr["sdf"].cpu().numpy()[fx["covered"]], fx["sdf"][fx["covered"]], **TOL)


@pytest.mark.parametrize("K,S,n", [(1, 8, 257), (1500, 8, 3001), (2048, 8, 1000), (64, 4, 513)])
def test_matches_oracle(K, S, n):
    """Ragged sizes; K > one staging chunk (1024); the shipped K=2048; another primitive resolution."""
    g = torch.Generator().manual_seed(K * 7 + n)
    srt = torch.cat([torch.rand(K, 1, generator=g) * 0.1 + 0.03, torch.rand(K, 3, generator=g) * 1.6 - 0.8], 1)
    feat = torch.randn(K, 6 * S ** 3, generator=g)
    x = torch.rand(n, 3, generator=g) * 2 - 1
    m = _module(srt, feat, K, S)
    out = m(x.cuda())
    ref = oracle.primsdf.query(x, srt, feat, S=S, dim_feat=6, inference=True)
    for k in ("tex", "mat"):
        np.testing.assert_allclose(out[k].cpu().numpy(), ref[k].numpy(), err_msg=k, **TOL)
    bad = ~np.isclose(out["sdf"].cpu().numpy(), ref["sdf"].numpy(), **TOL)[:, 0]
    # The nearest-primitive / nearest-voxel search of an uncovered point (primsdf.py:88-97) is an fp32 argmin: where two
    # candidates are closer than fp32 can tell apart, which one wins is rounding, not algorithm.  Only such points may differ.
    assert bad.mean() <= 0.01, f"{bad.sum()} of {n} sdf values differ"
    for i in np.nonzero(bad)[0]:
        assert is_fp32_tie(x[i].double(), srt.double(), S), f"point {i}: kernel {float(out['sdf'][i])} oracle {float(ref['sdf'][i])}"


def test_voxel_centres_reproduce_the_voxels():
    """Size-independent property at the shipped size: querying every primitive's own voxel centres of an isolated
    primitive returns its voxels (weights normalise to 1 up to the 1e-6 epsilon); checks the z/y/x axis convention."""
    K, S = 2048, 8
    g = torch.Generator().manual_seed(5)
    side = 13                                              # 13^3 = 2197 >= 2048 disjoint cells
    idx = torch.arange(K)
    centre = torch.stack([idx % side, (idx // side) % side, idx // (side * side)], 1).float() / side * 1.9 - 0.95 + 0.07
    scale = torch.full((K, 1), 0.06)
    srt = torch.cat([scale, centre], 1)
    feat = torch.rand(K, 6, S, S, S, generator=g)
    lin = torch.linspace(-1, 1, S)[1:-1]                   # interior voxel centres (w > 0 there)
    zz, yy, xx = torch.meshgrid(lin, lin, lin, indexing="ij")
    local = torch.stack([xx, yy, zz], -1).reshape(-1, 3)   # x indexes W, z indexes D (grid_sample convention)
    pts = (centre[:, None, :] + scale[:, None, :] * local[None]).reshape(-1, 3)
    m = _module(srt, feat.reshape(K, -1), K, S)
    out = m(pts.cuda())
    want = feat[:, :, 1:-1, 1:-1, 1:-1].reshape(K, 6, -1).permute(0, 2, 1).reshape(-1, 6)
    got = torch.cat([out["sdf"], out["tex"], out["mat"]], 1).cpu()
    w = 1 - local.abs().max(1).values                      # the single covering weight
    np.testing.assert_allclose(got.numpy(), (want * (w / (w + 1e-6)).repeat(K)[:, None]).numpy(), rtol=1e-4, atol=1e-5)


def test_errors_and_empty():
    m = _module(torch.rand(4, 4) + 0.1, torch.randn(4, 6 * 512), 4)
    assert m(torch.zeros(0, 3).cuda())["sdf"].shape == (0, 1)
    with pytest.raises(ValueError):
        m(torch.zeros(5, 2).cuda())
    with pytest.raises(_lib.TpxError):
        m(torch.zeros(5, 3))                               # host points: no CPU path


@pytest.mark.parametrize("cap", [8 << 20, 2048])
def test_grid_query_identical_to_exhaustive(cap):
    """The grid-binned kernel must reproduce the exhaustive one BIT FOR BIT (same visits in the same ascending order, same argmin):
    points inside and outside the grid's box, covered and uncovered, and a workspace too small for the lists (exhaustive fallback)."""
    K, S, n = 2048, 8, 20000
    g = torch.Generator().manual_seed(77)
    d = torch.randn(K, 3, generator=g)
    pos = d / d.norm(dim=1, keepdim=True) * (0.55 + 0.1 * torch.rand(K, 1, generator=g))
    srt = torch.cat([0.03 + 0.05 * torch.rand(K, 1, generator=g), pos], 1).cuda().contiguous()
    feat = torch.randn(K, 6 * S ** 3, generator=g).cuda()
    x = (torch.rand(n, 3, generator=g) * 2.6 - 1.3).cuda()          # a share of the points lies outside [-1, 1]^3
    x[:4000] = (pos[torch.randint(0, K, (4000,), generator=g)] + 0.02 * torch.randn(4000, 3, generator=g)).cuda()   # covered points
    lib = _lib.lib()
    ref = torch.empty(n, 6, device="cuda")
    out = torch.full((n, 6), 7.0, device="cuda")
    st = _lib.stream_ptr()
    _lib.check(lib.tpx_primsdf_query(x.data_ptr(), srt.data_ptr(), feat.data_ptr(), n, K, S, 6, 1, ref.data_ptr(), st))
    nbytes = int(lib.tpx_primsdf_grid_bytes(cap))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.tpx_primsdf_grid_build(srt.data_ptr(), K, ws.data_ptr(), nbytes, st))
    _lib.check(lib.tpx_primsdf_query_grid(x.data_ptr(), srt.data_ptr(), feat.data_ptr(), ws.data_ptr(), nbytes, n, K, S, 6, 1, out.data_ptr(), st))
    torch.cuda.synchronize()
    hdr = ws[:40].view(torch.int32).cpu()      # GridHdr: 5 floats, then total_cover, total_near, overflow, cap, K
    print("grid lists: cover", int(hdr[5]), "near", int(hdr[6]), "overflow", int(hdr[7]), "cap", int(hdr[8]))
    assert int(hdr[7]) == (1 if cap == 2048 else 0)
    assert (ref[:, 0].abs() > 0).float().mean() > 0.5 and (ref[:4000, 1:].abs().sum(1) > 0).float().mean() > 0.9   # the test exercises both branches
    assert torch.equal(out, ref)
