"""CPU: the texture-bake oracle (oracle/bake.py) against the reference fixture tests/golden/texture_bake.npz and against the
rasterisation contract, the nvdiffrast binding of install(), and the bake entry points without a GPU."""
import os
import sys

import numpy as np
import pytest
import torch

import oracle
import tpxl_b200
from oracle import bake as obake
from tpxl_b200 import _lib, bake


@pytest.fixture(scope="module")
def fx(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "texture_bake.npz")))


def check_inpaint(out, src, d2, pre, mask, want_d2, want_post=None):
    """``out`` / ``src`` / ``d2`` are an inpaint of ``pre`` under ``mask``; ``want_d2`` [H,W] is the squared distance another
    implementation found per written texel (-1 = not written).  Equidistant sources are checked to be ties, not compared."""
    H, W = mask.shape
    assert np.array_equal(src >= 0, want_d2 >= 0), "the sets of written texels differ"
    assert not (mask & (src >= 0)).any()
    wi, wj = np.nonzero(src >= 0)
    si, sj = src[wi, wj] // W, src[wi, wj] % W
    assert mask[si, sj].all(), "a source lies outside the mask"
    assert np.array_equal((si - wi) ** 2 + (sj - wj) ** 2, d2[wi, wj])
    assert np.array_equal(d2[wi, wj], want_d2[wi, wj]), "nearest distances differ"
    assert np.array_equal(out[wi, wj], pre[si, sj])
    keep = src < 0
    assert np.array_equal(out[keep], pre[keep]), "a texel outside the padded region changed"
    if want_post is not None:
        same = (out[wi, wj] == want_post[wi, wj]).all(1)
        for i, j in zip(wi[~same], wj[~same]):                           # the other implementation chose another texel: it must be a tie
            ci, cj = np.nonzero(mask & (((np.arange(H)[:, None] - i) ** 2 + (np.arange(W)[None, :] - j) ** 2) == d2[i, j]))
            assert len(ci) > 1 and any(np.array_equal(pre[a, b], want_post[i, j]) for a, b in zip(ci, cj)), (i, j)
        assert np.array_equal(out[keep], want_post[keep])


def test_oracle_inpaint_reproduces_the_reference_padding(fx):
    mask, pre = fx["mask"], fx["feats_pre"]
    assert mask.shape == (128, 128) and 0.2 < mask.mean() < 0.8 and (fx["inpaint_d2"] >= 0).sum() > 1000
    out, src, d2 = obake.inpaint(pre, mask, 32)
    check_inpaint(out, src, d2, pre, mask, fx["inpaint_d2"].astype(np.int64), fx["feats_post"])
    assert np.array_equal(out[mask], pre[mask])
    # smallest (row, col) among equidistant sources
    m = np.zeros((5, 5), bool)
    m[0, 2] = m[2, 0] = m[2, 4] = m[4, 2] = True
    f = np.arange(25, dtype=np.float32).reshape(5, 5, 1)
    out, src, d2 = obake.inpaint(f, m, 2)
    assert src[2, 2] == 0 * 5 + 2 and d2[2, 2] == 4 and out[2, 2, 0] == f[0, 2, 0]
    assert src[1, 1] == 0 * 5 + 2 and d2[1, 1] == 2                      # (0,2) and (2,0) tie: the smaller row
    # L1 ball: a texel at L1 distance 3 stays untouched with pad 2 although its Euclidean distance is below 3
    m = np.zeros((7, 7), bool)
    m[0, 0] = True
    _, src, _ = obake.inpaint(np.zeros((7, 7, 1), np.float32), m, 2)
    assert src[1, 1] == 0 and src[0, 2] == 0 and src[1, 2] == -1 and src[2, 1] == -1
    assert np.array_equal(src >= 0, obake.dilate_cross(m, 2) & ~m)


def test_oracle_dilation_is_scipys(fx):
    from scipy.ndimage import binary_dilation
    for it in (1, 3, 32):
        assert np.array_equal(obake.dilate_cross(fx["mask"], it), binary_dilation(fx["mask"], iterations=it))


def test_oracle_query_reproduces_the_reference_texels(fx):
    """oracle.primsdf.query at the fixture's texel positions gives the reference's pre-inpaint feats."""
    h, w = fx["mask"].shape
    rast, tri, _ = obake.rasterize_uv(fx["vt"], fx["ft"], h, w)
    assert np.array_equal(tri >= 0, fx["mask"])
    xyz = torch.from_numpy(obake.interpolate(fx["v"], rast, fx["f"])).float()[torch.from_numpy(fx["mask"])]
    out = oracle.primsdf.query(xyz, torch.from_numpy(fx["srt"]), torch.from_numpy(fx["feat"]), S=8, dim_feat=6, inference=True)
    want = fx["feats_pre"][fx["mask"]] / 255.0
    got = torch.cat([out["tex"], torch.zeros_like(out["tex"][:, :1]), out["mat"]], 1).numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-5)
    assert (want.max(0)[[0, 1, 2, 4, 5]] > 0.5).all() and (want[:, 3] == 0).all()
    assert (fx["feats_pre"][~fx["mask"]] == 0).all()


QUAD = np.array([[0.125, 0.125], [0.875, 0.125], [0.875, 0.875], [0.125, 0.875]], np.float32)


def test_rasteriser_contract_shared_edge_overlap_winding_degenerate():
    H = W = 16
    # two triangles sharing the diagonal, whose texel centres (i == j) lie exactly on it
    ft = np.array([[0, 1, 2], [0, 2, 3]])
    rast, tri, margin = obake.rasterize_uv(QUAD, ft, H, W)
    inside = np.zeros((H, W), bool)
    inside[2:14, 2:14] = True
    assert np.array_equal(tri >= 0, inside), "hole or spill on the quad"
    ii, jj = np.nonzero(inside)
    assert (tri[ii, jj][jj > ii] == 0).all() and (tri[ii, jj][jj < ii] == 1).all()
    assert (tri[ii, jj][jj == ii] == 0).all(), "a centre on the shared edge belongs to both: the lower index wins"
    assert (margin[ii, jj][jj == ii] == 0).all() and (margin[ii, jj][np.abs(jj - ii) > 0] > 1e-3).all()
    alone = [obake.rasterize_uv(QUAD, ft[k:k + 1], H, W)[1] >= 0 for k in (0, 1)]
    assert np.array_equal(alone[0] | alone[1], inside) and np.array_equal(alone[0] & alone[1], inside & np.eye(H, dtype=bool))
    # both windings give the same coverage, and barycentrics that follow the vertices
    r2, t2, _ = obake.rasterize_uv(QUAD, ft[:, ::-1], H, W)
    assert np.array_equal(t2, tri)
    np.testing.assert_allclose(obake.interpolate(QUAD, r2, ft[:, ::-1]), obake.interpolate(QUAD, rast, ft), atol=1e-12)
    # (u, v) weigh vertices 0 and 1: interpolating the uv coordinates returns the texel centre
    uv = obake.interpolate(QUAD, rast, ft)
    np.testing.assert_allclose(uv[ii, jj], np.stack([(jj + 0.5) / W, (ii + 0.5) / H], 1), atol=1e-12)
    assert (rast[..., 2] == 0).all() and np.array_equal(rast[..., 3], tri + 1) and (rast[~inside] == 0).all()
    # overlap: lowest index wins; degenerate and out-of-range triangles are ignored
    ft3 = np.array([[0, 0, 1], [0, 1, 2], [0, 2, 3], [0, 1, 3], [0, 1, 7], [-1, 1, 2]])
    _, tri3, _ = obake.rasterize_uv(QUAD, ft3, H, W)
    assert np.array_equal(tri3 >= 0, inside) and set(np.unique(tri3)) == {-1, 1, 2}
    assert np.array_equal(tri3[inside], tri[inside] + 1)


def test_rasteriser_row_zero_is_v_zero_and_sizes():
    tri_low = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 0.25]], np.float32)       # hugs v = 0
    _, tri, _ = obake.rasterize_uv(tri_low, np.array([[0, 1, 2]]), 8, 12)
    rows = np.nonzero((tri >= 0).any(1))[0]
    assert rows.min() == 0 and rows.max() <= 1 and tri.shape == (8, 12)
    # sub-texel triangle: covers the one centre it contains, or nothing
    c = np.array([(5 + 0.5) / 12, (3 + 0.5) / 8])
    small = (c + np.array([[-0.01, -0.01], [0.02, -0.01], [-0.01, 0.02]])).astype(np.float32)
    _, tri, _ = obake.rasterize_uv(small, np.array([[0, 1, 2]]), 8, 12)
    assert (tri >= 0).sum() == 1 and tri[3, 5] == 0
    _, tri, _ = obake.rasterize_uv(small + np.float32(0.03), np.array([[0, 1, 2]]), 8, 12)
    assert (tri >= 0).sum() == 0


def test_install_binds_nvdiffrast_only_on_request():
    saved = {k: sys.modules.pop(k, None) for k in ("nvdiffrast", "nvdiffrast.torch")}
    try:
        tpxl_b200.install()
        tpxl_b200.install(mcubes=True)
        assert "nvdiffrast" not in sys.modules and "nvdiffrast.torch" not in sys.modules
        sys.modules.pop("mcubes", None)
        tpxl_b200.install(nvdiffrast=True)
        assert "mcubes" not in sys.modules
        import nvdiffrast.torch as dr
        assert sys.modules["nvdiffrast"].torch is dr
        assert callable(dr.rasterize) and callable(dr.interpolate)
        dr.RasterizeCudaContext()
        dr.RasterizeGLContext()
    finally:
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
        sys.modules.pop("mcubes", None)


def test_entry_points_validate_and_refuse_the_cpu():
    raw = _lib.load_library()
    assert raw.tpx_texture_inpaint_bytes(1024, 1024) >= 2 * 1024 * 1024
    assert raw.tpx_texture_inpaint_bytes(0, 8) == 0 and raw.tpx_texture_inpaint_bytes(8, 8193) == 0
    assert raw.tpx_uv_rasterize(None, 0, None, 0, 8, 8, None, None, None) == -1 and b"null" in raw.tpx_last_error()
    assert raw.tpx_texture_inpaint(None, None, 8, 8, 6, 32, None, 0, None, None) == -1
    assert raw.tpx_primsdf_bake(None, 8, 8, None, 0, None, 0, None, None, None, 0, 1, 8, 6, None, None, None) == -1
    assert raw.tpx_rast_interpolate(None, 0, 3, None, 0, None, 8, 8, None, None) == -1
    vt, ft = torch.rand(6, 2), torch.tensor([[0, 1, 2], [3, 4, 5]])
    rast, feats, mask = torch.zeros(8, 8, 4), torch.zeros(8, 8, 6), torch.zeros(8, 8, dtype=torch.bool)
    m = tpxl_b200.PrimSDF(num_prims=4).eval()
    for call in (lambda: bake.rasterize_uv(vt[:, :1], ft, 8, 8), lambda: bake.rasterize_uv(vt, ft.float(), 8, 8), lambda: bake.rasterize_uv(vt, ft[:, :2], 8, 8),
                 lambda: bake.rasterize_uv(vt, ft, 0, 8), lambda: bake.rasterize_uv(vt, ft, 8, 8193), lambda: bake.rasterize_uv(vt.long(), ft, 8, 8),
                 lambda: bake.interpolate(vt, rast[..., :3], ft), lambda: bake.interpolate(vt[0], rast, ft), lambda: bake.interpolate(vt, rast.double(), ft),
                 lambda: bake.inpaint(feats, mask[:4]), lambda: bake.inpaint(feats.double(), mask), lambda: bake.inpaint(feats, mask.float()),
                 lambda: bake.inpaint(feats, mask, pad=-1), lambda: bake.inpaint(feats[:, :, :3], mask),
                 lambda: m.bake_texture(torch.rand(6, 3), ft, vt, ft[:1]), lambda: m.bake_texture(torch.rand(6, 2), ft, vt, ft),
                 lambda: m.bake_texture(torch.rand(6, 3), ft, vt, ft, resolution=(8, 0))):
        with pytest.raises(ValueError):
            call()
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for call in (lambda: bake.rasterize_uv(vt, ft, 8, 8), lambda: bake.interpolate(vt, rast, ft), lambda: bake.inpaint(feats, mask),
                 lambda: m.bake_texture(torch.rand(6, 3), ft, vt, ft, resolution=8)):
        with pytest.raises(_lib.TpxError):
            call()
    tpxl_b200.install(nvdiffrast=True)
    try:
        import nvdiffrast.torch as dr
        with pytest.raises(_lib.TpxError):
            dr.rasterize(dr.RasterizeCudaContext(), torch.zeros(1, 6, 4), ft.int(), (8, 8))
    finally:
        sys.modules.pop("nvdiffrast", None)
        sys.modules.pop("nvdiffrast.torch", None)
