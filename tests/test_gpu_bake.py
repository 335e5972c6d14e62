"""-m gpu: texture bake — the UV rasteriser / interpolation (tpx_uv_rasterize, tpx_rast_interpolate) and the seam padding
(tpx_texture_inpaint) against the float64 oracle, the fused texel query (tpx_primsdf_bake) against PrimSDF.forward over the masked,
chunked texel positions, PrimSDF.bake_texture against the reference fixture, and the nvdiffrast binding."""
import os
import sys

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import bake as obake
from test_bake_host import check_inpaint
from tpxl_b200 import _lib, bake, synth

pytestmark = pytest.mark.gpu
AMBIGUOUS = 1e-5          # |min barycentric| below which a coverage decision may flip under fp32 rounding


@pytest.fixture(scope="module")
def fx(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "texture_bake.npz")))


def _fixture_module(fx):
    m = tpxl_b200.PrimSDF(num_prims=fx["srt"].shape[0], dim_feat=6, prim_shape=8).eval()
    m.srt_param.data = torch.from_numpy(fx["srt"])
    m.feat_param.data = torch.from_numpy(fx["feat"])
    return m.cuda()


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


def _raster_cases(fx):
    rng = np.random.default_rng(7)
    yield "fixture", fx["vt"], fx["ft"], 128, 128
    vt, ft = synth.cell_atlas(100_000, 1)
    yield "100k_small", vt.numpy(), ft.numpy(), 1024, 1024
    quad = np.array([[0.01, 0.02], [0.99, 0.03], [0.98, 0.97], [0.02, 0.99]], np.float32)
    yield "quad_2048", quad, np.array([[0, 1, 2], [0, 2, 3]], np.int32), 2048, 2048
    yield "exact_quad", np.array([[0, 0], [1, 0], [1, 1], [0, 1]], np.float32), np.array([[0, 1, 2], [2, 3, 0]], np.int32), 64, 64
    yield "nonsquare", rng.random((300, 2), dtype=np.float32), rng.integers(0, 300, (150, 3)).astype(np.int32), 96, 160
    yield "overlapping", (rng.random((60, 2), dtype=np.float32) * 1.4 - 0.2), rng.integers(0, 60, (40, 3)).astype(np.int32), 200, 120
    ft_bad = rng.integers(0, 50, (80, 3)).astype(np.int32)
    ft_bad[::7, 1] = 50
    ft_bad[3::11, 2] = -1
    ft_bad[5::13, 0] = 2 ** 31 - 1
    yield "out_of_range", rng.random((50, 2), dtype=np.float32), ft_bad, 64, 64


def test_rasterize_and_interpolate_match_the_oracle(fx):
    side = torch.cuda.Stream()
    for name, vt, ft, H, W in _raster_cases(fx):
        dvt, dft = torch.from_numpy(vt).cuda(), torch.from_numpy(ft).cuda()
        rast, winner = bake._rasterize(dvt, dft, H, W)
        assert torch.equal(bake.rasterize_uv(dvt, dft.long(), H, W), rast), name            # int64 triangles are narrowed
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            again = bake.rasterize_uv(dvt, dft, H, W)
        torch.cuda.current_stream().wait_stream(side)
        assert torch.equal(again, rast), f"{name}: a call on a side stream differs"
        r, win = rast.cpu().numpy(), winner.cpu().numpy()
        assert rast.shape == (H, W, 4) and np.array_equal(r[..., 3], (win + 1).astype(np.float32)) and (r[..., 2] == 0).all()
        assert (r[win < 0] == 0).all()
        orast, otri, margin = obake.rasterize_uv(vt, ft, H, W)
        differ = win != otri
        covered = int((otri >= 0).sum())
        assert covered > 0 and not (differ & (margin >= AMBIGUOUS)).any(), f"{name}: {int((differ & (margin >= AMBIGUOUS)).sum())} unambiguous texels differ"
        if name != "exact_quad":                                         # there every centre of the diagonal sits on the shared edge by construction
            assert ((margin < AMBIGUOUS) & ((otri >= 0) | (win >= 0))).sum() < 0.005 * covered, name
        same = ~differ & (otri >= 0)
        err = float(np.abs(r[same][:, :2] - orast[same][:, :2]).max())
        print(f"{name}: {covered} texels covered, {int(differ.sum())} ambiguous differ, max |bary - oracle| = {err:.2e}")
        assert err <= 1e-5, (name, err)
        if name == "exact_quad":                                         # centres on the shared diagonal: no hole, the lower index wins
            assert (win >= 0).all() and (np.diag(win) == 0).all()
        # interpolation of a 5-channel attribute given the same rast
        tri = np.where((ft >= 0) & (ft < len(vt)), ft, 0).astype(np.int32)
        attr = np.random.default_rng(1).standard_normal((len(vt), 5)).astype(np.float32)
        out = bake.interpolate(torch.from_numpy(attr).cuda(), rast, torch.from_numpy(tri).cuda())
        want = obake.interpolate(attr, r, tri)
        assert out.shape == (H, W, 5) and float(np.abs(out.cpu().numpy() - want).max()) <= 1e-6 * max(1.0, float(np.abs(attr).max()))
        assert (out.cpu().numpy()[win < 0] == 0).all()


def test_interpolate_skips_out_of_range_attribute_indices():
    vt = torch.tensor([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0], [1.0, 1.0]], device="cuda")
    ft = torch.tensor([[0, 1, 2], [1, 3, 2]], dtype=torch.int32, device="cuda")
    rast = bake.rasterize_uv(vt, ft, 16, 16)
    tri = torch.tensor([[0, 1, 2], [1, 9, 2]], dtype=torch.int32, device="cuda")
    out = bake.interpolate(torch.ones(4, 2, device="cuda"), rast, tri)
    first = rast[..., 3] == 1
    assert first.any() and (~first).any() and (out[first] == 1).all() and (out[~first] == 0).all()


def _chunked_forward_path(m, v, f, vt, ft, h, w):
    """inference.py:172-198 through this package: rasterise, interpolate positions and mask, masked forward in 8192-point chunks, * 255."""
    rast = bake.rasterize_uv(vt, ft, h, w)
    xyzs = bake.interpolate(v, rast, f).view(-1, 3)
    mask = (bake.interpolate(torch.ones_like(v[:, :1]), rast, f) > 0).view(-1)
    feats = torch.zeros(h * w, 6, device="cuda")
    chunks = []
    with torch.no_grad():
        for c in torch.split(xyzs[mask], 8192):
            p = m(c)
            chunks.append(torch.cat([p["tex"], torch.zeros_like(p["tex"][:, :1]), p["mat"]], -1))
    feats[mask] = torch.cat(chunks, 0)
    return feats.view(h, w, 6) * 255, mask.view(h, w)


def test_bake_pre_inpaint_is_bit_identical_to_forward_on_the_fixture(fx):
    m = _fixture_module(fx)
    v, f, vt, ft = [torch.from_numpy(fx[k]).cuda() for k in ("v", "f", "vt", "ft")]
    want, wmask = _chunked_forward_path(m, v, f, vt, ft, 128, 128)
    feats, mask = m.bake_texture(v, f, vt, ft, resolution=128, pad=0)
    assert feats.shape == (128, 128, 6) and mask.dtype == torch.bool and torch.equal(mask, wmask)
    assert torch.equal(feats, want), f"{int((feats != want).any(-1).sum())} texels differ"
    agree = mask.cpu().numpy() == fx["mask"]
    assert agree.mean() > 0.995
    err = np.abs(feats.cpu().numpy() - fx["feats_pre"])[agree]
    print(f"fixture: masks agree on {agree.mean():.4f} of the texels, max |feats - reference| = {err.max():.3e}")
    assert err.max() <= 2e-5 * 255
    # the exhaustive loop (no binned lists) gives the same texels
    lib = _lib.lib()
    rast = bake.rasterize_uv(vt, ft, 128, 128)
    ex, em = torch.empty(128, 128, 6, device="cuda"), torch.empty(128, 128, dtype=torch.uint8, device="cuda")
    srt, feat = m.srt_param.data.contiguous(), m.feat_param.data.contiguous()
    _lib.check(lib.tpx_primsdf_bake(rast.data_ptr(), 128, 128, v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], srt.data_ptr(), feat.data_ptr(), None, 0,
                                    srt.shape[0], 8, 6, ex.data_ptr(), em.data_ptr(), _lib.stream_ptr()))
    assert torch.equal(ex, feats) and torch.equal(em.bool(), mask)


def test_bake_pre_inpaint_is_bit_identical_to_forward_on_the_synthetic_shell():
    m = _shell_module()
    verts, faces = m.extract_mesh(128)
    F = faces.shape[0]
    assert F > 10_000
    v = verts[faces].reshape(-1, 3).contiguous()                        # inference.py:144-148: per-corner vertices
    f = torch.arange(3 * F, device="cuda").reshape(-1, 3)
    vt, ft = [t.cuda() for t in synth.cell_atlas(F, 5)]
    want, wmask = _chunked_forward_path(m, v, f, vt, ft, 1024, 1024)
    feats, mask = m.bake_texture(v, f, vt, ft, resolution=1024, pad=0)
    assert int(mask.sum()) > 100_000 and torch.equal(mask, wmask)
    assert torch.equal(feats, want), f"{int((feats != want).any(-1).sum())} texels differ"
    assert float(feats.max()) == 255.0 and float(feats[..., 3].abs().max()) == 0.0
    again, _ = m.bake_texture(v, f.int(), vt, ft.long(), resolution=(1024, 1024), pad=0)
    assert torch.equal(again, feats)
    rect, rmask = m.bake_texture(v, f, vt, ft, resolution=(256, 512), pad=4)
    assert rect.shape == (256, 512, 6) and rmask.shape == (256, 512)


def _seeded_mask(n, seed):
    """Islands, holes, one-texel specks and mask touching the image border."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n]
    m = np.zeros((n, n), bool)
    for _ in range(40):
        cy, cx, r = rng.uniform(0, n), rng.uniform(0, n), rng.uniform(n * 0.01, n * 0.08)
        m |= (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
    for _ in range(15):
        cy, cx, r = rng.uniform(0, n), rng.uniform(0, n), rng.uniform(n * 0.005, n * 0.03)
        m &= ~((yy - cy) ** 2 + (xx - cx) ** 2 < r * r)
    s = rng.integers(0, n, (200, 2))
    m[s[:, 0], s[:, 1]] = True
    m[0, :n // 3] = True
    m[n // 2:, n - 1] = True
    return m


def _inpaint_against_oracle(feats, mask, pad):
    H, W = mask.shape
    d = torch.from_numpy(feats).cuda()
    out, src = bake.inpaint(d, torch.from_numpy(mask).cuda(), pad, return_source=True)
    assert out is d
    out, src = out.cpu().numpy(), src.cpu().numpy().astype(np.int64)
    oout, osrc, od2 = obake.inpaint(feats, mask, pad)
    assert np.array_equal(src, osrc), f"pad {pad}: {int((src != osrc).sum())} sources differ (tie rule: smallest (row, col))"
    wi, wj = np.nonzero(src >= 0)
    d2 = np.full((H, W), -1, dtype=np.int64)
    d2[wi, wj] = (src[wi, wj] // W - wi) ** 2 + (src[wi, wj] % W - wj) ** 2
    check_inpaint(out, src, d2, feats, mask, od2)
    assert np.array_equal(out, oout)
    return out


def test_inpaint_matches_the_oracle(fx):
    for pad in (0, 1, 32, 64):
        out = _inpaint_against_oracle(fx["feats_pre"], fx["mask"], pad)
        if pad == 0:
            assert np.array_equal(out, fx["feats_pre"])
    small = _seeded_mask(256, 11)[:200]                                  # non-square
    f = np.random.default_rng(2).random((200, 256, 3), dtype=np.float32)
    for pad in (1, 64):
        _inpaint_against_oracle(f, small, pad)
    big = _seeded_mask(1024, 3)
    f = np.random.default_rng(0).random((1024, 1024, 6), dtype=np.float32)
    out = _inpaint_against_oracle(f, big, 32)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        again = bake.inpaint(torch.from_numpy(f).cuda(), torch.from_numpy(big.astype(np.uint8)).cuda(), 32)
    side.synchronize()
    assert np.array_equal(again.cpu().numpy(), out)
    for m in (np.zeros((64, 48), bool), np.ones((64, 48), bool)):         # nothing to pad from / nothing to pad
        g = np.random.default_rng(4).random((64, 48, 6), dtype=np.float32)
        out, src = bake.inpaint(torch.from_numpy(g).cuda(), torch.from_numpy(m).cuda(), 32, return_source=True)
        assert np.array_equal(out.cpu().numpy(), g) and (src == -1).all()


def test_bake_texture_end_to_end_against_the_reference_fixture(fx):
    m = _fixture_module(fx)
    v, f, vt, ft = [torch.from_numpy(fx[k]).cuda() for k in ("v", "f", "vt", "ft")]
    pre, mask = m.bake_texture(v, f, vt, ft, resolution=128, pad=0)
    post, mask2 = m.bake_texture(v, f, vt, ft, resolution=128)
    assert torch.equal(mask, mask2) and np.array_equal(mask.cpu().numpy(), fx["mask"]), "kernel and oracle masks differ on the fixture"
    pre, post = pre.cpu().numpy(), post.cpu().numpy()
    # same written set, same nearest distances, each value a pre-inpaint mask value at that distance; reference values within the
    # query tolerance wherever the kd-tree took the same texel
    _, src = bake.inpaint(torch.from_numpy(pre).cuda(), mask, 32, return_source=True)
    src = src.cpu().numpy().astype(np.int64)
    wi, wj = np.nonzero(src >= 0)
    d2 = np.full(src.shape, -1, dtype=np.int64)
    d2[wi, wj] = (src[wi, wj] // 128 - wi) ** 2 + (src[wi, wj] % 128 - wj) ** 2
    check_inpaint(post, src, d2, pre, fx["mask"], fx["inpaint_d2"].astype(np.int64))
    close = np.abs(post - fx["feats_post"]).max(-1) <= 2e-5 * 255
    assert close[fx["mask"]].all() and close[src < 0].all()
    for i, j in zip(*np.nonzero(~close)):                                # the kd-tree chose another equidistant texel
        ci, cj = np.nonzero(fx["mask"] & (((np.arange(128)[:, None] - i) ** 2 + (np.arange(128)[None, :] - j) ** 2) == d2[i, j]))
        assert len(ci) > 1 and any(np.abs(fx["feats_pre"][a, b] - fx["feats_post"][i, j]).max() == 0 for a, b in zip(ci, cj)), (i, j)
    print(f"fixture end to end: {len(wi)} texels padded, {int((~close).sum())} resolved a tie differently from the kd-tree")


def test_nvdiffrast_binding_runs_the_reference_call_shapes(fx):
    saved = {k: sys.modules.pop(k, None) for k in ("nvdiffrast", "nvdiffrast.torch")}
    try:
        tpxl_b200.install(nvdiffrast=True)
        import nvdiffrast.torch as dr
        glctx = dr.RasterizeCudaContext()
        v = torch.from_numpy(fx["v"]).float().contiguous().cuda()
        f = torch.from_numpy(fx["f"].astype(np.int64)).cuda()
        vt = torch.from_numpy(fx["vt"]).float().contiguous().cuda()
        ft = torch.from_numpy(fx["ft"].astype(np.int64)).int().contiguous().cuda()
        uv = vt * 2.0 - 1.0                                             # inference.py:163-164
        uv = torch.cat((uv, torch.zeros_like(uv[..., :1]), torch.ones_like(uv[..., :1])), dim=-1)
        h, w = 128, 96
        rast, _ = dr.rasterize(glctx, uv.unsqueeze(0), ft, (h, w))
        xyzs, _ = dr.interpolate(v.unsqueeze(0), rast, f.int())
        mask, _ = dr.interpolate(torch.ones_like(v[:, :1]).unsqueeze(0), rast, f.int())
        assert rast.shape == (1, h, w, 4) and xyzs.shape == (1, h, w, 3) and mask.shape == (1, h, w, 1)
        want = bake.rasterize_uv((uv[:, :2] + 1.0) * 0.5, ft, h, w)
        assert torch.equal(rast[0], want) and torch.equal(xyzs[0], bake.interpolate(v, want, f))
        direct = bake.rasterize_uv(vt, ft, h, w)                         # (vt * 2 - 1 + 1) / 2 rounds: only texels on an edge may move
        assert float((direct[..., 3] != want[..., 3]).float().mean()) < 0.005
        assert torch.equal(mask[0, ..., 0] > 0, want[..., 3] > 0)
        bad = uv.clone()
        bad[0, 3] = 2.0
        with pytest.raises(NotImplementedError):
            dr.rasterize(glctx, bad.unsqueeze(0), ft, (h, w))
        with pytest.raises(NotImplementedError):
            dr.rasterize(glctx, uv.unsqueeze(0).repeat(2, 1, 1), ft, (h, w))
    finally:
        for k, val in saved.items():
            sys.modules.pop(k, None)
            if val is not None:
                sys.modules[k] = val


def test_c_abi_rejects_bad_arguments():
    lib = _lib.lib()
    t = torch.zeros(64, device="cuda")
    st = _lib.stream_ptr()
    assert lib.tpx_uv_rasterize(t.data_ptr(), 4, t.data_ptr(), 1, 0, 8, t.data_ptr(), t.data_ptr(), st) == -3
    assert lib.tpx_uv_rasterize(t.data_ptr(), 4, t.data_ptr(), 1 << 24, 8, 8, t.data_ptr(), t.data_ptr(), st) == -3 and b"2^24" in lib.tpx_last_error()
    assert lib.tpx_rast_interpolate(t.data_ptr(), 4, 0, t.data_ptr(), 1, t.data_ptr(), 2, 2, t.data_ptr(), st) == -3
    assert lib.tpx_texture_inpaint(t.data_ptr(), t.data_ptr(), 2, 2, 6, 8193, t.data_ptr(), 256, None, st) == -3
    assert lib.tpx_texture_inpaint(t.data_ptr(), t.data_ptr(), 8, 8, 1, 4, t.data_ptr(), 16, None, st) == -1 and b"workspace" in lib.tpx_last_error()
    assert lib.tpx_primsdf_bake(t.data_ptr(), 2, 2, t.data_ptr(), 1, t.data_ptr(), 1, t.data_ptr(), t.data_ptr(), None, 0, 1, 8, 5, t.data_ptr(), t.data_ptr(), st) == -3
