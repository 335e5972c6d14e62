"""-m gpu: the preview renders of tpxl_b200.visualize against THE REFERENCE'S OWN dva/visualize.py (staged byte-identical under
oracle/_ref/, loader oracle.visualize.reference_visualize), on the same H100.

  * tpx_colored_boxes in both layouts equals the reference's generate_colored_boxes run on the GPU, bit for bit (NaN where it is NaN),
    and leaves numpy's global generator where the reference leaves it;
  * the rgb payload equals the prim_rgba the reference's statements build on the GPU, bit for bit; the material payload its torch
    restatement;
  * tpx_raymarch_preview_views equals per-view tpx_raymarch_preview calls, bit for bit;
  * after tpxl_b200.install(), the reference's dva/visualize.py imports and its frames and summary JPGs equal the drop-in's, bit for
    bit and byte for byte;
  * against the reference's dva/visualize.py over its own RayMarcher (compiled extensions), every drop-in frame stays within the image
    bounds of tests/test_gpu_raymarch_ref.py, measured as its _check measures them.
"""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import visualize as ov
from tpxl_b200 import _lib
from tpxl_b200 import visualize as tv
from tpxl_b200.ray_marcher import colored_boxes, generate_colored_boxes, march_camera, march_views

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_raymarch_ref import IMG_REL, PIX_MAX, PIX_SHARE  # noqa: E402

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ov.available("reference"), reason="the reference's dva/visualize.py and ray marcher are not staged")
needs_vis = pytest.mark.skipif(not ov.available("ours"), reason="the reference's dva/visualize.py is not staged")
VR = 10000.0


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and bool(torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0))) and \
        bool(torch.equal(torch.isnan(a), torch.isnan(b)))


def _recon(B=1, P=2048, S=8, seed=3):
    """A recon_param of the shipped layout [B, P, 4 + 6 S^3]: primitives of scale 0.05 on a shell of radius 0.5, sdf near 0."""
    g = torch.Generator().manual_seed(seed)
    S3 = S ** 3
    d = torch.randn(B, P, 3, generator=g)
    pos = d / d.norm(dim=-1, keepdim=True) * 0.5
    scale = 0.045 + 0.01 * torch.rand(B, P, 1, generator=g)
    sdf = torch.rand(B, P, S3, generator=g) * 0.02 - 0.004
    rest = torch.rand(B, P, 5 * S3, generator=g)
    return torch.cat([scale, pos, sdf, rest], dim=-1).cuda()


class _Capture:
    def __init__(self, H, W):
        self.image_height, self.image_width, self.volradius, self.calls = H, W, VR, []

    def __call__(self, prim_rgba, prim_pos, prim_rot, prim_scale, K, RT):
        self.calls.append(prim_rgba.detach().clone())
        return {"rgba_image": torch.zeros(prim_rgba.shape[0], 4, self.image_height, self.image_width, device=prim_rgba.device)}


@needs_ref
@pytest.mark.parametrize("K,S,B", [(2048, 8, 1), (6, 4, 1), (6, 5, 2), (6, 8, 2)] + [(6, s, 1) for s in (2, 3, 6, 7, 9, 11, 12, 16)])
def test_colored_boxes_match_the_reference_on_the_gpu(K, S, B):
    tpl = torch.zeros(B, K, 4, S, S, S, device="cuda")
    rot = torch.eye(3, device="cuda")[None, None].repeat(B, K, 1, 1)
    with ov.reference_visualize("reference") as (vis, _):
        np.random.seed(1)
        ref = vis.generate_colored_boxes(tpl, rot)
        st_ref = np.random.get_state()
    np.random.seed(1)
    ours = generate_colored_boxes(tpl, rot)
    st = np.random.get_state()
    assert np.array_equal(st[1], st_ref[1]) and st[2] == st_ref[2]
    chl = colored_boxes(B, K, S, tpxl_b200.ray_marcher.box_colors(K), 10000.0, True, "cuda")
    torch.cuda.synchronize()
    diff = ~((ours == ref) | (torch.isnan(ours) & torch.isnan(ref)))
    assert not bool(diff.any()), f"{int(diff.sum())} elements differ, first at {diff.nonzero()[:4].tolist()}"
    assert _same(chl, ref.permute(0, 1, 3, 4, 5, 2).contiguous())
    assert bool(torch.isnan(ref).any()) == bool(torch.isnan(ours).any())


@needs_ref
@pytest.mark.parametrize("B,P,S", [(1, 2048, 8), (2, 6, 5), (1, 6, 4)])
def test_payload_matches_the_reference_statements(B, P, S):
    recon = _recon(B, P, S, seed=11 + S)
    with ov.reference_visualize("reference") as (vis, _):
        rm = _Capture(64, 64)
        vis.visualize_primvolume(_tmpjpg(), {}, recon, rm, "cuda")
    ref = rm.calls[0].permute(0, 1, 3, 4, 5, 2).contiguous()
    assert _same(tv.primvolume_payload(recon, "rgb"), ref)
    mat = tv.primvolume_payload(recon, "mat")
    assert _same(mat, ov.payload(recon, "mat"))
    assert torch.equal(mat[..., 3], ref[..., 3]) and bool((mat[..., 0] == 0).all())


def _tmpjpg():
    return os.path.join(tempfile.mkdtemp(), "x.jpg")


def _scene(B, V, H):
    recon = _recon(B)
    rm = tpxl_b200.RayMarcher(H, H, VR)
    angles = torch.linspace(1.5, 3.5, V + 1)[:V] * torch.pi
    Rt = tv.orbit_extrinsics(rm, B, angles).cuda()
    K = tv.preview_intrinsics(rm, B).cuda()
    return recon, rm, Rt, K


@pytest.mark.parametrize("H", [256, 518])
@pytest.mark.parametrize("V", [1, 16, 61])
def test_views_launch_equals_per_view_launches(V, H):
    """One tpx_raymarch_preview_views launch of V views against V tpx_raymarch_preview calls, bit for bit."""
    recon, rm, Rt, K = _scene(1, V, H)
    tpl = tv.primvolume_payload(recon, "rgb")
    pos = (recon[:, :, 1:4] * VR / VR).contiguous()
    rot = torch.eye(3, device="cuda")[None, None].repeat(1, recon.shape[1], 1, 1).contiguous()
    scale = (1 / recon[:, :, 0:1].repeat(1, 1, 3)).contiguous()
    cams = [march_camera(Rt[v].clone(), K, "cuda") for v in range(V)]
    cam = tuple(torch.cat([c[i] for c in cams], 0).contiguous() for i in range(4))
    geom = (H, H, VR, 1.0 / VR, 8.0, 8.0)
    one = march_views(tpl, pos, rot, scale, cam, V, *geom)
    each = torch.empty_like(one)
    for v, c in enumerate(cams):           # the existing single-view entry, one call per view
        _lib.check(_lib.lib().tpx_raymarch_preview(tpl.data_ptr(), pos.data_ptr(), rot.data_ptr(), scale.data_ptr(), *[t.data_ptr() for t in c], 1,
                                                   tpl.shape[1], tpl.shape[2], H, H, VR, 1.0 / VR, 8.0, 8.0, each[v].data_ptr(), _lib.stream_ptr()),
                   "tpx_raymarch_preview")
    torch.cuda.synchronize()
    assert float(one[..., 3].amax()) > 0.3
    assert torch.equal(one, each)


def _frames(stub, folder, name):
    return np.stack(stub.frames[os.path.join(folder, name)], 0)


@needs_vis
@pytest.mark.parametrize("B", [1, 2])
def test_reference_visualize_after_install_equals_the_drop_in(tmp_path, B):
    """The regression: after install() the reference's dva/visualize.py imports (ImportError before generate_colored_boxes existed);
    its video frames (15 -> 16 views) and its single-view and multi-view summary JPGs equal the drop-in's exactly.  B = 2 covers the
    set-major cameras, two primitive sets in one march and the view-major order of the frames."""
    tpxl_b200.install()
    recon = _recon(B)
    rm = tpxl_b200.RayMarcher(256, 256, VR).cuda()
    ref_dir, our_dir = tmp_path / "ref", tmp_path / "ours"
    ref_dir.mkdir()
    our_dir.mkdir()
    with ov.reference_visualize("ours") as (vis, stub):
        vis.visualize_video_primvolume(str(ref_dir), {}, recon, 15, rm, "cuda")
        vis.visualize_primvolume(str(ref_dir / "one.jpg"), {}, recon, rm, "cuda")
        vis.visualize_multiview_primvolume(str(ref_dir / "multi.jpg"), {}, recon, 4, rm, "cuda")
        ref_rgb, ref_prim = _frames(stub, str(ref_dir), "rgb.mp4"), _frames(stub, str(ref_dir), "prim.mp4")
    stub = ov.imageio_stub()
    saved = sys.modules.get("imageio")
    sys.modules["imageio"] = stub
    try:
        tv.visualize_video_primvolume(str(our_dir), {}, recon, 15, rm, "cuda")
    finally:
        if saved is None:
            del sys.modules["imageio"]
        else:
            sys.modules["imageio"] = saved
    tv.visualize_primvolume(str(our_dir / "one.jpg"), {}, recon, rm, "cuda")
    tv.visualize_multiview_primvolume(str(our_dir / "multi.jpg"), {}, recon, 4, rm, "cuda")
    rgb, prim, mat = (_frames(stub, str(our_dir), n) for n in ("rgb.mp4", "prim.mp4", "mat.mp4"))
    assert ref_rgb.shape == (16 * B, 256, 256, 3) and rgb.shape == ref_rgb.shape and mat.shape == rgb.shape
    assert ref_rgb.max() > 100 and ref_prim.max() > 100
    assert np.array_equal(rgb, ref_rgb) and np.array_equal(prim, ref_prim)
    for name in ("one.jpg", "multi.jpg"):
        assert (ref_dir / name).read_bytes() == (our_dir / name).read_bytes(), name


def _figures(img, rimg):
    """tests/test_gpu_raymarch_ref.py's _check figures on frames [N, H, W, 4] (channels last here): relative L2 over the batch, value
    range per channel over the batch, the largest channel deviation per pixel over that range."""
    rel = float((img - rimg).norm() / rimg.norm())
    rng = (rimg.amax(dim=(0, 1, 2)) - rimg.amin(dim=(0, 1, 2))).clamp(min=1e-6).view(1, 1, 1, 4)
    dev = ((img - rimg).abs() / rng).amax(-1)
    return rel, float((dev > 1e-3).float().mean()), float(dev.max())


@needs_ref
@pytest.mark.parametrize("H,views,B", [(256, 15, 1), (518, 4, 1), (256, 4, 2)])
def test_drop_in_frames_within_the_reference_ray_marcher_bounds(H, views, B):
    """The drop-in's rgba frames against those of the reference's dva/visualize.py over its own RayMarcher and extensions (captured
    at the march's output, before the uint8 conversion): _check's figures on all frames of a kind, and on every frame alone."""
    recon = _recon(B)
    with ov.reference_visualize("reference") as (vis, _):
        rm_ref = vis.RayMarcher(H, H, VR, dt=1.0).cuda()
        outs = []
        real = rm_ref.forward

        def capture(*a, **k):
            res = real(*a, **k)
            outs.append(res["rgba_image"].permute(0, 2, 3, 1).clone())
            return res

        rm_ref.forward = capture
        vis.visualize_video_primvolume(tempfile.mkdtemp(), {}, recon, views, rm_ref, "cuda")
    ref = {"rgb": torch.cat(outs[0::2], 0), "boxes": torch.cat(outs[1::2], 0)}
    rm = tpxl_b200.RayMarcher(H, H, VR)
    angles = torch.linspace(1.5, 3.5, views + 1) * torch.pi
    frames = tv.render_views(recon, rm, tv.orbit_extrinsics(rm, B, angles).cuda(), tv.preview_intrinsics(rm, B).cuda(), kinds=("rgb", "boxes"),
                             alpha=True)
    for kind in ("rgb", "boxes"):
        img, rimg = frames[kind], ref[kind]
        assert img.shape == rimg.shape == ((views + 1) * B, H, H, 4)
        alpha = rimg[..., 3]
        assert float(alpha.max()) > 0.3 and float((alpha > 0).float().mean()) > 0.05, kind          # the scene is actually rendered
        rel, share, worst = _figures(img, rimg)
        print(f"{kind} H={H} B={B}: all frames rel-L2 {rel:.2e}, share {share:.2e}, worst {worst:.2e}")
        assert rel <= IMG_REL and share <= PIX_SHARE and worst <= PIX_MAX, (kind, rel, share, worst)
        for f in range(img.shape[0]):
            rel, share, worst = _figures(img[f:f + 1], rimg[f:f + 1])
            assert rel <= IMG_REL and share <= PIX_SHARE and worst <= PIX_MAX, (kind, f, rel, share, worst)


def test_material_frames():
    """mat frames are finite, their alpha is the rgb frames' alpha bit for bit, and their red channel is 0."""
    recon, rm, Rt, K = _scene(2, 16, 256)
    B, P = recon.shape[:2]
    pos = (recon[:, :, 1:4] * VR / VR).contiguous()
    rot = torch.eye(3, device="cuda")[None, None].repeat(B, P, 1, 1).contiguous()
    scale = (1 / recon[:, :, 0:1].repeat(1, 1, 3)).contiguous()
    cams = [march_camera(Rt[v].clone(), K, "cuda") for v in range(16)]
    cam = tuple(torch.stack([c[i] for c in cams], 1).reshape(B * 16, *cams[0][i].shape[1:]).contiguous() for i in range(4))
    geom = (256, 256, VR, 1.0 / VR, 8.0, 8.0)
    rgb = march_views(tv.primvolume_payload(recon, "rgb"), pos, rot, scale, cam, 16, *geom)
    mat = march_views(tv.primvolume_payload(recon, "mat"), pos, rot, scale, cam, 16, *geom)
    assert bool(torch.isfinite(mat).all()) and torch.equal(mat[..., 3], rgb[..., 3]) and bool((mat[..., 0] == 0).all())
    assert float(mat[..., 1].amax()) > 10 and float(rgb[..., 3].amax()) > 0.3
    frames = tv.render_views(recon, rm, Rt, K, kinds=("mat",))["mat"]
    assert frames.shape == (16 * B, 256, 256, 3) and bool((frames[..., 0] == 0).all())
