"""CPU: the preview payloads' oracle and the package's host code against the reference's own dva/visualize.py and
generate_colored_boxes (fixture tests/golden/visualize.npz, tests/golden/make_visualize_golden.py), the C entries' argument checks and
device guard, and the dva.visualize binding of install()."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tpxl_b200
from oracle import visualize as ov
from tpxl_b200 import _lib
from tpxl_b200 import visualize as tv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOX_CASES = [(6, 4, 1), (6, 5, 2), (6, 8, 1), (6, 8, 2), (2048, 8, 1)]
PAYLOAD_CASES = [(1, 6, 4), (2, 6, 5), (1, 6, 8), (2, 6, 8)]
VIDEO_CASES = [(1, 15, 256), (2, 15, 256), (1, 60, 518), (2, 60, 518)]


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(os.path.join(golden_dir, "visualize.npz"))


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True)


def _rng_after(fx, tag):
    st = np.random.get_state()
    return np.array_equal(st[1], fx[tag + "_rng_keys"]) and st[2] == int(fx[tag + "_rng_pos"])


@pytest.mark.parametrize("K,S,B", BOX_CASES)
def test_box_oracle_matches_the_reference(fx, K, S, B):
    """Colours, template and numpy's global generator state after the call, bit for bit; at odd S the centre voxel's colour is NaN
    (a zero normal), in the reference and the oracle alike."""
    tag = f"boxes_K{K}_S{S}_B{B}"
    np.random.seed(999)
    colors = ov.box_colors(K)
    assert _rng_after(fx, tag)
    t = ov.box_template(B, K, S, colors).numpy()
    if K > 64:
        assert _same(t[:, [0, 1, 1023, 2047]], fx[tag + "_prims"]) and _same(t[0, :, :, 0, 0, 0], fx[tag + "_corner"])
    else:
        assert _same(t, fx[tag])
    c = S // 2
    assert bool(np.isnan(t[:, :, :3, c, c, c]).all()) == (S % 2 == 1)
    assert bool(np.isnan(t[:, :, 3]).any()) is False


@pytest.mark.parametrize("K", [6, 2048])
def test_package_box_colors_draw_as_the_reference(fx, K):
    """tpxl_b200.ray_marcher.box_colors (the host half of generate_colored_boxes): np.random.rand(K, 3) * 255.0 gives the reference's
    3 K scalar draws and leaves the same global generator state."""
    S, B = (8, 1) if K > 64 else (4, 1)
    tag = f"boxes_K{K}_S{S}_B{B}"
    np.random.seed(999)
    colors = tpxl_b200.ray_marcher.box_colors(K)
    assert _rng_after(fx, tag)
    np.random.seed(999)
    assert torch.equal(colors, ov.box_colors(K))


@pytest.mark.parametrize("B,P,S", PAYLOAD_CASES)
def test_payload_oracle_matches_the_reference(fx, B, P, S):
    """The rgb payload is the reference's prim_rgba (channels-last); the material payload shares its alpha and has a zero red channel."""
    tag = f"payload_B{B}_P{P}_S{S}"
    recon = torch.from_numpy(fx[tag + "_recon"])
    rgb = ov.payload(recon, "rgb")
    assert _same(rgb.numpy(), np.ascontiguousarray(fx[tag + "_prim_rgba"].transpose(0, 1, 3, 4, 5, 2)))
    mat = ov.payload(recon, "mat")
    assert torch.equal(mat[..., 3], rgb[..., 3]) and bool((mat[..., 0] == 0).all())
    S3 = S ** 3
    want = recon[:, :, 4 + 4 * S3:].reshape(B, P, 2, S, S, S).permute(0, 1, 3, 4, 5, 2) * 255
    assert torch.equal(mat[..., 1:3], want)
    # the front camera of visualize_primvolume, built by the package's host code
    rm = tpxl_b200.RayMarcher(518, 518, 10000.0)
    assert _same(tv.front_extrinsics(rm, B).numpy(), fx[tag + "_RT"]) and _same(tv.preview_intrinsics(rm, B).numpy(), fx[tag + "_K"])
    # the box template of render_mvp_boxes on this payload
    np.random.seed(5)
    assert _same(ov.box_template(B, P, S, ov.box_colors(P)).numpy(), fx[tag + "_boxes"])


@pytest.mark.parametrize("B,V,H", VIDEO_CASES)
def test_orbit_cameras_match_the_reference(fx, B, V, H):
    """The per-view extrinsics and the intrinsics of visualize_video_primvolume (16 views at 256^2 as app.py, 61 at 518^2 as
    inference.py), from the oracle and from the package's host code, bit for bit."""
    tag = f"video_B{B}_V{V + 1}_H{H}"
    angles = torch.linspace(1.5, 3.5, V + 1) * torch.pi
    rm = tpxl_b200.RayMarcher(H, H, 10000.0)
    assert _same(ov.orbit_poses(5 * 10000.0, angles, B).numpy(), fx[tag + "_RT"])
    assert _same(tv.orbit_extrinsics(rm, B, angles).numpy(), fx[tag + "_RT"])
    assert _same(ov.intrinsics(H, H, B).numpy(), fx[tag + "_K"]) and _same(tv.preview_intrinsics(rm, B).numpy(), fx[tag + "_K"])


def test_new_entries_check_arguments_then_device():
    """tpx_colored_boxes, tpx_primvolume_payload and tpx_raymarch_preview_views reject bad arguments before any CUDA call, and with
    valid arguments fail at the device guard when there is no usable device."""
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses below must never reach a GPU")
    import __graft_entry__
    __graft_entry__._load_build_module().build()
    lib = _lib.load_library()
    P = 1 << 20
    bad = [
        (lib.tpx_colored_boxes, (None, 1, 6, 8, 1e4, 0, P, None), -1),
        (lib.tpx_colored_boxes, (P, 1, 6, 1, 1e4, 0, P, None), -3),          # S >= 2
        (lib.tpx_colored_boxes, (P, 1, 6, 8, 1e4, 2, P, None), -1),          # unknown layout
        (lib.tpx_colored_boxes, (P, 1, 6, 8, 1e4, 1, P + 4, None), -1),      # channels-last output not 16-B aligned
        (lib.tpx_primvolume_payload, (P, 1, 6, 8, 2, P, None), -1),          # unknown mode
        (lib.tpx_primvolume_payload, (P, 0, 6, 8, 0, P, None), -3),
        (lib.tpx_primvolume_payload, (P, 1, 6, 8, 0, P + 4, None), -1),
        (lib.tpx_raymarch_preview_views, (P, P, P, P, P, P, P, P, 6, 4, 2, 8, 8, 8, 1.0, 0.01, 8.0, 8.0, P, None), -3),   # 4 does not divide 6
        (lib.tpx_raymarch_preview_views, (P, P, P, P, P, P, P, P, 6, 0, 2, 8, 8, 8, 1.0, 0.01, 8.0, 8.0, P, None), -3),
    ]
    for fn, args, rc in bad:
        assert fn(*args) == rc, (fn.__name__, args, lib.tpx_last_error())
    good = [
        (lib.tpx_colored_boxes, (P, 2, 6, 8, 1e4, 0, P, None)),
        (lib.tpx_colored_boxes, (P, 2, 6, 5, 1e4, 1, P, None)),
        (lib.tpx_primvolume_payload, (P, 2, 6, 8, 1, P, None)),
        (lib.tpx_raymarch_preview_views, (P, P, P, P, P, P, P, P, 6, 3, 2, 8, 8, 8, 1.0, 0.01, 8.0, 8.0, P, None)),
    ]
    for fn, args in good:
        assert fn(*args) == -2 and b"cudaGetDevice" in lib.tpx_last_error(), (fn.__name__, lib.tpx_last_error())
    assert ctypes.c_int is _lib.SIGNATURES["tpx_colored_boxes"][0]


def test_visualize_module_imports_without_the_encoders():
    """cv2, torchvision and imageio are imported only by the functions that write files."""
    code = ("import sys\nfor m in ('cv2', 'torchvision', 'imageio'):\n    sys.modules[m] = None\n"
            "import tpxl_b200\nfrom tpxl_b200 import visualize\nassert callable(visualize.render_views)\nprint('ok')\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, env={**os.environ, "PYTHONPATH": ROOT})
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


def test_install_binds_dva_visualize():
    """install() binds dva.visualize to the drop-in, and dva.ray_marcher carries generate_colored_boxes (what the reference's
    dva/visualize.py imports from it).  The from-imports inference.py:12,15 and app.py:17-18 use resolve from sys.modules without a
    dva package; install() adds none, so a reference checkout put on sys.path afterwards still provides the rest of dva."""
    code = ("import sys\nimport tpxl_b200\ntpxl_b200.install()\nfrom dva.ray_marcher import RayMarcher, generate_colored_boxes\n"
            "from dva.visualize import visualize_primvolume, visualize_video_primvolume\nimport tpxl_b200.visualize as tv\n"
            "assert visualize_primvolume is tv.visualize_primvolume and visualize_video_primvolume is tv.visualize_video_primvolume\n"
            "assert sys.modules['dva.visualize'] is tv and generate_colored_boxes is tpxl_b200.ray_marcher.generate_colored_boxes\n"
            "assert 'dva' not in sys.modules or hasattr(sys.modules['dva'], '__file__')\nprint('ok')\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, env={**os.environ, "PYTHONPATH": ROOT})
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


@pytest.mark.skipif(not ov.available("ours"), reason="dva/visualize.py is not staged (python oracle/stage_visualize.py where the reference exists)")
def test_reference_visualize_imports_over_the_package_ray_marcher():
    """The reference's own dva/visualize.py imports over tpxl_b200.ray_marcher (what install() binds as dva.ray_marcher): it needs
    RayMarcher and generate_colored_boxes from it.  The loader leaves no dva or imageio behind."""
    before = {k for k in sys.modules if k.split(".")[0] in ("dva", "imageio")}
    with ov.reference_visualize("ours") as (vis, stub):
        assert vis.generate_colored_boxes is tpxl_b200.ray_marcher.generate_colored_boxes and vis.RayMarcher is tpxl_b200.RayMarcher
        assert vis.imageio is stub
    assert {k for k in sys.modules if k.split(".")[0] in ("dva", "imageio")} == before
