"""Time the preview videos (2048 primitives of 8^3, volradius 10000, dt 1): the 61-view inference.py turntable at 518^2 and the
16-view app.py turntable at 256^2, three ways:
  ref       the reference's dva/visualize.py with its host generate_colored_boxes (over this package's RayMarcher);
  ref+boxes the same with this package's generate_colored_boxes (what tpxl_b200.install() gives the reference's module);
  drop-in   tpxl_b200.visualize.visualize_video_primvolume (payload and box kernels, one march per kind; also renders mat.mp4);
and the march alone: V per-view tpx_raymarch_preview launches against one tpx_raymarch_preview_views launch.  Each figure is a host
clock around the call ending in a synchronise (and CUDA events for the march alone); video encoding is replaced by a stub that keeps
the frames.  The reference's module needs the staged copy under oracle/_ref (oracle/stage_visualize.py); without it those rows are
"not measured".
"""
import os
import subprocess
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import tpxl_b200  # noqa: E402
from tpxl_b200 import visualize as tv  # noqa: E402
from tpxl_b200.ray_marcher import march_camera, march_views  # noqa: E402

REF = os.path.join(ROOT, "oracle", "_ref")
VR = 10000.0


def _imageio_stub():
    stub = types.ModuleType("imageio")

    class _W:
        def append_data(self, frame):
            pass

        def close(self):
            pass

    stub.get_writer = lambda path, **kw: _W()
    return stub


def _reference_visualize(generate_colored_boxes):
    """The staged dva/visualize.py over this package's RayMarcher and the given generate_colored_boxes, or None."""
    if not os.path.exists(os.path.join(REF, "dva", "visualize.py")):
        return None
    import importlib.util
    rm_mod = types.ModuleType("dva.ray_marcher")
    rm_mod.RayMarcher, rm_mod.generate_colored_boxes = tpxl_b200.RayMarcher, generate_colored_boxes
    pkg = types.ModuleType("dva")
    pkg.__path__ = [os.path.join(REF, "dva")]
    saved = {k: sys.modules.get(k) for k in ("dva", "dva.ray_marcher", "imageio")}
    sys.modules.update({"dva": pkg, "dva.ray_marcher": rm_mod, "imageio": _imageio_stub()})
    try:
        spec = importlib.util.spec_from_file_location("dva.visualize", os.path.join(REF, "dva", "visualize.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    mod.imageio = _imageio_stub()
    return mod


def _reference_host_boxes():
    """The reference's generate_colored_boxes (a Python loop over the primitives) from the staged dva/ray_marcher.py, taken out of the
    module source so its extensions are not needed."""
    path = os.path.join(REF, "dva", "ray_marcher.py")
    if not os.path.exists(path):
        return None
    src = open(path).read()
    body = src[src.index("def generate_colored_boxes"):]
    ns = {"th": torch, "np": np}
    exec(compile(body, path, "exec"), ns)
    return ns["generate_colored_boxes"]


def _recon(P=2048, S=8, seed=3):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(1, P, 3, generator=g)
    pos = d / d.norm(dim=-1, keepdim=True) * 0.5
    scale = 0.045 + 0.01 * torch.rand(1, P, 1, generator=g)
    sdf = torch.rand(1, P, S ** 3, generator=g) * 0.02 - 0.004
    return torch.cat([scale, pos, sdf, torch.rand(1, P, 5 * S ** 3, generator=g)], dim=-1).cuda()


def _time(fn, reps=2, warm=True):
    if warm:
        fn()
        torch.cuda.synchronize()
    best = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best.append(time.perf_counter() - t0)
    return min(best) * 1e3


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q}")
    recon = _recon()
    ref_boxes, our_boxes = _reference_host_boxes(), tpxl_b200.ray_marcher.generate_colored_boxes
    for name, views, H in (("inference.py", 60, 518), ("app.py", 15, 256)):
        rm = tpxl_b200.RayMarcher(H, H, VR).cuda()
        out = tempfile.mkdtemp()
        rows = {}
        for label, gcb in (("ref+boxes", our_boxes), ("ref", ref_boxes)):       # the slow host loop last, unwarmed: kernels are warm by then
            mod = _reference_visualize(gcb) if gcb is not None else None
            rows[label] = _time(lambda: mod.visualize_video_primvolume(out, {}, recon, views, rm, "cuda"), reps=1, warm=label != "ref") if mod else None
        sys.modules["imageio"] = _imageio_stub()
        rows["drop-in"] = _time(lambda: tv.visualize_video_primvolume(out, {}, recon, views, rm, "cuda"))
        fmt = lambda v: "not measured" if v is None else f"{v:.1f} ms"  # noqa: E731
        print(f"{name} video, {views + 1} views at {H}^2: " + ", ".join(f"{k} {fmt(v)}" for k, v in rows.items()))

        # the march alone: rgb payload, V cameras
        V = views + 1
        angles = torch.linspace(1.5, 3.5, V) * torch.pi
        Rt, K = tv.orbit_extrinsics(rm, 1, angles).cuda(), tv.preview_intrinsics(rm, 1).cuda()
        tpl = tv.primvolume_payload(recon, "rgb")
        pos = recon[:, :, 1:4].contiguous()
        rot = torch.eye(3, device="cuda")[None, None].repeat(1, 2048, 1, 1).contiguous()
        scale = (1 / recon[:, :, 0:1].repeat(1, 1, 3)).contiguous()
        cams = [march_camera(Rt[v].clone(), K, "cuda") for v in range(V)]
        cam = tuple(torch.cat([c[i] for c in cams], 0).contiguous() for i in range(4))
        geom = (H, H, VR, 1.0 / VR, 8.0, 8.0)
        res = {}
        for label, fn in (("per-view", lambda: [march_views(tpl, pos, rot, scale, c, 1, *geom) for c in cams]),
                          ("one launch", lambda: march_views(tpl, pos, rot, scale, cam, V, *geom))):
            fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ts = []
            for _ in range(3):
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
            res[label] = ts
        print(f"  march, {V} views at {H}^2: " + ", ".join(f"{k} {min(v):.1f} ms (max {max(v):.1f})" for k, v in res.items()))


if __name__ == "__main__":
    main()
