#!/usr/bin/env python
"""Time mesh extraction at R = 128, 256 and 512 on the synthetic object of tools/primsdf_perf.py (2048 primitives on a noisy
sphere shell):
  * PrimSDF.sdf_grid (binned lists cached, as after the first call);
  * marching cubes on that grid (tpx_mc_count + tpx_mc_emit, including the counts readback between them);
  * PrimSDF.extract_mesh wall time (sdf grid + marching cubes + the counts readback, host clock around a synchronise);
  * the path inference.py:107-119 takes through this package today: PrimSDF.forward over linspace / meshgrid points in 8192-point
    chunks, then grid.cpu() (PyMCubes itself is not timed: it is not part of this package).
Device times are CUDA events.  Prints the card name and power limit, and V and F."""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tpxl_b200  # noqa: E402
from tpxl_b200 import mesh  # noqa: E402


def shell_module(K=2048, S=8):
    g = torch.Generator().manual_seed(0)
    d = torch.randn(K, 3, generator=g)
    pos = d / d.norm(dim=1, keepdim=True) * (0.55 + 0.1 * torch.rand(K, 1, generator=g))
    srt = torch.cat([0.03 + 0.05 * torch.rand(K, 1, generator=g), pos], 1)
    m = tpxl_b200.PrimSDF(num_prims=K, dim_feat=6, prim_shape=S).eval()
    m.srt_param.data = srt
    m.feat_param.data = torch.randn(K, 6 * S ** 3, generator=g)
    return m.cuda()


def device_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def wall_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps, out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q}")
    m = shell_module()
    for R in [int(r) for r in os.environ.get("RES", "128,256,512").split(",")]:
        reps = 10 if R <= 256 else 3
        t_grid, grid = device_ms(lambda: m.sdf_grid(R), reps)
        t_mc, (v, f) = device_ms(lambda: mesh.marching_cubes(grid, 0.0), reps)
        t_ex, _ = wall_ms(lambda: m.extract_mesh(R), reps)
        xx = torch.linspace(-1, 1, R, device="cuda")

        def chunked():
            pts = torch.stack(torch.meshgrid(xx, xx, xx, indexing="ij"), dim=-1).reshape(-1, 3)
            with torch.no_grad():
                dists = torch.cat([m(c)["sdf"].detach() for c in torch.split(pts, 8192)], 0)
            return dists.reshape(R, R, R).cpu()

        t_ref, ref = wall_ms(chunked, 1 if R >= 512 else 3)
        same = bool(torch.equal(ref, grid.cpu()))
        print(f"R={R:4d}  sdf_grid {t_grid:8.2f} ms | marching cubes (count+emit) {t_mc:7.2f} ms  V={v.shape[0]} F={f.shape[0]} | "
              f"extract_mesh wall {t_ex:8.2f} ms | chunked forward + grid.cpu() wall {t_ref:9.2f} ms (grid identical: {same})")
        del grid, v, f, ref
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
