#!/usr/bin/env python
"""Time mesh clean-up and decimation at R = 128, 256 and 512 on the synthetic object of tools/mesh_perf.py (2048 primitives on a
noisy sphere shell), the geometry branch of extract_texmesh (inference.py:119-129: marching cubes, clean_mesh's component filter
with min_f = 8 / min_d = 5, decimate_mesh to 100 000 faces):
  * F in: the marching-cubes face count;
  * the component filter (remove_small_components(8, 0.05), device events, counts readback included);
  * decimation to 100 000 faces: wall time on the host clock around a synchronise (the entry point synchronises once per round),
    the number of rounds and the face count after each;
  * the error figures of tests/test_gpu_decimate.py: share of face normals that agree with the sdf-grid gradient at the centroid,
    and |trilinear sdf| at the output vertices in voxels (voxel = 2 / (R - 1)).
Prints the card name, power limit and clock (nvidia-smi) in the same run."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mesh_perf import shell_module  # noqa: E402
from tpxl_b200 import mesh  # noqa: E402


def trilinear(grid, p, R):
    u = np.clip((p + 1) / 2 * (R - 1), 0, R - 1 - 1e-9)
    i = np.floor(u).astype(np.int64)
    t = u - i
    out = np.zeros(len(p))
    for c in range(8):
        o = np.array([(c >> 2) & 1, (c >> 1) & 1, c & 1])
        out += np.prod(np.where(o[None] == 1, t, 1 - t), 1) * grid[i[:, 0] + o[0], i[:, 1] + o[1], i[:, 2] + o[2]]
    return out


def error_figures(grid, v, f, R):
    g = grid.cpu().numpy().astype(np.float64)
    p = v.cpu().numpy().astype(np.float64)
    tri = p[f.cpu().numpy()]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    c = tri.mean(1)
    h = 1.0 / (R - 1)
    grad = np.stack([trilinear(g, c + h * e, R) - trilinear(g, c - h * e, R) for e in np.eye(3)], 1)
    agree = float((np.einsum("ij,ij->i", n, grad) > 0).mean())
    err = np.abs(trilinear(g, p, R)) * (R - 1) / 2
    return agree, float(err.mean()), float(err.max())


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q}")
    m = shell_module()
    target = int(os.environ.get("TARGET", "100000"))
    for R in [int(r) for r in os.environ.get("RES", "128,256,512").split(",")]:
        grid = m.sdf_grid(R)
        v0, f0 = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
        reps = 5 if R <= 256 else 2
        mesh.remove_small_components(v0, f0, 8, 0.05)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            v1, f1 = mesh.remove_small_components(v0, f0, 8, 0.05)
        e1.record()
        torch.cuda.synchronize()
        t_cc = e0.elapsed_time(e1) / reps
        mesh._decimate(v1, f1, target)                 # warm-up (module load, CUB tuning)
        torch.cuda.synchronize()
        walls = []
        for _ in range(reps):
            trace = []
            t0 = time.perf_counter()
            v2, f2 = mesh._decimate(v1, f1, target, trace)
            torch.cuda.synchronize()
            walls.append((time.perf_counter() - t0) * 1e3)
        agree, emean, emax = error_figures(grid, v2, f2, R)
        print(f"R={R:4d}  F in {f0.shape[0]:9d} | filter {t_cc:7.2f} ms -> F {f1.shape[0]} | decimate to {target}: wall {np.median(walls):8.1f} ms "
              f"(min {min(walls):.1f}, max {max(walls):.1f}, {reps} runs), {len(trace)} rounds -> F {f2.shape[0]}, V {v2.shape[0]}")
        print(f"        normals agreeing with the grid gradient {agree:.5f} | |sdf| at vertices: mean {emean:.4f} max {emax:.3f} voxels")
        print(f"        F after each round: {trace}")
        del grid, v0, f0, v1, f1, v2, f2
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
