#!/usr/bin/env python
"""Time mesh clean-up at R = 128, 256 and 512 on the synthetic object of tools/mesh_perf.py (2048 primitives on a noisy sphere
shell): the reference-faithful clean_mesh(v, t, v_pct=1, min_f=8, min_d=5, repair=True, remesh=False) of inference.py:126, stage by
stage, then decimation to 100 000 faces with and without it.
  * per stage (weld = close-vertex merge + duplicate / null faces, component filter, repair): device-event time, the face count after
    it, and the weld's merge rounds;
  * decimation to 100 000 faces from the cleaned mesh and from today's default chain (component filter only): wall time on the host
    clock around a synchronise, rounds, faces out;
  * the error figures of tools/decimate_perf.py for both: share of face normals agreeing with the sdf-grid gradient, and |trilinear
    sdf| at the output vertices in voxels.  The merge moves vertices by up to r (1 % of the diagonal), so this figure is expected to grow.
Prints the card name, power limit and clock (nvidia-smi) in the same run."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from decimate_perf import error_figures  # noqa: E402
from mesh_perf import shell_module  # noqa: E402
from tpxl_b200 import mesh  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def decimated(v, f, target, reps):
    mesh._decimate(v, f, target)
    torch.cuda.synchronize()
    walls = []
    for _ in range(reps):
        trace = []
        t0 = time.perf_counter()
        out = mesh._decimate(v, f, target, trace)
        torch.cuda.synchronize()
        walls.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(walls)), len(trace), out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q}")
    m = shell_module()
    target = int(os.environ.get("TARGET", "100000"))
    for R in [int(r) for r in os.environ.get("RES", "128,256,512").split(",")]:
        reps = 5 if R <= 256 else 2
        grid = m.sdf_grid(R)
        v0, f0 = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
        info = {}
        t_w, (v1, f1) = timed(lambda: mesh._weld(v0, f0, 0.01, info), reps)
        t_c, (v2, f2) = timed(lambda: mesh._remove_small(v1, f1, 8, 0.05), reps)
        t_r, (v3, f3) = timed(lambda: mesh._repair(v2, f2), reps)
        print(f"R={R:4d}  F in {f0.shape[0]:9d} | weld {t_w:8.2f} ms, {info['rounds']} rounds -> F {f1.shape[0]} | components {t_c:7.2f} ms -> F {f2.shape[0]} "
              f"| repair {t_r:7.2f} ms -> F {f3.shape[0]}, V {v3.shape[0]} (from {v2.shape[0]})")
        t_b, (vb, fb) = timed(lambda: mesh._remove_small(v0, f0, 8, 0.05), reps)
        for name, (v, f) in (("cleaned", (v3, f3)), ("component filter only", (vb, fb))):
            wall, rounds, (vd, fd) = decimated(v, f, target, reps)
            agree, emean, emax = error_figures(grid, vd, fd, R)
            print(f"        decimate {name} ({f.shape[0]} faces) to {target}: wall {wall:8.1f} ms, {rounds} rounds -> F {fd.shape[0]} | normals agreeing "
                  f"{agree:.5f} | |sdf| at vertices mean {emean:.4f} max {emax:.3f} voxels")
        del grid, v0, f0, v1, f1, v2, f2, v3, f3, vb, fb
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
