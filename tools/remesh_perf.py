#!/usr/bin/env python
"""Time isotropic remeshing at R = 128, 256 and 512 on the synthetic object of tools/mesh_perf.py (2048 primitives on a noisy sphere
shell), the geometry branch of extract_texmesh with "Remesh: Yes" (inference.py:119-129: marching cubes, the component filter with
min_f = 8 / min_d = 5, decimate_mesh(v, t, 100000, remesh=True)):
  * the filter and the decimation to 100 000 faces (their own tools time them; here they only make the input);
  * mesh.remesh at 1 % of the box diagonal, 3 iterations: wall time of the call and, per iteration, of the split and of the relax
    (collapse rounds, flip rounds, smoothing, projection), host clock around a synchronise (the entry points synchronise per round);
  * rounds per phase, F after each phase, V, and the share of edges in [4/5 L, 4/3 L] and of valence-6 vertices before and after.
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


def shares(v, f, L):
    V, F = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    a, b = F.ravel(), np.roll(F, -1, 1).ravel()
    E = np.unique(np.minimum(a, b) << 32 | np.maximum(a, b))
    ln = np.linalg.norm(V[E >> 32] - V[E & 0xFFFFFFFF], axis=1)
    val = np.bincount(np.concatenate([E >> 32, E & 0xFFFFFFFF]), minlength=len(V))
    return float(((ln >= 0.8 * L) & (ln <= 4 / 3 * L)).mean()), float((val[np.unique(F)] == 6).mean())


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q}")
    m = shell_module()
    for R in [int(r) for r in os.environ.get("RES", "128,256,512").split(",")]:
        grid = m.sdf_grid(R)
        v0, f0 = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
        v1, f1 = mesh._remove_small(v0, f0, 8, 0.05)
        vd, fd = mesh._decimate(v1, f1, 100000)
        d = vd.max(0).values.double() - vd.min(0).values.double()
        L = 0.01 * float(torch.sqrt((d * d).sum()))
        mesh.remesh(vd, fd, L, 1)                          # warm-up (module load, CUB tuning)
        torch.cuda.synchronize()
        walls, info = [], None
        for _ in range(3):
            info = []
            t0 = time.perf_counter()
            vr, fr = mesh.remesh(vd, fd, L, 3, info=info)
            torch.cuda.synchronize()
            walls.append((time.perf_counter() - t0) * 1e3)
        sb, sa = shares(vd, fd, L), shares(vr, fr, L)
        print(f"R={R:4d}  F mc {f0.shape[0]:9d} -> filter {f1.shape[0]} -> decimate {fd.shape[0]} | remesh L = {L:.5f} (1 % diag), 3 it: wall "
              f"{np.median(walls):8.1f} ms (min {min(walls):.1f}, max {max(walls):.1f}, 3 runs) -> F {fr.shape[0]}, V {vr.shape[0]}")
        for i, r in enumerate(info):
            print(f"        it {i}: split {r['split_ms']:7.1f} ms -> F {r['F'][0]}, V slots {r['V']} | relax {r['relax_ms']:7.1f} ms: "
                  f"{r['collapse_rounds']} collapse rounds -> F {r['F'][1]}, {r['flip_rounds']} flip rounds, smoothing, projection")
        print(f"        edges in [4/5 L, 4/3 L]: {sb[0]:.3f} -> {sa[0]:.3f} | valence 6: {sb[1]:.3f} -> {sa[1]:.3f}")
        del grid, v0, f0, v1, f1, vd, fd, vr, fr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
