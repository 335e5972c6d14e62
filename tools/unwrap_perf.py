#!/usr/bin/env python
"""Stage-by-stage device time of PrimSDF.extract_texmesh (the fast-unwrap branch of inference.py:90-222) on the 2048-primitive shell of
tools/mesh_perf.py: R = 256, 100 000 target faces, 1024^2 atlas.  Stages: noise filter, sdf grid + marching cubes, component filter,
decimation, vertex normals, unwrap (with its one count readback), bake.  CUDA events around each stage, after one warm-up pass; prints
the card name and power limit from the same run."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mesh_perf import shell_module  # noqa: E402
from tpxl_b200 import PrimSDF, mesh, unwrap  # noqa: E402


def stages(m, R=256, target=100000, atlas=1024):
    ev = [torch.cuda.Event(enable_timing=True)]
    ev[0].record()
    names = []

    def mark(name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev.append(e)
        names.append(name)

    keep = m.noise_filter_mask()
    mark("noise filter")
    sub = PrimSDF(num_prims=0)
    sub.srt_param.data, sub.feat_param.data = m.srt_param.detach()[keep].contiguous(), m.feat_param.detach()[keep].contiguous()
    sub.eval()
    grid = sub.sdf_grid(R)
    v, f = mesh._mesh(grid, 0.0, origin=(-1.0,) * 3, spacing=(2.0 / (R - 1),) * 3)
    mark("sdf grid + marching cubes")
    v, f = mesh._remove_small(v, f, 8, 0.05)
    mark("components")
    v, f = mesh._decimate(v, f, target)
    mark("decimate")
    n = unwrap.compute_vertex_normal(v, f)
    mark("vertex normals")
    uv, idx = unwrap.box_projection_uv_unwrap(v, n, f, 0.02)
    mark("unwrap")
    vt = uv[idx].reshape(-1, 2)
    ft = torch.arange(3 * f.shape[0], device=v.device).reshape(-1, 3)
    sub.bake_texture(v[f].reshape(-1, 3), ft, vt, ft, atlas)
    mark("bake")
    torch.cuda.synchronize()
    return [(nm, ev[i].elapsed_time(ev[i + 1])) for i, nm in enumerate(names)], f.shape[0], uv.shape[0]


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q}")
    m = shell_module()
    stages(m)
    for rep in range(3):
        t, F, U = stages(m)
        print(f"run {rep}: F {F} U {U} | " + " | ".join(f"{nm} {ms:.2f} ms" for nm, ms in t) + f" | total {sum(ms for _, ms in t):.1f} ms")


if __name__ == "__main__":
    main()
