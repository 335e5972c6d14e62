#!/usr/bin/env python
"""Golden SDF grid for mesh extraction (DESIGN.md §1 f-5), produced by RUNNING THE REFERENCE'S OWN STATEMENTS.

Run in the build container only (needs /root/reference):

    python tests/golden/make_mesh_golden.py

The grid extract_texmesh meshes is built by a statement block of ``inference.py`` (:107-116: linspace / meshgrid points, PrimSDF.forward
in ``batch_size`` chunks, sdf column, reshape to R^3), not by a function, and ``inference.py`` cannot be imported here (rembg,
nvdiffrast, ... at module level).  This script reads exactly that block from the reference file AT RUN TIME (nothing of it is stored in
this repository) and executes it on the CPU with the reference's own ``models.primsdf.PrimSDF`` (``trimesh`` stubbed as in
make_golden.py, ``tqdm`` as the identity), mc_resolution 40 and batch_size 8192 (8 chunks), on a seeded shell of 96 primitives whose
sdf voxels sample a sphere.  srt, feat and the grid go to tests/golden/primsdf_grid.npz; tests/test_mesh_host.py holds
oracle.primsdf.query to it and tests/test_gpu_mesh.py holds PrimSDF.sdf_grid to it.
"""
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference"
REF_FILE = os.path.join(REF, "inference.py")
OUT = os.path.join(ROOT, "tests", "golden", "primsdf_grid.npz")
RES, BATCH, K, S = 40, 8192, 96, 8


def reference_block() -> str:
    lines = open(REF_FILE).read().split("\n")
    start = next(i for i, l in enumerate(lines) if l.strip() == "with torch.no_grad():" and "linspace" in lines[i + 1])
    end = next(i for i in range(start, len(lines)) if lines[i].strip().startswith("grid = dists.reshape("))
    return textwrap.dedent("\n".join(lines[start:end + 1]))


def shell(seed: int = 2024):
    """96 primitives on a noisy sphere shell; channel 0 samples the sphere |x| = 0.55, the colour / material channels are zero (the
    grid reads channel 0 only, and zeros keep the fixture small)."""
    rs = np.random.RandomState(seed)
    d = rs.standard_normal((K, 3))
    pos = d / np.linalg.norm(d, axis=1, keepdims=True) * (0.55 + 0.04 * rs.uniform(-1, 1, (K, 1)))
    scale = rs.uniform(0.12, 0.2, (K, 1))
    srt = np.concatenate([scale, pos], 1).astype(np.float32)
    lin = np.linspace(-1, 1, S)
    zz, yy, xx = np.meshgrid(lin, lin, lin, indexing="ij")            # voxel [z, y, x] sits at local (x, y, z)
    local = np.stack([xx, yy, zz], -1).reshape(-1, 3)
    world = pos[:, None, :] + scale[:, None, :] * local[None]
    sdf = np.linalg.norm(world, axis=-1) - 0.55
    feat = np.zeros((K, 6, S ** 3))
    feat[:, 0] = sdf
    return srt, feat.reshape(K, -1).astype(np.float32)


def main():
    sys.modules.setdefault("trimesh", types.ModuleType("trimesh"))
    sys.path.insert(0, REF)
    from models.primsdf import PrimSDF  # noqa: E402
    block = compile(reference_block(), REF_FILE + ":<extract_texmesh sdf grid block>", "exec")
    srt, feat = shell()
    model = PrimSDF(num_prims=K, dim_feat=6, prim_shape=S).eval()
    model.srt_param.data = torch.from_numpy(srt)
    model.feat_param.data = torch.from_numpy(feat)
    ns = dict(torch=torch, tqdm=lambda x: x, model=model, device="cpu", args=types.SimpleNamespace(mc_resolution=RES, batch_size=BATCH))
    exec(block, ns)
    grid = ns["grid"].numpy()
    assert grid.shape == (RES, RES, RES) and grid.dtype == np.float32
    np.savez_compressed(OUT, srt=srt, feat=feat, grid=grid)
    print("wrote", OUT, os.path.getsize(OUT), "bytes; inside fraction", float((grid < 0).mean()), "chunks", -(-RES ** 3 // BATCH))


if __name__ == "__main__":
    main()
