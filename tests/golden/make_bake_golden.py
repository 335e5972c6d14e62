#!/usr/bin/env python
"""Golden texture bake (DESIGN.md §1 f-6), produced by RUNNING THE REFERENCE'S OWN STATEMENTS.

Run in the build container only (needs /root/reference, scipy and scikit-learn):

    python tests/golden/make_bake_golden.py

extract_texmesh bakes its texture in a statement block of ``inference.py`` (:176-211: the masked PrimSDF.forward over the covered texels
in ``batch_size`` chunks, * 255, then binary_dilation / binary_erosion / a kd-tree nearest-neighbour search for the seam padding), not
in a function, and ``inference.py`` cannot be imported here (rembg, nvdiffrast, ... at module level).  This script reads exactly that
block from the reference file AT RUN TIME (nothing of it is stored in this repository) and executes it on the CPU with the reference's
own ``models.primsdf.PrimSDF``, scipy and scikit-learn (``trimesh`` stubbed as in make_golden.py), batch_size 8192, on:
  * a seeded shell of 96 primitives whose sdf voxels sample a sphere and whose colour / material voxels are smooth, non-zero fields;
  * the oracle marching-cubes mesh of its 24^3 sdf grid (the reference's PrimSDF evaluates the grid);
  * UVs from the reference's own fast-unwrap statements (:142-150: ``compute_vertex_normal`` + ``box_projection_uv_unwrap`` of
    utils/uv_unwrap.py and the per-corner re-indexing), also read and executed at run time;
  * a 128 x 128 atlas; ``rast`` comes from oracle.bake.rasterize_uv (nvdiffrast cannot run here), ``xyzs`` / ``mask`` from
    oracle.bake.interpolate as :173-174 derive them.
tests/golden/texture_bake.npz receives srt, feat, v, f, vt, ft, mask, the pre- and post-inpaint feats, and for every inpainted texel
the squared distance to the source texel the kd-tree chose.
"""
import os
import sys
import textwrap
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference"
REF_FILE = os.path.join(REF, "inference.py")
OUT = os.path.join(ROOT, "tests", "golden", "texture_bake.npz")
RES, ATLAS, BATCH, K, S = 24, 128, 8192, 96, 8


def reference_lines(first, last) -> str:
    """The statements from the first line matching ``first`` through the next line matching ``last`` (predicates on stripped lines)."""
    lines = open(REF_FILE).read().split("\n")
    start = next(i for i, l in enumerate(lines) if first(l.strip()))
    end = next(i for i in range(start, len(lines)) if last(lines[i].strip()))
    return textwrap.dedent("\n".join(lines[start:end + 1]))


def shell(seed: int = 2025):
    """96 primitives on a noisy sphere shell; channel 0 samples the sphere |x| = 0.55, channels 1-5 smooth fields of the world position
    quantised to 1/64 (so the fixture compresses), reaching below 0 and above 1 so the clip of PrimSDF.forward is exercised."""
    rs = np.random.RandomState(seed)
    d = rs.standard_normal((K, 3))
    pos = d / np.linalg.norm(d, axis=1, keepdims=True) * (0.55 + 0.04 * rs.uniform(-1, 1, (K, 1)))
    scale = rs.uniform(0.12, 0.2, (K, 1))
    srt = np.concatenate([scale, pos], 1).astype(np.float32)
    lin = np.linspace(-1, 1, S)
    zz, yy, xx = np.meshgrid(lin, lin, lin, indexing="ij")            # voxel [z, y, x] sits at local (x, y, z)
    local = np.stack([xx, yy, zz], -1).reshape(-1, 3)
    world = pos[:, None, :] + scale[:, None, :] * local[None]
    feat = np.zeros((K, 6, S ** 3))
    feat[:, 0] = np.linalg.norm(world, axis=-1) - 0.55
    phase = rs.uniform(0, 2 * np.pi, (5, 3))
    for c in range(5):
        field = 0.5 + 0.6 * np.sin(3.0 * world @ np.array([1.0, 0.7, -0.4]) * (1 + 0.2 * c) + phase[c, 0]) * np.cos(2.0 * world[..., (c + 1) % 3] + phase[c, 1])
        feat[:, 1 + c] = np.round(field * 64) / 64
    return srt, feat.reshape(K, -1).astype(np.float32)


def main():
    sys.modules.setdefault("trimesh", types.ModuleType("trimesh"))
    sys.path.insert(0, REF)
    from models.primsdf import PrimSDF  # noqa: E402
    from scipy.ndimage import binary_dilation, binary_erosion  # noqa: E402
    from sklearn.neighbors import NearestNeighbors  # noqa: E402
    from utils.uv_unwrap import box_projection_uv_unwrap, compute_vertex_normal  # noqa: E402
    from oracle import bake as obake, mesh as omesh  # noqa: E402

    srt, feat = shell()
    model = PrimSDF(num_prims=K, dim_feat=6, prim_shape=S).eval()
    model.srt_param.data = torch.from_numpy(srt)
    model.feat_param.data = torch.from_numpy(feat)
    xx = torch.linspace(-1, 1, RES)
    pts = torch.stack(torch.meshgrid(xx, xx, xx, indexing="ij"), dim=-1).reshape(-1, 3)
    with torch.no_grad():
        grid = model(pts)["sdf"].reshape(RES, RES, RES).numpy()
    verts, tris = omesh.marching_cubes(grid, 0.0)
    verts = verts / (RES - 1.0) * 2.0 - 1.0                               # inference.py:122-124

    device = "cpu"
    ns = dict(torch=torch, np=np, device=device, compute_vertex_normal=compute_vertex_normal, box_projection_uv_unwrap=box_projection_uv_unwrap,
              v=torch.from_numpy(verts).float().contiguous(), f=torch.from_numpy(tris.astype(np.int64)).contiguous())
    unwrap = reference_lines(lambda l: l.startswith("v_normal = compute_vertex_normal("), lambda l: l.startswith("vt_np = uv_flat"))
    exec(compile(unwrap, REF_FILE + ":<extract_texmesh fast unwrap>", "exec"), ns)
    v, f = ns["v"], ns["f"]
    vt = torch.from_numpy(ns["vt_np"].astype(np.float32)).float().contiguous()          # inference.py:161-162
    ft = torch.from_numpy(ns["ft_np"].astype(np.int64)).int().contiguous()
    assert v.shape[0] == vt.shape[0] == 3 * f.shape[0] and float(vt.min()) >= 0 and float(vt.max()) <= 1

    h = w = ATLAS
    rast, _, _ = obake.rasterize_uv(vt.numpy(), ft.numpy(), h, w)
    xyzs = torch.from_numpy(obake.interpolate(v.numpy(), rast, f.numpy())).float().reshape(1, h, w, 3)
    mask = torch.from_numpy(obake.interpolate(np.ones((v.shape[0], 1)), rast, f.numpy())).float().reshape(1, h, w, 1)
    covered = (mask > 0).reshape(h, w).numpy()

    ns = dict(torch=torch, np=np, device=device, model=model, xyzs=xyzs, mask=mask, h=h, w=w, fp16=True, args=types.SimpleNamespace(batch_size=BATCH),
              binary_dilation=binary_dilation, binary_erosion=binary_erosion, NearestNeighbors=NearestNeighbors)
    query = reference_lines(lambda l: l == "xyzs = xyzs.view(-1, 3)", lambda l: l == "feats = (feats * 255)")
    pad = reference_lines(lambda l: l == "mask = mask.cpu().numpy()", lambda l: l.startswith("feats[tuple(inpaint_coords.T)] ="))
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")                                   # torch.cuda.amp.autocast on a machine without CUDA is a no-op
        exec(compile(query, REF_FILE + ":<extract_texmesh masked query>", "exec"), ns)
        feats_pre = ns["feats"].copy()
        exec(compile(pad, REF_FILE + ":<extract_texmesh seam padding>", "exec"), ns)
    feats_post = ns["feats"]
    assert np.array_equal(ns["mask"], covered) and feats_pre.shape == (h, w, 6) and feats_pre.dtype == np.float32
    chosen = ns["search_coords"][ns["indices"][:, 0]]
    inpaint_d2 = np.full((h, w), -1, dtype=np.int64)
    inpaint_d2[tuple(ns["inpaint_coords"].T)] = ((ns["inpaint_coords"] - chosen) ** 2).sum(1)
    np.savez_compressed(OUT, srt=srt, feat=feat, v=v.numpy(), f=f.numpy().astype(np.int32), vt=vt.numpy(), ft=ft.numpy(), mask=covered,
                        feats_pre=feats_pre, feats_post=feats_post, inpaint_d2=inpaint_d2.astype(np.int32))
    print("wrote", OUT, os.path.getsize(OUT), "bytes; triangles", f.shape[0], "covered texels", int(covered.sum()), "inpainted", int((inpaint_d2 >= 0).sum()),
          "chunks", -(-int(covered.sum()) // BATCH), "nonzero channels", (feats_pre.reshape(-1, 6).max(0) > 0).tolist())


if __name__ == "__main__":
    main()
