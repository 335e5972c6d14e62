#!/usr/bin/env python
"""Golden vectors for the PrimSDF query GRADIENTS, produced by running the reference's own ``models.primsdf.PrimSDF`` under CPU
autograd (the module PrimSDFLoss, dva/losses.py:102-148, differentiates when it fits primitives to a mesh).

Run in the build container only (needs /root/reference):

    python tests/golden/make_primsdf_grad_golden.py

The reference class is imported unchanged, with ``trimesh`` (imported but unused on this path) stubbed as make_golden.py does.
Leaves: the points x, ``srt_param`` and ``feat_param``; the outputs (sdf, tex, mat) are concatenated to [n,6] and back-propagated
with a seeded upstream gradient G, in training mode (uncovered points get nothing) and in eval mode (the nearest-voxel fill).
Two scenes:
  * "base": the scene and points of primsdf.npz (read from that file, not stored again);
  * "cons": a constructed scene, S = 5, dyadic positions and scales so that l = (x - pos) / s and the voxel lattice are exact:
    inf-norm ties on two and on three axes, a point at a primitive's centre, points on voxel planes, a point on a box boundary,
    uncovered points (one exactly on the nearest voxel, d = 0) and random points on a 1/64 lattice.  Uncovered points whose
    nearest primitive or nearest voxel is tied are dropped, so the fill's choice is unambiguous.
Everything goes to tests/golden/primsdf_grad.npz; tests/test_primsdf_grad_host.py holds the oracle to it.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
OUT = os.path.join(HERE, "primsdf_grad.npz")


def cons_scene():
    srt = np.array([[0.5, 0.0, 0.0, 0.0], [0.5, 0.75, 0.0, 0.0], [0.25, -0.5, 0.5, 0.25], [0.125, -0.375, -0.5, 0.625],
                    [0.25, 0.5, -0.625, -0.5], [0.5, -0.25, 0.25, -0.75]], np.float32)
    special = np.array([[0.0, 0.0, 0.0],          # centre of primitive 0: three-axis tie at l = 0
                        [0.25, 0.25, 0.125],      # l0 = (0.5, 0.5, 0.25): two-axis tie; on primitive 1's boundary (w = 0)
                        [0.25, -0.25, 0.25],      # l0 = (0.5, -0.5, 0.5): three-axis tie
                        [0.125, 0.0, -0.25],      # voxel planes l = 0 (y) and l = -0.5 (z)
                        [0.375, 0.0625, -0.0625], # covered by primitives 0 and 1
                        [-0.25, 0.75, 0.5],       # uncovered, exactly on primitive 2's corner voxel (d = 0)
                        [0.875, 0.875, -0.875], [-0.9375, -0.75, 0.5], [0.9375, 0.5, 0.9375]], np.float32)
    rs = np.random.RandomState(2025)
    pts = np.concatenate([special, (rs.randint(-64, 65, size=(400, 3)) / 64.0).astype(np.float32)])
    feat = rs.standard_normal(size=(len(srt), 6 * 5 ** 3)).astype(np.float32) * 0.6 + 0.4
    return srt, feat, pts


def unambiguous(pts, srt, S):
    """Drop uncovered points whose nearest centre or nearest voxel (of the nearest primitive) is tied, in fp64."""
    x, pos, s = pts.astype(np.float64), srt[:, 1:4].astype(np.float64), srt[:, 0].astype(np.float64)
    l = (x[:, None] - pos[None]) / s[None, :, None]
    covered = (1 - np.abs(l).max(-1) > 0).any(1)
    lin = np.linspace(-1, 1, S)
    grid = np.stack(np.meshgrid(lin, lin, lin, indexing="ij"), -1)[..., ::-1].reshape(-1, 3)
    keep = np.ones(len(x), bool)
    for i in np.nonzero(~covered)[0]:
        d = np.linalg.norm(x[i] - pos, axis=1)
        o = np.sort(d)
        k = int(d.argmin())
        dv = np.sort(np.linalg.norm(x[i] - (pos[k] + s[k] * grid), axis=1))
        keep[i] = (len(o) < 2 or o[1] - o[0] > 1e-6) and dv[1] - dv[0] > 1e-6
    return pts[keep]


def main():
    sys.path.insert(0, REF)
    sys.modules.setdefault("trimesh", types.ModuleType("trimesh"))
    from models.primsdf import PrimSDF              # noqa: E402
    base = np.load(os.path.join(HERE, "primsdf.npz"))
    scenes = {"base": (base["srt"], base["feat"], base["pts"], 8), "cons": (*cons_scene(), 5)}
    out = {}
    for name, (srt, feat, pts, S) in scenes.items():
        if name == "cons":
            pts = unambiguous(pts, srt, S)
            out["cons_srt"], out["cons_feat"], out["cons_pts"] = srt, feat, pts
        G = np.random.RandomState(7 if name == "base" else 8).standard_normal(size=(len(pts), 6)).astype(np.float32)
        out[f"{name}_G"] = G
        for mode in ("train", "eval"):
            m = PrimSDF(num_prims=len(srt), dim_feat=6, prim_shape=S)
            m.train(mode == "train")
            m.srt_param.data = torch.from_numpy(srt.copy())
            m.feat_param.data = torch.from_numpy(feat.copy())
            x = torch.from_numpy(pts.copy()).requires_grad_(True)
            preds = m(x)
            o = torch.cat([preds["sdf"], preds["tex"], preds["mat"]], 1)
            o.backward(torch.from_numpy(G))
            out[f"{name}_{mode}_out"] = o.detach().numpy()
            out[f"{name}_{mode}_grad_x"] = x.grad.numpy()
            out[f"{name}_{mode}_grad_srt"] = m.srt_param.grad.numpy()
            out[f"{name}_{mode}_grad_feat"] = m.feat_param.grad.numpy()
            assert all(np.isfinite(v).all() for k, v in out.items() if k.startswith(f"{name}_{mode}"))
        cov = int((1 - np.abs((pts[:, None] - srt[None, :, 1:4]) / srt[None, :, :1]).max(-1) > 0).any(1).sum())
        print(name, len(pts), "points,", cov, "covered")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
