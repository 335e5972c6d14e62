#!/usr/bin/env python
"""Golden box-projection unwrap and noise filter (DESIGN.md §1 f-8), produced by RUNNING THE REFERENCE'S OWN CODE.

Run in the build container only (needs /root/reference with jaxtyping importable):

    python tests/golden/make_unwrap_golden.py

Imports the reference's utils/uv_unwrap.py at run time and calls its stage functions one by one (compute_vertex_normal,
_box_assign_vertex_to_cube_face, _rotate_uv_slices_consistent_space, _assign_faces_uv_to_atlas_index, _find_slice_offset_and_scale,
_distribute_individual_uvs_in_atlas, _get_unique_face_uv) and box_projection_uv_unwrap as a whole, on the CPU in fp32, on:
  * ``torus``: a torus around the x axis (its inner wall sends faces to the overlap slices 6-11);
  * ``spheres``: three spheres on the x axis (faces hidden twice reach slot 12);
  * ``shell``: the indexed mesh of the texture-bake fixture (tests/golden/texture_bake.npz, per-corner vertices merged back).
The noise filter is the statement block of inference.py:92-99, read from the reference file at run time and executed on two seeded
srt arrays: 2048 primitives with isolated outliers, and 64 spread ones where some have nothing nearer than 1 and match themselves.
Nothing of the reference is stored.  The script asserts that no decision lies within the oracle's ambiguity margins (oracle/unwrap.py),
so the fixture comparisons can require equal decisions.
"""
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "unwrap.npz")
PAD = 0.02
PROJECT_TOL = 1e-6


def sdf_mesh(fn, R):
    from oracle import mesh as omesh
    lin = np.linspace(-1, 1, R)
    X, Y, Z = np.meshgrid(lin, lin, lin, indexing="ij")
    v, f = omesh.marching_cubes(fn(X, Y, Z).astype(np.float32), 0.0)
    return (v / (R - 1.0) * 2 - 1).astype(np.float32), f.astype(np.int64)


def meshes():
    """Off-centre shapes with a small ripple: a lattice-symmetric surface gives exact ties of |d - 3 r| that no fp32 restatement can
    promise to resolve like torch's norm."""
    def ripple(x, y, z):
        return 0.013 * np.sin(5.1 * x + 0.3) * np.cos(4.3 * y - 0.7) * np.sin(3.7 * z + 1.1)
    torus = sdf_mesh(lambda x, y, z: np.sqrt((np.sqrt((y + 0.021) ** 2 + (z - 0.017) ** 2) - 0.55) ** 2 + (x - 0.013) ** 2) - 0.22 + ripple(x, y, z), 44)
    spheres = sdf_mesh(lambda x, y, z: np.minimum.reduce([np.sqrt((x - c) ** 2 + (y - 0.011) ** 2 + (z + 0.019) ** 2) - 0.26 for c in (-0.617, 0.003, 0.623)])
                       + ripple(x, y, z), 48)
    b = np.load(os.path.join(ROOT, "tests", "golden", "texture_bake.npz"))
    uv, inv = np.unique(b["v"], axis=0, return_inverse=True)
    shell = (uv.astype(np.float32), inv.reshape(-1)[b["f"].astype(np.int64)].reshape(-1, 3))
    return {"torus": torus, "spheres": spheres, "shell": shell}


def srts():
    rs = np.random.RandomState(7)
    K = 2048
    d = rs.standard_normal((K, 3))
    pos = d / np.linalg.norm(d, axis=1, keepdims=True) * 0.5 + 0.01 * rs.standard_normal((K, 3))
    out = rs.choice(K, 24, replace=False)
    pos[out] *= rs.uniform(1.3, 1.9, (24, 1))
    big = np.concatenate([rs.uniform(0.02, 0.05, (K, 1)), pos], 1).astype(np.float32)
    spread = np.concatenate([rs.uniform(0.3, 0.7, (64, 1)), rs.uniform(-3, 3, (64, 3))], 1).astype(np.float32)
    return {"dense": big, "spread": spread}


def reference_noise_filter(srt):
    src = open(os.path.join(REF, "inference.py")).read().split("\n")
    start = next(i for i, l in enumerate(src) if l.strip().startswith("prim_position = raw_srt_param"))
    end = next(i for i in range(start, len(src)) if src[i].strip().startswith("prim_mask = "))
    ns = dict(torch=torch, raw_srt_param=torch.from_numpy(srt))
    exec(compile(textwrap.dedent("\n".join(src[start:end + 1])), "inference.py:<noise filter>", "exec"), ns)
    return ns["prim_mask"].numpy(), ns["min_indices"].numpy()


def main():
    sys.modules.setdefault("trimesh", types.ModuleType("trimesh"))
    sys.path.insert(0, REF)
    import utils.uv_unwrap as U  # noqa: E402
    from oracle import unwrap as ou  # noqa: E402

    data = {}
    for name, (v, f) in meshes().items():
        vt, ftt = torch.from_numpy(v), torch.from_numpy(f)
        n = U.compute_vertex_normal(vt, ftt)
        bbox = torch.stack([vt.min(0).values, vt.max(0).values])
        fuv, fidx = U._box_assign_vertex_to_cube_face(vt, n, ftt, bbox)
        proj = fuv.clone()
        ruv = U._rotate_uv_slices_consistent_space(vt, n, ftt, fuv.clone(), fidx)
        asg = U._assign_faces_uv_to_atlas_index(vt, ftt, ruv, fidx)
        ox, oy, dx, dy = U._find_slice_offset_and_scale(asg)
        placed = U._distribute_individual_uvs_in_atlas(ruv.clone(), asg, ox, oy, dx, dy, PAD)
        uv, vidx = U._get_unique_face_uv(placed)
        uv_all, vidx_all = U.box_projection_uv_unwrap(vt, n, ftt, PAD)
        assert torch.equal(uv, uv_all) and torch.equal(vidx, vidx_all), name
        # no decision within the oracle's margins, staged on the reference's own previous stage
        _, _, pm = ou.project(v, n.numpy(), f)
        oa, am = ou.assign(v, f, ruv.numpy(), fidx.numpy())
        assert np.array_equal(oa, asg.numpy()), name
        assert pm.min() > PROJECT_TOL and not ou.ambiguous(am).any(), (name, pm.min(), {k: x[x > 0].min() for k, x in am.items()})
        counts = np.bincount(asg.numpy(), minlength=13)
        print(f"{name}: V {len(v)} F {len(f)} U {len(uv)} slots {counts.tolist()} margins {pm.min():.3g} {[f"{k} {x[x > 0].min():.3g}" for k, x in am.items()]}")
        data.update({f"{name}_v": v, f"{name}_f": f.astype(np.int32), f"{name}_normals": n.numpy(), f"{name}_slice": fidx.numpy().astype(np.int8),
                     f"{name}_face_uv": proj.numpy(), f"{name}_rot_uv": ruv.numpy(), f"{name}_assign": asg.numpy().astype(np.int8),
                     f"{name}_placed": placed.numpy().reshape(-1, 3, 2), f"{name}_uv": uv.numpy(), f"{name}_vidx": vidx.numpy().astype(np.int32)})
    for name, srt in srts().items():
        keep, nn = reference_noise_filter(srt)
        print(f"noise {name}: K {len(srt)} kept {int(keep.sum())} self-matches {int((nn == np.arange(len(srt))).sum())}")
        data.update({f"noise_{name}_srt": srt, f"noise_{name}_keep": keep, f"noise_{name}_nn": nn.astype(np.int32)})
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
