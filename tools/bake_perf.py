#!/usr/bin/env python
"""Time the texture bake on the synthetic object of tools/primsdf_perf.py (2048 primitives on a noisy sphere shell): the mesh of
PrimSDF.extract_mesh(256) in the per-corner layout of extract_texmesh's fast-unwrap branch, a seeded one-cell-per-triangle atlas
(synth.cell_atlas), atlases of 1024^2 and 2048^2, for the whole mesh and for every n-th triangle of it down to 100 000:
  * each of the four kernels (UV rasteriser, attribute interpolation, fused texel query, seam padding) and PrimSDF.bake_texture end to
    end, device time from CUDA events (3 warm-ups, 20 repetitions);
  * the path inference.py:172-211 takes through this package without the fused kernels: rasterise + two interpolations on the GPU,
    PrimSDF.forward over the masked texels in 8192-point chunks with the mask gather / scatter, the device -> host copy of feats and
    mask, and — if scipy and scikit-learn import — the reference's binary_dilation / binary_erosion / kd-tree padding on the host
    (host clock around a synchronise); otherwise that leg prints "not measured".
Needs a GPU.  Prints the card name and power limit, triangles, texels covered and bytes moved."""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tpxl_b200  # noqa: E402
from tpxl_b200 import _lib, bake, synth  # noqa: E402

WARMUP, REPS = 3, 20


def shell_module(K=2048, S=8):
    g = torch.Generator().manual_seed(0)
    d = torch.randn(K, 3, generator=g)
    pos = d / d.norm(dim=1, keepdim=True) * (0.55 + 0.1 * torch.rand(K, 1, generator=g))
    srt = torch.cat([0.03 + 0.05 * torch.rand(K, 1, generator=g), pos], 1)
    m = tpxl_b200.PrimSDF(num_prims=K, dim_feat=6, prim_shape=S).eval()
    m.srt_param.data = srt
    m.feat_param.data = torch.randn(K, 6 * S ** 3, generator=g)
    return m.cuda()


def device_ms(fn, reps=REPS, warmup=WARMUP):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def wall_ms(fn, reps, warmup=1):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps, out


def host_padding(feats, mask, pad=32):
    """inference.py:200-211 as written there (numpy in, numpy out)."""
    from scipy.ndimage import binary_dilation, binary_erosion
    from sklearn.neighbors import NearestNeighbors
    import numpy as np
    inpaint_region = binary_dilation(mask, iterations=pad)
    inpaint_region[mask] = 0
    search_region = mask.copy()
    not_search_region = binary_erosion(search_region, iterations=3)
    search_region[not_search_region] = 0
    search_coords = np.stack(np.nonzero(search_region), axis=-1)
    inpaint_coords = np.stack(np.nonzero(inpaint_region), axis=-1)
    knn = NearestNeighbors(n_neighbors=1, algorithm="kd_tree").fit(search_coords)
    _, indices = knn.kneighbors(inpaint_coords)
    feats[tuple(inpaint_coords.T)] = feats[tuple(search_coords[indices[:, 0]].T)]
    return feats


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bake_perf needs a GPU: there is nothing to time without one")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name()} | nvidia-smi: {q}")
    m = shell_module()
    lib = _lib.lib()
    verts, all_faces = m.extract_mesh(256)
    srt, feat = m.srt_param.data.contiguous(), m.feat_param.data.contiguous()
    ws = m._grid_workspace(srt, srt.shape[0], srt.device)
    # the whole mesh (random voxels make it very dense: sub-texel triangles), and every n-th triangle of it down to the 100 000 faces
    # extract_texmesh decimates to before it unwraps
    cases = [(all_faces, R) for R in (1024, 2048)] + [(all_faces[::max(all_faces.shape[0] // 100_000, 1)][:100_000], R) for R in (1024, 2048)]
    for faces, R in cases:
        F = faces.shape[0]
        v = verts[faces].reshape(-1, 3).contiguous()
        f = torch.arange(3 * F, dtype=torch.int32, device="cuda").reshape(-1, 3)
        vt, ft = [t.cuda() for t in synth.cell_atlas(F, 5)]
        ones = torch.ones_like(v[:, :1])
        t_rast, (rast, _) = device_ms(lambda: bake._rasterize(vt, ft, R, R))
        t_interp, xyz = device_ms(lambda: bake.interpolate(v, rast, f))
        feats = torch.empty(R, R, 6, device="cuda")
        mask = torch.empty(R, R, dtype=torch.uint8, device="cuda")
        t_query, _ = device_ms(lambda: _lib.check(lib.tpx_primsdf_bake(rast.data_ptr(), R, R, v.data_ptr(), v.shape[0], f.data_ptr(), F, srt.data_ptr(), feat.data_ptr(),
                                                                        ws.data_ptr(), ws.numel(), srt.shape[0], 8, 6, feats.data_ptr(), mask.data_ptr(), _lib.stream_ptr())))
        pre = feats.clone()
        t_pad, _ = device_ms(lambda: bake.inpaint(feats.copy_(pre), mask, 32))
        t_copy, _ = device_ms(lambda: feats.copy_(pre))
        t_bake, (out, omask) = device_ms(lambda: m.bake_texture(v, f, vt, ft, resolution=R))
        covered = int(mask.sum())
        moved = R * R * (16 + 4) + R * R * (6 * 4 + 1) + R * R * 2 * 2          # rast + winner written, feats + mask written, row scratch written and read
        print(f"atlas {R}^2  F={F}  covered texels={covered} ({covered / R / R:.1%})  padded texels={int(((out != pre).any(-1)).sum())}")
        print(f"  kernels (device ms): rasterise {t_rast:.3f} | interpolate [Nv,3] {t_interp:.3f} | fused texel query {t_query:.3f} | "
              f"seam padding {t_pad - t_copy:.3f} (pad 32) | bake_texture end to end {t_bake:.3f}  (~{moved / 1e6:.0f} MB of atlas buffers written)")

        def chunked():
            r = bake.rasterize_uv(vt, ft, R, R)
            xyzs = bake.interpolate(v, r, f).view(-1, 3)
            mk = (bake.interpolate(ones, r, f) > 0).view(-1)
            ft6 = torch.zeros(R * R, 6, device="cuda")
            parts = []
            with torch.no_grad():
                for c in torch.split(xyzs[mk], 8192):
                    p = m(c)
                    parts.append(torch.cat([p["tex"], torch.zeros_like(p["tex"][:, :1]), p["mat"]], -1))
            ft6[mk] = torch.cat(parts, 0)
            return ft6.view(R, R, 6), mk.view(R, R)

        t_chunk, (cf, cm) = wall_ms(chunked, 3)
        t_d2h, (hf, hm) = wall_ms(lambda: ((cf * 255).cpu().numpy(), cm.cpu().numpy()), 3)
        same = bool(torch.equal(cf * 255, pre))
        line = (f"  replaced path (wall ms): rasterise + interpolate + chunked forward ({-(-covered // 8192)} chunks) + gather / scatter {t_chunk:.2f} "
                f"(texels identical: {same}) | feats + mask to the host ({(hf.nbytes + hm.nbytes) / 1e6:.0f} MB) {t_d2h:.2f} | ")
        try:
            t0 = time.perf_counter()
            host_padding(hf, hm)
            line += f"scipy dilation / erosion + scikit-learn kd-tree on the host {(time.perf_counter() - t0) * 1e3:.0f} (one run)"
        except ImportError as e:
            line += f"host padding not measured ({e.name} does not import here)"
        print(line)
        del rast, xyz, feats, mask, pre, out, omask, cf, cm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
