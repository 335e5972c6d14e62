"""Oracle restatement of the MVP ray-march preview (TEST INFRASTRUCTURE — see oracle/__init__.py).

PINNED to the reference's own pure-PyTorch ray-marcher, not to its CUDA extension: `dva/mvp/extensions/mvpraymarch` is an sm_70 torch
extension that needs a GPU and its own build, neither available where the fixtures are made.  The reference's gradcheck script carries
a plain PyTorch implementation of the same forward pass as the arm its CUDA kernel is checked against (mvpraymarch.py:391-475);
tests/golden/make_raymarch_golden.py EXECUTES that block from /root/reference on the CPU over a seeded scene and stores inputs + image
in tests/golden/raymarch_ref.npz.  tests/test_oracle_golden.py holds `raymarch_dense` (the restatement of that block) to the fixture
at 2.4e-7 and the kernel-shaped restatement `raymarch` at 1.3e-6, and additionally `raymarch` to `raymarch_dense` on a camera scene.
The CUDA-only parts (the per-warp hit list, its order and 512-entry cap, the start-at-first-hit stepping and compute_raydirs' slab
test) have no pure-PyTorch counterpart; they are pinned by running the reference's own CUDA extensions on the GPU against the kernel
(tests/test_gpu_raymarch_ref.py), and the list order by the reference's tree walk on the host (tests/test_raymarch_grad_host.py).

Restates (file:line under /root/reference):
  * convert_camera_parameters            dva/ray_marcher.py:24-33
  * RayMarcher.forward                   dva/ray_marcher.py:142-229   (pixel grid, pos / volradius, dt / volradius, "fixedorder" BVH, chlast)
  * compute_raydirs_forward_kernel       dva/mvp/extensions/utils/utils_kernel.cu:15-55
  * ray_subset_fixedbvh                  dva/mvp/extensions/mvpraymarch/utils.h:728-824   (per-warp hit list: a primitive is listed if ANY ray of the
                                          8x4-pixel warp hits its box; in the tree's leaf order, fixedorder_visit; at most maxhitboxes = 512; rtminmax from the
                                          ray's own hits)
  * raymarch_subset_forward_kernel       .../mvpraymarch_subset_kernel.h:14-101  (start at the first step before the first hit, fixed steps, stop
                                          after the last hit or at saturation)
  * PrimTransfSRT.forward / valid        .../primtransf.h:104-131      (y = (R^T-rows . (x - t)) * s, strictly inside (-1, 1)^3)
  * PrimSamplerTW<false>.forward         .../primsampler.h:44-66       (trilinear channels-last sample, alpha *= exp(-fadescale * sum |y|^fadeexp))
  * PrimAccumAdditive.forward_prim       .../primaccum.h:63-79         (additive alpha with saturation at 1)
"""
from __future__ import annotations

import torch


def convert_camera_parameters(Rt: torch.Tensor, K: torch.Tensor):
    R = Rt[:, :3, :3]
    t = -R.permute(0, 2, 1).bmm(Rt[:, :3, 3].unsqueeze(2)).squeeze(2)
    return dict(campos=t, camrot=R, focal=K[:, :2, :2], princpt=K[:, :2, 2])


def compute_raydirs(campos, camrot, focal, princpt, H: int, W: int, volradius: float):
    """campos [N,3], camrot [N,3,3], focal [N,2] (diagonal), princpt [N,2] -> raypos, raydir [N,H,W,3], tminmax [N,H,W,2]."""
    N = campos.shape[0]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    pix = torch.stack([xs, ys], -1)[None].expand(N, H, W, 2)
    pc = (pix - princpt[:, None, None, :]) / focal[:, None, None, :]
    d = torch.cat([pc, torch.ones(N, H, W, 1)], -1)
    raydir = camrot[:, None, None, 0, :] * d[..., 0:1] + camrot[:, None, None, 1, :] * d[..., 1:2] + camrot[:, None, None, 2, :] * d[..., 2:3]
    raydir = raydir / raydir.norm(dim=-1, keepdim=True)
    raypos = (campos / volradius)[:, None, None, :].expand(N, H, W, 3).contiguous()
    t1 = (-1.0 - raypos) / raydir
    t2 = (1.0 - raypos) / raydir
    tmin = torch.minimum(t1, t2).amax(-1)
    tmax = torch.maximum(t1, t2).amin(-1)
    return raypos, raydir, torch.stack([tmin.clamp(min=0.0), tmax], -1)


def _local(x, pos, rot, scale):
    """PrimTransfSRT.forward for one primitive: x [...,3] -> y0 [...,3]."""
    xmt = x - pos
    r = rot[0] * xmt[..., 0:1] + rot[1] * xmt[..., 1:2] + rot[2] * xmt[..., 2:3]
    return r * scale


def _sample_chlast(tpl, y):
    """tpl [D,H,W,4]; y [...,3] in (-1,1) -> [...,4]  (grid_sample_chlast_forward, utils.h:407-500, no border clipping)."""
    D, Hh, Ww = tpl.shape[:3]
    ix = (((y[..., 0] + 1) / 2).clamp(-100, 100)) * (Ww - 1)
    iy = (((y[..., 1] + 1) / 2).clamp(-100, 100)) * (Hh - 1)
    iz = (((y[..., 2] + 1) / 2).clamp(-100, 100)) * (D - 1)
    x0, y0, z0 = ix.floor().long(), iy.floor().long(), iz.floor().long()
    out = torch.zeros(*y.shape[:-1], 4, dtype=tpl.dtype)
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                xi, yi, zi = x0 + dx, y0 + dy, z0 + dz
                w = (1 - (ix - xi).abs()) * (1 - (iy - yi).abs()) * (1 - (iz - zi).abs())
                ok = (xi >= 0) & (xi < Ww) & (yi >= 0) & (yi < Hh) & (zi >= 0) & (zi < D)
                v = tpl[zi.clamp(0, D - 1), yi.clamp(0, Hh - 1), xi.clamp(0, Ww - 1)]
                out = out + torch.where(ok[..., None], v * w[..., None], torch.zeros_like(v))
    return out


def fixedorder_visit(K: int) -> list[int]:
    """The order in which ray_subset_fixedbvh lists primitives: its depth-first, left-first walk of build_accel(fixedorder=True)'s
    implicit heap (node i has children 2i+1, 2i+2; leaf node i is primitive i - (K - 1)) reaches the leaves of the deeper level first,
    so it is ascending order rotated by r = 2^ceil(log2 K) - K: [r, ..., K-1, 0, ..., r-1], ascending only when K is a power of two."""
    r = (1 << (K - 1).bit_length()) - K
    return [(j + r) % K for j in range(K)]


def slab_hits(raypos, raydir, primpos, primrot, primscale):
    """The exact per-ray test of ray_subset_fixedbvh: hit [K,H,W] (the ray's LINE meets primitive k's box; no t >= 0 condition) and
    the ray's rtminmax over its hits, rt_min / rt_max [H,W] (+inf / -inf without one)."""
    H, W = raypos.shape[:2]
    K = primpos.shape[0]
    rt_min = torch.full((H, W), float("inf"))
    rt_max = torch.full((H, W), -float("inf"))
    hit = torch.zeros(K, H, W, dtype=torch.bool)
    for k in range(K):
        r0 = _local(raypos, primpos[k], primrot[k], primscale[k])                       # forward2: origin with the translation ...
        rd = _local(raydir, torch.zeros(3), primrot[k], primscale[k])                  # ... direction without
        ird = 1.0 / rd
        t0, t1 = (-1.0 - r0) * ird, (1.0 - r0) * ird
        trmin = torch.minimum(t0, t1).amax(-1)
        trmax = torch.maximum(t0, t1).amin(-1)
        h = trmin <= trmax
        hit[k] = h
        rt_min = torch.where(h, torch.minimum(rt_min, trmin), rt_min)
        rt_max = torch.where(h, torch.maximum(rt_max, trmax), rt_max)
    return hit, rt_min, rt_max


def hit_lists(hit, block=(8, 16), maxhitboxes=512):
    """hit [K,H,W] bool (the exact slab test per primitive and ray) -> (warp_id [H,W], listed [warps, K] bool, order): a primitive is
    listed for a warp if ANY of its rays hits it and it is among the first maxhitboxes such primitives in `fixedorder_visit` order,
    which is also the order the march visits them in."""
    K, H, W = hit.shape
    bx, by = block
    # warp of pixel (h, w): thread id in the (bx, by) block = (h % by) * bx + (w % bx); 32 threads per warp
    hh, ww = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    wpb = (bx * by) // 32
    warp_id = ((hh // by) * ((W + bx - 1) // bx) + (ww // bx)) * wpb + ((hh % by) * bx + (ww % bx)) // 32
    nw = int(warp_id.max()) + 1
    cnt = torch.zeros(nw, K, dtype=torch.int32)
    cnt.index_put_((warp_id.reshape(-1).repeat(K), torch.arange(K).repeat_interleave(H * W)), hit.reshape(-1).int(), accumulate=True)
    order = fixedorder_visit(K)
    listed = (cnt > 0)[:, order]
    listed = listed & ~(listed.long().cumsum(1) > maxhitboxes)                      # the first maxhitboxes in visiting order survive
    out = torch.zeros_like(listed)
    out[:, order] = listed
    return warp_id, out, order


def raymarch(raypos, raydir, stepsize, tminmax, template, primpos, primrot, primscale, fadescale=8.0, fadeexp=8.0, block=(8, 16), maxhitboxes=512):
    """Kernel-shaped restatement for ONE batch element.  raypos/raydir [H,W,3], tminmax [H,W,2], template [K,D,H,W,4] channels-last,
    primpos [K,3] (already / volradius), primrot [K,3,3], primscale [K,3].  Returns rgba [H,W,4]."""
    H, W = raypos.shape[:2]
    K = primpos.shape[0]
    # ---- hit lists (ray_subset_fixedbvh, sync = true, sortboxes = false) ----
    hit, rt_min, rt_max = slab_hits(raypos, raydir, primpos, primrot, primscale)
    warp_id, listed, order = hit_lists(hit, block, maxhitboxes)
    rt_min = torch.maximum(rt_min, tminmax[..., 0])
    rt_max = torch.minimum(rt_max, tminmax[..., 1])
    # ---- march ----
    t = tminmax[..., 0].clone()
    pos = raypos + raydir * tminmax[..., 0:1]
    incs = torch.floor((rt_min - t) / stepsize)
    nohit = ~torch.isfinite(incs)
    incs = torch.where(nohit, torch.zeros_like(incs), incs)
    t = t + incs * stepsize
    pos = pos + raydir * incs[..., None] * stepsize
    rgba = torch.zeros(H, W, 4)
    sat = torch.zeros(H, W, dtype=torch.bool)
    alive = ~nohit
    active_k = [k for k in order if bool(listed[:, k].any())]
    while bool((alive & ~(t > rt_max + 1e-5) & ~sat).any()):
        for k in active_k:
            y0 = _local(pos, primpos[k], primrot[k], primscale[k])
            valid = ((y0 > -1.0) & (y0 < 1.0)).all(-1) & listed[warp_id, k] & ~sat & (t < rt_max + 1e-5) & alive
            if not bool(valid.any()):
                continue
            s = _sample_chlast(template[k], y0)
            fade = torch.exp(-fadescale * (y0.abs() ** fadeexp).sum(-1))
            alpha = s[..., 3] * fade
            newalpha = rgba[..., 3] + alpha * stepsize
            contrib = torch.where(valid, newalpha.clamp(max=1.0) - rgba[..., 3], torch.zeros_like(alpha))
            rgba = rgba + torch.cat([s[..., :3], torch.ones_like(alpha)[..., None]], -1) * contrib[..., None]
            sat = sat | (valid & (newalpha >= 1.0))
        t = t + stepsize
        pos = pos + raydir * stepsize
    return rgba


def saturating_overlap(raypos, raydir, stepsize, tminmax, template, primpos, primrot, primscale, fadescale=8.0, fadeexp=8.0):
    """[H,W] int: how many primitives a ray is inside of at the step where its accumulated alpha first reaches 1 (0 if it never does),
    on raymarch_dense's steps.  Where this is 2 or more, the primitive visited first takes the step's remaining alpha and supplies the
    ray's final colour, so the image depends on the visiting order; every other ray sums the same samples in any order."""
    H, W = raypos.shape[:2]
    K = primpos.shape[0]
    acc = torch.zeros(H, W)
    out = torch.zeros(H, W, dtype=torch.int64)
    pos0, t0 = raypos + raydir * tminmax[..., 0:1], tminmax[..., 0]
    step = 0
    t, pos = t0.clone(), pos0.clone()
    while bool((t < tminmax[..., 1]).any()):
        live = (t < tminmax[..., 1]) & (out == 0)
        n = torch.zeros(H, W, dtype=torch.int64)
        add = torch.zeros(H, W)
        for k in range(K):
            y0 = _local(pos, primpos[k], primrot[k], primscale[k])
            inside = ((y0 >= -1.0) & (y0 <= 1.0)).all(-1) & live
            s = _sample_chlast(template[k], y0.clamp(-1, 1))
            add = add + torch.where(inside, s[..., 3] * torch.exp(-fadescale * (y0.abs() ** fadeexp).sum(-1)) * stepsize, torch.zeros_like(add))
            n = n + inside.long()
        acc = acc + add
        out = torch.where(live & (acc >= 1.0), n, out)
        step += 1
        t = t0 + stepsize * step
        pos = pos0 + raydir * stepsize * step
    return out


def raymarch_dense(raypos, raydir, stepsize, tminmax, template, primpos, primrot, primscale, fadescale=8.0, fadeexp=8.0):
    """The reference's pure-PyTorch ray-marcher (mvpraymarch.py:391-475, accum == 0, no warp field), one batch element: every ray
    visits every primitive at every step from tminmax[0] to tminmax[1]; positions are t0 + stepsize * step."""
    H, W = raypos.shape[:2]
    K = primpos.shape[0]
    rgba = torch.zeros(H, W, 4)
    pos0 = raypos + raydir * tminmax[..., 0:1]
    t0 = tminmax[..., 0]
    step = 0
    t, pos = t0.clone(), pos0.clone()
    while bool((t < tminmax[..., 1]).any()):
        for k in range(K):
            y0 = _local(pos, primpos[k], primrot[k], primscale[k])
            fade = torch.exp(-fadescale * (y0.abs() ** fadeexp).sum(-1))
            valid1 = ((y0 >= -1.0) & (y0 <= 1.0)).all(-1)
            valid = (t >= tminmax[..., 0]) & (t < tminmax[..., 1])
            v = (valid & valid1).float()
            if not bool((valid & valid1).any()):
                continue
            s = _sample_chlast(template[k], y0.clamp(-1, 1))
            alpha = s[..., 3] * fade * stepsize * v
            newalpha = rgba[..., 3] + alpha
            contrib = (newalpha.clamp(max=1.0) - rgba[..., 3]) * v
            rgba = rgba + contrib[..., None] * torch.cat([s[..., :3] * v[..., None], torch.ones_like(alpha)[..., None]], -1)
        step += 1
        t = t0 + stepsize * step
        pos = pos0 + raydir * stepsize * step
    return rgba


def ray_marcher_forward(prim_rgba, prim_pos, prim_rot, prim_scale, K, RT, image_height, image_width, volradius, dt=1.0, fadescale=8.0, fadeexp=8.0):
    """RayMarcher.forward (dva/ray_marcher.py:142-229, eval, ray_subsample_factor = 1): prim_rgba [B,K,4,S,S,S] -> rgba_image [B,4,H,W]."""
    cam = convert_camera_parameters(RT, K)
    focal = torch.diagonal(cam["focal"], dim1=1, dim2=2)
    raypos, raydir, tminmax = compute_raydirs(cam["campos"], cam["camrot"], focal, cam["princpt"], image_height, image_width, volradius)
    tpl = prim_rgba.permute(0, 1, 3, 4, 5, 2).contiguous()
    out = [raymarch(raypos[b], raydir[b], dt / volradius, tminmax[b], tpl[b], prim_pos[b] / volradius, prim_rot[b], prim_scale[b], fadescale, fadeexp)
           for b in range(prim_rgba.shape[0])]
    return torch.stack(out, 0).permute(0, 3, 1, 2)
