"""Oracle of the MVP ray-march GRADIENTS and of subsampled rays (TEST INFRASTRUCTURE — see oracle/__init__.py).

Autograd through a kernel-shaped restatement of the forward march (oracle/raymarch.py's `raymarch`, with the same per-warp hit lists,
start step and saturation), which is what the reference's CUDA backward differentiates: MVPRaymarch.backward (mvpraymarch.py:152-213)
-> raymarch_subset_backward_kernel with forwarddir = true (mvpraymarch_subset_kernel.h:103-217, primaccum.h:81-98,
primsampler.h:68-91, primtransf.h:155-179).  tests/test_raymarch_grad_host.py holds it, through oracle.raymarch.raymarch_dense, to
tests/golden/raymarch_grad.npz: the gradients of the reference's own pure-PyTorch marcher under autograd (mvpraymarch.py:391-467),
produced by tests/golden/make_raymarch_grad_golden.py.

Restates (file:line under /root/reference):
  * compute_raydirs_forward_kernel with pixelcoords   dva/mvp/extensions/utils/utils_kernel.cu:15-55
  * subsample_pixel_coords / resize_pixel_coords     dva/ray_marcher.py:33-73 (their pixel grids are the `pixelcoords` argument)
  * MVPRaymarch forward + backward                    dva/mvp/extensions/mvpraymarch/mvpraymarch.py:74-213
"""
from __future__ import annotations

import torch

from .raymarch import _local, _sample_chlast, compute_raydirs, convert_camera_parameters, hit_lists, slab_hits


def compute_raydirs_at(campos, camrot, focal, princpt, pixelcoords, volradius: float):
    """compute_raydirs_forward_kernel with the pixelcoords argument (utils_kernel.cu:31): pixelcoords [N,h,w,2] (x, y) -> raypos,
    raydir [N,h,w,3], tminmax [N,h,w,2].  The same arithmetic as oracle.raymarch.compute_raydirs, which is this on the full pixel grid."""
    N, h, w = pixelcoords.shape[:3]
    pc = (pixelcoords - princpt[:, None, None, :]) / focal[:, None, None, :]
    d = torch.cat([pc, torch.ones(N, h, w, 1)], -1)
    raydir = camrot[:, None, None, 0, :] * d[..., 0:1] + camrot[:, None, None, 1, :] * d[..., 1:2] + camrot[:, None, None, 2, :] * d[..., 2:3]
    raydir = raydir / raydir.norm(dim=-1, keepdim=True)
    raypos = (campos / volradius)[:, None, None, :].expand(N, h, w, 3).contiguous()
    t1 = (-1.0 - raypos) / raydir
    t2 = (1.0 - raypos) / raydir
    tmin = torch.minimum(t1, t2).amax(-1)
    tmax = torch.maximum(t1, t2).amin(-1)
    return raypos, raydir, torch.stack([tmin.clamp(min=0.0), tmax], -1)


def raymarch_grad(raypos, raydir, stepsize, tminmax, template, primpos, primrot, primscale, fadescale=8.0, fadeexp=8.0, block=(8, 16), maxhitboxes=512):
    """oracle.raymarch.raymarch for autograd: the same per-warp hit lists, start step and saturation, with the discrete part (hit
    lists, rtminmax, the floor-based start step) evaluated without autograd.  Those carry no gradient in the kernel either, and the slab
    test divides by the ray direction in the primitive's frame, whose backward is 0 * inf = nan on a ray parallel to a box face."""
    H, W = raypos.shape[:2]
    K = primpos.shape[0]
    with torch.no_grad():
        hit, rt_min, rt_max = slab_hits(raypos, raydir, primpos, primrot, primscale)
        warp_id, listed, order = hit_lists(hit, block, maxhitboxes)
        rt_min = torch.maximum(rt_min, tminmax[..., 0])
        rt_max = torch.minimum(rt_max, tminmax[..., 1])
        t = tminmax[..., 0].clone()
        incs = torch.floor((rt_min - t) / stepsize)
        nohit = ~torch.isfinite(incs)
        incs = torch.where(nohit, torch.zeros_like(incs), incs)
        pos = raypos + raydir * tminmax[..., 0:1]
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


def ray_marcher_backward(prim_rgba, prim_pos, prim_rot, prim_scale, K, RT, image_height, image_width, volradius, grad_rgba, dt=1.0, fadescale=8.0, fadeexp=8.0,
                         pixelcoords=None):
    """RayMarcher.forward + backward (dva/ray_marcher.py:142-229, mvpraymarch.py:74-213) by autograd through `raymarch_grad`:
    prim_rgba [B,K,4,S,S,S], prim_pos [B,K,3] (world units), prim_rot, prim_scale; grad_rgba [B,4,h,w] the upstream gradient of
    rgba_image; pixelcoords [B,h,w,2] (the subsampled grid) or None for every pixel.  Returns (rgba_image [B,4,h,w], grads) with grads
    the gradients of <rgba_image, grad_rgba> w.r.t. (prim_rgba, prim_pos, prim_rot, prim_scale) in the callers' layout and units.  The
    camera gets none."""
    leaves = [t.detach().clone().requires_grad_(True) for t in (prim_rgba, prim_pos, prim_rot, prim_scale)]
    rgba, pos, rot, scale = leaves
    cam = convert_camera_parameters(RT, K)
    focal = torch.diagonal(cam["focal"], dim1=1, dim2=2)
    if pixelcoords is None:
        raypos, raydir, tminmax = compute_raydirs(cam["campos"], cam["camrot"], focal, cam["princpt"], image_height, image_width, volradius)
    else:
        raypos, raydir, tminmax = compute_raydirs_at(cam["campos"], cam["camrot"], focal, cam["princpt"], pixelcoords, volradius)
    tpl = rgba.permute(0, 1, 3, 4, 5, 2).contiguous()
    p = pos / volradius
    out = torch.stack([raymarch_grad(raypos[b], raydir[b], dt / volradius, tminmax[b], tpl[b], p[b], rot[b], scale[b], fadescale, fadeexp)
                       for b in range(prim_rgba.shape[0])], 0).permute(0, 3, 1, 2)
    out.backward(grad_rgba)
    return out.detach(), [t.grad for t in leaves]
