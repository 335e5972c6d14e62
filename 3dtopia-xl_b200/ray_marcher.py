"""Host-side mirror of the reference's preview renderer ``dva.ray_marcher.RayMarcher`` (SURVEY.md §8f-1), backed by libtpx_b200.

Same constructor kwargs (``RayMarcher(config.image_height, config.image_width, **config.rm)``, inference.py:282-286) and the same
``forward(prim_rgba, prim_pos, prim_rot, prim_scale, K, RT) -> {"rgba_image": [B,4,H,W], "pixel_coords": ...}``, so
``dva.visualize.visualize_primvolume`` / ``visualize_video_primvolume`` run unchanged on top of it.  The reference's forward is
``compute_raydirs`` + ``mvpraymarch`` from an sm_70 torch extension that has to be compiled and imported at module import time; here
one sm_90a kernel (csrc/raymarch.cu) does both, so the extension is not needed at all.

Gradients: when autograd is on and any of ``prim_rgba`` / ``prim_pos`` / ``prim_rot`` / ``prim_scale`` requires grad, the march runs as
a ``torch.autograd.Function`` (the reference's ``MVPRaymarch``, mvpraymarch.py:74-213) over ``tpx_raymarch_forward`` /
``tpx_raymarch_backward``; the volradius division, the channels-last permute and the fp32 cast stay in torch around it, so the gradients
arrive in the caller's layout, units and dtype.  The camera gets no gradient, as in the reference.  Otherwise the no-grad preview runs.
``ray_subsample_factor > 1`` marches every f-th pixel from a per-image offset: drawn as ``subsample_pixel_coords`` draws it in training,
``f // 2`` in eval (dva/ray_marcher.py:33-73, 174-190).

``generate_colored_boxes`` (dva/ray_marcher.py:232-279, what ``dva.visualize`` imports beside ``RayMarcher``) builds the box template
in one launch (tpx_colored_boxes); ``march_views`` marches many cameras of one primitive set in one launch for ``tpxl_b200.visualize``.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import _lib


def convert_camera_parameters(Rt: torch.Tensor, K: torch.Tensor):
    """dva/ray_marcher.py:24-33."""
    R = Rt[:, :3, :3]
    t = -R.permute(0, 2, 1).bmm(Rt[:, :3, 3].unsqueeze(2)).squeeze(2)
    return dict(campos=t, camrot=R, focal=K[:, :2, :2], princpt=K[:, :2, 2])


def march_camera(RT: torch.Tensor, K: torch.Tensor, dev) -> tuple:
    """(campos, camrot, focal, princpt) as the march reads them, computed on `dev` from extrinsics [B,3,4] and intrinsics [B,3,3] by
    the reference's torch statements (convert_camera_parameters, then the focal diagonal), fp32 and contiguous."""
    with torch.no_grad():
        cam = convert_camera_parameters(RT.to(dev).float(), K.to(dev).float())
        f32 = lambda t: t.to(dev).float().contiguous()  # noqa: E731
        return f32(cam["campos"]), f32(cam["camrot"]), f32(torch.diagonal(cam["focal"], dim1=1, dim2=2)), f32(cam["princpt"])


def march_views(tpl: torch.Tensor, pos: torch.Tensor, rot: torch.Tensor, scale: torch.Tensor, cam, views: int, H: int, W: int, volradius: float,
                stepsize: float, fadescale: float, fadeexp: float) -> torch.Tensor:
    """No-grad preview march of `views` cameras per primitive set in one launch (tpx_raymarch_preview_views): tpl [N,K,S,S,S,4] fp32
    channels-last, pos [N,K,3] (/ volradius), rot [N,K,3,3], scale [N,K,3], ``cam`` = march_camera's four tensors for N * views
    cameras, set-major (camera n belongs to set n // views) -> rgba [N * views, H, W, 4].  Each image is tpx_raymarch_preview's."""
    N, K, S = tpl.shape[0], tpl.shape[1], tpl.shape[2]
    out = torch.empty(N * views, H, W, 4, dtype=torch.float32, device=tpl.device)
    with torch.cuda.device(tpl.device):
        _lib.check(_lib.lib().tpx_raymarch_preview_views(tpl.data_ptr(), pos.data_ptr(), rot.data_ptr(), scale.data_ptr(), *[c.data_ptr() for c in cam],
                                                         N * views, views, K, S, H, W, float(volradius), float(stepsize), float(fadescale), float(fadeexp),
                                                         out.data_ptr(), _lib.stream_ptr()), "tpx_raymarch_preview_views")
    return out


def box_colors(K: int, seed: int = 123456) -> torch.Tensor:
    """The per-primitive colours of generate_colored_boxes: ``np.random.seed(seed)`` then ``np.random.rand(K, 3) * 255.0`` rounded to
    fp32 [K,3] on the host.  The draws are the 3 K scalar ``np.random.rand()`` calls of the reference's loop, in its order, and numpy's
    global generator is left where the reference leaves it."""
    np.random.seed(seed)
    return torch.from_numpy((np.random.rand(K, 3) * 255.0).astype(np.float32))


def colored_boxes(N: int, K: int, S: int, colors: torch.Tensor, alpha: float, chlast: bool, device) -> torch.Tensor:
    """tpx_colored_boxes: the lit box template for N copies of K primitives of S^3 with `colors` [K,3] fp32 -> [N,K,S,S,S,4] when
    `chlast` (the march's layout), else [N,K,4,S,S,S] (the reference's)."""
    shape = (N, K, S, S, S, 4) if chlast else (N, K, 4, S, S, S)
    out = torch.empty(shape, dtype=torch.float32, device=device)
    colors = colors.to(device=device, dtype=torch.float32).contiguous()
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().tpx_colored_boxes(colors.data_ptr(), N, K, S, float(alpha), _lib.LAYOUT_CHLAST if chlast else _lib.LAYOUT_NCDHW,
                                                out.data_ptr(), _lib.stream_ptr()), "tpx_colored_boxes")
    return out


def generate_colored_boxes(template: torch.Tensor, prim_rot: torch.Tensor, alpha: float = 10000.0, seed: int = 123456) -> torch.Tensor:
    """dva/ray_marcher.py:232-279 in one launch: a [N,K,4,S,S,S] template of the shape (not the values) of `template`, every primitive a
    box of one random colour shaded by a fixed light, alpha `alpha`.  Reseeds numpy's global generator with `seed` and draws the
    colours as the reference does (box_colors).  `prim_rot` is unused, as in the reference."""
    if template.dim() != 6 or template.shape[2] != 4 or not (template.shape[3] == template.shape[4] == template.shape[5]):
        raise ValueError(f"template must be [N, K, 4, S, S, S], got {tuple(template.shape)}")
    if template.dtype != torch.float32:
        raise ValueError(f"template must be fp32 (the box template is computed in fp32), got {template.dtype}")
    if not template.is_cuda:
        raise _lib.TpxError("generate_colored_boxes runs on CUDA only (no CPU path)")
    N, K, S = template.shape[0], template.shape[1], template.shape[-1]
    return colored_boxes(N, K, S, box_colors(K, seed), alpha, False, template.device)


def subsample_offsets(batch_size: int, ray_subsample_factor: int, training: bool) -> list[tuple[int, int]]:
    """Per-image (x0, y0) of subsample_pixel_coords (training: two ``torch.randint(0, f - 1, size=())`` draws per image, x0 first, on the
    default host generator, so x0, y0 are in [0, f - 2]) or resize_pixel_coords (eval: f // 2), dva/ray_marcher.py:33-73."""
    f = ray_subsample_factor
    if not training:
        return [(f // 2, f // 2)] * batch_size
    out = []
    for _ in range(batch_size):
        x0 = int(torch.randint(0, f - 1, size=()))
        y0 = int(torch.randint(0, f - 1, size=()))
        out.append((x0, y0))
    return out


def offset_pixel_coords(base_pixel_coords: torch.Tensor, offsets, ray_subsample_factor: int) -> torch.Tensor:
    """The reference's slice of the pixel grid for each offset: [B, H // f, W // f, 2]."""
    f = ray_subsample_factor
    H, W = base_pixel_coords.shape[:2]
    SH, SW = H // f, W // f
    return torch.stack([base_pixel_coords[y0:y0 + f * SH:f, x0:x0 + f * SW:f, :] for x0, y0 in offsets], 0)


class _RayMarchFunction(torch.autograd.Function):
    """MVPRaymarch (mvpraymarch.py:74-213) over the C entries: tpl [N,K,S,S,S,4] fp32 channels-last, pos [N,K,3] (/ volradius), rot
    [N,K,3,3], scale [N,K,3] -> rgba [N,h,w,4].  ``cam`` = (campos, camrot, focal, princpt), ``geom`` = (H, W, volradius, stepsize,
    fadescale, fadeexp, stride), ``offsets`` device int32 [N,2] or None."""

    @staticmethod
    def forward(ctx, tpl, pos, rot, scale, cam, geom, offsets):
        N, K, S = tpl.shape[0], tpl.shape[1], tpl.shape[2]
        H, W, volradius, stepsize, fadescale, fadeexp, stride = geom
        rgba = torch.empty(N, H // stride, W // stride, 4, dtype=torch.float32, device=tpl.device)
        save = any(ctx.needs_input_grad[:4])         # raysat is only needed by the backward
        raysat = torch.empty(N, H // stride, W // stride, 3, dtype=torch.float32, device=tpl.device) if save else None
        with torch.cuda.device(tpl.device):
            _lib.check(_lib.lib().tpx_raymarch_forward(tpl.data_ptr(), pos.data_ptr(), rot.data_ptr(), scale.data_ptr(), *[c.data_ptr() for c in cam], N, K, S, H, W,
                                                       volradius, stepsize, fadescale, fadeexp, stride, _lib.ptr(offsets), rgba.data_ptr(), _lib.ptr(raysat),
                                                       _lib.stream_ptr()), "tpx_raymarch_forward")
        if save:
            ctx.save_for_backward(tpl, pos, rot, scale, raysat, *cam, *([] if offsets is None else [offsets]))
        ctx.geom = geom
        return rgba

    @staticmethod
    def backward(ctx, grad_rgba):
        tpl, pos, rot, scale, raysat, *rest = ctx.saved_tensors
        cam, offsets = rest[:4], (rest[4] if len(rest) > 4 else None)
        H, W, volradius, stepsize, fadescale, fadeexp, stride = ctx.geom
        N, K, S = tpl.shape[0], tpl.shape[1], tpl.shape[2]
        grad_rgba = grad_rgba.float().contiguous()
        g_tpl, g_pos, g_rot, g_scale = (torch.zeros_like(t) for t in (tpl, pos, rot, scale))
        with torch.cuda.device(tpl.device):
            _lib.check(_lib.lib().tpx_raymarch_backward(tpl.data_ptr(), pos.data_ptr(), rot.data_ptr(), scale.data_ptr(), *[c.data_ptr() for c in cam], N, K, S, H, W,
                                                        volradius, stepsize, fadescale, fadeexp, stride, _lib.ptr(offsets), raysat.data_ptr(),
                                                        grad_rgba.data_ptr(), g_tpl.data_ptr(), g_pos.data_ptr(), g_rot.data_ptr(), g_scale.data_ptr(),
                                                        _lib.stream_ptr()), "tpx_raymarch_backward")
        return g_tpl, g_pos, g_rot, g_scale, None, None, None


class RayMarcher(nn.Module):
    def __init__(self, image_height, image_width, volradius, fadescale=8.0, fadeexp=8.0, dt=1.0, ray_subsample_factor=1, accum=2, termthresh=0.99,
                 blocksize=None, with_t_img=True, chlast=False, assets=None):
        super().__init__()
        self.image_height, self.image_width = image_height, image_width
        self.volradius, self.dt = volradius, dt
        self.fadescale, self.fadeexp = fadescale, fadeexp
        self.blocksize = (8, 16) if blocksize is None else blocksize
        self.with_t_img, self.chlast, self.accum, self.termthresh = with_t_img, chlast, accum, termthresh
        self.ray_subsample_factor = ray_subsample_factor
        self.register_buffer("base_pixel_coords", self._pix(image_height, image_width), persistent=False)

    @staticmethod
    def _pix(h, w, device=None):
        ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32, device=device), torch.arange(w, dtype=torch.float32, device=device), indexing="ij")
        return torch.stack([xs, ys], dim=-1)

    def resize(self, h: int, w: int):
        self.image_height, self.image_width = h, w
        self.base_pixel_coords = self._pix(h, w, self.base_pixel_coords.device)

    def forward(self, prim_rgba, prim_pos, prim_rot, prim_scale, K, RT, ray_subsample_factor=None):
        f = self.ray_subsample_factor if ray_subsample_factor is None else ray_subsample_factor
        if tuple(self.blocksize) != (8, 16):
            raise NotImplementedError("blocksize (8, 16) only: the per-warp hit list of 8 x 4 pixels is part of the reference's result")
        if not prim_rgba.is_cuda:
            raise _lib.TpxError("RayMarcher runs on CUDA only (no CPU path)")
        B, Kp, C, S = prim_rgba.shape[0], prim_rgba.shape[1], prim_rgba.shape[2], prim_rgba.shape[-1]
        if C != 4 or prim_rgba.shape[3] != S or prim_rgba.shape[4] != S:
            raise ValueError(f"prim_rgba must be [B, K, 4, S, S, S], got {tuple(prim_rgba.shape)}")
        H, W = self.image_height, self.image_width
        if f < 1 or H // f < 1 or W // f < 1:
            raise ValueError(f"ray_subsample_factor {f} does not fit a {H} x {W} image")
        grad = torch.is_grad_enabled() and any(t.requires_grad for t in (prim_rgba, prim_pos, prim_rot, prim_scale))
        dev = prim_rgba.device
        cam = march_camera(RT, K, dev)
        if f > 1:
            offsets = subsample_offsets(int(B), f, self.training)
            pixel_coords = offset_pixel_coords(self.base_pixel_coords, offsets, f)
            offsets = torch.tensor(offsets, dtype=torch.int32).to(dev)
        else:
            offsets, pixel_coords = None, self.base_pixel_coords[None].expand(B, -1, -1, -1).contiguous()
        with torch.set_grad_enabled(grad):
            tpl = prim_rgba.float().permute(0, 1, 3, 4, 5, 2).contiguous()
            pos = (prim_pos / self.volradius).to(dev).float().contiguous()
            rot, scale = prim_rot.to(dev).float().contiguous(), prim_scale.to(dev).float().contiguous()
        geom = (H, W, float(self.volradius), float(self.dt / self.volradius), float(self.fadescale), float(self.fadeexp), f)
        if grad or f > 1:
            out = _RayMarchFunction.apply(tpl, pos, rot, scale, cam, geom, offsets)
        else:
            out = torch.empty(B, H, W, 4, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().tpx_raymarch_preview(tpl.data_ptr(), pos.data_ptr(), rot.data_ptr(), scale.data_ptr(), *[c.data_ptr() for c in cam], B, Kp, S,
                                                           H, W, float(self.volradius), geom[3], float(self.fadescale), float(self.fadeexp), out.data_ptr(),
                                                           _lib.stream_ptr()), "tpx_raymarch_preview")
        return {"rgba_image": out.permute(0, 3, 1, 2), "pixel_coords": pixel_coords}
