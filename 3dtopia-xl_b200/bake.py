"""Texture bake on the GPU: UV-space rasterisation, attribute interpolation and seam padding (csrc/texture_bake.cu through
include/tpx.h) — the pieces of extract_texmesh's texture block (inference.py:163-211) that the reference takes from nvdiffrast, scipy
and scikit-learn.  ``PrimSDF.bake_texture`` strings them together with the fused texel query; ``install(nvdiffrast=True)`` binds
``nvdiffrast.torch`` to the forward-only, UV-space subset below.  See INTEGRATION.md for the rasterisation contract and how it
relates to nvdiffrast's.

Images are [H, W, ...] with row 0 at v = 0 (nvdiffrast's bottom-up rows), ``rast`` is nvdiffrast's (u, v, 0, triangle_id + 1).
CUDA tensors only: there is no CPU path.
"""
from __future__ import annotations

import types

import torch

from . import _lib

_INDEX_LIMIT = 1 << 31


def _need_cuda(what: str, *tensors: torch.Tensor) -> None:
    for t in tensors:
        if not t.is_cuda:
            raise _lib.TpxError(f"{what} runs on CUDA only (no CPU path): pass CUDA tensors")


def _check_rows(t, cols: int | None, name: str) -> None:
    if not isinstance(t, torch.Tensor) or t.dim() != 2 or (cols is not None and t.shape[1] != cols) or t.shape[1] < 1 or not t.is_floating_point():
        raise ValueError(f"{name} must be a floating-point [N,{cols if cols is not None else 'C'}] tensor, got {_describe(t)}")


def _check_triangles(t, name: str) -> None:
    if not isinstance(t, torch.Tensor) or t.dim() != 2 or t.shape[1] != 3 or t.dtype not in (torch.int32, torch.int64):
        raise ValueError(f"{name} must be an int32 / int64 [F,3] tensor, got {_describe(t)}")


def _describe(t) -> str:
    return f"{t.dtype} {tuple(t.shape)}" if isinstance(t, torch.Tensor) else type(t).__name__


def _narrow(t: torch.Tensor, name: str) -> torch.Tensor:
    """[F,3] int32 / int64 -> contiguous int32; int64 values of 2^31 or more are refused (one device -> host read, int64 only)."""
    if t.dtype == torch.int64:
        if t.numel() and int(t.abs().max()) >= _INDEX_LIMIT:
            raise ValueError(f"{name} holds an index of 2^31 or more")
        t = t.int()
    return t.contiguous()


def _size(height, width) -> tuple[int, int]:
    h, w = int(height), int(width)
    if not (1 <= h <= 8192 and 1 <= w <= 8192):
        raise ValueError(f"atlas size must be 1..8192 per side, got {h} x {w}")
    return h, w


def _rasterize(vt: torch.Tensor, ft: torch.Tensor, h: int, w: int):
    """vt fp32 [Nt,2], ft int32 [F,3], both contiguous CUDA -> (rast fp32 [h,w,4], winner int32 [h,w])."""
    lib = _lib.lib()
    rast = torch.empty(h, w, 4, dtype=torch.float32, device=vt.device)
    winner = torch.empty(h, w, dtype=torch.int32, device=vt.device)
    with torch.cuda.device(vt.device):
        _lib.check(lib.tpx_uv_rasterize(vt.data_ptr(), vt.shape[0], ft.data_ptr(), ft.shape[0], h, w, rast.data_ptr(), winner.data_ptr(), _lib.stream_ptr()),
                   "tpx_uv_rasterize")
    return rast, winner


def rasterize_uv(vt: torch.Tensor, ft: torch.Tensor, height: int, width: int) -> torch.Tensor:
    """Rasterise the UV layout (vt [Nt,2] in [0,1], ft [F,3]) into a height x width atlas: rast fp32 [height, width, 4] =
    (u, v, 0, triangle_id + 1), zeros where no triangle covers the texel centre; (u, v) weigh vertices 0 and 1 of the triangle.
    What ``dr.rasterize(glctx, cat(vt * 2 - 1, 0, 1)[None], ft, (h, w))[0][0]`` is used for at inference.py:163-172."""
    _check_rows(vt, 2, "vt")
    _check_triangles(ft, "ft")
    h, w = _size(height, width)
    _need_cuda("rasterize_uv", vt, ft)
    return _rasterize(vt.detach().float().contiguous(), _narrow(ft, "ft"), h, w)[0]


def interpolate(attr: torch.Tensor, rast: torch.Tensor, tri: torch.Tensor) -> torch.Tensor:
    """Per-texel attribute: out fp32 [H,W,C] = u a0 + v a1 + (1 - u - v) a2 over the triangle ``tri[id]`` of attr [N,C]; zeros where
    rast[..., 3] == 0 (``dr.interpolate``, inference.py:173-174)."""
    _check_rows(attr, None, "attr")
    _check_triangles(tri, "tri")
    if not isinstance(rast, torch.Tensor) or rast.dim() != 3 or rast.shape[2] != 4 or rast.dtype != torch.float32:
        raise ValueError(f"rast must be a float32 [H,W,4] tensor, got {_describe(rast)}")
    h, w = _size(rast.shape[0], rast.shape[1])
    _need_cuda("interpolate", attr, rast, tri)
    attr, tri, rast = attr.detach().float().contiguous(), _narrow(tri, "tri"), rast.contiguous()
    lib = _lib.lib()
    out = torch.empty(h, w, attr.shape[1], dtype=torch.float32, device=rast.device)
    with torch.cuda.device(rast.device):
        _lib.check(lib.tpx_rast_interpolate(attr.data_ptr(), attr.shape[0], attr.shape[1], tri.data_ptr(), tri.shape[0], rast.data_ptr(), h, w, out.data_ptr(),
                                            _lib.stream_ptr()), "tpx_rast_interpolate")
    return out


def inpaint(feats: torch.Tensor, mask: torch.Tensor, pad: int = 32, return_source: bool = False):
    """Seam padding, in place: every texel of feats [H,W,C] outside ``mask`` [H,W] (bool / uint8) within ``pad`` 4-connected steps of it
    takes the value of the Euclidean-nearest mask texel (smallest (row, col) among equidistant ones): inference.py:200-211 with
    pad = 32.  Returns feats, or (feats, src int32 [H,W]) with the flat index of each written texel's source and -1 elsewhere."""
    if not isinstance(feats, torch.Tensor) or feats.dim() != 3 or feats.dtype != torch.float32 or feats.shape[2] < 1 or not feats.is_contiguous():
        raise ValueError(f"feats must be a contiguous float32 [H,W,C] tensor, got {_describe(feats)}")
    if not isinstance(mask, torch.Tensor) or mask.shape != feats.shape[:2] or mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"mask must be a bool / uint8 [H,W] tensor matching feats, got {_describe(mask)}")
    if not 0 <= int(pad) <= 8192:
        raise ValueError(f"pad must be 0..8192, got {pad}")
    h, w = _size(feats.shape[0], feats.shape[1])
    _need_cuda("inpaint", feats, mask)
    m8 = mask.contiguous().view(torch.uint8)
    lib = _lib.lib()
    with torch.cuda.device(feats.device):
        nbytes = int(lib.tpx_texture_inpaint_bytes(h, w))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=feats.device)
        src = torch.empty(h, w, dtype=torch.int32, device=feats.device) if return_source else None
        _lib.check(lib.tpx_texture_inpaint(feats.data_ptr(), m8.data_ptr(), h, w, feats.shape[2], int(pad), ws.data_ptr(), nbytes, _lib.ptr(src),
                                           _lib.stream_ptr()), "tpx_texture_inpaint")
    return (feats, src) if return_source else feats


# ---- the nvdiffrast.torch names extract_texmesh uses (inference.py:22,31,172-174) ----------------------------------------------------
class _Context:
    """Stands in for RasterizeCudaContext / RasterizeGLContext: the kernels keep no state between calls."""

    def __init__(self, *args, **kwargs):
        pass


def _dr_rasterize(glctx, pos, tri, resolution, ranges=None, grad_db=True):
    """``dr.rasterize`` for UV-space positions: pos [1,N,4] = (x, y, z, 1) in clip space, uv = (xy + 1) / 2; z is ignored (the lowest
    triangle index wins an overlap).  Returns (rast [1,h,w,4], rast_db zeros)."""
    if ranges is not None or pos.dim() != 3 or pos.shape[0] != 1 or pos.shape[2] != 4:
        raise NotImplementedError("rasterize: only one instance of [1,N,4] clip-space positions is covered (the UV-space use of extract_texmesh)")
    _need_cuda("rasterize", pos, tri)
    if bool((pos[..., 3] != 1).any()):
        raise NotImplementedError("rasterize: positions with w != 1 need a 3-D rasteriser; this one covers UV space only")
    h, w = resolution
    rast = rasterize_uv((pos[0, :, :2].float() + 1.0) * 0.5, tri, h, w).unsqueeze(0)
    return rast, torch.zeros_like(rast)


def _dr_interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
    """``dr.interpolate`` forward: attr [1,N,C], rast [1,h,w,4] -> (out [1,h,w,C], None)."""
    if rast_db is not None or diff_attrs is not None or attr.dim() != 3 or attr.shape[0] != 1 or rast.dim() != 4 or rast.shape[0] != 1:
        raise NotImplementedError("interpolate: only attr [1,N,C] with rast [1,h,w,4] and no attribute derivatives is covered")
    return interpolate(attr[0], rast[0], tri).unsqueeze(0), None


def nvdiffrast_modules():
    """(``nvdiffrast``, ``nvdiffrast.torch``) modules exposing the forward-only UV-space subset extract_texmesh imports."""
    pkg = types.ModuleType("nvdiffrast", "UV-space rasteriser of 3dtopia-xl_b200 (tpxl_b200.bake) under the nvdiffrast import name.")
    pkg.__path__ = []
    dr = types.ModuleType("nvdiffrast.torch", pkg.__doc__)
    dr.RasterizeCudaContext = dr.RasterizeGLContext = _Context
    dr.rasterize, dr.interpolate = _dr_rasterize, _dr_interpolate
    pkg.torch = dr
    return pkg, dr
