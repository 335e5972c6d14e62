"""Box-projection UV unwrap on the GPU (csrc/uv_unwrap.cu through include/tpx.h): drop-ins for ``compute_vertex_normal`` and
``box_projection_uv_unwrap`` of utils/uv_unwrap.py, the fast-unwrap branch of extract_texmesh (inference.py:140-150, app.py's
"Faster" choice).  ``install(uv_unwrap=True)`` binds them as ``utils.uv_unwrap``.  The contract, quirks included, is DESIGN.md §1 f-8.

CUDA tensors in give CUDA tensors out; a CPU tensor raises TpxError (there is no CPU path); malformed input (shapes, dtypes, an index
outside [0, V)) raises ValueError; faces may be int32 or int64.
"""
from __future__ import annotations

import ctypes as C
import types

import torch

from . import _lib, bake

TAP_NAMES = ("slice", "face_uv", "angle", "rot_uv", "assign", "placed")


def _check(v: torch.Tensor, f: torch.Tensor, what: str, n: torch.Tensor | None = None):
    """-> (v fp32 contiguous, f int32 contiguous, n fp32 contiguous or None) after the checks of the module docstring."""
    bake._check_rows(v, 3, "vertex_positions")
    bake._check_triangles(f, "triangle_idxs")
    if n is not None:
        bake._check_rows(n, 3, "vertex_normals")
        if n.shape[0] != v.shape[0]:
            raise ValueError(f"vertex_normals has {n.shape[0]} rows for {v.shape[0]} vertices")
    bake._need_cuda(what, v, f, *([] if n is None else [n]))
    if f.device != v.device or (n is not None and n.device != v.device):
        raise ValueError("vertices, normals and faces must be on one device")
    V, F = v.shape[0], f.shape[0]
    if V >= (1 << 31) - 1 or F >= (1 << 31) // 3:
        raise ValueError(f"{V} vertices / {F} faces: too large (V < 2^31 - 1, F < 2^31 / 3)")
    if F:
        lo, hi = torch.stack([f.min(), f.max()]).tolist()
        if lo < 0 or hi >= V:
            raise ValueError(f"a face index is outside [0, {V})")
    return (v.detach().float().contiguous(), f.to(torch.int32).contiguous(),
            None if n is None else n.detach().float().contiguous())


def _workspace(lib, V: int, F: int, dev) -> torch.Tensor:
    nbytes = int(lib.tpx_uv_unwrap_workspace_bytes(V, F))
    if nbytes == 0:
        raise ValueError(f"{V} vertices / {F} faces: too large for the unwrap")
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


def compute_vertex_normal(v_pos: torch.Tensor, t_pos_idx: torch.Tensor) -> torch.Tensor:
    """compute_vertex_normal (utils/uv_unwrap.py:65-85): area-weighted vertex normals fp32 [V,3], summed in the reference's scatter_add_
    order (deterministic, no float atomics), (0, 0, 1) where the sum is degenerate."""
    v, f, _ = _check(v_pos, t_pos_idx, "compute_vertex_normal")
    V, F = v.shape[0], f.shape[0]
    if F == 0:
        return torch.tensor([0.0, 0.0, 1.0], device=v.device).expand(V, 3).contiguous()
    lib = _lib.lib()
    out = torch.empty(V, 3, dtype=torch.float32, device=v.device)
    with torch.cuda.device(v.device):
        ws = _workspace(lib, V, F, v.device)
        _lib.check(lib.tpx_vertex_normals(v.data_ptr(), V, f.data_ptr(), F, ws.data_ptr(), ws.numel(), out.data_ptr(), _lib.stream_ptr()), "tpx_vertex_normals")
    return out


def _unwrap(v: torch.Tensor, n: torch.Tensor, f: torch.Tensor, island_padding: float, taps: dict | None):
    """Checked fp32 v / n and int32 f -> (uv fp32 [U,2], vtex_idx int64 [F,3]); ``taps`` (a dict) receives the stage outputs."""
    V, F = v.shape[0], f.shape[0]
    dev = v.device
    lib = _lib.lib()
    with torch.cuda.device(dev):
        ws = _workspace(lib, V, F, dev)
        counts = torch.empty(1, dtype=torch.int64, device=dev)
        tap_arr = None
        if taps is not None:
            bufs = {"slice": torch.empty(F, dtype=torch.int32, device=dev), "face_uv": torch.empty(F, 3, 2, device=dev),
                    "angle": torch.empty(6, device=dev), "rot_uv": torch.empty(F, 3, 2, device=dev),
                    "assign": torch.empty(F, dtype=torch.int32, device=dev), "placed": torch.empty(F, 3, 2, device=dev)}
            taps.update(bufs)
            tap_arr = (C.c_void_p * len(TAP_NAMES))(*[bufs[k].data_ptr() for k in TAP_NAMES])
        st = _lib.stream_ptr()
        _lib.check(lib.tpx_uv_unwrap(v.data_ptr(), n.data_ptr(), V, f.data_ptr(), F, float(island_padding), ws.data_ptr(), ws.numel(), counts.data_ptr(),
                                     tap_arr, st), "tpx_uv_unwrap")
        U = int(counts.item())                 # the one device -> host read: the number of unique uv rows is data-dependent
        if U < 0:
            raise ValueError(f"a face index is outside [0, {V})")
        uv = torch.empty(U, 2, dtype=torch.float32, device=dev)
        vidx = torch.empty(F, 3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_uv_unwrap_emit(V, F, ws.data_ptr(), ws.numel(), uv.data_ptr(), vidx.data_ptr(), st), "tpx_uv_unwrap_emit")
    return uv, vidx


def box_projection_uv_unwrap(vertex_positions: torch.Tensor, vertex_normals: torch.Tensor, triangle_idxs: torch.Tensor, island_padding: float,
                             taps: dict | None = None):
    """box_projection_uv_unwrap (utils/uv_unwrap.py:644-685): (uv fp32 [U,2], vtex_idx int64 [F,3]) with ``uv[vtex_idx]`` the per-corner
    atlas coordinates in [0, 1]; the rows of uv are the unique corner coordinates sorted by (u, v).  ``taps`` (a dict, optional) receives
    the stage outputs: slice int32 [F], face_uv [F,3,2] (projection), angle [6], rot_uv [F,3,2] (rotated, rescaled), assign int32 [F]
    (atlas slot 0..12), placed [F,3,2]."""
    v, f, n = _check(vertex_positions, triangle_idxs, "box_projection_uv_unwrap", vertex_normals)
    if not 0.0 <= float(island_padding) < 0.5:
        raise ValueError(f"island_padding must be in [0, 0.5), got {island_padding}")
    if f.shape[0] == 0:
        return torch.zeros(0, 2, device=v.device), torch.zeros(0, 3, dtype=torch.int64, device=v.device)
    return _unwrap(v, n, f, float(island_padding), taps)


def noise_filter(srt: torch.Tensor, return_nn: bool = False):
    """The primitive noise filter of extract_texmesh (inference.py:90-103) on srt [K,4] = (scale, x, y, z): keep bool [K] where the
    nearest other primitive (distance + 1 on the diagonal, so a primitive with nothing nearer than 1 matches itself; first index on ties)
    is closer than the two scales summed.  ``return_nn`` also returns that index (int64 [K])."""
    if not isinstance(srt, torch.Tensor) or srt.dim() != 2 or srt.shape[1] != 4 or not srt.is_floating_point():
        raise ValueError(f"srt must be a floating-point [K,4] tensor, got {bake._describe(srt)}")
    bake._need_cuda("noise_filter", srt)
    K = srt.shape[0]
    keep = torch.zeros(K, dtype=torch.uint8, device=srt.device)
    nn = torch.zeros(K, dtype=torch.int32, device=srt.device)
    if K:
        s = srt.detach().float().contiguous()
        lib = _lib.lib()
        with torch.cuda.device(s.device):
            _lib.check(lib.tpx_prim_noise_filter(s.data_ptr(), K, keep.data_ptr(), nn.data_ptr(), _lib.stream_ptr()), "tpx_prim_noise_filter")
    keep = keep.view(torch.bool)
    return (keep, nn.long()) if return_nn else keep


def uv_unwrap_module() -> types.ModuleType:
    """A module named ``utils.uv_unwrap`` exposing the two functions extract_texmesh imports (inference.py:142-143)."""
    m = types.ModuleType("utils.uv_unwrap", "GPU box-projection unwrap of 3dtopia-xl_b200 (tpxl_b200.unwrap) under the reference's import name.")
    m.compute_vertex_normal = compute_vertex_normal
    m.box_projection_uv_unwrap = box_projection_uv_unwrap
    return m
