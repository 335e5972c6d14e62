"""Mesh extraction on the GPU: marching cubes over a dense fp32 volume (csrc/marching_cubes.cu through include/tpx.h).

``marching_cubes(volume, isovalue)`` is the call extract_texmesh makes on the SDF grid (inference.py:119,
``mcubes.marching_cubes(grid.cpu().numpy(), 0.0)``); ``install(mcubes=True)`` binds it as ``mcubes.marching_cubes``.  Vertices are
in index units, component d along array axis d, shared between triangles; faces are int64 and wound so that the normal
(v1 - v0) x (v2 - v0) points toward increasing value (outward for an SDF that is negative inside).  See INTEGRATION.md for how
this differs from PyMCubes.
"""
from __future__ import annotations

import types

import numpy as np
import torch

from . import _lib

_INDEX_LIMIT = 1 << 31


def _mesh(vol: torch.Tensor, iso: float, origin=(0.0, 0.0, 0.0), spacing=(1.0, 1.0, 1.0)):
    """vol: CUDA fp32 contiguous [X,Y,Z] -> (verts fp32 [V,3], faces int64 [F,3]) on vol's device.  Reads the two counts back once."""
    X, Y, Z = vol.shape
    dev = vol.device
    if min(X, Y, Z) < 2:
        return torch.zeros(0, 3, dtype=torch.float32, device=dev), torch.zeros(0, 3, dtype=torch.int64, device=dev)
    lib = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(lib.tpx_mc_workspace_bytes(X, Y, Z))
        if nbytes == 0:
            raise _lib.TpxError(f"marching_cubes: volume {tuple(vol.shape)} has 2^31 or more points")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr()
        _lib.check(lib.tpx_mc_count(vol.data_ptr(), X, Y, Z, float(iso), ws.data_ptr(), nbytes, counts.data_ptr(), st), "tpx_mc_count")
        V, F = counts.tolist()                 # the one device -> host read (the mesh size is data-dependent, as for torch.nonzero)
        if V >= _INDEX_LIMIT or F >= _INDEX_LIMIT:
            raise _lib.TpxError(f"marching_cubes: {V} vertices / {F} triangles exceed 2^31")
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_mc_emit(vol.data_ptr(), X, Y, Z, float(iso), *[float(o) for o in origin], *[float(s) for s in spacing], ws.data_ptr(), nbytes,
                                   verts.data_ptr(), faces.data_ptr(), st), "tpx_mc_emit")
    return verts, faces


def marching_cubes(volume, isovalue: float = 0.0):
    """Isosurface of a dense [X,Y,Z] volume at ``isovalue`` (a value < isovalue is inside; equal is outside).

    * CUDA fp32 tensor -> (verts fp32 [V,3], faces int64 [F,3]) on its device;
    * numpy array -> (float64 [V,3], int64 [F,3]) numpy arrays, computed in fp32 on the current CUDA device (the
      ``mcubes.marching_cubes`` call of inference.py:119);
    * a CPU tensor, or any call without a GPU, raises TpxError (there is no CPU path); a volume that is not 3-D, or a tensor that
      is not fp32, raises ValueError; a dimension below 2 gives an empty mesh.
    """
    if isinstance(volume, torch.Tensor):
        if not volume.is_cuda:
            raise _lib.TpxError("marching_cubes runs on CUDA only (no CPU path): pass a CUDA tensor or a numpy array")
        if volume.dim() != 3:
            raise ValueError(f"volume must be [X,Y,Z], got {tuple(volume.shape)}")
        if volume.dtype != torch.float32:
            raise ValueError(f"volume must be float32, got {volume.dtype}")
        return _mesh(volume.contiguous(), isovalue)
    arr = np.asarray(volume)
    if arr.ndim != 3:
        raise ValueError(f"volume must be [X,Y,Z], got {arr.shape}")
    _lib.lib()                                 # raises TpxError without a GPU
    vol = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float32)).to(torch.device("cuda", torch.cuda.current_device()))
    verts, faces = _mesh(vol, isovalue)
    return verts.cpu().numpy().astype(np.float64), faces.cpu().numpy()


def mcubes_module() -> types.ModuleType:
    """A module named ``mcubes`` exposing ``marching_cubes``: what extract_texmesh imports (inference.py:119)."""
    m = types.ModuleType("mcubes", "GPU marching cubes of 3dtopia-xl_b200 (tpxl_b200.mesh) under the PyMCubes import name.")
    m.marching_cubes = marching_cubes
    return m
