"""Mesh extraction on the GPU: marching cubes over a dense fp32 volume (csrc/marching_cubes.cu through include/tpx.h).

``marching_cubes(volume, isovalue)`` is the call extract_texmesh makes on the SDF grid (inference.py:119,
``mcubes.marching_cubes(grid.cpu().numpy(), 0.0)``); ``install(mcubes=True)`` binds it as ``mcubes.marching_cubes``.  Vertices are
in index units, component d along array axis d, shared between triangles; faces are int64 and wound so that the normal
(v1 - v0) x (v2 - v0) points toward increasing value (outward for an SDF that is negative inside).  See INTEGRATION.md for how
this differs from PyMCubes.

``remove_small_components`` and ``decimate`` (csrc/mesh_simplify.cu) are the clean_mesh / decimate_mesh calls extract_texmesh makes
next (inference.py:126-129, pymeshlab there); see INTEGRATION.md for how they differ from pymeshlab.  ``clean_mesh`` and
``decimate_mesh`` are the whole utils/meshutils.py calls (close-vertex merge, duplicate / null faces, components, non-manifold repair);
``install(meshutils=True)`` binds them as ``utils.meshutils``.
"""
from __future__ import annotations

import ctypes as C
import math
import time
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


def _check_mesh(verts: torch.Tensor, faces: torch.Tensor, allow_repeat: bool = False):
    """ValueError unless verts is fp32 [V,3] and faces int64 [F,3] with every index in [0, V) and (unless allow_repeat) three distinct
    indices per face."""
    if verts.dim() != 2 or verts.shape[1] != 3 or verts.dtype != torch.float32:
        raise ValueError(f"verts must be float32 [V,3], got {verts.dtype} {tuple(verts.shape)}")
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype != torch.int64:
        raise ValueError(f"faces must be int64 [F,3], got {faces.dtype} {tuple(faces.shape)}")
    V, F = verts.shape[0], faces.shape[0]
    if V >= _INDEX_LIMIT or F >= _INDEX_LIMIT:
        raise ValueError(f"{V} vertices / {F} faces: each must be below 2^31")
    if F:
        if int(faces.min()) < 0 or int(faces.max()) >= V:
            raise ValueError(f"a face index is outside [0, {V})")
        if not allow_repeat and bool(((faces[:, 0] == faces[:, 1]) | (faces[:, 1] == faces[:, 2]) | (faces[:, 2] == faces[:, 0])).any()):
            raise ValueError("a face repeats a vertex index")


def _remove_small(verts: torch.Tensor, faces: torch.Tensor, min_faces: int, min_diameter: float):
    """CUDA verts fp32 [V,3] / faces int64 [F,3] (checked) -> the kept mesh on their device.  Reads the two counts back once."""
    dev = verts.device
    V, F = verts.shape[0], faces.shape[0]
    lib = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(lib.tpx_mesh_components_workspace_bytes(V, F))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr()
        _lib.check(lib.tpx_mesh_components_count(verts.data_ptr(), V, faces.data_ptr(), F, int(min_faces), float(min_diameter), ws.data_ptr(), nbytes,
                                                 counts.data_ptr(), st), "tpx_mesh_components_count")
        Vo, Fo = counts.tolist()
        if Vo < 0:
            raise ValueError("a face index is outside [0, V) or a face repeats an index")
        vo = torch.empty(Vo, 3, dtype=torch.float32, device=dev)
        fo = torch.empty(Fo, 3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_mesh_components_emit(verts.data_ptr(), V, F, ws.data_ptr(), nbytes, vo.data_ptr(), fo.data_ptr(), st), "tpx_mesh_components_emit")
    return vo, fo


def _decimate(verts: torch.Tensor, faces: torch.Tensor, target: int, trace: list | None = None):
    """CUDA verts / faces (checked) -> the decimated mesh on their device; ``trace`` (a list) receives the face count after each round."""
    dev = verts.device
    V, F = verts.shape[0], faces.shape[0]
    lib = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(lib.tpx_decimate_workspace_bytes(V, F))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(3, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr()
        cap = 4096 if trace is not None else 0
        buf = (C.c_int64 * max(cap, 1))()
        _lib.check(lib.tpx_decimate(verts.data_ptr(), V, faces.data_ptr(), F, int(target), ws.data_ptr(), nbytes, counts.data_ptr(),
                                    buf if cap else None, cap, st), "tpx_decimate")
        Vo, Fo, rounds = counts.tolist()
        if trace is not None:
            trace.extend(int(buf[i]) for i in range(min(rounds, cap)))
        vo = torch.empty(Vo, 3, dtype=torch.float32, device=dev)
        fo = torch.empty(Fo, 3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_decimate_emit(V, F, ws.data_ptr(), nbytes, vo.data_ptr(), fo.data_ptr(), st), "tpx_decimate_emit")
    return vo, fo


def _weld(verts: torch.Tensor, faces: torch.Tensor, merge_distance: float, info: dict | None = None):
    """CUDA verts / faces (range-checked; faces may repeat an index) -> the merged mesh without duplicate or null faces, on their
    device; ``info`` (a dict) receives the merge rounds."""
    dev = verts.device
    V, F = verts.shape[0], faces.shape[0]
    lib = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(lib.tpx_mesh_weld_workspace_bytes(V, F))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(3, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr()
        _lib.check(lib.tpx_mesh_weld_count(verts.data_ptr(), V, faces.data_ptr(), F, float(merge_distance), ws.data_ptr(), nbytes, counts.data_ptr(), st),
                   "tpx_mesh_weld_count")
        Vo, Fo, rounds = counts.tolist()
        if Vo < 0:
            raise ValueError("a face index is outside [0, V)")
        if info is not None:
            info["rounds"] = rounds
        vo = torch.empty(Vo, 3, dtype=torch.float32, device=dev)
        fo = torch.empty(Fo, 3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_mesh_weld_emit(verts.data_ptr(), V, F, ws.data_ptr(), nbytes, vo.data_ptr(), fo.data_ptr(), st), "tpx_mesh_weld_emit")
    return vo, fo


def _repair(verts: torch.Tensor, faces: torch.Tensor):
    """CUDA verts / faces (checked) -> the mesh with non-manifold edges and vertices repaired, on their device."""
    dev = verts.device
    V, F = verts.shape[0], faces.shape[0]
    lib = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(lib.tpx_mesh_repair_workspace_bytes(V, F))
        if nbytes == 0:
            raise ValueError(f"repair: {F} faces: must be below 2^30")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr()
        _lib.check(lib.tpx_mesh_repair_count(verts.data_ptr(), V, faces.data_ptr(), F, ws.data_ptr(), nbytes, counts.data_ptr(), st), "tpx_mesh_repair_count")
        Vo, Fo = counts.tolist()
        if Vo < 0:
            raise ValueError("a face index is outside [0, V) or a face repeats an index")
        vo = torch.empty(Vo, 3, dtype=torch.float32, device=dev)
        fo = torch.empty(Fo, 3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_mesh_repair_emit(verts.data_ptr(), V, F, ws.data_ptr(), nbytes, vo.data_ptr(), fo.data_ptr(), st), "tpx_mesh_repair_emit")
    return vo, fo


def _remesh(verts: torch.Tensor, faces: torch.Tensor, target_len: float, iterations: int, feature_deg: float, info: list | None = None):
    """CUDA verts / faces (checked) -> the remeshed, compacted mesh on their device; ``info`` (a list) receives per iteration
    dict(F=[faces after split, collapse, flip], V=vertex slots, collapse_rounds, flip_rounds, split_ms, relax_ms) (host clock around a
    synchronise)."""
    dev = verts.device
    V0, F0 = verts.shape[0], faces.shape[0]
    lib = _lib.lib()
    cosf = math.cos(math.radians(feature_deg))
    v, f = verts, faces
    with torch.cuda.device(dev):
        st = _lib.stream_ptr()
        gbytes = int(lib.tpx_remesh_grid_bytes(F0))
        nbytes = int(lib.tpx_remesh_workspace_bytes(V0, F0))
        if gbytes == 0 or nbytes == 0:
            raise ValueError(f"remesh: {F0} faces: must be below 2^28")
        grid = torch.empty(gbytes, dtype=torch.uint8, device=dev)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        creases = torch.empty(max(3 * F0, 1), dtype=torch.int64, device=dev)
        counts = torch.empty(3, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_remesh_begin(verts.data_ptr(), V0, faces.data_ptr(), F0, cosf, grid.data_ptr(), gbytes, ws.data_ptr(), nbytes,
                                        creases.data_ptr(), counts.data_ptr(), st), "tpx_remesh_begin")
        nC = int(counts[0])
        if nC < 0:
            raise ValueError("a face index is outside [0, V) or a face repeats an index")
        creases = creases[:nC]
        v = verts.clone()
        for _ in range(iterations):
            t0 = time.perf_counter()
            V, F = v.shape[0], f.shape[0]
            nbytes = int(lib.tpx_remesh_workspace_bytes(V, F))
            if nbytes == 0:
                raise _lib.TpxError(f"remesh: {V} vertices / {F} faces exceed the index range")
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(lib.tpx_remesh_split_count(v.data_ptr(), V, f.data_ptr(), F, creases.data_ptr(), nC, float(target_len), ws.data_ptr(), nbytes,
                                                  counts.data_ptr(), st), "tpx_remesh_split_count")
            Vs, Fs, nCs = counts.tolist()
            if Vs >= _INDEX_LIMIT or 2 * Fs >= _INDEX_LIMIT:
                raise _lib.TpxError(f"remesh: the split gives {Vs} vertices / {Fs} faces, over the index range")
            vs = torch.empty(Vs, 3, dtype=torch.float32, device=dev)
            fs = torch.empty(Fs, 3, dtype=torch.int64, device=dev)
            cs = torch.empty(max(nCs, 1), dtype=torch.int64, device=dev)
            _lib.check(lib.tpx_remesh_split_emit(v.data_ptr(), V, F, creases.data_ptr(), nC, nCs, ws.data_ptr(), nbytes, vs.data_ptr(), fs.data_ptr(),
                                                 cs.data_ptr(), st), "tpx_remesh_split_emit")
            v, f, creases, nC = vs, fs, cs[:nCs], nCs
            if info is not None:
                torch.cuda.synchronize(dev)
            t1 = time.perf_counter()
            nbytes = int(lib.tpx_remesh_workspace_bytes(Vs, Fs))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(lib.tpx_remesh_relax(v.data_ptr(), Vs, f.data_ptr(), Fs, creases.data_ptr(), nC, verts.data_ptr(), V0, F0, grid.data_ptr(), gbytes,
                                            float(target_len), cosf, ws.data_ptr(), nbytes, counts.data_ptr(), st), "tpx_remesh_relax")
            Fr, rc, rf = counts.tolist()
            if info is not None:
                info.append(dict(F=[Fs, Fr, Fr], V=Vs, collapse_rounds=rc, flip_rounds=rf, split_ms=round((t1 - t0) * 1e3, 2),
                                 relax_ms=round((time.perf_counter() - t1) * 1e3, 2)))
            f = f[:Fr]
    return _remove_small(v, f.contiguous(), 0, 0.0)          # the compaction: referenced vertices in ascending id, faces in order


def _closest(verts: torch.Tensor, faces: torch.Tensor, pts: torch.Tensor):
    """CUDA verts / faces (checked), pts fp32 [n,3] on their device -> (closest points fp32 [n,3], face ids int64 [n]) of the mesh: the
    projection step of ``remesh`` on its own, through the same grid."""
    dev = verts.device
    V, F, n = verts.shape[0], faces.shape[0], pts.shape[0]
    lib = _lib.lib()
    with torch.cuda.device(dev):
        gbytes, nbytes = int(lib.tpx_remesh_grid_bytes(F)), int(lib.tpx_remesh_workspace_bytes(V, F))
        if gbytes == 0 or nbytes == 0:
            raise ValueError(f"closest: {F} faces: must be below 2^28")
        grid = torch.empty(gbytes, dtype=torch.uint8, device=dev)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        creases = torch.empty(max(3 * F, 1), dtype=torch.int64, device=dev)
        counts = torch.empty(1, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr()
        _lib.check(lib.tpx_remesh_begin(verts.data_ptr(), V, faces.data_ptr(), F, 1.0, grid.data_ptr(), gbytes, ws.data_ptr(), nbytes, creases.data_ptr(),
                                        counts.data_ptr(), st), "tpx_remesh_begin")
        if int(counts[0]) < 0:
            raise ValueError("a face index is outside [0, V) or a face repeats an index")
        out = torch.empty(n, 3, dtype=torch.float32, device=dev)
        fid = torch.empty(n, dtype=torch.int64, device=dev)
        _lib.check(lib.tpx_remesh_closest(pts.data_ptr(), n, verts.data_ptr(), V, F, grid.data_ptr(), gbytes, out.data_ptr(), fid.data_ptr(), st),
                   "tpx_remesh_closest")
    return out, fid


def _clean(verts: torch.Tensor, faces: torch.Tensor, merge_distance: float, min_faces: int, min_diameter: float, repair: bool):
    """The steps of clean_mesh in the reference's order: weld / duplicate / null faces, components, then the non-manifold repair."""
    v, f = _weld(verts, faces, merge_distance)
    if min_faces > 0 or min_diameter > 0:
        v, f = _remove_small(v, f, min_faces, min_diameter)
    if repair:
        v, f = _repair(v, f)
    return v, f


def _mesh_call(fn, verts, faces, *args, allow_repeat: bool = False):
    """The marching_cubes convention: CUDA tensors in, CUDA tensors out; numpy in, numpy float64 / int64 out from the current device."""
    if isinstance(verts, torch.Tensor) or isinstance(faces, torch.Tensor):
        if not (isinstance(verts, torch.Tensor) and isinstance(faces, torch.Tensor)):
            raise ValueError("pass verts and faces both as tensors or both as numpy arrays")
        if not verts.is_cuda or not faces.is_cuda:
            raise _lib.TpxError("mesh clean-up runs on CUDA only (no CPU path): pass CUDA tensors or numpy arrays")
        if verts.device != faces.device:
            raise ValueError(f"verts on {verts.device}, faces on {faces.device}")
        verts, faces = verts.contiguous(), faces.contiguous()
        _check_mesh(verts, faces, allow_repeat)
        return fn(verts, faces, *args)
    v, f = np.asarray(verts), np.asarray(faces)
    if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3 or not np.issubdtype(f.dtype, np.integer):
        raise ValueError(f"verts must be [V,3] and faces integer [F,3], got {v.shape} and {f.dtype} {f.shape}")
    _lib.lib()                                 # raises TpxError without a GPU
    dev = torch.device("cuda", torch.cuda.current_device())
    vt = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(dev)
    ft = torch.from_numpy(np.ascontiguousarray(f, dtype=np.int64)).to(dev)
    _check_mesh(vt, ft, allow_repeat)
    vo, fo = fn(vt, ft, *args)
    return vo.cpu().numpy().astype(np.float64), fo.cpu().numpy()


def remove_small_components(verts, faces, min_faces: int = 8, min_diameter: float = 0.05):
    """Drop the small connected components of a triangle mesh: clean_mesh's remove_connected_component_by_face_number(min_f) and
    ..._by_diameter(PercentageValue(min_d)) (utils/meshutils.py:63-193, inference.py:126 with min_f = 8, min_d = 5).

    Faces are connected iff they share an undirected edge; a component is removed iff it has fewer than ``min_faces`` faces or its
    bounding-box diagonal is below ``min_diameter`` (a fraction, 0.05 for min_d = 5) times that of all referenced vertices.  Returns the
    vertices the kept faces use (ascending original id) and the kept faces (original order, remapped, winding unchanged).
    CUDA fp32 [V,3] / int64 [F,3] tensors give CUDA tensors; numpy arrays give float64 / int64 numpy arrays computed on the current
    device; a CPU tensor or a call without a GPU raises TpxError; malformed input (shapes, dtypes, an index outside [0, V), a face
    repeating an index) raises ValueError."""
    return _mesh_call(_remove_small, verts, faces, int(min_faces), float(min_diameter))


def decimate(verts, faces, target_faces: int):
    """Quadric-error edge-collapse decimation to ``target_faces`` faces: the GPU stand-in for decimate_mesh(v, t, target)
    (utils/meshutils.py:63-193, inference.py:129 with 100000).  Deterministic rounds of independent collapses (DESIGN.md §1 f-7);
    boundary and non-manifold vertices never move.  A reachable target ends at ``target_faces - 1`` or ``target_faces`` faces; if a
    round finds no valid collapse (e.g. a mesh of only boundary or tetrahedron-like pieces) the mesh is returned ABOVE the target.
    ``target_faces >= F`` returns the input (minus unreferenced vertices).  Inputs and outputs as ``remove_small_components``."""
    if int(target_faces) < 0:
        raise ValueError(f"target_faces must be >= 0, got {target_faces}")
    return _mesh_call(_decimate, verts, faces, int(target_faces))


def remesh(verts, faces, target_len: float, iterations: int = 3, feature_deg: float = 30.0, info: list | None = None):
    """Isotropic remeshing toward edges of length ``target_len``: the GPU stand-in for pymeshlab's
    meshing_isotropic_explicit_remeshing(iterations, targetlen) that decimate_mesh(..., remesh=True) runs after the decimation
    (utils/meshutils.py:101-105, inference.py:128-129, where targetlen is PercentageValue(1), 1 % of the box diagonal).  Per iteration,
    in VCG's order: split edges above 4/3 target_len, collapse edges below 4/5 target_len, flip edges toward valence 6 (4 at the
    border), one tangential smoothing pass, then project every moved vertex onto the closest point of the input mesh.  Border,
    non-manifold vertices and the ends of crease edges (faces meeting beyond ``feature_deg`` degrees) never move.  The rules are this
    package's reading of VCG (DESIGN.md §1 "Isotropic remeshing contract"), not checked against pymeshlab.  ``iterations = 0`` returns
    the input without its unreferenced vertices.  ``info`` (a list) receives per iteration the face counts after split, collapse and
    flip and the round counts.  Inputs and outputs as ``remove_small_components``; ValueError also for a ``target_len`` that is not
    finite and positive, ``iterations < 0`` or ``feature_deg`` outside [0, 180]."""
    L, it, fd = float(target_len), int(iterations), float(feature_deg)
    if not (math.isfinite(L) and L > 0):
        raise ValueError(f"target_len must be finite and > 0, got {target_len}")
    if it < 0:
        raise ValueError(f"iterations must be >= 0, got {iterations}")
    if not 0.0 <= fd <= 180.0:
        raise ValueError(f"feature_deg must be in [0, 180], got {feature_deg}")
    return _mesh_call(_remesh, verts, faces, L, it, fd, info)


def clean_mesh(verts, faces, v_pct=1, min_f=64, min_d=20, repair=True, remesh=True, remesh_size=0.01, remesh_iters=3):
    """clean_mesh of utils/meshutils.py:118-193 (called at inference.py:126 as clean_mesh(v, t, min_f=8, min_d=5, repair=True,
    remesh=False)), with its signature and defaults, on the GPU.  In the reference's order: unreferenced vertices dropped; vertices
    within ``v_pct`` % of the box diagonal merged greedily onto the earliest seed (skipped for v_pct = 0); faces that repeat an index,
    duplicate faces (same vertex set; the lowest face id stays) and zero-area faces removed; components below ``min_d`` % of the diagonal
    and below ``min_f`` faces removed; with ``repair``, faces removed from non-manifold edges and non-manifold vertices split.  The rules
    are this package's reading of pymeshlab / VCG (DESIGN.md §1 "clean-up contract").  ``remesh=True`` (the default, as in the
    reference) raises NotImplementedError; pass remesh=False as inference.py does, and call ``remesh`` for the isotropic remeshing
    (binding it here is left to a later change).
    Unlike ``remove_small_components`` the faces may repeat an index.  Output: the surviving vertices in ascending original id, then
    the split copies; the faces in their original order, remapped, winding unchanged; no face repeats an index, so the result feeds
    ``decimate``.  Inputs and outputs otherwise as ``remove_small_components``."""
    if remesh:
        raise NotImplementedError("clean_mesh: isotropic remeshing is not implemented; pass remesh=False (as inference.py:126 does)")
    if v_pct < 0 or min_f < 0 or min_d < 0:
        raise ValueError(f"v_pct, min_f and min_d must be >= 0, got {v_pct}, {min_f}, {min_d}")
    return _mesh_call(_clean, verts, faces, float(v_pct) / 100.0, int(min_f), float(min_d) / 100.0, bool(repair), allow_repeat=True)


def decimate_mesh(verts, faces, target=5e4, backend="pymeshlab", remesh=False, optimalplacement=True):
    """decimate_mesh of utils/meshutils.py:63-115 (inference.py:129): ``decimate`` to int(target) faces.  backend="pyfqmr",
    remesh=True and optimalplacement=False are not implemented and raise NotImplementedError (for remesh=True call ``remesh`` on the
    result; binding it here is left to a later change)."""
    if backend != "pymeshlab":
        raise NotImplementedError(f"decimate_mesh: backend {backend!r} is not implemented (the quadric decimation of `decimate` stands in for pymeshlab)")
    if remesh:
        raise NotImplementedError("decimate_mesh: isotropic remeshing is not implemented; pass remesh=False")
    if not optimalplacement:
        raise NotImplementedError("decimate_mesh: only optimal placement is implemented")
    return decimate(verts, faces, int(target))


def meshutils_module() -> types.ModuleType:
    """A module named ``utils.meshutils`` exposing ``clean_mesh`` and ``decimate_mesh``: what extract_texmesh imports (inference.py:126-129)."""
    m = types.ModuleType("utils.meshutils", "GPU mesh clean-up and decimation of 3dtopia-xl_b200 (tpxl_b200.mesh) under the reference's import name.")
    m.clean_mesh = clean_mesh
    m.decimate_mesh = decimate_mesh
    return m


def mcubes_module() -> types.ModuleType:
    """A module named ``mcubes`` exposing ``marching_cubes``: what extract_texmesh imports (inference.py:119)."""
    m = types.ModuleType("mcubes", "GPU marching cubes of 3dtopia-xl_b200 (tpxl_b200.mesh) under the PyMCubes import name.")
    m.marching_cubes = marching_cubes
    return m
