"""Host-side mirror of the reference's PrimSDF query field (SURVEY.md §8f-1), backed by libtpx_b200.

Drop-in for ``models.primsdf.PrimSDF`` (/root/reference/models/primsdf.py) on the inference path: same constructor
kwargs (configs/inference_dit.yml:22-30), the same two parameters ``srt_param [K,4]`` / ``feat_param [K, 6*S^3]`` (so
``load_state_dict`` of ``denoised.pt`` and the ``.data = filtered`` reassignment in inference.py:100-101 work), and
``forward(x[n,3]) -> {"sdf","tex","mat"}``.  The reference evaluates a dense [points x prims] weight matrix per 8192-point
chunk; the kernel visits every primitive per point in registers and samples only the covering ones.
Mesh-based initialisation (``_init_param``) is training-time and absent, as in the released reference (it is ``pass``).

Gradients: with ``differentiable=True``, autograd on, and any of ``x`` / ``srt_param`` / ``feat_param`` requiring grad, ``forward`` runs
as a ``torch.autograd.Function`` over the same query kernel and ``tpx_primsdf_query_backward``, so ``PrimSDFLoss``-style fitting
(dva/losses.py:102-148) and ``d sdf / d x`` (the field's normal) work through it.  Its outputs are bit-identical to the no-grad path's.
The backward is once-differentiable: a second derivative (``PrimSDFLoss``'s ``grad_l2`` term) raises.  Without ``differentiable``, every
call returns detached outputs, as before.  ``sdf_grid``, ``bake_texture`` and the ``extract_*`` methods carry no gradient.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib, bake, mesh, unwrap


class _PrimSDFFunction(torch.autograd.Function):
    """PrimSDF.forward (models/primsdf.py:52-109) under autograd: x [n,3], srt [K,4], feat [K, 6 S^3] in any float dtype -> fp32
    [n,6] = (sdf, rgb, roughness, metallic), with ``module`` supplying prim_shape, training (the uncovered-point fill) and the
    grid cache.  The backward walks the workspace the forward used (kept on ctx: the module may rebuild its grid before backward runs)."""

    @staticmethod
    def forward(ctx, x, srt_param, feat_param, module):
        xx, srt, feat = (t.detach().float().contiguous() for t in (x, srt_param, feat_param))
        out, ws = module._query(xx, srt, feat)
        ctx.save_for_backward(x, srt_param, feat_param)
        ctx.ws, ctx.S, ctx.dim_feat, ctx.inference = ws, module.prim_shape, module.dim_feat, 0 if module.training else 1
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if torch.is_grad_enabled():       # create_graph=True: a graph of the gradient was asked for
            raise RuntimeError("PrimSDF's backward is once_differentiable: a second derivative (create_graph=True, e.g. a loss on "
                               "d sdf / d x) is not supported")
        return _PrimSDFFunction._backward(ctx, grad_out)

    @staticmethod
    @once_differentiable
    def _backward(ctx, grad_out):
        x, srt_param, feat_param = ctx.saved_tensors
        xx, srt, feat = (t.detach().float().contiguous() for t in (x, srt_param, feat_param))
        need = ctx.needs_input_grad[:3]
        gx, gs, gf = (torch.zeros_like(t) if nd else None for t, nd in zip((xx, srt, feat), need))
        g = grad_out.float().contiguous()
        ws = ctx.ws
        with torch.cuda.device(xx.device):
            _lib.check(_lib.lib().tpx_primsdf_query_backward(xx.data_ptr(), srt.data_ptr(), feat.data_ptr(), _lib.ptr(ws), 0 if ws is None else ws.numel(),
                                                             xx.shape[0], srt.shape[0], ctx.S, ctx.dim_feat, ctx.inference, g.data_ptr(), _lib.ptr(gx),
                                                             _lib.ptr(gs), _lib.ptr(gf), _lib.stream_ptr()), "tpx_primsdf_query_backward")
        return (None if gx is None else gx.to(x.dtype), None if gs is None else gs.to(srt_param.dtype),
                None if gf is None else gf.to(feat_param.dtype), None)


class PrimSDF(nn.Module):
    def __init__(self, mesh_obj=None, f_sdf=None, geo_fn=None, asset_list=None, num_prims=1024, dim_feat=6, prim_shape=8, init_scale=0.05,
                 sdf2alpha_var=0.005, auto_scale_init=True, init_sampling="uniform", differentiable=False, **_unused):
        super().__init__()
        self.differentiable = differentiable   # forward records a graph (see _PrimSDFFunction) only when this is set
        self.num_prims, self.dim_feat, self.prim_shape = num_prims, dim_feat, prim_shape
        self.sdf2alpha_var = sdf2alpha_var
        self.auto_scale_init, self.init_sampling = auto_scale_init, init_sampling
        self.mesh_obj, self.f_sdf = mesh_obj, f_sdf
        self.srt_param = nn.parameter.Parameter(torch.zeros(num_prims, 1 + 3))
        self.feat_param = nn.parameter.Parameter(torch.zeros(num_prims, dim_feat * prim_shape ** 3))
        s3 = prim_shape ** 3
        self.geo_start_index, self.geo_end_index = 0, s3
        self.tex_start_index, self.tex_end_index = s3, 4 * s3
        self.mat_start_index, self.mat_end_index = 4 * s3, 6 * s3
        self._grid = None          # (key, srt tensor the grid was built from, workspace): rebuilt whenever srt_param changes
        self.grid_entries = 8 << 20   # capacity of the per-cell lists (int32 entries); over-full grids fall back to the exhaustive loop

    def forward(self, x: torch.Tensor):
        if x.dim() != 2 or x.shape[1] != 3:
            raise ValueError(f"x must be [n,3], got {tuple(x.shape)}")
        if not x.is_cuda or not self.srt_param.is_cuda:
            raise _lib.TpxError("PrimSDF query runs on CUDA only (no CPU path): move the module and the points to the GPU")
        if self.differentiable and torch.is_grad_enabled() and any(t.requires_grad for t in (x, self.srt_param, self.feat_param)):
            out = _PrimSDFFunction.apply(x, self.srt_param, self.feat_param, self)
        else:
            out, _ = self._query(x.detach().float().contiguous(), self.srt_param.detach().float().contiguous(),
                                 self.feat_param.detach().float().contiguous())
        return {"sdf": out[:, 0:1], "tex": out[:, 1:4], "mat": out[:, 4:6]}

    def _query(self, xx: torch.Tensor, srt: torch.Tensor, feat: torch.Tensor):
        """fp32 [n, dim_feat] query of the fp32 contiguous points, and the grid workspace it walked (None: exhaustive kernel)."""
        lib = _lib.lib()
        n, K = xx.shape[0], srt.shape[0]
        out = torch.empty(n, self.dim_feat, dtype=torch.float32, device=xx.device)
        ws = None
        with torch.cuda.device(xx.device):
            if K < 1 or K > 4096:      # outside the grid builder's range: exhaustive kernel
                _lib.check(lib.tpx_primsdf_query(xx.data_ptr(), srt.data_ptr(), feat.data_ptr(), n, K, self.prim_shape, self.dim_feat,
                                                 0 if self.training else 1, out.data_ptr(), _lib.stream_ptr()), "tpx_primsdf_query")
            else:
                ws = self._grid_workspace(srt, K, xx.device)
                _lib.check(lib.tpx_primsdf_query_grid(xx.data_ptr(), srt.data_ptr(), feat.data_ptr(), ws.data_ptr(), ws.numel(), n, K, self.prim_shape,
                                                      self.dim_feat, 0 if self.training else 1, out.data_ptr(), _lib.stream_ptr()), "tpx_primsdf_query_grid")
        return out, ws

    def _grid_workspace(self, srt: torch.Tensor, K: int, device) -> torch.Tensor:
        """The binned lists of the current srt_param (tpx_primsdf_grid_build), rebuilt only when srt_param changes."""
        lib = _lib.lib()
        key = (self.srt_param.data_ptr(), self.srt_param._version, K, str(device))
        if self._grid is None or self._grid[0] != key:
            nbytes = int(lib.tpx_primsdf_grid_bytes(self.grid_entries))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
            _lib.check(lib.tpx_primsdf_grid_build(srt.data_ptr(), K, ws.data_ptr(), nbytes, _lib.stream_ptr()), "tpx_primsdf_grid_build")
            self._grid = (key, self.srt_param.data, ws)     # holding the tensor keeps its address from being recycled under the key
        return self._grid[2]

    def sdf_grid(self, resolution: int, bound: float = 1.0) -> torch.Tensor:
        """sdf of the query on the resolution^3 lattice linspace(-bound, bound, resolution)^3: fp32 [R,R,R] on the module's device,
        grid[i,j,k] at (x, y, z) = (xx[i], xx[j], xx[k]).  Bit-identical to the grid extract_texmesh builds from ``forward`` over the
        meshgrid points (inference.py:107-116), without materialising them; the uncovered-point approximation follows
        ``self.training`` as in ``forward``."""
        R = int(resolution)
        if R < 1:
            raise ValueError(f"resolution must be >= 1, got {resolution}")
        if not self.srt_param.is_cuda:
            raise _lib.TpxError("PrimSDF query runs on CUDA only (no CPU path): move the module to the GPU")
        lib = _lib.lib()
        dev = self.srt_param.device
        srt = self.srt_param.detach().float().contiguous()
        feat = self.feat_param.detach().float().contiguous()
        K = srt.shape[0]
        grid = torch.empty(R, R, R, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            coords = torch.linspace(-bound, bound, R, device=dev)
            ws = self._grid_workspace(srt, K, dev) if 1 <= K <= 4096 else None
            _lib.check(lib.tpx_primsdf_sdf_grid(coords.data_ptr(), R, srt.data_ptr(), feat.data_ptr(), _lib.ptr(ws), 0 if ws is None else ws.numel(), K,
                                                self.prim_shape, self.dim_feat, 0 if self.training else 1, grid.data_ptr(), _lib.stream_ptr()),
                       "tpx_primsdf_sdf_grid")
        return grid

    def extract_mesh(self, resolution: int = 256, isovalue: float = 0.0, bound: float = 1.0, *, min_faces: int = 0, min_diameter: float = 0.0,
                     target_faces: int | None = None, merge_distance: float = 0.0, repair: bool = False, remesh_pct: float | None = None,
                     remesh_iters: int = 3):
        """Surface of the sdf field on the GPU: ``sdf_grid`` + marching cubes, in world coordinates (origin -bound, spacing
        2 bound / (R - 1)), i.e. inference.py:107-124 without the host copy.  Returns (verts fp32 [V,3], faces int64 [F,3]) on the
        module's device.  Then, in the order of inference.py:126-129 (clean_mesh, then decimate_mesh): when ``merge_distance`` > 0 or
        ``repair`` is set, the close-vertex merge (``merge_distance`` a fraction of the box diagonal, 0.01 for v_pct = 1; 0 merges
        nothing) with duplicate and zero-area faces removed; when ``min_faces`` > 0 or ``min_diameter`` > 0,
        ``mesh.remove_small_components`` with those thresholds; when ``repair`` is set, the non-manifold edge and vertex repair; when
        ``target_faces`` is set, ``mesh.decimate`` to it (see its note on unreachable targets); when ``remesh_pct`` is set,
        ``mesh.remesh`` with ``remesh_iters`` iterations toward ``remesh_pct`` % of the box diagonal of the mesh at that point
        (decimate_mesh(..., remesh=True), utils/meshutils.py:101-105: PercentageValue(1) is remesh_pct = 1).  As in inference.py:128-129,
        where the remesh belongs to the decimation call, with ``target_faces`` set it runs only when the mesh had more faces than that.
        ``extract_mesh(256, min_faces=8, min_diameter=0.05, target_faces=100000, merge_distance=0.01, repair=True)`` is the geometry of
        extract_texmesh as this package reads clean_mesh (DESIGN.md §1 "clean-up contract"; remeshing is off there).  The defaults run
        marching cubes only.  The primitive noise filter of extract_texmesh (:90-103) is ``noise_filter_mask``; ``extract_texmesh``
        runs it first."""
        R = int(resolution)
        if R < 2:
            raise ValueError(f"resolution must be >= 2, got {resolution}")
        if target_faces is not None and int(target_faces) < 0:
            raise ValueError(f"target_faces must be >= 0, got {target_faces}")
        if not merge_distance >= 0:
            raise ValueError(f"merge_distance must be >= 0, got {merge_distance}")
        grid = self.sdf_grid(R, bound)
        step = 2.0 * bound / (R - 1)
        v, f = mesh._mesh(grid, isovalue, origin=(-bound,) * 3, spacing=(step,) * 3)
        if merge_distance > 0 or repair:
            v, f = mesh._weld(v, f, float(merge_distance))
        if min_faces > 0 or min_diameter > 0:
            v, f = mesh._remove_small(v, f, int(min_faces), float(min_diameter))
        if repair:
            v, f = mesh._repair(v, f)
        if remesh_pct is not None and not (math.isfinite(remesh_pct) and remesh_pct > 0):
            raise ValueError(f"remesh_pct must be finite and > 0, got {remesh_pct}")
        decimated = target_faces is None or f.shape[0] > int(target_faces)
        if target_faces is not None:
            v, f = mesh._decimate(v, f, int(target_faces))
        if remesh_pct is not None and decimated and f.shape[0]:
            d = v.max(0).values.double() - v.min(0).values.double()
            diag = float(torch.sqrt((d * d).sum()))
            v, f = mesh.remesh(v, f, remesh_pct / 100.0 * diag, int(remesh_iters))
        return v, f

    def bake_texture(self, v, f, vt, ft, resolution=1024, pad: int = 32):
        """Texture atlas of the colour / material channels over a UV-unwrapped mesh, on the GPU: inference.py:163-211 in one call
        (rasterise the UV layout, interpolate the 3-D position of every covered texel, query this field there, pad the seams).
        ``v`` [Nv,3] / ``f`` [F,3] are the mesh, ``vt`` [Nt,2] in [0,1] / ``ft`` [F,3] its UV layout (``f`` and ``ft`` index different
        vertex arrays), as inference.py:161-162 hold them after either unwrap branch; ``resolution`` is an int or (h, w).
        Returns (feats fp32 [h,w,6] = 255 * (R, G, B, 0, roughness, metallic), mask bool [h,w] of the covered texels) on the module's
        device; row 0 is v = 0.  feats / 255 at a covered texel is bit-identical to ``forward`` at the position ``bake.interpolate``
        gives for it; ``pad`` = 0 leaves the uncovered texels zero."""
        h, w = (resolution, resolution) if isinstance(resolution, int) else resolution
        h, w = bake._size(h, w)
        bake._check_rows(v, 3, "v")
        bake._check_rows(vt, 2, "vt")
        bake._check_triangles(f, "f")
        bake._check_triangles(ft, "ft")
        if f.shape[0] != ft.shape[0]:
            raise ValueError(f"f and ft must list the same triangles, got {f.shape[0]} and {ft.shape[0]}")
        if not self.srt_param.is_cuda:
            raise _lib.TpxError("PrimSDF query runs on CUDA only (no CPU path): move the module to the GPU")
        lib = _lib.lib()
        dev = self.srt_param.device
        v, vt = v.detach().float().contiguous().to(dev), vt.detach().float().contiguous().to(dev)
        f, ft = bake._narrow(f.to(dev), "f"), bake._narrow(ft.to(dev), "ft")
        srt = self.srt_param.detach().float().contiguous()
        feat = self.feat_param.detach().float().contiguous()
        K = srt.shape[0]
        feats = torch.empty(h, w, 6, dtype=torch.float32, device=dev)
        mask = torch.empty(h, w, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            rast, _ = bake._rasterize(vt, ft, h, w)
            ws = self._grid_workspace(srt, K, dev) if 1 <= K <= 4096 else None
            _lib.check(lib.tpx_primsdf_bake(rast.data_ptr(), h, w, v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], srt.data_ptr(), feat.data_ptr(),
                                            _lib.ptr(ws), 0 if ws is None else ws.numel(), K, self.prim_shape, self.dim_feat, feats.data_ptr(),
                                            mask.data_ptr(), _lib.stream_ptr()), "tpx_primsdf_bake")
            bake.inpaint(feats, mask, pad)
        return feats, mask.view(torch.bool)

    def noise_filter_mask(self) -> torch.Tensor:
        """The primitive noise filter of extract_texmesh (inference.py:90-103) on ``srt_param``: bool [K] on the module's device, True
        for the primitives whose nearest neighbour is closer than the sum of the two scales (``unwrap.noise_filter``)."""
        if not self.srt_param.is_cuda:
            raise _lib.TpxError("the noise filter runs on CUDA only (no CPU path): move the module to the GPU")
        return unwrap.noise_filter(self.srt_param.detach())

    def extract_texmesh(self, resolution: int = 256, target_faces: int = 100000, atlas: int = 1024, island_padding: float = 0.02, min_faces: int = 8,
                        min_diameter: float = 0.05, merge_distance: float = 0.0, repair: bool = False, remesh: bool = False):
        """The fast-unwrap branch of extract_texmesh (inference.py:90-222) on the device, without touching this module's parameters:
        the noise filter, ``extract_mesh(resolution, min_faces=, min_diameter=, target_faces=, merge_distance=, repair=)`` of the kept
        primitives (the reference's clean_mesh is ``extract_texmesh(256, 100000, 1024, 0.02, 8, 0.05, merge_distance=0.01,
        repair=True)``; the defaults leave the close-vertex merge and the repair out; ``remesh=True`` is the "Remesh: Yes" of app.py, 3
        iterations of ``mesh.remesh`` at 1 % of the diagonal after the decimation, run only when the decimation ran), vertex normals,
        the box-projection unwrap, the per-corner re-indexing of :144-148 and ``bake_texture`` at ``atlas`` x ``atlas``.  Returns a dict
        of device tensors in the layout :222 hands to Mesh: ``v`` fp32 [V,3] / ``f`` int64 [F,3] (the indexed mesh), ``vt`` fp32 [3F,2],
        ``ft`` int64 [F,3] (= arange), ``albedo`` and ``metallicRoughness`` fp32 [atlas, atlas, 3] (feats / 255).  The caller's
        ``srt_param[:, 1:4] *= 0.85`` (inference.py:373) is not applied here."""
        keep = self.noise_filter_mask()
        sub = PrimSDF(num_prims=0, dim_feat=self.dim_feat, prim_shape=self.prim_shape, sdf2alpha_var=self.sdf2alpha_var)
        sub.grid_entries = self.grid_entries
        sub.srt_param.data = self.srt_param.detach()[keep].contiguous()
        sub.feat_param.data = self.feat_param.detach()[keep].contiguous()
        sub.train(self.training)
        v, f = sub.extract_mesh(resolution, min_faces=min_faces, min_diameter=min_diameter, target_faces=target_faces, merge_distance=merge_distance,
                                repair=repair, remesh_pct=1.0 if remesh else None)
        if f.shape[0] == 0:
            raise ValueError("the filtered field has no surface at this resolution")
        n = unwrap.compute_vertex_normal(v, f)
        uv, idx = unwrap.box_projection_uv_unwrap(v, n, f, island_padding)
        vt = uv[idx].reshape(-1, 2)
        ft = torch.arange(3 * f.shape[0], device=f.device, dtype=torch.int64).reshape(-1, 3)
        feats, _ = sub.bake_texture(v[f].reshape(-1, 3), ft, vt, ft, atlas)
        return {"v": v, "f": f, "vt": vt, "ft": ft, "albedo": feats[..., :3] / 255, "metallicRoughness": feats[..., 3:] / 255}

    def sdf2alpha(self, sdf):
        return torch.exp(-(sdf / self.sdf2alpha_var) ** 2)


def _column_view(param: str, lo, hi):
    """Read-only views of the two parameters under the reference's attribute names (models/primsdf.py:111-137).  ``lo`` / ``hi``
    are column bounds, or names of the per-instance ``*_start_index`` / ``*_end_index`` attributes."""
    def get(self):
        a = getattr(self, lo) if isinstance(lo, str) else lo
        b = getattr(self, hi) if isinstance(hi, str) else hi
        return getattr(self, param)[:, a:b]
    return property(get)


for _name, _param, _lo, _hi in (("pos", "srt_param", 1, 4), ("scale", "srt_param", 0, 1), ("feat", "feat_param", 0, None),
                                ("feat_geo", "feat_param", "geo_start_index", "geo_end_index"),
                                ("feat_tex", "feat_param", "tex_start_index", "tex_end_index"),
                                ("feat_mat", "feat_param", "mat_start_index", "mat_end_index")):
    setattr(PrimSDF, _name, _column_view(_param, _lo, _hi))
