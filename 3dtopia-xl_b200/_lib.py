"""ctypes binding of libtpx_b200.so (include/tpx.h).  No fallback: if the library or an H100 is missing the
product path raises."""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtpx_b200.so")
_lock = threading.Lock()
_lib = None

DTYPE_F32, DTYPE_F16 = 0, 1
LAYOUT_NCDHW, LAYOUT_CHLAST = 0, 1          # tpx_colored_boxes
PAYLOAD_RGB, PAYLOAD_MAT = 0, 1            # tpx_primvolume_payload
_vp, _i, _f, _sz, _i64 = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_int64


class DitConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("seq_length", "in_channels", "out_channels", "condition_channels", "hidden_size", "depth",
                                         "num_heads", "mlp_hidden")]


class VaeConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("latent_channels", "out_channels", "ch_mid", "ch_out", "attn_heads")]


class SamplerCoefs(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("sqrt_ab", "sqrt_1mab", "sqrt_recip_ab", "sqrt_recipm1_ab", "c_x0", "c_eps", "sigma", "nonzero",
                                         "coef1", "coef2", "min_log", "max_log")] + [("clip", C.c_int32)]


# name -> (restype, argtypes); mirrors include/tpx.h one to one and in its order (tests/test_abi.py checks every type)
SIGNATURES = {
    "tpx_version": (_i, []),
    "tpx_last_error": (C.c_char_p, []),
    "tpx_device_check": (_i, []),
    "tpx_launch_count": (_i64, []),
    "tpx_profile_begin": (_i, []),
    "tpx_profile_end": (_i, [C.POINTER(C.c_float), C.POINTER(_i64)]),
    "tpx_dit_create": (_i, [C.POINTER(DitConfig), C.POINTER(_vp)]),
    "tpx_dit_destroy": (None, [_vp]),
    "tpx_dit_set_weight": (_i, [_vp, C.c_char_p, _vp, _i, C.POINTER(_i64), _i, _vp]),
    "tpx_dit_get_weight": (_i, [_vp, C.c_char_p, _vp, _i, _vp]),
    "tpx_dit_finalize": (_i, [_vp, _vp]),
    "tpx_dit_cond_bytes": (_sz, [_vp, _i, _i]),
    "tpx_dit_workspace_bytes": (_sz, [_vp, _i]),
    "tpx_dit_set_cond": (_i, [_vp, _vp, _i, _i, _vp, _sz, _vp]),
    "tpx_dit_forward": (_i, [_vp, _vp, _vp, _i, _i, _f, _vp, _vp, _sz, _vp]),
    "tpx_dit_timesteps_bytes": (_sz, [_vp, _i]),
    "tpx_dit_set_timesteps": (_i, [_vp, C.POINTER(_i64), _i, _vp, _sz, _vp]),
    "tpx_dit_forward_step": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _vp, _sz, _vp]),
    "tpx_dit_debug_stage": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _sz, _vp]),
    "tpx_dit_debug_tap": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "tpx_sampler_step": (_i, [_i, _vp, _vp, _i, _vp, _i64, _i, C.POINTER(SamplerCoefs), _vp, _vp, _vp]),
    "tpx_latent_split": (_i, [_vp, _vp, _vp, _f, _i64, _i, _vp, _vp, _vp]),
    "tpx_primvolume_pack": (_i, [_vp, _vp, _i, _i64, _i, _i, _i, _vp, _vp]),
    "tpx_vae_create": (_i, [C.POINTER(VaeConfig), C.POINTER(_vp)]),
    "tpx_vae_destroy": (None, [_vp]),
    "tpx_vae_set_weight": (_i, [_vp, C.c_char_p, _vp, _i, C.POINTER(_i64), _i, _vp]),
    "tpx_vae_finalize": (_i, [_vp, _vp]),
    "tpx_vae_workspace_bytes": (_sz, [_vp, _i]),
    "tpx_vae_decode": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _sz, _vp]),
    "tpx_vae_debug_stage": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "tpx_vae_encoder_create": (_i, [C.POINTER(VaeConfig), C.POINTER(_vp)]),
    "tpx_vae_encoder_destroy": (None, [_vp]),
    "tpx_vae_encoder_set_weight": (_i, [_vp, C.c_char_p, _vp, _i, C.POINTER(_i64), _i, _vp]),
    "tpx_vae_encoder_finalize": (_i, [_vp, _vp]),
    "tpx_vae_encoder_workspace_bytes": (_sz, [_vp, _i]),
    "tpx_vae_encode": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _sz, _vp]),
    "tpx_vae_encode_debug_stage": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "tpx_linear": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "tpx_linear_gated": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _vp]),
    "tpx_linear_heads": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i, _vp]),
    "tpx_ln_modulate": (_i, [_vp, _i, _i, _f, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "tpx_attention": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "tpx_attention_tc": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _vp]),
    "tpx_cfg_combine": (_i, [_vp, _i64, _f, _vp, _vp]),
    "tpx_groupnorm_silu": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp, _vp]),
    "tpx_conv3d_k3": (_i, [_vp, _vp, _vp, _vp, _f, _vp, _i, _i, _i, _i, _vp]),
    "tpx_primsdf_query": (_i, [_vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp, _vp]),
    "tpx_primsdf_grid_bytes": (_sz, [_i64]),
    "tpx_primsdf_grid_build": (_i, [_vp, _i, _vp, _sz, _vp]),
    "tpx_primsdf_query_grid": (_i, [_vp, _vp, _vp, _vp, _sz, _i64, _i, _i, _i, _i, _vp, _vp]),
    "tpx_primsdf_query_backward": (_i, [_vp, _vp, _vp, _vp, _sz, _i64, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "tpx_primsdf_sdf_grid": (_i, [_vp, _i, _vp, _vp, _vp, _sz, _i, _i, _i, _i, _vp, _vp]),
    "tpx_raymarch_preview": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _f, _f, _vp, _vp]),
    "tpx_raymarch_forward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _f, _f, _i, _vp, _vp, _vp, _vp]),
    "tpx_raymarch_backward": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _f, _f, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                   _vp]),
    "tpx_raymarch_preview_views": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _f, _f, _f, _f, _vp, _vp]),
    "tpx_colored_boxes": (_i, [_vp, _i, _i, _i, _f, _i, _vp, _vp]),
    "tpx_primvolume_payload": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "tpx_mc_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "tpx_mc_count": (_i, [_vp, _i64, _i64, _i64, _f, _vp, _sz, _vp, _vp]),
    "tpx_mc_emit": (_i, [_vp, _i64, _i64, _i64, _f, _f, _f, _f, _f, _f, _f, _vp, _sz, _vp, _vp, _vp]),
    "tpx_mesh_components_workspace_bytes": (_sz, [_i64, _i64]),
    "tpx_mesh_components_count": (_i, [_vp, _i64, _vp, _i64, _i64, C.c_double, _vp, _sz, _vp, _vp]),
    "tpx_mesh_components_emit": (_i, [_vp, _i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "tpx_decimate_workspace_bytes": (_sz, [_i64, _i64]),
    "tpx_decimate": (_i, [_vp, _i64, _vp, _i64, _i64, _vp, _sz, _vp, _vp, _i64, _vp]),
    "tpx_decimate_emit": (_i, [_i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "tpx_mesh_weld_workspace_bytes": (_sz, [_i64, _i64]),
    "tpx_mesh_weld_count": (_i, [_vp, _i64, _vp, _i64, C.c_double, _vp, _sz, _vp, _vp]),
    "tpx_mesh_weld_emit": (_i, [_vp, _i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "tpx_mesh_repair_workspace_bytes": (_sz, [_i64, _i64]),
    "tpx_mesh_repair_count": (_i, [_vp, _i64, _vp, _i64, _vp, _sz, _vp, _vp]),
    "tpx_mesh_repair_emit": (_i, [_vp, _i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "tpx_remesh_workspace_bytes": (_sz, [_i64, _i64]),
    "tpx_remesh_grid_bytes": (_sz, [_i64]),
    "tpx_remesh_begin": (_i, [_vp, _i64, _vp, _i64, C.c_double, _vp, _sz, _vp, _sz, _vp, _vp, _vp]),
    "tpx_remesh_closest": (_i, [_vp, _i64, _vp, _i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "tpx_remesh_split_count": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, C.c_double, _vp, _sz, _vp, _vp]),
    "tpx_remesh_split_emit": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _sz, _vp, _vp, _vp, _vp]),
    "tpx_remesh_relax": (_i, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i64, _vp, _sz, C.c_double, C.c_double, _vp, _sz, _vp, _vp]),
    "tpx_uv_unwrap_workspace_bytes": (_sz, [_i64, _i64]),
    "tpx_vertex_normals": (_i, [_vp, _i64, _vp, _i64, _vp, _sz, _vp, _vp]),
    "tpx_uv_unwrap": (_i, [_vp, _vp, _i64, _vp, _i64, C.c_double, _vp, _sz, _vp, _vp, _vp]),
    "tpx_uv_unwrap_emit": (_i, [_i64, _i64, _vp, _sz, _vp, _vp, _vp]),
    "tpx_prim_noise_filter": (_i, [_vp, _i, _vp, _vp, _vp]),
    "tpx_uv_rasterize": (_i, [_vp, _i64, _vp, _i64, _i, _i, _vp, _vp, _vp]),
    "tpx_rast_interpolate": (_i, [_vp, _i64, _i, _vp, _i64, _vp, _i, _i, _vp, _vp]),
    "tpx_primsdf_bake": (_i, [_vp, _i, _i, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _sz, _i, _i, _i, _vp, _vp, _vp]),
    "tpx_texture_inpaint_bytes": (_sz, [_i, _i]),
    "tpx_texture_inpaint": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _sz, _vp, _vp]),
    "tpx_gelu_erf": (_i, [_vp, _i64, _vp]),
}


class TpxError(RuntimeError):
    pass


def load_library(path: str | None = None) -> C.CDLL:
    """dlopen the library and bind every prototype.  Works without a GPU (no compute is issued)."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        override = os.environ.get("TPX_LIB_PATH")       # tuning aid: A/B an older build of the library (symbols it lacks are skipped)
        p = path or override or LIB_PATH
        if not os.path.exists(p):
            raise TpxError(f"{p} not found: build it with `python 3dtopia-xl_b200/build.py` (there is no fallback path)")
        lib = C.CDLL(p)
        for name, (res, args) in SIGNATURES.items():
            if override and not path and not hasattr(lib, name):
                continue
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
        return lib


def lib() -> C.CDLL:
    """Library for the compute path: requires CUDA and an sm_90 device."""
    if not torch.cuda.is_available():
        raise TpxError("3dtopia-xl_b200 needs a CUDA device (sm_90a); no CPU fallback exists")
    return load_library()


def check(rc: int, what: str = "") -> int:
    if rc < 0:
        msg = load_library().tpx_last_error()
        raise TpxError(f"{what or 'libtpx_b200'} failed ({rc}): {msg.decode() if msg else ''}")
    return rc


def ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def dtype_tag(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return DTYPE_F32
    if t.dtype == torch.float16:
        return DTYPE_F16
    raise TpxError(f"unsupported tensor dtype {t.dtype} (fp32 / fp16 only)")


class Handle:
    """Owner of one C handle, made by ``create(&cfg, &h)`` on `dev`.  ``ptr`` is what the C entries take, and ctypes passes the owner
    itself as ``ptr`` (NULL once closed).  ``close()`` runs the given `destroy` at most once and never raises; dropping the owner closes
    it, also at interpreter shutdown (nothing is looked up then)."""

    def __init__(self, create, destroy, cfg, dev: torch.device):
        self.ptr, self._destroy = None, destroy
        h = C.c_void_p()
        with torch.cuda.device(dev):
            check(create(C.byref(cfg), C.byref(h)), create.__name__)
        self.ptr = h

    def close(self) -> None:
        h, self.ptr = self.ptr, None
        if h is not None:
            try:
                self._destroy(h)
            except Exception:
                pass

    __del__ = close

    @property
    def _as_parameter_(self):
        return self.ptr


class Scratch:
    """A device byte buffer that only grows: ``get(nbytes)`` returns (256-B aligned address, nbytes) inside it."""

    def __init__(self, dev: torch.device):
        self.dev, self.buf, self.addr = dev, None, 0

    def get(self, nbytes: int) -> tuple[int, int]:
        if self.buf is None or self.buf.numel() < nbytes + 256:
            self.buf = None                     # the old buffer goes back to the allocator before the larger one is taken
            self.buf = torch.empty(nbytes + 256, dtype=torch.uint8, device=self.dev)
            self.addr = (self.buf.data_ptr() + 255) & ~255
        return self.addr, nbytes


def check_state_dict(owner: str, shapes, state_dict, strict: bool, ignore_prefixes=()) -> tuple[list, list]:
    """The key and shape checks of nn.Module.load_state_dict against a (key -> shape) table: returns (missing, unexpected) and raises
    torch's RuntimeError on a size mismatch, or on missing / unexpected keys when `strict`.  Keys under `ignore_prefixes` are never
    unexpected."""
    missing = [k for k in shapes if k not in state_dict]
    unexpected = [k for k in state_dict if k not in shapes and not k.startswith(ignore_prefixes)]
    errs = [f"size mismatch for {k}: copying a param with shape {tuple(state_dict[k].shape)}, expected {tuple(s)}"
            for k, s in shapes.items() if k in state_dict and tuple(state_dict[k].shape) != tuple(s)]
    if strict and (missing or unexpected):
        errs.append(f"Missing key(s): {missing[:5]}{'...' if len(missing) > 5 else ''}; unexpected key(s): {unexpected[:5]}")
    if errs:
        raise RuntimeError(f"Error(s) in loading state_dict for {owner}:\n\t" + "\n\t".join(errs))
    return missing, unexpected


def read_checkpoint(path: str, key: str | None):
    """``torch.load(path, map_location='cpu')[key]`` (the whole file when `key` is None), memory-mapped so that a tensor is read only
    when it is used."""
    try:
        ck = torch.load(path, map_location="cpu", mmap=True, weights_only=True)
    except (RuntimeError, ValueError, TypeError):      # legacy (non-zipfile) serialisation cannot be memory-mapped
        ck = torch.load(path, map_location="cpu", weights_only=True)
    return ck[key] if key is not None else ck


def upload(handle, set_weight, finalize, tensors, dev: torch.device) -> None:
    """Load (key, tensor) pairs into a parameter handle on `dev` through its tpx_*_set_weight and tpx_*_finalize.  Each tensor is
    staged as a contiguous fp16 / fp32 copy on the device; the stream is synchronised before the staged copies are dropped, since
    the repack kernels read them."""
    with torch.cuda.device(dev):
        st = stream_ptr()
        keep = []
        for k, v in tensors:
            t = v.detach()
            if t.dtype not in (torch.float16, torch.float32):
                t = t.float()
            t = t.to(dev, non_blocking=True).contiguous()
            keep.append(t)
            shape = (C.c_int64 * t.dim())(*t.shape)
            check(set_weight(handle, k.encode(), t.data_ptr(), dtype_tag(t), shape, t.dim(), st), f"{set_weight.__name__}({k})")
        check(finalize(handle, st), finalize.__name__)
        torch.cuda.current_stream().synchronize()
