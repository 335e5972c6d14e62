"""Host-side mirror of the reference's DiT interface, backed by libtpx_b200 (sm_90a kernels).

Drop-in for ``models.dit_crossattn.DiT`` (/root/reference/models/dit_crossattn.py:111-213): same
constructor kwargs (configs/inference_dit.yml:52-62), same ``load_state_dict`` key names, same
``forward`` / ``forward_with_cfg`` signatures, so ``inference.py`` / ``app.py`` and the reference's own
sampler can call it unchanged.  All compute is CUDA; there is no CPU path.

What is different underneath (results stay within the fp16 tolerance of the reference, tests/):
  * parameters live once, as fp16, in a packed store owned by the C library (the reference keeps fp32
    modules and lets autocast re-cast ~905 M weights every forward);
  * cross-attention K/V of all blocks are computed once per conditioning tensor ``y`` and cached
    (the cache holds a strong reference to that tensor and compares identity + version counter), not once per step;
  * under ``forward_with_cfg`` the null-conditioned half of the batch does not run cross-attention at
    all: with an all-equal context the softmax is uniform and the branch equals a per-block constant;
  * the timestep embedding and all 29 adaLN modulation Linears depend only on ``t``: ``set_timesteps`` computes them once for a
    sampling schedule's timesteps (8 per pass over the 669 MB of adaLN weights) and a forward that is told its timestep on the
    host (``t_host=``, what ``SpacedDiffusion``'s loops do) reads the row instead of re-running them — bit-identical results.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict
from typing import Dict, Iterator, Optional, Sequence

import torch
import torch.nn as nn

from . import _lib
from .synth import dit_shapes


class DiT(nn.Module):
    def __init__(self, seq_length=2, in_channels=4, condition_channels=512, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4.0, cond_drop_prob=0.0, attn_proj_bias=False, learn_sigma=True, gradient_checkpointing=False):
        super().__init__()
        self.gradient_checkpointing = gradient_checkpointing
        self.learn_sigma = learn_sigma
        self.in_channels = in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.seq_length = seq_length
        self.num_heads = num_heads
        self.cond_drop_prob = cond_drop_prob
        self.hidden_size = hidden_size
        self.depth = depth
        self.condition_channels = condition_channels
        self.mlp_hidden = int(hidden_size * mlp_ratio)
        self._shapes = dit_shapes(in_channels=in_channels, condition_channels=condition_channels, hidden_size=hidden_size, depth=depth,
                                  mlp_ratio=mlp_ratio, attn_proj_bias=attn_proj_bias, cond_drop_prob=cond_drop_prob, learn_sigma=learn_sigma)
        # one tiny real parameter so `.to(device)`, `next(model.parameters()).device` (gaussian_diffusion.py:669) work
        self._anchor = nn.Parameter(torch.zeros(1), requires_grad=False)
        self._sd: Optional["OrderedDict[str, torch.Tensor]"] = None
        self._handle: Optional[_lib.Handle] = None
        self._handle_device = None
        self._ws: Dict[int, _lib.Scratch] = {}          # one per sequence count: debug_tap reads the one the last forward used
        self._cond_ws: Optional[_lib.Scratch] = None
        self._cond_key = None
        self._resident_only = False                     # True once the host copy was released (release_state_dict / load_checkpoint)
        self._cond_ref: Optional[torch.Tensor] = None   # strong reference to the cached y: its address cannot be recycled while cached
        self._ts_ws: Optional[_lib.Scratch] = None      # timestep table (set_timesteps): modulation rows of a schedule's timesteps
        self._ts_key: Optional[tuple] = None
        self.collapse_null_branch = True     # set False to run the null half through real cross-attention (tests)

    # ---- parameters: reference key names, values kept as given (CPU or GPU, fp16 or fp32) ----------------
    def _default_init(self) -> "OrderedDict[str, torch.Tensor]":
        """Same scheme as DiT.initialize_weights (dit_crossattn.py:158-182): xavier-uniform Linear weights, zero
        biases, N(0, 0.02) timestep MLP, zero adaLN / output layers, N(0,1) null embedding."""
        sd = OrderedDict()
        for k, shp in self._shapes.items():
            if k == "null_cond_embedding":
                sd[k] = torch.randn(shp)
            elif k.endswith(".bias") or "adaLN_modulation" in k or k.startswith("final_layer.linear"):
                sd[k] = torch.zeros(shp)
            elif k.startswith("t_embedder"):
                sd[k] = torch.randn(shp) * 0.02
            else:
                bound = math.sqrt(6.0 / (shp[0] + shp[1]))
                sd[k] = (torch.rand(shp) * 2 - 1) * bound
        return sd

    def state_dict(self, *args, **kwargs):
        if self._sd is None and self._handle is not None and self._resident_only:
            return self._export_all()              # host copy released: read the packed fp16 store back (reference key names / shapes)
        if self._sd is None:
            self._sd = self._default_init()
        return OrderedDict(self._sd)

    # ---- checkpoint ingestion without a retained copy (SURVEY.md §8f-4; inference.py:257-265) ------------------------
    def _export(self, key: str, dtype=torch.float16) -> torch.Tensor:
        t = torch.empty(self._shapes[key], dtype=dtype, device=self._handle_device)
        with torch.cuda.device(self._handle_device):
            _lib.check(_lib.lib().tpx_dit_get_weight(self._handle, key.encode(), t.data_ptr(), _lib.dtype_tag(t), _lib.stream_ptr()), f"get_weight({key})")
        return t

    def _export_all(self) -> "OrderedDict[str, torch.Tensor]":
        return OrderedDict((k, self._export(k)) for k in self._shapes)

    def _param(self, key: str) -> torch.Tensor:
        return self._sd[key] if self._sd is not None else self._export(key, torch.float32)

    def release_state_dict(self) -> None:
        """Drop the host mirror's references to the checkpoint tensors.  The packed fp16 store in the C library (1.8 GB for the shipped
        model) is then the only copy; ``state_dict()`` and ``.to(other_gpu)`` read it back through ``tpx_dit_get_weight``."""
        self._require_handle()
        self._sd, self._resident_only = None, True

    def load_checkpoint(self, path: str, key: Optional[str] = "ema", retain: bool = False):
        """``model.load_state_dict(torch.load(path, map_location='cpu')['ema'])`` (inference.py:260-262) without materialising the
        checkpoint twice: the file is memory-mapped, every tensor goes host -> device -> packed fp16 slot one at a time (fp16
        checkpoints such as model_sview_dit_fp16.pt are copied, never widened to fp32 modules), and with ``retain=False`` nothing but
        the packed store is kept.  The model must already be on its GPU (``.to('cuda')``)."""
        self._require_handle()
        out = self.load_state_dict(_lib.read_checkpoint(path, key))      # validates keys / shapes, ingests tensor by tensor
        if not retain:
            self.release_state_dict()
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        missing, unexpected = _lib.check_state_dict("DiT", self._shapes, state_dict, strict)
        base = self._sd if self._sd is not None else ((self._export_all() if self._resident_only and self._handle is not None else self._default_init()) if missing else OrderedDict())
        sd = OrderedDict()
        for k in self._shapes:
            sd[k] = state_dict[k].detach() if k in state_dict else base[k]
        self._sd, self._resident_only = sd, False
        if self._handle is not None:
            self._ingest()
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        dev = self._anchor.device
        if dev.type == "cuda" and (self._handle is None or self._handle_device != dev):
            self._create_handle(dev)
        return out

    def _create_handle(self, dev: torch.device):
        lib = _lib.lib()
        if self._sd is None and self._resident_only and self._handle is not None:
            self._sd = self._export_all()          # moving a released model to another GPU: carry the packed values over
            torch.cuda.synchronize(self._handle_device)
        self._handle = None                        # the old handle is freed before the new one is made
        cfg = _lib.DitConfig(self.seq_length, self.in_channels, self.out_channels, self.condition_channels, self.hidden_size, self.depth,
                             self.num_heads, self.mlp_hidden)
        self._handle, self._handle_device = _lib.Handle(lib.tpx_dit_create, lib.tpx_dit_destroy, cfg, dev), dev
        self._ws.clear()
        self._cond_ws, self._cond_key, self._cond_ref = _lib.Scratch(dev), None, None
        self._ts_ws, self._ts_key = _lib.Scratch(dev), None
        self._ingest()

    def _ingest(self):
        lib = _lib.lib()
        if self._sd is None:
            self._sd = self._default_init()
        released = self._resident_only
        _lib.upload(self._handle, lib.tpx_dit_set_weight, lib.tpx_dit_finalize, self._sd.items(), self._handle_device)
        self._cond_key, self._cond_ref = None, None
        self._ts_key = None                        # the C library dropped its timestep table with the first set_weight
        if released:                               # re-ingested after a device move of a released model: release again
            self._sd = None

    # ---- forward -------------------------------------------------------------------------------------------
    def _require_handle(self):
        if self._handle is None:
            raise _lib.TpxError("DiT is not on a CUDA device: call .to('cuda') first (this implementation has no CPU path)")

    def _workspace(self, n_seq: int):
        """(aligned address, bytes) of the workspace of n_seq sequences."""
        if n_seq not in self._ws:
            self._ws[n_seq] = _lib.Scratch(self._handle_device)
        return self._ws[n_seq].get(_lib.lib().tpx_dit_workspace_bytes(self._handle, n_seq))

    def _set_cond(self, y: torch.Tensor, with_null: bool):
        """(Re)compute the hoisted cross-attention K/V when the conditioning tensor changed.

        Identity of the cached conditioning = the tensor OBJECT (held alive here, so the caching allocator cannot hand its
        address to a later request's tensor — app.py:108-131 builds a fresh function-local y per request) + its version
        counter (in-place edits) + the view geometry (a different slice of the same storage is a different y)."""
        key = (y.data_ptr(), y._version, tuple(y.shape), tuple(y.stride()), y.dtype, with_null)
        if self._cond_ref is not None and key == self._cond_key and (y is self._cond_ref or y.untyped_storage().data_ptr() == self._cond_ref.untyped_storage().data_ptr()):
            return
        lib = _lib.lib()
        yy = y.detach().to(self._handle_device, torch.float32).contiguous()
        if with_null:
            null = self._param("null_cond_embedding").to(self._handle_device, torch.float32)
            yy = torch.cat([yy, null.expand_as(yy)], dim=0).contiguous()
        n_cross, M = yy.shape[0], yy.shape[1]
        self._cond_key = None                      # the store is rewritten below, and may move
        ws, nbytes = self._cond_ws.get(lib.tpx_dit_cond_bytes(self._handle, n_cross, M))
        _lib.check(lib.tpx_dit_set_cond(self._handle, yy.data_ptr(), n_cross, M, ws, nbytes, _lib.stream_ptr()), "tpx_dit_set_cond")
        self._cond_key, self._cond_ref = key, y

    def set_timesteps(self, timesteps: Sequence[int], force: bool = False) -> None:
        """Hoist TimestepEmbedder + every adaLN_modulation Linear (models/utils.py:27-64, dit_crossattn.py:40-43,54,66-69,75) out of a
        sampling loop: compute the modulation vectors of all of a schedule's ORIGINAL-schedule timesteps (``SpacedDiffusion.timestep_map``)
        once.  A later ``forward(..., t_host=t)`` / ``forward_with_cfg(..., t_host=t)`` with ``t`` among them reads its row; any other call
        computes them per step as before.  Recomputed only when the list changes (or ``force``); reloading weights drops the table."""
        self._require_handle()
        ts = tuple(int(v) for v in timesteps)
        if not ts:
            raise ValueError("set_timesteps: empty timestep list")
        if not force and ts == self._ts_key:
            return
        lib = _lib.lib()
        with torch.cuda.device(self._handle_device):
            nbytes = lib.tpx_dit_timesteps_bytes(self._handle, len(ts))
            if nbytes == 0:
                raise _lib.TpxError(f"set_timesteps: {len(ts)} timesteps is outside what the table holds (1..4096)")
            self._ts_key = None
            ws, nbytes = self._ts_ws.get(nbytes)
            arr = (C.c_int64 * len(ts))(*ts)
            _lib.check(lib.tpx_dit_set_timesteps(self._handle, arr, len(ts), ws, nbytes, _lib.stream_ptr()), "tpx_dit_set_timesteps")
        self._ts_key = ts

    def _prepare(self, x, t, y, use_cfg: int):
        """Validate one call's inputs and bring them to the device; (re)compute the conditioning store.  Returns x, t on the device,
        the sequence count and the workspace (aligned address, bytes)."""
        self._require_handle()
        if x.dim() != 3 or x.shape[1] != self.seq_length or x.shape[2] != self.in_channels:
            raise ValueError(f"x must be [B,{self.seq_length},{self.in_channels}], got {tuple(x.shape)}")
        if y.dim() != 3 or y.shape[0] != x.shape[0] or y.shape[2] != self.condition_channels:
            raise ValueError(f"y must be [B,M,{self.condition_channels}] with B={x.shape[0]}, got {tuple(y.shape)}")
        if not 1 <= x.shape[0] <= 8:
            raise _lib.TpxError(f"batch of {x.shape[0]} samples per forward: the H100 DiT handle runs 1..8 samples (2..16 sequences under CFG) per call; split larger batches")
        if use_cfg and self.cond_drop_prob <= 0:
            raise AttributeError("'DiT' object has no attribute 'null_cond_embedding'")   # as the reference would (dit_crossattn.py:208)
        B = x.shape[0]
        xx = x.detach().to(self._handle_device, torch.float32).contiguous()
        tt = t.detach().to(self._handle_device, torch.int64).contiguous()
        if tt.shape != (B,):
            raise ValueError(f"t must have shape [{B}], got {tuple(tt.shape)}")
        self._set_cond(y, with_null=(use_cfg == 2))
        n_seq = 2 * B if use_cfg else B
        return xx, tt, n_seq, *self._workspace(n_seq)

    def _run(self, x, t, y, use_cfg: int, cfg_scale: float, enable_amp: bool, t_host: Optional[int] = None):
        lib = _lib.lib()
        dev = self._handle_device
        with torch.cuda.device(dev):
            xx, tt, n_seq, ws, nbytes = self._prepare(x, t, y, use_cfg)
            B = xx.shape[0]
            out = torch.empty(B, self.seq_length, self.out_channels, dtype=torch.float16, device=dev)
            if t_host is not None and self._ts_key is not None and int(t_host) in self._ts_key:
                # the caller states (on the host) that every sample of the batch sits at timestep t_host and its modulation row is in the
                # table: no timestep MLP, no adaLN pass, and the device tensor t is not read
                _lib.check(lib.tpx_dit_forward_step(self._handle, xx.data_ptr(), int(t_host), B, use_cfg, float(cfg_scale), out.data_ptr(),
                                                    ws, nbytes, _lib.stream_ptr()), "tpx_dit_forward_step")
            else:
                _lib.check(lib.tpx_dit_forward(self._handle, xx.data_ptr(), tt.data_ptr(), B, use_cfg, float(cfg_scale), out.data_ptr(), ws,
                                               nbytes, _lib.stream_ptr()), "tpx_dit_forward")
        # the reference returns fp16 under autocast and fp32 otherwise (dit_crossattn.py:197-202)
        return out if enable_amp else out.float()

    def forward(self, x, t, y, precision_dtype=torch.float32, enable_amp=False, t_host: Optional[int] = None):
        """DiT.forward (dit_crossattn.py:184-202).  ``t_host`` (not a reference argument, optional): the caller's promise that every
        entry of ``t`` equals this Python int — lets the call use the table of ``set_timesteps`` (see there); results do not change.

        PRECISION: the kernels implement ONE contract, the reference's CUDA autocast(fp16) path (what inference.py / app.py run:
        ``precision: fp16`` + ``amp``).  ``enable_amp=False`` or ``precision_dtype != float16`` does NOT select an fp32 (or bf16)
        computation here: the same fp16-contract result is returned, cast to fp32 when amp is off, and a warning says so once."""
        self._precision_notice(precision_dtype, enable_amp)
        return self._run(x, t, y, 0, 0.0, enable_amp, t_host)

    _warned_precision = False

    def _precision_notice(self, precision_dtype, enable_amp):
        if (not enable_amp or precision_dtype not in (torch.float16, None)) and not DiT._warned_precision:
            DiT._warned_precision = True
            import warnings
            warnings.warn("tpxl_b200.DiT computes in the reference's fp16-autocast contract regardless of precision_dtype/enable_amp "
                          f"(got precision_dtype={precision_dtype}, enable_amp={enable_amp}); the output is fp16-accurate, returned as "
                          f"{'fp16' if enable_amp else 'fp32'}", stacklevel=3)

    def forward_with_cfg(self, x, t, y, cfg_scale=0.0, precision_dtype=torch.float32, enable_amp=False, t_host: Optional[int] = None):
        """DiT.forward_with_cfg (dit_crossattn.py:204-213).  Precision and ``t_host``: see forward()."""
        self._precision_notice(precision_dtype, enable_amp)
        return self._run(x, t, y, 1 if self.collapse_null_branch else 2, cfg_scale, enable_amp, t_host)

    # stop points of tpx_dit_debug_stage and buffers of tpx_dit_debug_tap (include/tpx.h)
    STAGES = {"embed": 0, "cross": 1, "self": 2, "mlp": 3}
    TAPS = {"residual": 0, "ao": 1, "mod": 2, "pre_cfg": 3}

    def debug_stage(self, x, t, y, stage: str, block: int = 0, use_cfg: int = 0) -> torch.Tensor:
        """Run the forward's schedule (use_cfg 0: forward; 1: forward_with_cfg; 2: forward_with_cfg with real cross-attention over the
        null context) up to `stage` ("embed", or "cross" / "self" / "mlp" of block `block`) with the same launches, and return the fp32
        residual stream [n_seq, N, D] there (parity tests).  The workspace's other buffers stay readable through debug_tap."""
        if stage not in self.STAGES:
            raise ValueError(f"stage must be one of {list(self.STAGES)}, got {stage!r}")
        lib = _lib.lib()
        with torch.cuda.device(self._handle_device):
            xx, tt, n_seq, ws, nbytes = self._prepare(x, t, y, use_cfg)
            _lib.check(lib.tpx_dit_debug_stage(self._handle, xx.data_ptr(), tt.data_ptr(), xx.shape[0], use_cfg, block, self.STAGES[stage], ws, nbytes,
                                               _lib.stream_ptr()), "tpx_dit_debug_stage")
        return self.debug_tap(n_seq, "residual")

    def debug_tap(self, n_seq: int, which: str, count: Optional[int] = None) -> torch.Tensor:
        """The leading `count` (default n_seq) sequences, or samples for "mod", of one buffer of the workspace of n_seq sequences, as the
        last forward or debug_stage left it: "residual" fp32 [count, N, D], "ao" fp16 [count, N, D], "mod" fp16 [count, Ltot],
        "pre_cfg" fp16 [count, N, out_channels] (tpx_dit_debug_tap)."""
        self._require_handle()
        count = n_seq if count is None else count
        N, D = self.seq_length, self.hidden_size
        shape, dtype = {"residual": ((count, N, D), torch.float32), "ao": ((count, N, D), torch.float16),
                        "mod": ((count, self.depth * 9 * D + 2 * D), torch.float16),
                        "pre_cfg": ((count, N, self.out_channels), torch.float16)}[which]
        out = torch.empty(shape, dtype=dtype, device=self._handle_device)
        with torch.cuda.device(self._handle_device):
            _lib.check(_lib.lib().tpx_dit_debug_tap(self._handle, self._workspace(n_seq)[0], n_seq, self.TAPS[which], count, out.data_ptr(),
                                                    _lib.stream_ptr()), "tpx_dit_debug_tap")
        return out

    def debug_timestep_table(self) -> torch.Tensor:
        """The modulation rows [K, Ltot] fp16 that set_timesteps computed, one per timestep in its order (a view of the table)."""
        if self._ts_key is None:
            raise _lib.TpxError("debug_timestep_table: no timestep table (call set_timesteps)")
        ws = self._ts_ws
        off = ws.addr - ws.buf.data_ptr()                                # the table opens the store (tpx_dit_set_timesteps)
        K, Ltot = len(self._ts_key), self.depth * 9 * self.hidden_size + 2 * self.hidden_size
        return ws.buf[off:off + K * Ltot * 2].view(torch.float16).view(K, Ltot)

    def debug_residual(self, n_seq: int) -> torch.Tensor:
        """fp32 residual stream [n_seq, N, D] left by the last forward (parity tests)."""
        return self.debug_tap(n_seq, "residual")
