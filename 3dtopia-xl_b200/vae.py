"""Host-side mirror of the reference's VAE interface, backed by libtpx_b200.

Drop-in for ``models.vae3d_dib.VAE`` (/root/reference/models/vae3d_dib.py:391-453): same constructor kwargs
(configs/inference_dit.yml:31-40), ``load_state_dict(sd['model_state_dict'])`` with the reference key names,
``decode(z[P,1,4,4,4]) -> [P,6,8,8,8]`` in z's dtype, returned as a fresh contiguous tensor (the caller mutates it in place,
inference.py:345-346).  ``encode(x[P,6,8,8,8])`` returns a ``DiagonalGaussianDistribution`` over the quant_conv output
[P,2,4,4,4] and ``forward(x, sample)`` is ``(decode(z), posterior)``; the encoder's tensors (encoder.* / quant_conv.*) are kept
from ``load_state_dict`` and uploaded to a handle of their own on the first ``encode``, so a decode-only user never pays for them.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from .synth import vae_decoder_shapes, vae_encoder_shapes

_ENCODER_PREFIXES = ("encoder.", "quant_conv.")


class DiagonalGaussianDistribution:
    """The posterior of VAE.encode (vae3d_dib.py:50-90), restated: ``parameters`` [B, 2C, ...] splits along dim 1 into the mean and
    the log-variance, which is clamped to [-30, 20]; ``std = exp(logvar / 2)``, ``var = exp(logvar)`` (zeros when deterministic).
    Everything is torch arithmetic on the parameters' device and dtype, so ``sample()`` draws from the same RNG stream, in the same
    shape and dtype, as the reference."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if self.deterministic:
            self.var = self.std = torch.zeros_like(self.mean, device=self.parameters.device, dtype=self.parameters.dtype)

    def sample(self) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, device=self.parameters.device, dtype=self.parameters.dtype)
        return self.mean + self.std * noise

    def kl(self, other: Optional["DiagonalGaussianDistribution"] = None, dims=(1, 2, 3, 4)) -> torch.Tensor:
        """KL divergence to N(0, 1) (or to ``other``), averaged over ``dims``."""
        if self.deterministic:
            return torch.Tensor([0.0])
        dims = list(dims)
        if other is None:
            return 0.5 * torch.mean(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=dims)
        return 0.5 * torch.mean(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0 - self.logvar + other.logvar,
                                dim=dims)

    def nll(self, sample: torch.Tensor, dims=(1, 2, 3, 4)) -> torch.Tensor:
        """Negative log-likelihood of ``sample``, summed over ``dims``."""
        if self.deterministic:
            return torch.Tensor([0.0])
        return 0.5 * torch.sum(math.log(2.0 * math.pi) + self.logvar + torch.pow(sample - self.mean, 2) / self.var, dim=list(dims))

    def mode(self) -> torch.Tensor:
        return self.mean


class VAE(nn.Module):
    def __init__(self, in_channels=1, latent_channels=16, out_channels=1, down_channels=(16, 32, 64, 128, 256), mid_attention=True,
                 up_channels=(256, 128, 64, 32, 16), layers_per_block=2, skip_scale=None, gradient_checkpointing=False):
        super().__init__()
        up_channels = tuple(up_channels)
        if not (latent_channels == 1 and up_channels == (256, 32) and mid_attention and layers_per_block == 2 and skip_scale is None):
            raise NotImplementedError("the H100 decoder kernel set covers the released configuration (configs/inference_dit.yml:31-40): "
                                      f"latent_channels=1, up_channels=[256,32], mid_attention, layers_per_block=2; got latent={latent_channels}, "
                                      f"up={list(up_channels)}, mid_attention={mid_attention}, layers={layers_per_block}")
        self.in_channels, self.latent_channels, self.out_channels = in_channels, latent_channels, out_channels
        self.up_channels = up_channels
        self.down_channels = tuple(down_channels)
        self.mid_attention, self.layers_per_block = mid_attention, layers_per_block
        self._shapes = vae_decoder_shapes(latent_channels=latent_channels, out_channels=out_channels, up_channels=up_channels,
                                          mid_attention=mid_attention, layers_per_block=layers_per_block)
        self._anchor = nn.Parameter(torch.zeros(1), requires_grad=False)
        self._sd: Optional["OrderedDict[str, torch.Tensor]"] = None
        self._extra = OrderedDict()   # encoder.* / quant_conv.* tensors, kept only so state_dict() round-trips
        self._handle: Optional[_lib.Handle] = None
        self._handle_device = None
        self._ws: Optional[_lib.Scratch] = None
        self._enc_handle: Optional[_lib.Handle] = None      # created and filled on the first encode after load_state_dict / .to()
        self._enc_ws: Optional[_lib.Scratch] = None

    def state_dict(self, *args, **kwargs):
        if self._sd is None:
            raise _lib.TpxError("VAE has no parameters yet: load_state_dict first (random initialisation of a decoder is not an inference path)")
        out = OrderedDict(self._extra)
        out.update(self._sd)
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        missing, unexpected = _lib.check_state_dict("VAE", self._shapes, state_dict, strict, _ENCODER_PREFIXES)
        self._sd = OrderedDict((k, state_dict[k].detach()) for k in self._shapes if k in state_dict)
        self._extra = OrderedDict((k, v) for k, v in state_dict.items() if k.startswith(_ENCODER_PREFIXES))
        self._enc_handle = None
        if self._handle is not None:
            self._ingest()
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def load_checkpoint(self, path: str, key: Optional[str] = "model_state_dict", encoder: bool = False):
        """``vae.load_state_dict(torch.load(path, map_location='cpu')['model_state_dict'])`` (inference.py:257-258) from a memory-mapped
        file: only decoder.* / post_quant_conv.* tensors are read and uploaded; the encoder half of the checkpoint is never touched
        unless ``encoder=True``, which also keeps its encoder.* / quant_conv.* tensors for ``encode``."""
        sd = _lib.read_checkpoint(path, key)
        return self.load_state_dict(OrderedDict((k, v) for k, v in sd.items() if encoder or not k.startswith(_ENCODER_PREFIXES)))

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        dev = self._anchor.device
        if dev.type == "cuda" and (self._handle is None or self._handle_device != dev):
            self._create_handle(dev)
        return out

    def _create_handle(self, dev):
        lib = _lib.lib()
        self._handle = self._enc_handle = None     # the old handles are freed before the new one is made
        cfg = _lib.VaeConfig(self.latent_channels, self.out_channels, self.up_channels[0], self.up_channels[1], 8)
        self._handle, self._handle_device = _lib.Handle(lib.tpx_vae_create, lib.tpx_vae_destroy, cfg, dev), dev
        self._ws, self._enc_ws = _lib.Scratch(dev), _lib.Scratch(dev)
        if self._sd is not None:
            self._ingest()

    def _ingest(self):
        lib = _lib.lib()
        _lib.upload(self._handle, lib.tpx_vae_set_weight, lib.tpx_vae_finalize, self._sd.items(), self._handle_device)

    def _latents(self, x: torch.Tensor, what: str) -> torch.Tensor:
        if self._handle is None:
            raise _lib.TpxError("VAE is not on a CUDA device: call .to('cuda') first (this implementation has no CPU path)")
        if self._sd is None:
            raise _lib.TpxError(f"VAE.{what} before load_state_dict")
        if x.dim() != 5 or tuple(x.shape[1:]) != (self.latent_channels, 4, 4, 4):
            raise ValueError(f"z must be [P,{self.latent_channels},4,4,4], got {tuple(x.shape)}")
        z = x.detach().to(self._handle_device)
        if z.dtype not in (torch.float16, torch.float32):
            z = z.float()
        return z.contiguous()

    def _workspace(self, lib, P: int, encoder: bool = False):
        """(256-B aligned address, bytes) of the decode scratch for P primitives, or of the encode scratch with `encoder`."""
        if encoder:
            return self._enc_ws.get(lib.tpx_vae_encoder_workspace_bytes(self._enc_handle, P))
        return self._ws.get(lib.tpx_vae_workspace_bytes(self._handle, P))

    def decode(self, x: torch.Tensor) -> torch.Tensor:
        """VAE.decode (vae3d_dib.py:437-440)."""
        z = self._latents(x, "decode")
        lib = _lib.lib()
        dev = self._handle_device
        P = z.shape[0]
        out = torch.empty(P, self.out_channels, 8, 8, 8, dtype=z.dtype, device=dev)
        if P == 0:
            return out
        with torch.cuda.device(dev):
            base, nbytes = self._workspace(lib, P)
            _lib.check(lib.tpx_vae_decode(self._handle, z.data_ptr(), _lib.dtype_tag(z), out.data_ptr(), _lib.dtype_tag(out), P, base, nbytes,
                                          _lib.stream_ptr()), "tpx_vae_decode")
        return out

    # (S^3, channels) of the activation after each stage of tpx_vae_debug_stage (include/tpx.h)
    STAGE_SHAPES = ((64, 256),) * 6 + ((512, 256),) + ((512, 32),) * 3

    def debug_stage(self, x: torch.Tensor, stage: int) -> torch.Tensor:
        """Channels-last fp16 activation [P, S^3, C] after decoder stage `stage` (0 conv_in ... 9 norm_out + SiLU), computed by
        the same launches decode makes up to that point (parity tests)."""
        if not 0 <= stage < len(self.STAGE_SHAPES):
            raise ValueError(f"stage must be in [0, {len(self.STAGE_SHAPES)}), got {stage}")
        z = self._latents(x, "debug_stage")
        lib = _lib.lib()
        dev = self._handle_device
        P = z.shape[0]
        tap = torch.empty(P, *self.STAGE_SHAPES[stage], dtype=torch.float16, device=dev)
        if P == 0:
            return tap
        with torch.cuda.device(dev):
            base, nbytes = self._workspace(lib, P)
            _lib.check(lib.tpx_vae_debug_stage(self._handle, z.data_ptr(), _lib.dtype_tag(z), P, stage, tap.data_ptr(), base, nbytes,
                                               _lib.stream_ptr()), "tpx_vae_debug_stage")
        return tap

    # ---- encoder -----------------------------------------------------------------------------------------------------
    # (S^3, channels) of the activation after each stage of tpx_vae_encode_debug_stage (include/tpx.h)
    ENC_STAGE_SHAPES = ((512, 32),) * 3 + ((64, 32),) + ((64, 256),) * 6

    def _encoder(self):
        """The encoder handle of the module's device, created and filled from the kept encoder.* / quant_conv.* tensors on first use."""
        if self._enc_handle is not None:
            return self._enc_handle
        shapes = vae_encoder_shapes(in_channels=self.in_channels, latent_channels=self.latent_channels, down_channels=self.down_channels,
                                    mid_attention=self.mid_attention, layers_per_block=self.layers_per_block)
        missing = [k for k in shapes if k not in self._extra]
        wrong = [f"{k} {tuple(self._extra[k].shape)} (expected {tuple(s)})" for k, s in shapes.items()
                 if k in self._extra and tuple(self._extra[k].shape) != tuple(s)]
        if missing or wrong:
            raise RuntimeError("VAE.encode needs the encoder's tensors (load_state_dict with encoder.* / quant_conv.* keys, or "
                               f"load_checkpoint(..., encoder=True)): missing {missing[:8]}{' ...' if len(missing) > 8 else ''}; "
                               f"mis-shaped {wrong[:8]}")
        lib = _lib.lib()
        dev = self._handle_device
        cfg = _lib.VaeConfig(self.latent_channels, self.in_channels, self.down_channels[1], self.down_channels[0], 8)
        h = _lib.Handle(lib.tpx_vae_encoder_create, lib.tpx_vae_encoder_destroy, cfg, dev)
        try:
            _lib.upload(h, lib.tpx_vae_encoder_set_weight, lib.tpx_vae_encoder_finalize, ((k, self._extra[k]) for k in shapes), dev)
        except Exception:
            h.close()
            raise
        self._enc_handle = h
        return h

    def _volumes(self, x: torch.Tensor, what: str):
        if self._handle is None:
            raise NotImplementedError(f"VAE.{what} runs on CUDA only: call .to('cuda') first (this implementation has no CPU path)")
        if self.down_channels != (32, 256) or self.in_channels != 6 or self.latent_channels != 1 or not self.mid_attention \
                or self.layers_per_block != 2:
            raise NotImplementedError("the H100 encoder kernel set covers the released configuration (configs/inference_dit.yml:31-40): "
                                      f"in_channels=6, down_channels=[32,256]; got in={self.in_channels}, down={list(self.down_channels)}")
        if x.dim() != 5 or tuple(x.shape[1:]) != (self.in_channels, 8, 8, 8):
            raise ValueError(f"x must be [P,{self.in_channels},8,8,8], got {tuple(x.shape)}")
        if x.dtype not in (torch.float16, torch.float32):
            raise ValueError(f"x must be fp32 or fp16, got {x.dtype}")
        if x.device != self._handle_device:
            raise ValueError(f"x is on {x.device}, the module on {self._handle_device}")
        return x.detach().contiguous(), self._encoder()

    def encode(self, x: torch.Tensor) -> DiagonalGaussianDistribution:
        """VAE.encode (vae3d_dib.py:431-435): x [P,6,8,8,8] fp32 / fp16 on the module's device -> the posterior over quant_conv(encoder(x))
        [P,2,4,4,4] in x's dtype (computed in fp16 with fp32 accumulation, as under autocast).  Enqueued on the current stream."""
        x, h = self._volumes(x, "encode")
        lib = _lib.lib()
        P = x.shape[0]
        out = torch.empty(P, 2 * self.latent_channels, 4, 4, 4, dtype=x.dtype, device=x.device)
        if P > 0:
            with torch.cuda.device(x.device):
                base, nbytes = self._workspace(lib, P, encoder=True)
                _lib.check(lib.tpx_vae_encode(h, x.data_ptr(), _lib.dtype_tag(x), out.data_ptr(), _lib.dtype_tag(out), P, base, nbytes,
                                              _lib.stream_ptr()), "tpx_vae_encode")
        return DiagonalGaussianDistribution(out)

    def debug_encode_stage(self, x: torch.Tensor, stage: int) -> torch.Tensor:
        """Channels-last fp16 activation [P, S^3, C] after encoder stage `stage` (0 conv_in, 1-2 down_blocks.0 res, 3 downsample, 4-5
        down_blocks.1 res, 6 mid res 0, 7 mid attention, 8 mid res 1, 9 norm_out + SiLU), computed by the same launches encode makes up
        to that point (parity tests)."""
        if not 0 <= stage < len(self.ENC_STAGE_SHAPES):
            raise ValueError(f"stage must be in [0, {len(self.ENC_STAGE_SHAPES)}), got {stage}")
        x, h = self._volumes(x, "debug_encode_stage")
        lib = _lib.lib()
        P = x.shape[0]
        tap = torch.empty(P, *self.ENC_STAGE_SHAPES[stage], dtype=torch.float16, device=x.device)
        if P > 0:
            with torch.cuda.device(x.device):
                base, nbytes = self._workspace(lib, P, encoder=True)
                _lib.check(lib.tpx_vae_encode_debug_stage(h, x.data_ptr(), _lib.dtype_tag(x), P, stage, tap.data_ptr(), base, nbytes,
                                                          _lib.stream_ptr()), "tpx_vae_encode_debug_stage")
        return tap

    def forward(self, x: torch.Tensor, sample: bool = True):
        """VAE.forward (vae3d_dib.py:442-453): (decode(z), posterior) with z = posterior.sample() or posterior.mode()."""
        posterior = self.encode(x)
        z = posterior.sample() if sample else posterior.mode()
        return self.decode(z), posterior
