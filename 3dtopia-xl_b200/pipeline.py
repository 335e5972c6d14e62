"""Sample -> decode pipeline of the reference's inference loop as product code (SURVEY.md §8a a13/a15, §8f-3, config #5).

What ``inference.py:313-349`` / ``app.py:108-140`` do around the hot path, behind one object:

    x_T, y  --DDIM/DDPM loop (DiT.forward_with_cfg + fused update)-->  latents [B, P, 68]
            --a13: / latent_nf * latent_std + latent_mean ; slice 0:4 | 4:68-->  srt [B, P, 4] , z [B*P, 1, 4, 4, 4]
            --VAE.decode-->  voxels [B*P, 6, 8, 8, 8]
            --a15: sdf / 5 ; (rgb, mat + 1) / 2 ; channel-major pack-->  recon_param [B, P, 4 + 3072]   (PrimSDF / ray-marcher layout)

a13 and a15 are one CUDA launch each (``tpx_latent_split`` / ``tpx_primvolume_pack``) whose index layout is bit-exact with the
reference's slicing / reshape / concat and whose arithmetic repeats its eager CUDA ops rounding by rounding.

Progressive previews (§8f-3, inference.py:325-349: decode + render every 10th step): with ``overlap=True`` the decode of step k is
enqueued on a side stream and runs while the main stream already executes DiT step k+1; the preview is handed to the caller one
step later, ordered behind the side stream by an event (no host synchronisation).  The yielded samples are identical either way.

All compute is CUDA through libtpx_b200; there is no CPU path.
"""
from __future__ import annotations

from typing import Dict, Iterator, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .diffusion import create_diffusion

VOX = 8 * 8 * 8


class LatentCodec:
    """a13 / a15 with the checkpoint's normalisation constants (configs/inference_dit.yml:63-65)."""

    def __init__(self, latent_mean: Optional[Sequence[float]] = None, latent_std: Optional[Sequence[float]] = None, latent_nf: float = 1.0):
        if (latent_mean is None) != (latent_std is None):
            raise ValueError("latent_mean and latent_std go together (inference.py:291-295)")
        self.perchannel_norm = latent_mean is not None
        # torch.Tensor(list) -> fp32, exactly what inference.py:292-293 builds
        self._mean = torch.tensor(list(latent_mean), dtype=torch.float32) if self.perchannel_norm else None
        self._std = torch.tensor(list(latent_std), dtype=torch.float32) if self.perchannel_norm else None
        self.latent_nf = float(latent_nf)
        # `tensor / python_float` on CUDA multiplies by the reciprocal rounded to the tensor's dtype
        self._inv_nf = float(np.float32(1.0) / np.float32(self.latent_nf))
        self._dev_consts: Dict[torch.device, tuple] = {}

    def _consts(self, dev):
        c = self._dev_consts.get(dev)
        if c is None:
            c = (self._mean.to(dev), self._std.to(dev)) if self.perchannel_norm else (None, None)
            self._dev_consts[dev] = c
        return c

    def split(self, sample: torch.Tensor):
        """sample [B, P, C] fp32 (the loop's ``samples["sample"]``) -> srt [B, P, 4] fp32, z [B*P, 1, 4, 4, 4] fp32."""
        if sample.dim() != 3 or sample.shape[-1] != 68:
            raise ValueError(f"sample must be [B, P, 68], got {tuple(sample.shape)}")
        if sample.device.type != "cuda":
            raise _lib.TpxError("LatentCodec.split runs on CUDA only (no CPU path)")
        if self.perchannel_norm and self._mean.numel() != sample.shape[-1]:
            raise AssertionError("latent_mean length != in_channels (inference.py:294)")
        B, P, C = sample.shape
        x = sample.to(torch.float32).contiguous()
        srt = torch.empty(B, P, 4, dtype=torch.float32, device=x.device)
        z = torch.empty(B * P, 1, 4, 4, 4, dtype=torch.float32, device=x.device)
        mean, std = self._consts(x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().tpx_latent_split(x.data_ptr(), _lib.ptr(mean), _lib.ptr(std), self._inv_nf, B * P, C, srt.data_ptr(), z.data_ptr(),
                                                   _lib.stream_ptr()), "tpx_latent_split")
        return srt, z

    def pack(self, srt: torch.Tensor, decoded: torch.Tensor) -> torch.Tensor:
        """srt [B, P, 4] fp32 + decoded [B*P, 6, 8, 8, 8] (fp32 or fp16) -> recon_param [B, P, 4 + 6*512] fp32.
        ``recon_param[..., :4]`` is the reference's ``recon_srt_param``, ``recon_param[..., 4:]`` its ``recon_feat_param``."""
        B, P = srt.shape[0], srt.shape[1]
        if decoded.dim() != 5 or decoded.shape[0] != B * P:
            raise ValueError(f"decoded must be [{B * P}, C, S, S, S], got {tuple(decoded.shape)}")
        vox = decoded.shape[2] * decoded.shape[3] * decoded.shape[4]
        F = decoded.shape[1] * vox
        d = decoded.contiguous()
        s = srt.to(torch.float32).contiguous()
        out = torch.empty(B, P, 4 + F, dtype=torch.float32, device=d.device)
        with torch.cuda.device(d.device):
            _lib.check(_lib.lib().tpx_primvolume_pack(s.data_ptr(), d.data_ptr(), _lib.dtype_tag(d), B * P, F, vox, 0 if self.perchannel_norm else 1,
                                                      out.data_ptr(), _lib.stream_ptr()), "tpx_primvolume_pack")
        return out


    # ---- the other direction: PrimX volumes -> latents (building a latent dataset, round-trip checks) ----------------------------
    # The reference ships no encoder-side preprocessing; these are the algebraic inverses of its sampling glue (inference.py:330, :335,
    # :343-346), a convention of this package.  Elementwise torch ops on the inputs' device.
    def unpack(self, recon_param: torch.Tensor):
        """Inverse of ``pack``: recon_param [B, P, 4 + 6*512] -> srt [B, P, 4] fp32, feats [B*P, 6, 8, 8, 8] fp32 with the sdf channel
        times 5 and the other five channels mapped back by x * 2 - 1 (and, without per-channel statistics, srt scale (s - 0.05) * 10)."""
        if recon_param.dim() != 3 or recon_param.shape[-1] != 4 + 6 * VOX:
            raise ValueError(f"recon_param must be [B, P, {4 + 6 * VOX}], got {tuple(recon_param.shape)}")
        B, P = recon_param.shape[:2]
        rp = recon_param.to(torch.float32)
        srt = rp[..., 0:4].clone()
        if not self.perchannel_norm:
            srt[..., 0:1] = (srt[..., 0:1] - 0.05) * 10
        feats = rp[..., 4:].reshape(B * P, 6, 8, 8, 8).clone()
        feats[:, 0:1] *= 5.0
        feats[:, 1:] = feats[:, 1:] * 2.0 - 1.0
        return srt, feats

    def merge(self, srt: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
        """Inverse of ``split``: srt [B, P, 4] + z [B*P, 1, 4, 4, 4] (or [B, P, 64]) -> sample [B, P, 68] fp32 in the DiT's normalised
        latent space: (p - latent_mean) / latent_std * latent_nf with per-channel statistics, else (srt, z * latent_nf)."""
        B, P = srt.shape[:2]
        if z.numel() != B * P * 64:
            raise ValueError(f"z must hold {B * P} latents of 64 values, got {tuple(z.shape)}")
        p = torch.cat([srt.to(torch.float32), z.reshape(B, P, 64).to(torch.float32)], dim=-1)
        if self.perchannel_norm:
            mean, std = (self._mean.to(p.device), self._std.to(p.device))
            return (p - mean) / std * self.latent_nf
        p[..., 4:] = p[..., 4:] * self.latent_nf
        return p


class PrimXPipeline:
    """DDIM/DDPM sampling + VAE decode of image-conditioned PrimX latents (config #2 / #3 / #5 of BASELINE.json).

    model / vae: ``tpxl_b200.DiT`` / ``tpxl_b200.VAE`` (already on the GPU).  ``diffusion_kwargs`` = the ``diffusion:`` block of
    configs/inference_dit.yml without ``timestep_respacing``."""

    def __init__(self, model, vae, diffusion_kwargs: Optional[dict] = None, latent_mean=None, latent_std=None, latent_nf: float = 1.0,
                 num_prims: int = 2048, cfg_scale: float = 6.0, ddim_steps: int = 25, precision: str = "fp16"):
        if precision not in ("fp16", "tf32"):
            raise NotImplementedError("{} precision is not supported".format(precision))     # inference.py:247
        self.model, self.vae = model, vae
        self.codec = LatentCodec(latent_mean, latent_std, latent_nf)
        self.diffusion_kwargs = dict(diffusion_kwargs or dict(noise_schedule="squaredcos_cap_v2", diffusion_steps=1000, parameterization="v"))
        self.diffusion_kwargs.pop("timestep_respacing", None)
        self.num_prims, self.cfg_scale, self.ddim_steps = num_prims, float(cfg_scale), int(ddim_steps)
        self.amp = precision == "fp16"
        self.precision_dtype = torch.float16 if self.amp else torch.float32
        self._side: Dict[torch.device, torch.cuda.Stream] = {}

    # ---- pieces --------------------------------------------------------------------------------------------------
    def make_diffusion(self, steps: Optional[int] = None):
        steps = self.ddim_steps if steps is None else steps
        return create_diffusion(timestep_respacing="ddim{}".format(steps) if steps > 0 else "", **self.diffusion_kwargs)

    def decode_latents(self, sample: torch.Tensor) -> torch.Tensor:
        """inference.py:326-348 for one yielded sample: [B, P, 68] -> recon_param [B, P, 3076].  Samples are decoded one at a time like
        the reference ("one-by-one to avoid oom"); primitives are independent, so the result does not depend on the chunking."""
        srt, z = self.codec.split(sample.reshape(sample.shape[0], self.num_prims, -1))
        P = self.num_prims
        decoded = torch.cat([self.vae.decode(z[b * P:(b + 1) * P]) for b in range(sample.shape[0])], dim=0) if sample.shape[0] > 1 else self.vae.decode(z)
        return self.codec.pack(srt, decoded)

    def encode_primvolume(self, recon_param: torch.Tensor, sample: bool = False) -> torch.Tensor:
        """PrimX volumes -> DiT latents, the inverse of ``decode_latents``: recon_param [B, P, 3076] -> [B, P, 68] (``LatentCodec.unpack``,
        VAE.encode, the posterior's mode or a sample, ``LatentCodec.merge``).  One asset at a time, like decoding."""
        srt, feats = self.codec.unpack(recon_param)
        B, P = srt.shape[:2]
        zs = []
        for b in range(B):
            post = self.vae.encode(feats[b * P:(b + 1) * P])
            zs.append(post.sample() if sample else post.mode())
        return self.codec.merge(srt, torch.cat(zs, dim=0))

    def _model_kwargs(self, y):
        kw = dict(y=y, precision_dtype=self.precision_dtype, enable_amp=self.amp)
        if self.cfg_scale > 0:                       # inference.py:319-320 (app.py:115 uses >= 0)
            kw["cfg_scale"] = self.cfg_scale
        return kw

    # ---- the loop ------------------------------------------------------------------------------------------------
    def sample_progressive(self, y: torch.Tensor, x_T: torch.Tensor, steps: Optional[int] = None, preview_every: int = 10,
                           overlap: bool = True) -> Iterator[dict]:
        """Generator over the previews the reference renders (every ``preview_every``-th step and the last, inference.py:326-328):
        yields ``{"step": sampled_count, "sample": latents, "recon_param": [B, P, 3076], "final": bool}`` in step order.
        ``preview_every <= 0`` decodes the final sample only (app.py)."""
        dev = x_T.device
        if dev.type != "cuda":
            raise _lib.TpxError("PrimXPipeline runs on CUDA only (no CPU path)")
        diffusion = self.make_diffusion(steps)
        sample_fn = diffusion.ddim_sample_loop_progressive if (self.ddim_steps if steps is None else steps) > 0 else diffusion.p_sample_loop_progressive
        fwd = self.model.forward_with_cfg if self.cfg_scale > 0 else self.model.forward
        last = diffusion.num_timesteps - 1
        main = torch.cuda.current_stream(dev)
        side = self._side.get(dev)
        if side is None:
            side = self._side[dev] = torch.cuda.Stream(device=dev)
        pending = None
        with torch.no_grad():
            count = -1
            for samples in sample_fn(fwd, tuple(x_T.shape), x_T, clip_denoised=False, model_kwargs=self._model_kwargs(y), progress=False, device=dev):
                count += 1
                # DiT step `count` and its update are enqueued on the main stream at this point
                if pending is not None:
                    step_k, lat_k, recon_k, done = pending
                    pending = None
                    main.wait_event(done)            # later main-stream work (the caller's renderer, step count+1 ...) runs after the decode
                    recon_k.record_stream(main)
                    yield {"step": step_k, "sample": lat_k, "recon_param": recon_k, "final": False}
                wanted = count == last or (preview_every > 0 and count % preview_every == 0)
                if not wanted:
                    continue
                lat = samples["sample"]
                if overlap and count != last:
                    ready = torch.cuda.Event()
                    ready.record(main)
                    side.wait_event(ready)
                    with torch.cuda.stream(side):
                        recon = self.decode_latents(lat)
                        done = torch.cuda.Event()
                        done.record(side)
                    lat.record_stream(side)
                    pending = (count, lat, recon, done)
                else:
                    yield {"step": count, "sample": lat, "recon_param": self.decode_latents(lat), "final": count == last}

    def __call__(self, y: torch.Tensor, x_T: torch.Tensor, steps: Optional[int] = None) -> Dict[str, torch.Tensor]:
        """app.py:108-140: run the whole loop, decode the final sample.  -> recon_param [B, P, 3076] + the two views the reference
        saves (``srt_param`` [B, P, 4], ``feat_param`` [B, P, 3072])."""
        out = None
        for out in self.sample_progressive(y, x_T, steps=steps, preview_every=0, overlap=False):
            pass
        rp = out["recon_param"]
        return {"sample": out["sample"], "recon_param": rp, "srt_param": rp[..., 0:4], "feat_param": rp[..., 4:]}

    # ---- config #3 / #5: samples sharded over the GPUs of the box -------------------------------------------------
    def generate_sharded(self, y_all: torch.Tensor, num_samples: int, samples_per_forward: int = 1, seed: int = 42, steps: Optional[int] = None,
                         group=None) -> Optional[torch.Tensor]:
        """``num_samples`` image-conditioned generations, sample s on rank s mod G, ``samples_per_forward`` local samples batched
        into one forward (config #5: 4 -> 8 sequences per forward under CFG).  ``y_all`` [num_samples, M, Dc] conditioning tokens
        (host or device).  Noise is drawn on one CPU generator in the reference's order (shard.draw_noise), so results do not
        depend on the number of GPUs.  No collective inside the loops; one all_gather of the packed volumes at the end.
        Returns recon_param [num_samples, P, 3076] on rank 0 (None elsewhere)."""
        from . import shard
        dev = next(self.model.parameters()).device

        def per_batch(indices, x_T):
            y = y_all[indices].to(dev, torch.float32).contiguous()
            return self(y, x_T.to(dev), steps=steps)["recon_param"]

        return shard.run_sharded_batched(num_samples, per_batch, batch=samples_per_forward, seed=seed, num_prims=self.num_prims, channels=68, group=group)
