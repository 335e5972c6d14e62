"""Oracle restatement of the cross-attention DiT (TEST INFRASTRUCTURE — see oracle/__init__.py).

Restates, as pure functions over a reference-keyed ``state_dict``:
  * DiT.forward            /root/reference/models/dit_crossattn.py:184-202
  * DiT.forward_with_cfg   /root/reference/models/dit_crossattn.py:204-213
  * DiTBlock._forward      /root/reference/models/dit_crossattn.py:51-58
  * FinalLayer.forward     /root/reference/models/dit_crossattn.py:74-78
  * MemEffCrossAttention   /root/reference/models/attention.py:96-114   (q pre-scaled by Dh^-1/2 AND the
                           attention core scales by Dh^-1/2 again => logits are q.k/Dh)
  * MemEffAttention        /root/reference/models/attention.py:48-59
  * TimestepEmbedder       /root/reference/models/utils.py:41-64  (cos first, then sin)
  * Mlp (GELU-tanh)        /root/reference/models/utils.py:94-101
  * modulate               /root/reference/models/utils.py:19-20
  * xformers.ops.memory_efficient_attention (third-party, un-vendored, unpinned; README.md:67):
    restated from its published contract softmax(Q K^T * Dh^-1/2) V on [B,N,H,Dh] tensors, fp32 softmax.

Two precision policies:
  ``fp32``  every op in fp32 — what the reference computes on a CPU (autocast('cuda') is inert there).
  ``fp16``  emulates the reference's CUDA autocast(fp16) contract (SURVEY.md §8a "precision contract")
            by rounding to fp16 at exactly the points autocast does, with fp32 accumulation inside
            each Linear / attention.  Runs on any device.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def r16(x: Tensor) -> Tensor:
    """Round to fp16 and come back: fp64 stays fp64 (so the policies can run in fp64 with fp16 rounding points), anything else
    comes back as fp32."""
    return x.to(torch.float16).to(torch.float64 if x.dtype == torch.float64 else torch.float32)


class Policy:
    def __init__(self, name: str = "fp32"):
        assert name in ("fp32", "fp16")
        self.amp = name == "fp16"

    # nn.Linear under autocast: input, weight, bias cast to fp16, fp32 accumulate, one rounding of the result.
    def linear(self, x: Tensor, w: Tensor, b: Tensor | None) -> Tensor:
        if not self.amp:
            return F.linear(x, w, b)
        y = F.linear(r16(x), r16(w), None if b is None else r16(b))
        return r16(y)

    def rnd(self, x: Tensor) -> Tensor:
        return r16(x) if self.amp else x


def timestep_embedding(t: Tensor, dim: int = 256, max_period: float = 10000.0, dtype: torch.dtype = torch.float32) -> Tensor:
    """models/utils.py:41-59.  The reference evaluates the sinusoid in fp32; dtype=torch.float64 gives the exact one."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=dtype) / half).to(t.device)
    args = t[:, None].to(dtype) * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def t_embedder(sd: Dict[str, Tensor], t: Tensor, dtype: torch.dtype = torch.float32) -> Tensor:
    """models/utils.py:61-64 — always fp32 (outside the autocast region, dit_crossattn.py:192); the sinusoid in `dtype`, cast to the
    weights' dtype."""
    w0 = sd["t_embedder.mlp.0.weight"]
    h = F.linear(timestep_embedding(t, dtype=dtype).to(w0.dtype), w0, sd["t_embedder.mlp.0.bias"])
    h = F.silu(h)
    return F.linear(h, sd["t_embedder.mlp.2.weight"], sd["t_embedder.mlp.2.bias"])


def attention_core(q: Tensor, k: Tensor, v: Tensor, pol: Policy) -> Tensor:
    """xformers memory_efficient_attention contract: q,k,v [B,N,H,Dh] -> [B,N,H,Dh]; scale Dh^-1/2."""
    scale = q.shape[-1] ** -0.5
    qh, kh, vh = (pol.rnd(a).permute(0, 2, 1, 3) for a in (q, k, v))
    if not pol.amp and q.device.type == "cpu" and q.shape[1] * k.shape[1] > (1 << 20):
        # same fp32 math through torch's fused CPU kernel (no [B,H,N,M] score tensor): keeps the CPU baseline honest
        return F.scaled_dot_product_attention(qh, kh, vh, scale=scale).permute(0, 2, 1, 3)
    s = torch.matmul(qh, kh.transpose(-1, -2)) * scale
    p = torch.softmax(s, dim=-1)
    o = torch.matmul(p, vh)
    return pol.rnd(o.permute(0, 2, 1, 3))


def modulate(x: Tensor, shift: Tensor, scale: Tensor, pol: Policy) -> Tensor:
    """models/utils.py:19-20.  Under autocast shift/scale are fp16, so (1 + scale) is an fp16 op."""
    return x * pol.rnd(1 + scale).unsqueeze(1) + shift.unsqueeze(1)


def layer_norm(x: Tensor) -> Tensor:
    """nn.LayerNorm(elementwise_affine=False, eps=1e-6) (dit_crossattn.py:32) — fp32 under autocast."""
    return F.layer_norm(x, (x.shape[-1],), eps=1e-6)


def cross_attention(sd, pre: str, x: Tensor, y: Tensor, H: int, pol: Policy, taps: dict | None = None) -> Tensor:
    """models/attention.py:96-114.  taps (optional): receives "ao", the attention core's output [B,N,D] before proj."""
    B, N, D = x.shape
    M = y.shape[1]
    Dh = D // H
    q = pol.linear(x, sd[pre + "to_q.weight"], sd.get(pre + "to_q.bias"))
    q = pol.rnd((Dh ** -0.5) * q).reshape(B, N, H, Dh)
    k = pol.linear(y, sd[pre + "to_k.weight"], sd.get(pre + "to_k.bias")).reshape(B, M, H, Dh)
    v = pol.linear(y, sd[pre + "to_v.weight"], sd.get(pre + "to_v.bias")).reshape(B, M, H, Dh)
    o = attention_core(q, k, v, pol).reshape(B, N, D)
    if taps is not None:
        taps["ao"] = o
    return pol.linear(o, sd[pre + "proj.weight"], sd.get(pre + "proj.bias"))


def self_attention(sd, pre: str, x: Tensor, H: int, pol: Policy, taps: dict | None = None) -> Tensor:
    """models/attention.py:48-59.  taps: as for cross_attention."""
    B, N, D = x.shape
    qkv = pol.linear(x, sd[pre + "qkv.weight"], sd.get(pre + "qkv.bias")).reshape(B, N, 3, H, D // H)
    q, k, v = torch.unbind(qkv, 2)
    o = attention_core(q, k, v, pol).reshape(B, N, D)
    if taps is not None:
        taps["ao"] = o
    return pol.linear(o, sd[pre + "proj.weight"], sd.get(pre + "proj.bias"))


def mlp(sd, pre: str, x: Tensor, pol: Policy) -> Tensor:
    """models/utils.py:94-101 with nn.GELU(approximate='tanh') (dit_crossattn.py:38)."""
    h = pol.linear(x, sd[pre + "fc1.weight"], sd[pre + "fc1.bias"])
    h = pol.rnd(F.gelu(h, approximate="tanh"))
    return pol.linear(h, sd[pre + "fc2.weight"], sd[pre + "fc2.bias"])


def block_modulation(sd, i: int, t_emb: Tensor, pol: Policy):
    """The 9 adaLN chunks of block i (dit_crossattn.py:54): (shift, scale, gate) x (mca, msa, mlp), each [B, D]."""
    p = f"blocks.{i}."
    mod = pol.linear(F.silu(t_emb), sd[p + "adaLN_modulation.1.weight"], sd[p + "adaLN_modulation.1.bias"])
    return mod.chunk(9, dim=1)


# The three branches of DiTBlock._forward (dit_crossattn.py:55-57).  Each returns its increment, the gated amount it adds to the
# residual stream x; mod_chunks are the block's 9 chunks.  They compute in the dtype of x and sd (fp64 for the stage tests).
def cross_branch(sd, i: int, x: Tensor, y: Tensor, mod_chunks, H: int, pol: Policy, taps: dict | None = None) -> Tensor:
    sh, sc, g = mod_chunks[0:3]
    return pol.rnd(g.unsqueeze(1) * cross_attention(sd, f"blocks.{i}.crossattn.", modulate(layer_norm(x), sh, sc, pol), y, H, pol, taps))


def self_branch(sd, i: int, x: Tensor, mod_chunks, H: int, pol: Policy, taps: dict | None = None) -> Tensor:
    sh, sc, g = mod_chunks[3:6]
    return pol.rnd(g.unsqueeze(1) * self_attention(sd, f"blocks.{i}.attn.", modulate(layer_norm(x), sh, sc, pol), H, pol, taps))


def mlp_branch(sd, i: int, x: Tensor, mod_chunks, pol: Policy) -> Tensor:
    sh, sc, g = mod_chunks[6:9]
    return pol.rnd(g.unsqueeze(1) * mlp(sd, f"blocks.{i}.mlp.", modulate(layer_norm(x), sh, sc, pol), pol))


def dit_block(sd, i: int, x: Tensor, y: Tensor, t_emb: Tensor, H: int, pol: Policy) -> Tensor:
    """models/dit_crossattn.py:51-58 — order is cross-attn, self-attn, MLP."""
    m = block_modulation(sd, i, t_emb, pol)
    x = x + cross_branch(sd, i, x, y, m, H, pol)
    x = x + self_branch(sd, i, x, m, H, pol)
    x = x + mlp_branch(sd, i, x, m, pol)
    return x


def final_modulation(sd, t_emb: Tensor, pol: Policy):
    """(shift, scale) of the final layer (dit_crossattn.py:75), each [B, D]."""
    mod = pol.linear(F.silu(t_emb), sd["final_layer.adaLN_modulation.1.weight"], sd["final_layer.adaLN_modulation.1.bias"])
    return mod.chunk(2, dim=1)


def final_apply(sd, x: Tensor, shift: Tensor, scale: Tensor, pol: Policy) -> Tensor:
    """models/dit_crossattn.py:76-78 on given modulation chunks."""
    return pol.linear(modulate(layer_norm(x), shift, scale, pol), sd["final_layer.linear.weight"], sd["final_layer.linear.bias"])


def final_layer(sd, x: Tensor, t_emb: Tensor, pol: Policy) -> Tensor:
    """models/dit_crossattn.py:74-78."""
    shift, scale = final_modulation(sd, t_emb, pol)
    return final_apply(sd, x, shift, scale, pol)


def depth_of(sd) -> int:
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))


def forward(sd: Dict[str, Tensor], x: Tensor, t: Tensor, y: Tensor, num_heads: int,
            precision: str = "fp32", return_blocks: bool = False):
    """DiT.forward (dit_crossattn.py:184-202).  x [B,N,Cin] fp32, t [B] int, y [B,M,Dc] fp32."""
    pol = Policy(precision)
    sd = {k: v.float() for k, v in sd.items()}
    h = F.linear(x, sd["x_embedder.weight"], sd["x_embedder.bias"])       # fp32, outside autocast (:191)
    t_emb = t_embedder(sd, t)                                             # fp32 (:192)
    blocks = []
    for i in range(depth_of(sd)):
        h = dit_block(sd, i, h, y, t_emb, num_heads, pol)
        if return_blocks:
            blocks.append(h.clone())
    out = final_layer(sd, h, t_emb, pol)
    return (out, blocks) if return_blocks else out


def forward_with_cfg(sd, x: Tensor, t: Tensor, y: Tensor, cfg_scale: float, num_heads: int,
                     precision: str = "fp32") -> Tensor:
    """DiT.forward_with_cfg (dit_crossattn.py:204-213): batch = [cond ; uncond], guidance on ALL channels."""
    pol = Policy(precision)
    combined = torch.cat([x, x], dim=0)
    combined_t = torch.cat([t, t], dim=0)
    y_null = sd["null_cond_embedding"].float().expand_as(y)
    combined_y = torch.cat([y, y_null], dim=0)
    out = forward(sd, combined, combined_t, combined_y, num_heads, precision)
    cond, uncond = torch.split(out, len(out) // 2, dim=0)
    return pol.rnd(uncond + pol.rnd(cfg_scale * pol.rnd(cond - uncond)))


def uncond_cross_constant(sd, i: int, precision: str = "fp32") -> Tensor:
    """Identity used by the CUDA path (SURVEY §8a a8): when every context row equals the null embedding the
    softmax is uniform, so cross-attention output == proj(to_v(null)) for every query."""
    pol = Policy(precision)
    sd = {k: v.float() for k, v in sd.items()}
    p = f"blocks.{i}.crossattn."
    v = pol.linear(sd["null_cond_embedding"][None], sd[p + "to_v.weight"], sd.get(p + "to_v.bias"))
    return pol.linear(v, sd[p + "proj.weight"], sd.get(p + "proj.bias"))[0]
