"""Oracle restatement of the PrimSDF point query's BACKWARD (TEST INFRASTRUCTURE — see oracle/__init__.py).

The gradient of /root/reference/models/primsdf.py:52-109 (PrimSDF.forward, what PrimSDFLoss in dva/losses.py:102-148 differentiates),
written out with the loop structure of tpx_primsdf_query_backward instead of autograd: pass 1 recomputes the box weights, the
trilinear samples and the raw normalised output o; the upstream gradient of the clipped channels (1..5) is masked where o lies
outside [0, 1]; pass 2 emits, per covering (point, primitive) pair, the feature scatter and the weight / local-position chain;
uncovered points at inference get the nearest-voxel fill's gradient.  Vectorised over the covering pairs; any float dtype.
"""
from __future__ import annotations

import torch

from .primsdf import local_grid


def _corners(lj: torch.Tensor, S: int):
    """Trilinear cell of covered local positions lj [P,3] (x indexes W, z indexes D; align_corners=True): the flat voxel index of
    the 8 corners [P,8], their weights [P,8] and the weights' derivatives along x, y, z [P,8,3] per unit of l."""
    hs = 0.5 * (S - 1)
    f = (lj + 1) * hs
    i0 = f.floor().long().clamp(max=S - 2)
    a = f - i0
    b = 1 - a
    idx, wt, dw = [], [], []
    for c in range(8):
        dz, dy, dx = c >> 2, (c >> 1) & 1, c & 1
        wx, wy, wz = (a[:, 0] if dx else b[:, 0]), (a[:, 1] if dy else b[:, 1]), (a[:, 2] if dz else b[:, 2])
        sx, sy, sz = (1 if dx else -1), (1 if dy else -1), (1 if dz else -1)
        idx.append(((i0[:, 2] + dz) * S + (i0[:, 1] + dy)) * S + i0[:, 0] + dx)
        wt.append(wx * wy * wz)
        dw.append(torch.stack([sx * wy * wz, sy * wx * wz, sz * wx * wy], -1) * hs)
    return torch.stack(idx, 1), torch.stack(wt, 1), torch.stack(dw, 1)


def query_backward(x: torch.Tensor, srt: torch.Tensor, feat: torch.Tensor, grad_out: torch.Tensor, S: int = 8, dim_feat: int = 6,
                   inference: bool = True):
    """x [n,3], srt [K,4] = (scale, tx, ty, tz), feat [K, dim_feat*S^3], grad_out [n, dim_feat] (the upstream gradient of
    (sdf, tex, mat) concatenated).  Returns (grad_x [n,3], grad_srt [K,4], grad_feat [K, dim_feat*S^3])."""
    n, K, S3 = x.shape[0], srt.shape[0], S ** 3
    pos, s = srt[:, 1:4], srt[:, 0]
    local = (x[:, None, :] - pos[None]) / s[None, :, None]
    w = 1 - local.abs().amax(-1)
    ib, ip = torch.where(w > 0)
    # pass 1: the forward's sums
    lj, wj = local[ib, ip], w[ib, ip]
    idx, cw, dcw = _corners(lj, S)
    vol = feat.reshape(K, dim_feat, S3)[ip]                                  # [P, C, S^3]
    fv = torch.gather(vol, 2, idx[:, None, :].expand(-1, dim_feat, -1))     # [P, C, 8]
    v = (fv * cw[:, None, :]).sum(-1)                                        # [P, C]
    W = torch.zeros(n, dtype=x.dtype, device=x.device).index_add_(0, ib, wj) + 1e-6
    o = torch.zeros(n, dim_feat, dtype=x.dtype, device=x.device).index_add_(0, ib, wj[:, None] * v) / W[:, None]
    g = grad_out.clone()
    g[:, 1:] = torch.where((o[:, 1:] >= 0) & (o[:, 1:] <= 1), g[:, 1:], torch.zeros_like(g[:, 1:]))
    # pass 2: per covering pair
    gv = g[ib] * (wj / W[ib])[:, None]                                        # dL/dv_jc
    gw = (g[ib] * (v - o[ib])).sum(1) / W[ib]                                 # dL/dw_j
    dv = torch.einsum("pck,pkd->pcd", fv, dcw)                                # dv_jc / dl
    am = lj.abs()
    tie = (am == am.amax(-1, keepdim=True)).to(x.dtype)
    gl = (gv[:, :, None] * dv).sum(1) - gw[:, None] * torch.sign(lj) * tie / tie.sum(-1, keepdim=True)
    gl = gl / s[ip][:, None]
    grad_x = torch.zeros_like(x).index_add_(0, ib, gl)
    grad_srt = torch.zeros_like(srt)
    grad_srt[:, 1:4].index_add_(0, ip, -gl)
    grad_srt[:, 0].index_add_(0, ip, -(gl * lj).sum(1))
    grad_feat = torch.zeros_like(feat).reshape(-1)
    flat = (ip * dim_feat * S3)[:, None, None] + (torch.arange(dim_feat, device=x.device) * S3)[None, :, None] + idx[:, None, :]
    grad_feat.index_add_(0, flat.reshape(-1), (gv[:, :, None] * cw[:, None, :]).reshape(-1))
    grad_feat = grad_feat.reshape(K, -1)
    # uncovered points at inference: sdf = f + |x - c| sign(f) at the nearest voxel c of the nearest primitive
    covered = torch.zeros(n, dtype=torch.bool, device=x.device)
    covered[ib] = True
    miss = torch.nonzero(~covered)[:, 0]
    if inference and K > 0 and len(miss):
        xm = x[miss]
        near = (xm[:, None, :] - pos[None]).norm(dim=-1).argmin(1)
        grid = local_grid(S).to(x)
        e = xm[:, None, :] - (pos[near][:, None, :] + s[near][:, None, None] * grid[None])
        d = e.norm(dim=-1)
        dmin, vi = d.min(1)
        u = e[torch.arange(len(miss), device=x.device), vi] / torch.where(dmin > 0, dmin, torch.ones_like(dmin))[:, None]
        h = (g[miss, 0] * torch.sign(feat[near, vi]))[:, None] * u
        grad_feat.index_put_((near, vi), g[miss, 0], accumulate=True)
        grad_x.index_add_(0, miss, h)
        grad_srt[:, 1:4].index_add_(0, near, -h)
        grad_srt[:, 0].index_add_(0, near, -(h * grid[vi]).sum(1))
    return grad_x, grad_srt, grad_feat
