#!/usr/bin/env python
"""Time PrimSDF(differentiable=True) forward and backward (tpx_primsdf_query_grid + tpx_primsdf_query_backward, all three gradients)
with CUDA events: 2048 primitives of 8^3 on the shell scene of tools/primsdf_perf.py, n = 2^18 and 2^21 points, half near the
surface (where fitting samples them) and half uniform in [-1, 1]^3, training mode.  Also times a dense torch autograd formulation of
the same query (the reference's [points x prims] weight matrix + grid_sample, restated here; tools do not use oracle/) at 2^18 on
the same GPU.  Prints the card, its power limit and max SM clock from the same run."""
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tpxl_b200  # noqa: E402


def dense_query(x, srt, feat, S=8, C=6):
    """models/primsdf.py:52-109 in training mode: dense weight matrix, gather of the covering pairs, grid_sample, index_add_."""
    local = (x[:, None, :] - srt[None, :, 1:4]) / srt[None, :, 0:1]
    w = F.relu(1 - torch.norm(local, p=float("inf"), dim=-1))
    w = w / (w.sum(-1, keepdim=True) + 1e-6)
    ib, ip = torch.where(w > 0)
    samp = F.grid_sample(feat[ip].reshape(-1, C, S, S, S), local[ib, ip].reshape(-1, 1, 1, 1, 3), mode="bilinear", padding_mode="zeros",
                         align_corners=True).reshape(-1, C)
    out = torch.zeros(x.shape[0], C, device=x.device).index_add_(0, ib, samp * w[ib, ip][:, None])
    return torch.cat([out[:, :1], out[:, 1:].clip(0.0, 1.0)], 1)


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q.splitlines()[0] if q else torch.cuda.get_device_name()}")
    K, S = 2048, 8
    g = torch.Generator().manual_seed(0)
    d = torch.randn(K, 3, generator=g)
    pos = d / d.norm(dim=1, keepdim=True) * (0.55 + 0.1 * torch.rand(K, 1, generator=g))
    srt = torch.cat([0.03 + 0.05 * torch.rand(K, 1, generator=g), pos], 1)
    feat = torch.randn(K, 6 * S ** 3, generator=g)
    m = tpxl_b200.PrimSDF(num_prims=K, dim_feat=6, prim_shape=S, differentiable=True).train()
    m.srt_param.data, m.feat_param.data = srt, feat
    m = m.cuda()
    for logn in (18, 21):
        n = 1 << logn
        x = torch.rand(n, 3, generator=g) * 2 - 1
        x[: n // 2] = pos[torch.randint(0, K, (n // 2,), generator=g)] + 0.05 * torch.randn(n // 2, 3, generator=g)
        x = x.cuda().requires_grad_(True)
        G = torch.randn(n, 6, device="cuda")

        def fwd():
            with torch.no_grad():
                return m(x)

        def fwd_bwd():
            o = m(x)
            torch.cat([o["sdf"], o["tex"], o["mat"]], 1).backward(G)

        reps = 20 if logn == 18 else 5
        t_f = timed(fwd, reps)
        t_fb = timed(fwd_bwd, reps)
        with torch.no_grad():
            cov = float((m(x)["tex"].sum(1) != 0).float().mean())
        print(f"n = 2^{logn}: forward {t_f:.3f} ms, forward + backward {t_fb:.3f} ms (backward ~{t_fb - t_f:.3f} ms), covered {cov:.3f}")
        if logn == 18:
            sp, fp = m.srt_param.detach().clone().requires_grad_(True), m.feat_param.detach().clone().requires_grad_(True)
            xd = x.detach().clone().requires_grad_(True)

            def dense_fwd_bwd():
                dense_query(xd, sp, fp, S).backward(G)

            t_d = timed(lambda: dense_query(xd.detach(), sp.detach(), fp.detach(), S), 5)
            t_db = timed(dense_fwd_bwd, 5)
            print(f"  dense torch autograd: forward {t_d:.3f} ms, forward + backward {t_db:.3f} ms")


if __name__ == "__main__":
    main()
