"""Time the ray-march preview, the saving forward (tpx_raymarch_forward with raysat) and the backward (tpx_raymarch_backward) with CUDA
events, at the shipped primitive count (2048 primitives of 8^3 on a shell, volradius 10000, dt 1) for 256^2 (app.py) and 518^2
(inference.py), N = 1 and 4.  Prints one line per configuration and the GPU it ran on.

    python tools/raymarch_grad_perf.py [--iters 10]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import tpxl_b200  # noqa: E402
from tpxl_b200 import _lib  # noqa: E402


def scene(N, H, W):
    K, S, volradius = 2048, 8, 10000.0
    g = torch.Generator().manual_seed(3)
    d = torch.randn(N, K, 3, generator=g)
    pos = d / d.norm(dim=-1, keepdim=True) * 0.5
    rgba = torch.rand(N, K, 4, S, S, S, generator=g) * 255.0
    rgba[:, :, 3] = 255.0 * torch.exp(-(torch.rand(N, K, S, S, S, generator=g) * 0.02 / 0.005) ** 2)
    R = torch.eye(3)[None, None].repeat(N, K, 1, 1)
    scale = torch.full((N, K, 3), 1.0 / 0.05)
    RT = torch.tensor([[[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, 5 * volradius]]]).repeat(N, 1, 1)
    Kc = torch.tensor([[[2084.9526697685183 * H / 1024, 0, 512.0 * H / 1024], [0, 2084.9526697685183 * W / 1024, 512.0 * W / 1024], [0, 0, 1.0]]]).repeat(N, 1, 1)
    return rgba, pos * volradius, R, scale, Kc, RT, volradius


def timed(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"GPU: {q.splitlines()[0] if q else torch.cuda.get_device_name()}")
    L = _lib.lib()
    for H in (256, 518):
        for N in (1, 4):
            rgba, pos, R, scale, Kc, RT, volradius = scene(N, H, H)
            cam = tpxl_b200.ray_marcher.convert_camera_parameters(RT.cuda(), Kc.cuda())
            c = [t.float().contiguous() for t in (cam["campos"], cam["camrot"], torch.diagonal(cam["focal"], dim1=1, dim2=2), cam["princpt"])]
            tpl = rgba.cuda().permute(0, 1, 3, 4, 5, 2).contiguous()
            p, r, s = (pos.cuda() / volradius).contiguous(), R.cuda().contiguous(), scale.cuda().contiguous()
            K, S = tpl.shape[1], tpl.shape[2]
            out = torch.empty(N, H, H, 4, device="cuda")
            raysat = torch.empty(N, H, H, 3, device="cuda")
            G = torch.randn(N, H, H, 4, generator=torch.Generator().manual_seed(1)).cuda()
            grads = [torch.zeros_like(t) for t in (tpl, p, r, s)]
            common = [tpl.data_ptr(), p.data_ptr(), r.data_ptr(), s.data_ptr(), *[t.data_ptr() for t in c], N, K, S, H, H, volradius, 1.0 / volradius, 8.0, 8.0]
            st = _lib.stream_ptr()

            def preview():
                _lib.check(L.tpx_raymarch_preview(*common, out.data_ptr(), st))

            def forward():
                _lib.check(L.tpx_raymarch_forward(*common, 1, None, out.data_ptr(), raysat.data_ptr(), st))

            def backward():
                _lib.check(L.tpx_raymarch_backward(*common, 1, None, raysat.data_ptr(), G.data_ptr(), *[g.data_ptr() for g in grads], st))

            t_prev, t_fwd = timed(preview, args.iters), timed(forward, args.iters)
            t_bwd = timed(backward, args.iters)          # accumulates into the same buffers: only the time matters here
            al = out[..., 3]
            print(f"{H}x{H} N={N} K={K} S={S}: preview {t_prev:.3f} ms, saving forward {t_fwd:.3f} ms, backward {t_bwd:.3f} ms "
                  f"(backward / forward {t_bwd / t_fwd:.2f}; covered {float((al > 0).float().mean()):.2f}, saturated {float((raysat[..., 0] >= 0).float().mean()):.2f})")


if __name__ == "__main__":
    main()
