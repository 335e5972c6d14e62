"""Micro-benchmarks of the hot kernels through the C ABI (device-timed: CUDA events per call, torch.profiler for the kernel alone)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tpxl_b200 import _lib
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from gpu_util import linear, st

def timeit(fn, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters

def card():
    """Name, power limit and max SM clock of GPU 0 (read-only nvidia-smi query): a time means little without them."""
    import subprocess
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def kernel_us(fn, name, iters=50):
    """Mean device time per call of the kernels whose name contains `name` (torch.profiler, CUDA activity): excludes the output
    memsets tpx_linear_heads issues before its GEMM.  Calls are synchronised one by one: back to back, a kernel launched with
    programmatic dependent launch starts while its predecessor drains, and its span would include that wait."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5): fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
            torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA and name in e.name]
    return sum(e.time_range.elapsed_us() for e in ev) / iters


def dit_gemms(lib):
    """The six linears of one DiT block as dit_forward issues them at the headline size (CFG: 2 x 2048 tokens, hidden 1152, 16 heads
    of 72 padded to 80, MLP 4608): the same epilogues, the gate row with batch stride 0, the head-split outputs (V transposed), the
    automatic tile (cross q: 144, as the DiT passes it)."""
    S, N, D, H, Dh, DhP, Dm = 2, 2048, 1152, 16, 72, 80, 4608
    r = lambda *s: torch.randn(*s, device="cuda").half()
    h, hid, mod = r(S * N, D), r(S * N, Dm), r(1, 9 * D)
    xres = torch.randn(S * N, D, device="cuda")
    q, k = torch.zeros(S, H, N, DhP, device="cuda").half(), torch.zeros(S, H, N, DhP, device="cuda").half()
    vT = torch.zeros(S, H, DhP, N, device="cuda").half()
    Wq, Wqkv, Wp, W1, W2 = r(D, D) * D ** -0.5, r(3 * D, D) * D ** -0.5, r(D, D) * D ** -0.5, r(Dm, D) * D ** -0.5, r(D, Dm) * Dm ** -0.5
    b3, b1 = r(3 * D), r(Dm)
    gate = mod[:, 2 * D:3 * D]
    hid_out = torch.empty(S * N, Dm, device="cuda", dtype=torch.float16)

    def heads_call(M, W, nw, scale, tile):
        return lambda: _lib.check(lib.tpx_linear_heads(h.data_ptr(), D, W.data_ptr(), b3.data_ptr(), q.data_ptr(), k.data_ptr() if nw == 3 else None,
                                                       vT.data_ptr() if nw == 3 else None, M, nw * D, D, D, H, Dh, DhP, N, scale, tile, 2 if nw == 3 else -1, N, st()))

    def gated_call(A, M, W, K):
        return lambda: _lib.check(lib.tpx_linear_gated(A.data_ptr(), K, W.data_ptr(), b3.data_ptr(), gate.data_ptr(), 0, 1, N, xres.data_ptr(), D, M, D, K, 0, st()))

    fc1 = lambda: _lib.check(lib.tpx_linear(h.data_ptr(), D, W1.data_ptr(), b1.data_ptr(), hid_out.data_ptr(), Dm, S * N, Dm, D, 1, 1.0, 0, st()))
    cases = [("cross q (heads, q scaled)", N, D, D, heads_call(N, Wq, 1, Dh ** -0.5, 144), h[:N], Wq),
             ("cross proj (gated)", N, D, D, gated_call(h, N, Wp, D), h[:N], Wp),
             ("self qkv (heads, V^T)", S * N, 3 * D, D, heads_call(S * N, Wqkv, 3, 1.0, 0), h, Wqkv),
             ("self proj (gated)", S * N, D, D, gated_call(h, S * N, Wp, D), h, Wp),
             ("fc1 (GELU)", S * N, Dm, D, fc1, h, W1),
             ("fc2 (gated)", S * N, D, Dm, gated_call(hid, S * N, W2, Dm), hid, W2)]
    tot_us = tot_cb = 0.0
    for name, M, Nn, K, fn, A, W in cases:
        fl = 2.0 * M * Nn * K
        us = kernel_us(fn, "gemm_tc_kernel")
        call = timeit(fn, iters=50) * 1e3
        cb = timeit(lambda: A @ W.t(), iters=50) * 1e3
        tot_us += us; tot_cb += cb
        print(f"dit {name:28s} M={M:5d} N={Nn:5d} K={K:5d}: kernel {us:8.1f} us {fl / us / 1e6:7.1f} TFLOP/s (call {call:8.1f} us) | "
              f"cublas fp16 out {cb:8.1f} us {fl / cb / 1e6:7.1f} TFLOP/s", flush=True)
    print(f"dit block, six linears: {tot_us:8.1f} us (cublas {tot_cb:8.1f} us)", flush=True)


def main():
    lib = _lib.lib()
    print("card:", card(), flush=True)
    dit_gemms(lib)
    for (M, N, K) in [(4096, 1152, 1152), (4096, 3456, 1152), (4096, 4608, 1152), (4096, 1152, 4608), (2048, 1152, 1152)]:
        A = torch.randn(M, K, device="cuda").half(); W = torch.randn(N, K, device="cuda").half() * K ** -0.5; b = torch.randn(N, device="cuda").half()
        for tile in (128, 144, 192, 256):
            for act in (0, 1):
                try:
                    ms = timeit(lambda: linear(A, W, b, act=act, tile_n=tile))
                except _lib.TpxError as e:    # a library built without this width
                    print(f"linear M={M} N={N} K={K} tile={tile} act={act}: {e}", flush=True)
                    continue
                print(f"linear M={M} N={N} K={K} tile={tile} act={act}: {ms*1e3:8.1f} us  {2*M*N*K/ms/1e9:8.1f} TFLOP/s", flush=True)
        ms = timeit(lambda: A @ W.t())
        print(f"cublas M={M} N={N} K={K}: {ms*1e3:8.1f} us  {2*M*N*K/ms/1e9:8.1f} TFLOP/s", flush=True)
    # attention
    for (B, H, Nq, Nk, Dh, DhP) in [(2, 16, 2048, 2048, 72, 80), (1, 16, 2048, 1370, 72, 80)]:
        q = torch.randn(B, H, Nq, DhP, device="cuda").half(); k = torch.randn(B, H, Nk, DhP, device="cuda").half(); v = torch.randn(B, H, Nk, DhP, device="cuda").half()
        o = torch.empty(B, Nq, H * Dh, device="cuda", dtype=torch.float16)
        ms = timeit(lambda: lib.tpx_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), B, H, Nq, Nk, Dh, DhP, Dh ** -0.5, st()))
        fl = 4.0 * B * H * Nq * Nk * Dh
        print(f"attention B={B} Nq={Nq} Nk={Nk}: {ms*1e3:8.1f} us  {fl/ms/1e9:8.1f} TFLOP/s (algorithmic, Dh=72)", flush=True)
        NkPad = (Nk + 7) // 8 * 8
        vT = torch.zeros(B, H, DhP, NkPad, device="cuda", dtype=torch.float16); vT[..., :Nk] = v.transpose(-1, -2)
        ms = timeit(lambda: lib.tpx_attention_tc(q.data_ptr(), k.data_ptr(), vT.data_ptr(), o.data_ptr(), B, H, Nq, Nk, NkPad, Dh, Dh ** -0.5, st()))
        print(f"attention_tc B={B} Nq={Nq} Nk={Nk}: {ms*1e3:8.1f} us  {fl/ms/1e9:8.1f} TFLOP/s (algorithmic, Dh=72)", flush=True)
        qq, kk, vv = (t[..., :Dh].contiguous() for t in (q, k, v))
        ms = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qq, kk, vv))
        print(f"torch sdpa same shape: {ms*1e3:8.1f} us  {fl/ms/1e9:8.1f} TFLOP/s", flush=True)
    # LN
    x = torch.randn(4096, 1152, device="cuda"); mod = torch.randn(1, 3 * 1152, device="cuda").half(); out = torch.empty(4096, 1152, device="cuda", dtype=torch.float16)
    ms = timeit(lambda: lib.tpx_ln_modulate(x.data_ptr(), 4096, 1152, 1e-6, mod.data_ptr(), mod[:, 1152:].data_ptr(), 3456, 2048, 1, out.data_ptr(), None, None, 0, st()))
    print(f"ln_modulate 4096x1152: {ms*1e3:8.1f} us  {(4096*1152*6)/ms/1e6:8.1f} GB/s", flush=True)

main()
