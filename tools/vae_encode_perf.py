"""Time tpxl_b200.VAE.encode at 2048 and 8 x 2048 primitives (fp16 in/out) with CUDA events after warm-up, beside VAE.decode of 2048
primitives in the same run; print the per-kernel-class device times of one profiled encode, the TFLOP/s of the encoder's algorithmic
work, and the card's name and power limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C

import torch

import tpxl_b200
from tpxl_b200 import _lib, synth


def encoder_flops_per_primitive() -> int:
    """Multiply-adds x 2 of every convolution / linear / attention product of Encoder.forward + quant_conv (vae3d_dib.py:310-327)."""
    conv = lambda vox, cin, cout, taps=27: 2 * vox * cin * cout * taps
    f = conv(512, 6, 32)                                         # conv_in
    f += 2 * 2 * conv(512, 32, 32)                               # down_blocks.0: two blocks, two convs each
    f += conv(64, 32, 32)                                        # downsample (stride 2: 64 outputs)
    f += conv(64, 32, 256) + conv(64, 256, 256) + conv(64, 32, 256, 1)   # down_blocks.1.nets.0 + shortcut
    f += 3 * 2 * conv(64, 256, 256)                              # down_blocks.1.nets.1, mid res 0 / 1
    f += 2 * 64 * 256 * 768 + 2 * 2 * 64 * 64 * 256 + 2 * 64 * 256 * 256   # attention: qkv, QK^T + PV, proj
    f += conv(64, 256, 2) + conv(64, 2, 2, 1)                    # conv_out, quant_conv
    return f


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=20).stdout.strip()
    except Exception as e:   # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q or torch.cuda.get_device_name(0)


def timed(fn, iters):
    for _ in range(3):
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
    dev = "cuda:0"
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    sd = synth.synth_state_dict(synth.vae_encoder_shapes(**synth.FULL_VAE), 103)
    sd.update(synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 104))
    vae = tpxl_b200.VAE(**synth.FULL_VAE)
    vae.load_state_dict(sd)
    vae = vae.to(dev)
    print("card (name, power limit):", card(), flush=True)
    z = torch.randn(2048, 1, 4, 4, 4, device=dev).half()
    fpp = encoder_flops_per_primitive()
    with torch.no_grad():
        x = vae.decode(z)
        print(f"decode 2048 primitives: {timed(lambda: vae.decode(z), iters):.3f} ms", flush=True)
        for P in (2048, 8 * 2048):
            xp = x.repeat(P // 2048, 1, 1, 1, 1)
            ms = timed(lambda: vae.encode(xp), iters)
            print(f"encode {P} primitives: {ms:.3f} ms, {fpp * P / ms / 1e9:.1f} TFLOP/s of {fpp / 1e9:.3f} GFLOP per primitive", flush=True)
        lib = _lib.lib()
        lib.tpx_profile_begin()
        vae.encode(x)
        ms = (C.c_float * 8)()
        n = (C.c_int64 * 8)()
        lib.tpx_profile_end(ms, n)
        names = ["gemm", "attention", "ln", "gemv", "elementwise", "conv_gemm", "groupnorm", "vae_misc"]
        print("encode 2048 per class (ms, launches):", {names[i]: (round(ms[i], 3), n[i]) for i in range(8) if n[i]}, flush=True)


if __name__ == "__main__":
    main()
