"""The precision contract of the per-kernel entry points (DESIGN §5), one rounding point at a time, and operands that make it testable
bit for bit.

Every emulation takes fp64 arrays and goes through float32 exactly where the kernel does: an fp32 operation is its fp64 result
rounded to fp32 (correct for +, -, x: fp64 carries more than 2 x 24 + 2 bits), and ``h`` is fp32 -> fp16 round-to-nearest-even.
``h`` asserts that its input is an fp32 value, so an emulation that silently carries more precision than the kernel fails loudly.

Exact operands (``exact_linear``): A and W hold small integers times a power of two, the bias a multiple of their products' unit,
and K * max|a| * max|w| + max|b| stays below 2^22 units.  Every partial sum of acc + bias is then an fp32 number, so the tensor
cores' order, grouping or truncation cannot change it, and the fp16 output depends on the contract's rounding points alone.  The
integer ranges are as wide as that budget allows, so the sum keeps 14-20 significant bits and nearly every element is rounded.
"""
import math

import numpy as np

F16_MAX = 65504.0


def is_f32(x):
    x = np.asarray(x, dtype=np.float64)
    return np.all((x.astype(np.float32).astype(np.float64) == x) | ~np.isfinite(x))


def f32(x):
    """Round an fp64 result to fp32 (one fp32 operation)."""
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def h(x):
    """fp32 -> fp16, round to nearest even, back as fp64.  The input must already be an fp32 value."""
    x = np.asarray(x, dtype=np.float64)
    assert is_f32(x), "h() of a value that is not an fp32 number: the emulation carries more precision than the kernel"
    return x.astype(np.float32).astype(np.float16).astype(np.float64)


def ulp16(x):
    """Spacing of fp16 numbers at |x| (2^-24 in the subnormal range)."""
    a = np.abs(np.asarray(x, dtype=np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.exp2(e - 10)


def gelu_tanh(x):
    x = np.asarray(x, dtype=np.float64)
    return 0.5 * x * (1.0 + np.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


# ---- the contract's rounding points ------------------------------------------------------------------------------------------
def acc_bias(acc, bias):
    """acc + bias in fp32 (exact for exact operands; asserted)."""
    y = np.asarray(acc, dtype=np.float64) + (0.0 if bias is None else np.asarray(bias, dtype=np.float64))
    assert is_f32(y), "acc + bias is not exact in fp32: the operands break the exactness precondition"
    return y


def linear_store(y, post_scale=1.0):
    """EPI_STORE: h(acc + b) rounded once; with a post-scale, h(h(y) * s) (the scaled value re-rounded)."""
    if post_scale == 1.0:
        return h(y)
    return h(f32(h(y) * np.float64(np.float32(post_scale))))


def linear_gelu(y):
    """EPI_GELU: GELU-tanh of the fp16-rounded value, rounded to fp16 (the exact GELU; the kernel is within one ulp of it)."""
    return h(f32(gelu_tanh(h(y))))


def gated(x0, gate, y):
    """EPI_GATED: x0 + h(gate * h(y)) with one fp32 add (gate * h(y) of two fp16 numbers is exact in fp32)."""
    return f32(np.asarray(x0, dtype=np.float64) + h(f32(np.asarray(gate, dtype=np.float64) * h(y))))


def resid_scale(y, resid, alpha):
    """EPI_RESID_SCALE: (acc + bias + resid) in fp32, times alpha in fp32, then one fp16 rounding."""
    s = f32(y + np.asarray(resid, dtype=np.float64))
    return h(f32(s * np.float64(np.float32(alpha))))


def ln_modulate(x, shift, scale, eps):
    """LayerNorm in fp64 of the fp32 row, times h(1 + scale) (rounded to fp16: an fp16 op under autocast), plus shift, to fp16."""
    x = np.asarray(x, dtype=np.float64)
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    ln = (x - mu) / np.sqrt(var + np.float64(np.float32(eps)))
    m = h(f32(1.0 + np.asarray(scale, dtype=np.float64)))
    return ln, m, (ln * m + shift).astype(np.float16).astype(np.float64)


# ---- plausible wrong policies (what the exact-operand tests must be able to tell apart) -------------------------------------
def wrong_double_round(acc, bias):
    """h(h(acc) + b): the bias added after a first rounding."""
    return h(f32(h(f32(acc)) + bias))


def wrong_post_scale(y, post_scale):
    """h(y * s): no re-rounding of the scaled value."""
    return h(f32(y * np.float64(np.float32(post_scale))))


def wrong_gelu(y):
    """GELU of the unrounded value."""
    return h(f32(gelu_tanh(y)))


def wrong_gated(x0, gate, y):
    """x0 + h(gate * y): no inner rounding of the branch."""
    return f32(np.asarray(x0, dtype=np.float64) + h(f32(np.asarray(gate, dtype=np.float64) * y)))


def wrong_resid_scale(y, resid, alpha):
    """h((h(acc + b) + resid) * alpha): rounded before the residual is added."""
    return h(f32(f32(h(y) + resid) * np.float64(np.float32(alpha))))


def wrong_ln_modulate(x, shift, scale, eps):
    """(1 + scale) not rounded to fp16."""
    ln, _, _ = ln_modulate(x, shift, scale, eps)
    m = f32(1.0 + np.asarray(scale, dtype=np.float64))
    return (ln * m + shift).astype(np.float16).astype(np.float64)


# ---- exact operands ----------------------------------------------------------------------------------------------------------
SPAN_BITS = 22   # K * max|a| * max|w| and max|b| each below 2^21 units of a * w: every partial sum of acc + bias below 2^22 units


def exact_linear(rng, M, N, K, target_std=6.0, span_bits=SPAN_BITS):
    """(A [M,K], W [N,K], bias [N]) fp16-representable fp64 arrays whose products sum exactly in fp32 in any order.

    a = ia 2^-sa, w = iw 2^-sw with |ia|, |iw| <= I (I <= 1023, so fp16 holds them exactly), bias = ib 2^-(sa+sw) with ib an 11-bit
    integer times a power of two; K I^2 < 2^(span_bits-1) and |ib| < 2^(span_bits-1).  The scale puts the output's standard
    deviation near target_std (the GELU cases ask for most |y| within [-4, 4])."""
    half = 2.0 ** (span_bits - 1)
    I = int(min(1023, math.floor(math.sqrt((half - 1) / K))))
    assert I >= 1, K
    std_units = math.sqrt(K) * I * I / 3.0
    S = max(0, int(round(math.log2(std_units / target_std))))
    sa = S // 2
    sw = S - sa
    A = rng.integers(-I, I + 1, size=(M, K)).astype(np.float64) * 2.0 ** -sa
    W = rng.integers(-I, I + 1, size=(N, K)).astype(np.float64) * 2.0 ** -sw
    # bias: an 11-bit integer times 2^t units, |bias| about the output's spread, |ib| < 2^(span_bits-1)
    t = max(0, int(math.floor(math.log2(max(std_units, 1024.0) / 1024.0))))
    ib = rng.integers(-1023, 1024, size=N).astype(np.float64) * 2.0 ** t
    assert np.abs(ib).max() < half
    b = ib * 2.0 ** -S
    for arr in (A, W, b):
        assert np.all(arr.astype(np.float16).astype(np.float64) == arr)
    return A, W, b


def gated_operands(rng, M, N, G):
    """fp32 residual (moderate, never near zero after the update) and fp16 gates of both signs in [1/8, 2)."""
    x0 = f32(rng.standard_normal((M, N)) * 4.0 + np.sign(rng.standard_normal((M, N))) * 8.0)
    gate = h(f32(rng.uniform(0.125, 2.0, size=(G, N)) * np.sign(rng.standard_normal((G, N)))))
    return x0, gate


def resid_operand(rng, shape):
    return h(f32(rng.standard_normal(shape) * 4.0))


def ln_operands(rng, rows, D):
    """fp32 rows, fp16 shift, and fp16 scales for which 1 + scale is not an fp16 number (|scale| in [2^-9, 2^-3] with low bits)."""
    x = f32(rng.standard_normal((rows, D)) * 3.0 + rng.standard_normal((rows, 1)) * 2.0)
    shift = h(f32(rng.standard_normal(D) * 0.5))
    scale = h(f32(rng.uniform(2.0 ** -9, 2.0 ** -3, size=D) * np.sign(rng.standard_normal(D))))
    return x, shift, scale


def exact_sum_check(A, W, b, orders=3, seed=0):
    """The exactness precondition: the fp64 sum equals an fp32 running sum in several permuted orders (and the fp32 pairwise sum)."""
    ref = A @ W.T + b
    rng = np.random.default_rng(seed)
    K = A.shape[1]
    prods = (A[:, None, :] * W[None, :, :]).astype(np.float32)   # exact: 11 x 11-bit products
    assert np.all(prods.astype(np.float64) == A[:, None, :] * W[None, :, :])
    for _ in range(orders):
        perm = rng.permutation(K)
        s = b.astype(np.float32)[None, :].repeat(A.shape[0], 0)
        for k in perm:
            s = (s + prods[:, :, k]).astype(np.float32)
        if not np.array_equal(s.astype(np.float64), ref):
            return False
    pw = prods.sum(-1, dtype=np.float32) + b.astype(np.float32)   # numpy's pairwise fp32 reduction, bias last
    return bool(np.array_equal(pw.astype(np.float64), ref))


def exact_conv3d(rng, P, S, C, Cout, target_std=6.0, span_bits=SPAN_BITS):
    """Channels-last x [P,S,S,S,C], W [Cout, 27 C] (k = tap C + c), bias [Cout]: exact operands of a 3x3x3 convolution (K = 27 C)."""
    A, W, b = exact_linear(rng, P * S ** 3, Cout, 27 * C, target_std, span_bits)
    return A[:, :C].reshape(P, S, S, S, C), W, b   # one voxel row holds C of a row's 27 C draws: the same grid and range


def conv3d_ref(x, W, bias):
    """fp64 3x3x3 / pad 1 convolution, channels-last [P,S,S,S,C] -> [P,S,S,S,Cout]; W [Cout, 27 C] with k = ((kz 3 + ky) 3 + kx) C + c."""
    P, S, _, _, C = x.shape
    Cout = W.shape[0]
    xp = np.zeros((P, S + 2, S + 2, S + 2, C))
    xp[:, 1:-1, 1:-1, 1:-1] = x
    Wt = W.reshape(Cout, 27, C)
    out = np.zeros((P, S, S, S, Cout))
    for tap in range(27):
        kz, ky, kx = tap // 9, (tap // 3) % 3, tap % 3
        out += xp[:, kz:kz + S, ky:ky + S, kx:kx + S] @ Wt[:, tap].T
    return out + bias
