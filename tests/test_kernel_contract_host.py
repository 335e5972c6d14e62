"""CPU: the precision-contract emulations (oracle/contract.py) on hand-worked cases, the exact-operand generators' precondition, and
the power of the bit-exact GPU checks: on the operands tests/test_gpu_kernel_contract.py draws, every plausible wrong rounding policy
differs from the contract on a stated share of the elements, so a kernel that followed it would fail there."""
import math

import numpy as np
import pytest

from oracle import contract as C

E = 2.0 ** -11   # half an fp16 ulp at 1


def test_h_ties_to_even_and_rejects_non_fp32():
    assert C.h(1 + E) == 1.0                       # tie, 1.0 is even
    assert C.h(1 + 3 * E) == 1 + 4 * E             # tie, 1 + 2^-9 is even
    assert C.h(1 + E + 2.0 ** -23) == 1 + 2 * E    # just above the tie
    assert C.h(2049.0) == 2048.0 and C.h(2051.0) == 2052.0
    with np.errstate(over="ignore"):
        assert C.h(65520.0) == np.inf              # the overflow threshold rounds up
    with pytest.raises(AssertionError):
        C.h(1 + 2.0 ** -30)                        # not an fp32 number: the emulation would carry more than the kernel


def test_rounding_points_hand_worked():
    # h(acc + b) once: 2048 + 1 is a tie that goes to 2048; rounding acc first (2049 -> 2048) then adding 1 gives 2049 -> 2048 too,
    # but 2047.5 + 1.5: once -> 2049 -> 2048; twice -> h(2047.5) = 2048, + 1.5 -> 2049.5 -> 2050
    y = C.acc_bias(np.array([2047.5]), np.array([1.5]))
    assert C.linear_store(y)[0] == 2048.0
    assert C.wrong_double_round(np.array([2047.5]), np.array([1.5]))[0] == 2050.0
    # post-scale re-rounds the rounded value: h(h(2049) * 0.75) = h(1536) vs h(2049 * 0.75) = h(1536.75) = 1537
    assert C.linear_store(np.array([2049.0]), 0.75)[0] == 1536.0
    assert C.wrong_post_scale(np.array([2049.0]), 0.75)[0] == 1537.0
    # gated: x0 + h(g * h(y)), one fp32 add
    assert C.gated(np.array([1.0]), np.array([0.75]), np.array([2049.0]))[0] == 1537.0         # 1 + h(0.75 * 2048)
    assert C.wrong_gated(np.array([1.0]), np.array([0.75]), np.array([2049.0]))[0] == 1538.0   # 1 + h(1536.75)
    # RESID_SCALE rounds (acc + b + r) * alpha once: 2046.5 + 3 = 2049.5 -> 2050; rounding first: h(2046.5) = 2046 (tie), + 3 = 2049 -> 2048
    assert C.resid_scale(np.array([2046.5]), np.array([3.0]), 1.0)[0] == 2050.0
    assert C.wrong_resid_scale(np.array([2046.5]), np.array([3.0]), 1.0)[0] == 2048.0
    # GELU on the rounded value
    assert C.linear_gelu(np.array([0.0]))[0] == 0.0
    assert abs(C.linear_gelu(np.array([3.0]))[0] - C.gelu_tanh(3.0)) <= C.ulp16(3.0) / 2
    # LayerNorm-modulate: h(1 + scale); 1 + 2^-11 rounds to 1
    x = np.array([[1.0, -1.0, 1.0, -1.0]])
    ln, m, y = C.ln_modulate(x, np.zeros(4), np.full(4, 2.0 ** -11), 0.0)
    assert np.all(m == 1.0) and np.allclose(ln, x) and np.all(y == x)
    assert np.all(C.wrong_ln_modulate(x * 0.75, np.zeros(4), np.full(4, 2.0 ** -11), 0.0) == C.ln_modulate(x * 0.75, np.zeros(4), np.full(4, 2.0 ** -11), 0.0)[2])


@pytest.mark.parametrize("K", [8, 16, 32, 40, 72, 200, 1152, 4608, 27 * 32, 27 * 256])
def test_exact_operands_sum_exactly(K):
    rng = np.random.default_rng(K)
    A, W, b = C.exact_linear(rng, 4, 8, K)
    assert C.exact_sum_check(A, W, b, orders=3, seed=K)
    y = A @ W.T + b
    assert C.is_f32(y)
    # most outputs carry more bits than fp16 keeps (the rounding points are exercised)
    A2, W2, b2 = C.exact_linear(np.random.default_rng(K + 1), 64, 64, K)
    y2 = A2 @ W2.T + b2
    assert np.mean(C.h(y2) != y2) > 0.6, K


def test_exact_conv_operands():
    rng = np.random.default_rng(3)
    x, W, b = C.exact_conv3d(rng, 2, 4, 32, 16)
    y = C.conv3d_ref(x, W, b)
    assert C.is_f32(y) and np.mean(C.h(y) != y) > 0.6
    # against a direct loop over one output voxel at a corner (halo taps) and one inside
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (1, 1), (0, 0)))
    for (p, z, yy, xx) in [(0, 0, 0, 0), (1, 2, 1, 3)]:
        patch = xp[p, z:z + 3, yy:yy + 3, xx:xx + 3].reshape(27 * 32)
        assert np.array_equal(W @ patch + b, y[p, z, yy, xx])


# ---- power of the GPU checks -------------------------------------------------------------------------------------------------
POST_SCALE = float(np.float32(72 ** -0.5))
RESID_ALPHA = float(np.float32(math.sqrt(0.5)))


def _power_table():
    """Share of elements on which each wrong policy differs from the contract, on the GPU test's own operand draws."""
    rows = []
    for K in (8, 40, 200, 1152, 4608):
        A, W, b = C.exact_linear(np.random.default_rng(1000 + K), 300, 136, K)
        acc = A @ W.T
        y = C.acc_bias(acc, b)
        rows.append((f"store K={K}: h(h(acc)+b)", np.mean(C.wrong_double_round(acc, b) != C.linear_store(y))))
        rows.append((f"post-scale K={K}: h(y s)", np.mean(C.wrong_post_scale(y, POST_SCALE) != C.linear_store(y, POST_SCALE))))
        Ag, Wg, bg = C.exact_linear(np.random.default_rng(2000 + K), 300, 136, K, target_std=2.0)
        yg = C.acc_bias(Ag @ Wg.T, bg)
        rows.append((f"gelu K={K}: gelu(y)", np.mean(C.wrong_gelu(yg) != C.linear_gelu(yg))))
    rng = np.random.default_rng(7)
    A, W, b = C.exact_linear(rng, 640, 576, 72)
    y = C.acc_bias(A @ W.T, b)
    x0, gate = C.gated_operands(np.random.default_rng(8), 640, 576, 2)
    g = gate[(np.arange(640) // 100) % 2]
    rows.append(("gated: x0 + h(g y)", np.mean(C.wrong_gated(x0, g, y) != C.gated(x0, g, y))))
    x, Wc, bc = C.exact_conv3d(np.random.default_rng(9), 3, 8, 32, 32)
    yc = C.conv3d_ref(x, Wc, bc)
    assert C.is_f32(yc)
    r = C.resid_operand(np.random.default_rng(10), yc.shape)
    rows.append(("resid-scale: h(h(y) + r)", np.mean(C.wrong_resid_scale(yc, r, RESID_ALPHA) != C.resid_scale(yc, r, RESID_ALPHA))))
    xl, sh, sc = C.ln_operands(np.random.default_rng(11), 64, 1152)
    rows.append(("ln-modulate: 1 + scale unrounded",
                 np.mean(C.wrong_ln_modulate(xl, sh, sc, 1e-6) != C.ln_modulate(xl, sh, sc, 1e-6)[2])))
    return rows


def test_wrong_policies_are_caught():
    rows = _power_table()
    print("\nshare of elements where the wrong policy differs from the contract:")
    for name, share in rows:
        print(f"  {name:42s} {share:.3f}")
    for name, share in rows:
        assert share > 0.05, (name, share)


def test_ln_fingerprint_scales():
    _, _, sc = C.ln_operands(np.random.default_rng(11), 4, 1152)
    assert np.mean(C.h(C.f32(1 + sc)) != 1 + sc) > 0.9
