"""GPU: the per-kernel entry points element by element against the precision contract (DESIGN §5, oracle/contract.py).

Exact operands (oracle.contract.exact_linear: every partial sum of acc + bias is an fp32 number) make the GEMM's output a function of
the contract's rounding points alone, so tpx_linear (store, post-scale), tpx_linear_heads, tpx_linear_gated and tpx_conv3d_k3 are
compared bit for bit with the host emulation, over tile widths, epilogues, ragged M / N / K (K tails through the TMA's zero fill),
strided operands with NaN in the unread columns, and sentinels around every output.  tests/test_kernel_contract_host.py shows that
each plausible wrong rounding policy differs from the contract on 20-34 % of these elements.

Bounded, not exact:
  GELU: every element within 1 fp16 ulp of h(gelu(h(y))), and a share of exact matches above GELU_MATCH (the kernel's MUFU
        ex2 / rcp GELU is within ~2e-7 of exact: 99.989-99.996 % measured; GELU of the unrounded value matches on 66-67 %);
  random operands: |got - y| <= ulp16(y) + K 2^-23 sum|a w| + |b| 2^-24 per element;
  attention: per element ulp16(o*) + (2^-11 + 4 eps_s + 2^-20) sum pi|v| + 2^-25 sum|v| / l against fp64 softmax attention, and
        per (b, head, 64-row tile) rel-L2 <= 2.5 x the fp16-P policy's + 1e-4;
  LayerNorm-modulate: per element 1 ulp16 of the fp64 policy + 2^-18 (|LN m| + |shift|) + the fp32 mean's error over sigma (a row
        offset by 1e3 reaches 0.99 of this bound); on scales where h(1 + scale) != 1 + scale
        the kernel matches the contract on a share above LN_MATCH and the unrounded alternative on a clearly smaller share.
"""
import math

import numpy as np
import pytest
import torch

from oracle import contract as C
from tpxl_b200 import _lib
from gpu_util import st
import parity

pytestmark = pytest.mark.gpu

GELU_MATCH = 0.999   # measured 0.99989-0.99996 on an H100 80GB HBM3 (700 W)
LN_MATCH = 0.99      # measured 0.9974-0.9996 (the unrounded alternative: 0.69-0.72)
POST_SCALE = float(np.float32(72 ** -0.5))
ALPHA = float(np.float32(math.sqrt(0.5)))
S16 = 0x7E5A            # fp16 sentinel bit pattern (a NaN payload no kernel produces)
S32 = 0x7FC0BEEF        # fp32 sentinel bit pattern


def lib():
    return _lib.lib()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def d16(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.float16).cuda()


def host(t):
    return t.double().cpu().numpy()


def sentinel16(*shape):
    return torch.full(shape, S16, dtype=torch.int16, device="cuda").view(torch.float16)


def bits16(t):
    return t.view(torch.int16)


def strided_a(A, lda):
    """A [M, K] inside an [M, lda] buffer whose unread columns hold NaN."""
    M, K = A.shape
    buf = torch.full((M, lda), float("nan"), dtype=torch.float16, device="cuda")
    buf[:, :K] = d16(A)
    return buf


def run_linear(A, W, b, act, post_scale, tile, pad_k=24, pad_n=16, extra_rows=3):
    """tpx_linear on strided A (lda = K + pad_k) into an [M + extra_rows, N + pad_n] sentinel buffer; returns (out [M, N] fp64,
    whether every byte outside [M, N] kept its sentinel)."""
    M, K = A.shape
    N = W.shape[0]
    lda, ldo = K + pad_k, N + pad_n
    a = strided_a(A, lda)
    w, bb = d16(W), d16(b)
    out = sentinel16(M + extra_rows, ldo)
    _lib.check(lib().tpx_linear(a.data_ptr(), lda, w.data_ptr(), bb.data_ptr(), out.data_ptr(), ldo, M, N, K, act, post_scale, tile, st()),
               f"tpx_linear M={M} N={N} K={K} tile={tile}")
    torch.cuda.synchronize()
    o = out[:M, :N]
    mask = torch.ones(M + extra_rows, ldo, dtype=torch.bool, device="cuda")
    mask[:M, :N] = False
    untouched = bool(torch.all(bits16(out)[mask] == S16))
    return host(o), untouched


TILES = [(0, "store"), (0, "scale"), (0, "gelu"), (32, "store"), (32, "scale")] + [(t, e) for t in (128, 144, 192, 256) for e in ("store", "scale", "gelu")]
MS = [1, 8, 127, 128, 129, 300]
NS = [8, 136, 1152, 1160]
KS = [8, 16, 32, 40, 72, 200, 1152, 4608]


def check_case(M, N, K, tile, epi, seed):
    gelu = epi == "gelu"
    A, W, b = C.exact_linear(np.random.default_rng(seed), M, N, K, target_std=2.0 if gelu else 6.0)
    s = POST_SCALE if epi == "scale" else 1.0
    got, untouched = run_linear(A, W, b, 1 if gelu else 0, s, tile)
    y = C.acc_bias(A @ W.T, b)
    where = f"M={M} N={N} K={K} tile={tile} {epi}"
    assert untouched, f"{where}: wrote outside the output"
    if not gelu:
        ref = C.linear_store(y, s)
        bad = got != ref
        assert not bad.any(), f"{where}: {int(bad.sum())} of {bad.size} elements differ from the contract, e.g. got {got[bad][:4]} want {ref[bad][:4]}"
        return None
    ref = C.linear_gelu(y)
    err = np.abs(got - ref)
    assert np.all(err <= C.ulp16(ref)), f"{where}: GELU off by more than one ulp: max {err.max()}"
    return np.mean(got == ref), np.mean(got == C.wrong_gelu(y)), got.size


@pytest.mark.parametrize("tile,epi", TILES)
def test_linear_exact_k_sweep(tile, epi):
    """Every K (tails of 8 .. 56 columns zero-filled by the TMA, K = 32 included) at a ragged M and N."""
    stats = [check_case(129, 136, K, tile, epi, 1000 + K if epi != "gelu" else 2000 + K) for K in KS]
    _gelu_share(stats, f"K sweep tile {tile}")


@pytest.mark.parametrize("tile,epi", TILES)
def test_linear_exact_m_sweep(tile, epi):
    """M from one row to just over one and two waves of 128-row tiles on every SM."""
    ms = MS + [128 * sms() + 1, 256 * sms() + 1]
    stats = [check_case(M, 136, 72, tile, epi, 3000 + M) for M in ms]
    _gelu_share(stats, f"M sweep tile {tile}")


@pytest.mark.parametrize("tile,epi", TILES)
def test_linear_exact_n_sweep(tile, epi):
    stats = [check_case(300, N, 200, tile, epi, 4000 + N) for N in NS]
    _gelu_share(stats, f"N sweep tile {tile}")


def _gelu_share(stats, what):
    stats = [s for s in stats if s is not None]
    if not stats:
        return
    n = sum(s[2] for s in stats)
    match = sum(s[0] * s[2] for s in stats) / n
    wrong = sum(s[1] * s[2] for s in stats) / n
    print(f"\nGELU {what}: exact matches {match:.5f} (GELU of the unrounded value would match {wrong:.3f})")
    assert match >= GELU_MATCH and match - wrong > 0.2, (match, wrong)


@pytest.mark.parametrize("K", [32, 40, 1152])
def test_linear_random_operands_bounded(K):
    rng = np.random.default_rng(K)
    for (M, N) in [(1, 8), (129, 1160), (300, 136)]:
        A = C.h(C.f32(rng.standard_normal((M, K))))
        W = C.h(C.f32(rng.standard_normal((N, K)) / math.sqrt(K)))
        b = C.h(C.f32(rng.standard_normal(N)))
        for tile in (0, 32, 128, 144, 192, 256):
            got, untouched = run_linear(A, W, b, 0, 1.0, tile)
            y = A @ W.T + b
            bound = C.ulp16(y) + K * 2.0 ** -23 * (np.abs(A) @ np.abs(W).T) + np.abs(b) * 2.0 ** -24
            frac = float((np.abs(got - y) / bound).max())
            print(f"\nrandom operands M={M} N={N} K={K} tile={tile}: worst element at {frac:.3f} of its bound")
            assert untouched and frac <= 1.0, (M, N, K, tile, frac)


def test_uninstantiated_tile_widths_fail_cleanly():
    """An explicit width with no kernel for its epilogue returns TPX_ERR_SHAPE with the message and writes nothing."""
    A, W, b = C.exact_linear(np.random.default_rng(5), 64, 64, 64)
    a, w, bb = d16(A), d16(W), d16(b)
    for tile, act in [(32, 1), (16, 0), (64, 0), (200, 0)]:
        out = sentinel16(64, 64)
        rc = lib().tpx_linear(a.data_ptr(), 64, w.data_ptr(), bb.data_ptr(), out.data_ptr(), 64, 64, 64, 64, act, 1.0, tile, st())
        torch.cuda.synchronize()
        assert rc == -3 and b"no kernel instantiated" in lib().tpx_last_error(), (tile, act, rc)
        assert torch.all(bits16(out) == S16)
    outs = [sentinel16(1, 2, 64, 80) for _ in range(3)]
    w = torch.zeros(3 * 144, 64, dtype=torch.float16, device="cuda")
    rc = lib().tpx_linear_heads(a.data_ptr(), 64, w.data_ptr(), None, outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), 64, 3 * 144,
                                64, 144, 2, 72, 80, 64, 1.0, 200, 2, 64, st())
    torch.cuda.synchronize()
    assert rc == -3 and all(torch.all(bits16(o) == S16) for o in outs), "a failed head-split call must not clear its outputs"


# ---- head split ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Dh,Nseq,tile,K", [(72, 64, 144, 72), (72, 64, 192, 200), (72, 64, 0, 32), (72, 100, 128, 72), (64, 100, 0, 72), (64, 64, 0, 32)])
def test_linear_heads_exact(Dh, Nseq, tile, K):
    """Bulk 24-column stores (Dh 72, Nseq % 32 == 0, tile 144 / 192) and the per-thread path (the others); V transposed with a row
    length past the sequence; q post-scaled.  Every element of the three outputs is pinned: the values, zeros in d >= Dh, zeros in the
    transposed V's token columns [Nseq, ld) on the bulk path (which clears the outputs first) and their old contents on the per-thread
    path (include/tpx.h); the elements after each output keep their sentinels."""
    B, H, DhP = 3, 8, 80
    D = H * Dh
    M, N = B * Nseq, 3 * D
    vt_ld = (Nseq + 8 + 7) // 8 * 8 + 8
    A, W, b = C.exact_linear(np.random.default_rng(Dh + Nseq + K), M, N, K)
    a, w, bb = strided_a(A, K + 8), d16(W), d16(b)
    tail = 64
    sizes = [B * H * Nseq * DhP, B * H * Nseq * DhP, B * H * DhP * vt_ld]
    bufs = [sentinel16(n + tail) for n in sizes]
    _lib.check(lib().tpx_linear_heads(a.data_ptr(), K + 8, w.data_ptr(), bb.data_ptr(), bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(),
                                      M, N, K, D, H, Dh, DhP, Nseq, POST_SCALE, tile, 2, vt_ld, st()), "tpx_linear_heads")
    torch.cuda.synchronize()
    y = C.acc_bias(A @ W.T, b).reshape(B, Nseq, 3, H, Dh)
    want = [np.zeros((B, H, Nseq, DhP)), np.zeros((B, H, Nseq, DhP)), np.zeros((B, H, DhP, vt_ld))]
    if not (Dh % 24 == 0 and Nseq % 32 == 0):
        want[2][..., Nseq:] = np.nan   # the per-thread path leaves the token columns [Nseq, ld) as they were: the sentinel
    want[0][..., :Dh] = C.linear_store(y[:, :, 0], POST_SCALE).transpose(0, 2, 1, 3)
    want[1][..., :Dh] = C.linear_store(y[:, :, 1]).transpose(0, 2, 1, 3)
    want[2][:, :, :Dh, :Nseq] = C.linear_store(y[:, :, 2]).transpose(0, 2, 3, 1)
    for i in range(3):
        got = host(bufs[i][:sizes[i]]).reshape(want[i].shape)
        keep = np.isnan(want[i])
        assert torch.all(bits16(bufs[i][:sizes[i]]).view(want[i].shape)[torch.from_numpy(keep).cuda()] == S16), f"output {i}: columns >= Nseq written"
        bad = (got != want[i]) & ~keep
        assert not bad.any(), f"output {i}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0]}"
        assert torch.all(bits16(bufs[i][sizes[i]:]) == S16), f"output {i}: written past its end"


# ---- gated residual ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tile,rpb,K", [(128, 100, 72), (144, 128, 72), (192, 100, 200), (0, 256, 32), (144, 100, 32)])
def test_linear_gated_exact(tile, rpb, K):
    """x0 + h(g h(y)), then the second launch's update, bit for bit: per-row gates (rows_per_batch 100: looked up per row) or per-tile
    gates (a multiple of 128: staged in shared memory), the % gate_batches wrap (5 row batches over 2 gate rows), ldx > N with
    sentinels in the padding columns and rows."""
    G, nb = 2, 5
    M, N = nb * rpb, 576
    A, W, b = C.exact_linear(np.random.default_rng(tile + rpb + K), M, N, K)
    x0, gate = C.gated_operands(np.random.default_rng(tile + rpb + K + 1), M, N, G)
    gstride = N + 40
    gbuf = torch.zeros(G, gstride, dtype=torch.float16, device="cuda")
    gbuf[:, :N] = d16(gate)
    ldx = N + 8
    x = torch.full((M + 2, ldx), S32, dtype=torch.int32, device="cuda").view(torch.float32)
    x[:M, :N] = torch.from_numpy(x0).float().cuda()
    a, w, bb = strided_a(A, K + 16), d16(W), d16(b)
    for _ in range(2):
        _lib.check(lib().tpx_linear_gated(a.data_ptr(), K + 16, w.data_ptr(), bb.data_ptr(), gbuf.data_ptr(), gstride, G, rpb, x.data_ptr(), ldx, M, N,
                                          K, tile, st()), "tpx_linear_gated")
    torch.cuda.synchronize()
    y = C.acc_bias(A @ W.T, b)
    g = gate[(np.arange(M) // rpb) % G]
    want = C.gated(C.gated(x0, g, y), g, y)
    got = host(x[:M, :N])
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} elements differ, first at {np.argwhere(bad)[0]}"
    mask = torch.ones(M + 2, ldx, dtype=torch.bool, device="cuda")
    mask[:M, :N] = False
    assert torch.all(x.view(torch.int32)[mask] == S32), "wrote outside [M, N]"


# ---- convolution -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,C_,Cout,P,resid", [(8, 32, 32, 3, False), (8, 32, 32, 5, True), (8, 256, 32, 3, True), (4, 32, 256, 3, False),
                                               (4, 256, 256, 5, False), (4, 256, 256, 3, True)])
def test_conv3d_k3_exact(S, C_, Cout, P, resid):
    """The halo kernel (S 8, Cout 32) and the implicit-GEMM conv (S 4, Cout 256), store and RESID_SCALE, every halo tap, bit for bit
    against the fp64 convolution with zero padding."""
    x, W, b = C.exact_conv3d(np.random.default_rng(S + C_ + Cout + P), P, S, C_, Cout)
    y = C.conv3d_ref(x, W, b)
    assert C.is_f32(y)
    r = C.resid_operand(np.random.default_rng(P), y.shape) if resid else None
    n = P * S ** 3 * Cout
    out = sentinel16(n + 64)
    xr, wr, br = d16(x), d16(W), d16(b)
    rr = d16(r) if resid else None
    _lib.check(lib().tpx_conv3d_k3(xr.data_ptr(), wr.data_ptr(), br.data_ptr(), _lib.ptr(rr), ALPHA if resid else 1.0, out.data_ptr(), P, S, C_, Cout,
                                   st()), "tpx_conv3d_k3")
    torch.cuda.synchronize()
    want = C.resid_scale(y, r, ALPHA) if resid else C.h(y)
    got = host(out[:n]).reshape(want.shape)
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} elements differ, first at {np.argwhere(bad)[0]}"
    assert torch.all(bits16(out[n:]) == S16)


# ---- LayerNorm-modulate ------------------------------------------------------------------------------------------------------
def run_ln(x, shift, scale, rows_per_batch=None, pre=None):
    rows, D = x.shape
    xd = torch.from_numpy(x).float().cuda()
    out = sentinel16(rows * D + 64)
    sh, sc = d16(shift[None]), d16(scale[None])
    pg = pc = None
    if pre is not None:
        pg, pc = d16(pre[0][None]), d16(pre[1])
    _lib.check(lib().tpx_ln_modulate(xd.data_ptr(), rows, D, 1e-6, sh.data_ptr(), sc.data_ptr(), D, rows, 1, out.data_ptr(), _lib.ptr(pg), _lib.ptr(pc),
                                     0, st()), "tpx_ln_modulate")
    torch.cuda.synchronize()
    assert torch.all(bits16(out[rows * D:]) == S16)
    return host(out[:rows * D]).reshape(rows, D), host(xd)


@pytest.mark.parametrize("D", list(range(128, 2049, 128)))
def test_ln_modulate_every_width(D):
    rng = np.random.default_rng(D)
    x, shift, scale = C.ln_operands(rng, 40, D)
    x[1] += 1000.0                                  # an offset row
    x[2] = 0.0                                       # a constant row (LN = 0: the output is the shift)
    x = C.f32(x)
    pre = None
    if D == 1152:                                    # the CFG pre-add: x += h(gate * const) in fp32 before the norm
        pre = (C.h(C.f32(rng.standard_normal(D))), C.h(C.f32(rng.standard_normal(D))))
    got, xnew = run_ln(x, shift, scale, pre=pre)
    if pre is not None:
        x = C.f32(x + C.h(C.f32(pre[0] * pre[1])))
        assert np.array_equal(xnew, x), "the pre-add must be written back to the residual"
    ln, m, want = C.ln_modulate(x, shift, scale, 1e-6)
    # plus the fp32 mean's own error (a lane's serial sum of D/32 terms, then a 5-level butterfly), which the offset row scales up
    sd = np.sqrt(((x - x.mean(-1, keepdims=True)) ** 2).mean(-1, keepdims=True) + 1e-6)
    e_mean = (D / 32 + 5) * 2.0 ** -24 * np.abs(x).max(-1, keepdims=True)
    bound = C.ulp16(want) + 2.0 ** -18 * (np.abs(ln * m) + np.abs(shift)) + np.abs(m) * e_mean / sd
    err = np.abs(got - want)
    print(f"\nln_modulate D={D}: worst element at {float((err / bound).max()):.3f} of its bound")
    assert np.all(err <= bound), (D, float((err / bound).max()))
    if pre is None:
        assert np.array_equal(got[2], C.h(C.f32(shift))), "constant row"
    match = np.mean(got == want)
    wrong = np.mean(got == C.wrong_ln_modulate(x, shift, scale, 1e-6))
    print(f"\nln_modulate D={D}: matches the contract on {match:.4f}, the unrounded (1 + scale) on {wrong:.4f}")
    assert match >= LN_MATCH and match - wrong > 0.15, (match, wrong)


# ---- attention ---------------------------------------------------------------------------------------------------------------
def attention_inputs(B, H, Nq, Nk, Dh, tile, seed, gap=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, H, Nq, Dh, generator=g, device="cuda", dtype=torch.float64)
    k = torch.randn(B, H, Nk, Dh, generator=g, device="cuda", dtype=torch.float64)
    v = torch.randn(B, H, Nk, Dh, generator=g, device="cuda", dtype=torch.float64)
    if gap:
        # rows with a large first component against keys whose first component flips sign after the first key tile: the logit gap
        # across tiles is about 470, so one side underflows to zero after the rescale (gap > 0: later tiles win; < 0: the first)
        q[:, :, ::2, 0] = 100.0
        k[:, :, :, 0] = 20.0 * (1 if gap > 0 else -1)
        k[:, :, :min(tile, Nk), 0] *= -1
    return q.half(), k.half(), v.half()


def attention_ref(q, k, v, scale):
    """fp64 softmax attention, its per-element bound terms, and the fp16-P policy (P = h(exp(s - max)), l = the unrounded sum)."""
    qd, kd, vd = q.double(), k.double(), v.double()
    s = scale * qd @ kd.transpose(-1, -2)
    e = torch.exp(s - s.amax(-1, keepdim=True))
    l = e.sum(-1, keepdim=True)
    pi = e / l
    o = pi @ vd
    Dh = q.shape[-1]
    eps_s = scale * Dh * 2.0 ** -24 * (qd.abs() @ kd.abs().transpose(-1, -2)).amax(-1, keepdim=True)
    bound = (2.0 ** -11 + 4 * eps_s + 2.0 ** -20) * (pi @ vd.abs()) + 2.0 ** -25 * vd.abs().sum(-2, keepdim=True) / l
    pol = ((e.float().half().double() @ vd) / l).float().half().double()
    return o, bound, pol


def check_attention(got, o, bound, pol, what):
    """got [B, Nq, H, Dh] against o [B, H, Nq, Dh]: per element, and per (b, head, 64-row query tile) against the policy."""
    got = got.double().permute(0, 2, 1, 3)
    frac, _ = parity.check_elementwise(f"{what}: per element", got, o, parity.ulp16(o) + bound)
    B, H, Nq, Dh = o.shape
    worst = parity.check(f"{what}: per query tile", *(t.reshape(B * H, Nq, Dh) for t in (got, pol, o)),
                         {"query tile": parity.block(64)})["query tile"]
    print(f"\n{what}: worst element at {frac:.3f} of its bound, worst query tile at {worst:.3f}")


NKS = [1, 8, 127, 128, 129, 2047, 2048, 2049]


@pytest.mark.parametrize("Nk", NKS)
@pytest.mark.parametrize("gap", [0, 1, -1])
def test_attention_tc_contract(Nk, gap):
    B, H, Nq, Dh, DhP = 1, 2, 130, 72, 80
    if gap and Nk < 129:
        pytest.skip("one key tile: no gap across tiles")
    scale = Dh ** -0.5
    q, k, v = attention_inputs(B, H, Nq, Nk, Dh, 128, Nk * 7 + gap, gap)
    nkp = (Nk + 7) // 8 * 8 + 8
    qp = torch.zeros(B, H, Nq, DhP, dtype=torch.float16, device="cuda")
    kp = torch.zeros(B, H, Nk, DhP, dtype=torch.float16, device="cuda")
    qp[..., :Dh], kp[..., :Dh] = q, k
    outs = []
    for fill in (0.0, 6e4):
        vT = torch.zeros(B, H, DhP, nkp, dtype=torch.float16, device="cuda")
        if fill:
            vT[:] = fill * (1 - 2 * (torch.arange(nkp, device="cuda") % 2)).half()   # +-6e4 everywhere, then the real block
        vT[:, :, :Dh, :Nk] = v.transpose(-1, -2)
        out = sentinel16(B * Nq * H * Dh + 64)
        _lib.check(lib().tpx_attention_tc(qp.data_ptr(), kp.data_ptr(), vT.data_ptr(), out.data_ptr(), B, H, Nq, Nk, nkp, Dh, scale, st()), "attention_tc")
        torch.cuda.synchronize()
        assert torch.all(bits16(out[B * Nq * H * Dh:]) == S16)
        outs.append(out[:B * Nq * H * Dh])
    assert torch.equal(bits16(outs[0]), bits16(outs[1])), "padding rows / key columns changed the output"
    o, bound, pol = attention_ref(q, k, v, scale)
    check_attention(outs[0].view(B, Nq, H, Dh), o, bound, pol, f"attention_tc Nk={Nk} gap={gap}")


@pytest.mark.parametrize("Nk", NKS)
@pytest.mark.parametrize("Dh,DhP,gap", [(72, 80, 0), (64, 64, 0), (72, 80, 1), (72, 80, -1), (30, 32, 0)])
def test_attention_contract(Nk, Dh, DhP, gap):
    """The mma.sync kernel.  Its padding contract (include/tpx.h): q and k columns d >= Dh must be zero (q k^T runs over all DhP);
    v columns d >= Dh never reach an output, so NaN there must leave the output bit-identical."""
    B, H, Nq = 2, 2, 130
    if gap and Nk < 65:
        pytest.skip("one key tile: no gap across tiles")
    scale = Dh ** -0.5
    q, k, v = attention_inputs(B, H, Nq, Nk, Dh, 64, Nk * 11 + Dh + gap, gap)
    pads = [torch.zeros(B, H, n, DhP, dtype=torch.float16, device="cuda") for n in (Nq, Nk, Nk)]
    for p_, t in zip(pads, (q, k, v)):
        p_[..., :Dh] = t
    outs = []
    for vfill in (0.0, float("nan")):
        vp = pads[2].clone()
        vp[..., Dh:] = vfill
        out = sentinel16(B * Nq * H * Dh + 64)
        _lib.check(lib().tpx_attention(pads[0].data_ptr(), pads[1].data_ptr(), vp.data_ptr(), out.data_ptr(), B, H, Nq, Nk, Dh, DhP, scale, st()),
                   "attention")
        torch.cuda.synchronize()
        assert torch.all(bits16(out[B * Nq * H * Dh:]) == S16)
        outs.append(out[:B * Nq * H * Dh])
    assert torch.equal(bits16(outs[0]), bits16(outs[1])), "v's padding columns reached the output"
    o, bound, pol = attention_ref(q, k, v, scale)
    check_attention(outs[0].view(B, Nq, H, Dh), o, bound, pol, f"attention Nk={Nk} Dh={Dh} gap={gap}")
