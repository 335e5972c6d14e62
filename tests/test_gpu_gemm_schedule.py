"""GPU: the ping-pong schedule of the wgmma GEMM (linear tiles 128 / 144: each consumer warpgroup owns whole tiles) against fp32 torch
math, and bit for bit against the cooperative schedule (tiles 192 / 256: both warpgroups share a tile), which sums every output element
over the same k-blocks in the same order."""
import pytest
import torch

from tpxl_b200 import _lib
from gpu_util import linear, linear_ref, rel_l2, st

pytestmark = pytest.mark.gpu

H, DH, DHP = 16, 72, 80
D = H * DH


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def heads(A, W, b, n_seq, post_scale=1.0, tile=0, vt=True):
    """tpx_linear_heads over [q | k | v] (or q alone when W has D rows); V transposed as [b, head, DhP, tokens] when vt."""
    M, K = A.shape
    nwhich = W.shape[0] // D
    B = M // n_seq
    outs = [torch.full((B, H, n_seq, DHP), 7.0, dtype=torch.float16, device="cuda") for _ in range(nwhich)]
    if vt and nwhich == 3:
        outs[2] = torch.full((B, H, DHP, n_seq), 7.0, dtype=torch.float16, device="cuda")
    ptrs = [o.data_ptr() for o in outs] + [None] * (3 - nwhich)
    _lib.check(_lib.lib().tpx_linear_heads(A.data_ptr(), K, W.data_ptr(), b.data_ptr(), *ptrs, M, W.shape[0], K, D, H, DH, DHP, n_seq, post_scale, tile,
                                           2 if (vt and nwhich == 3) else -1, n_seq, st()), "tpx_linear_heads")
    return outs


def heads_check(outs, A, W, b, n_seq, post_scale=1.0, vt=True):
    M = A.shape[0]
    ref = linear_ref(A, W, b).float().reshape(M // n_seq, n_seq, len(outs), H, DH)
    for w, got in enumerate(outs):
        r = ref[:, :, w].permute(0, 2, 1, 3)
        if w == 0 and post_scale != 1.0:
            r = (r * post_scale).half().float()
        if vt and w == 2:
            assert torch.all(got[:, :, DH:, :] == 0)
            got = got[:, :, :DH, :].transpose(-1, -2)
        else:
            assert torch.all(got[..., DH:] == 0)
            got = got[..., :DH]
        assert rel_l2(got, r) < 2e-3, w


def gated(A, W, b, gate, gate_bstride, gate_batches, rows_per_batch, x, tile=0, times=1):
    M, K = A.shape
    N = W.shape[0]
    for _ in range(times):
        _lib.check(_lib.lib().tpx_linear_gated(A.data_ptr(), K, W.data_ptr(), b.data_ptr(), gate.data_ptr(), gate_bstride, gate_batches, rows_per_batch,
                                               x.data_ptr(), N, M, N, K, tile, st()), "tpx_linear_gated")
    return x


def gated_update(A, W, b, gate_rows):
    return (gate_rows.float() * linear_ref(A, W, b).float()).half().float()


@pytest.mark.parametrize("tile", [128, 144])
@pytest.mark.parametrize("M,N", [(300, 1152), (1370, 1160)])
def test_store_gelu_and_post_scale(tile, M, N):
    """Ragged rows and (N = 1160) ragged columns; 128 takes the bulk-store epilogue, 144 the per-thread one."""
    K = 320
    A, W, b = _rand(M, K, seed=1), _rand(N, K, scale=K ** -0.5, seed=2), _rand(N, seed=3)
    s = DH ** -0.5
    for kw in (dict(), dict(act=1), dict(post_scale=s)):
        out = linear(A, W, b, tile_n=tile, **kw)
        assert rel_l2(out, linear_ref(A, W, b, **kw)) < 2e-3, kw


@pytest.mark.parametrize("tile", [128, 144])
def test_identity_exact(tile):
    M, K = 300, 288
    A = _rand(M, K, seed=4)
    out = linear(A, torch.eye(K, device="cuda").half(), None, tile_n=tile)
    torch.cuda.synchronize()
    assert torch.equal(out, A)


@pytest.mark.parametrize("tile", [128, 144])
def test_heads_transposed_v_and_scaled_q(tile):
    """144 stores 24-column head groups in bulk; 128 (not a multiple of 24) takes the per-thread head split."""
    B, N, K = 2, 256, 256
    A, W, b = _rand(B * N, K, seed=8), _rand(3 * D, K, scale=1 / 16, seed=9), _rand(3 * D, seed=10)
    s = DH ** -0.5
    heads_check(heads(A, W, b, N, s, tile), A, W, b, N, s)


@pytest.mark.parametrize("tile", [128, 144])
def test_gated_uniform_gate_two_launches(tile):
    """Sequences of 256 rows: the gate row is uniform over a tile (staged in shared memory); two launches accumulate."""
    B, N, K = 2, 256, 320
    A, W, b = _rand(B * N, K, seed=11), _rand(D, K, scale=K ** -0.5, seed=12), _rand(D, seed=13)
    gate = _rand(1, 3 * D, seed=14)[:, D:2 * D]
    x0 = torch.randn(B * N, D, device="cuda")
    x = gated(A, W, b, gate, 0, 1, N, x0.clone(), tile, times=2)
    upd = gated_update(A, W, b, gate)
    ref = (x0 + upd) + upd
    assert rel_l2(x, ref) < 1e-3 and (x - ref).abs().max() < 4e-2


@pytest.mark.parametrize("tile", [128, 144])
def test_gated_per_row_gate_ragged(tile):
    """Sequences of 200 rows (a tile straddles two gate rows) and N = 1160 (a partial last column tile)."""
    B, N, Dn, K = 3, 200, 1160, 192
    A, W, b = _rand(B * N, K, seed=51), _rand(Dn, K, scale=K ** -0.5, seed=52), _rand(Dn, seed=53)
    gate = _rand(B, Dn, seed=54)
    x0 = torch.randn(B * N, Dn, device="cuda")
    x = gated(A, W, b, gate, Dn, B, N, x0.clone(), tile, times=2)
    upd = gated_update(A, W, b, gate.repeat_interleave(N, 0))
    ref = (x0 + upd) + upd
    assert rel_l2(x, ref) < 1e-3 and (x - ref).abs().max() < 4e-2


@pytest.mark.parametrize("rounds", [0, 1, 2, 3])
def test_tiles_per_cta(rounds):
    """Fewer tiles than SMs (rounds 0), and tile counts just over 1 / 2 / 3 x the SM count, so CTAs hold one to four tiles and both
    odd and even counts occur.  Each result equals the cooperative schedule's bit for bit."""
    N, K = 1152, 256
    sms = _sms()
    mt = 2 if rounds == 0 else (rounds * sms) // 8 + 1          # 8 column tiles of 144 (9 of 128) per row of tiles
    M = 128 * mt - 40
    A, W, b = _rand(M, K, seed=21), _rand(N, K, scale=K ** -0.5, seed=22), _rand(N, seed=23)
    out = linear(A, W, b, act=1, tile_n=128)
    assert torch.equal(out, linear(A, W, b, act=1, tile_n=256))
    assert rel_l2(out, linear_ref(A, W, b, act=1)) < 2e-3
    gate = _rand(1, N, seed=24)
    x0 = torch.randn(M, N, device="cuda")
    x = gated(A, W, b, gate, 0, 1, M, x0.clone(), 144)
    assert torch.equal(x, gated(A, W, b, gate, 0, 1, M, x0.clone(), 192))
    assert rel_l2(x, x0 + gated_update(A, W, b, gate)) < 1e-3


def test_dit_shapes_match_fp32_and_the_cooperative_schedule():
    """The six linears of a DiT block at the headline size (2 x 2048 tokens with CFG, hidden 1152, MLP 4608) with the automatic tile,
    as dit_forward issues them: bit-equal to the cooperative schedule at 192 / 256 and within 2e-3 of fp32."""
    S, N, Dm = 2, 2048, 4 * D
    s = DH ** -0.5
    h = _rand(S * N, D, seed=31)
    hid = _rand(S * N, Dm, scale=0.5, seed=32)
    mod = _rand(1, 9 * D, seed=33)
    # cross q (sequence 0 only; the DiT passes 144), self qkv with transposed V
    for M, nw, tile in ((N, 1, 144), (S * N, 3, 0)):
        W, b = _rand(nw * D, D, scale=D ** -0.5, seed=34 + nw), _rand(nw * D, seed=36 + nw)
        A = h[:M]
        q_scale = s if nw == 1 else 1.0
        got = heads(A, W, b, N, q_scale, tile)
        heads_check(got, A, W, b, N, q_scale)
        for g, c in zip(got, heads(A, W, b, N, q_scale, 192)):
            assert torch.equal(g, c)
    # cross proj, self proj, fc2: gated residual with the batch-stride-0 gate row
    for M, A, K, seed in ((N, h[:N], D, 40), (S * N, h, D, 41), (S * N, hid, Dm, 42)):
        W, b = _rand(D, K, scale=K ** -0.5, seed=seed), _rand(D, seed=seed + 10)
        gate = mod[:, 2 * D:3 * D]
        x0 = torch.randn(M, D, device="cuda")
        x = gated(A, W, b, gate, 0, 1, N, x0.clone())
        assert torch.equal(x, gated(A, W, b, gate, 0, 1, N, x0.clone(), 192))
        assert rel_l2(x, x0 + gated_update(A, W, b, gate)) < 2e-3
    # fc1
    W1, b1 = _rand(Dm, D, scale=D ** -0.5, seed=43), _rand(Dm, seed=44)
    out = linear(h, W1, b1, act=1)
    assert torch.equal(out, linear(h, W1, b1, act=1, tile_n=256))
    assert rel_l2(out, linear_ref(h, W1, b1, act=1)) < 2e-3
