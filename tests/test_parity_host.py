"""CPU: the parity rule of tests/parity.py on hand-built tensors: what each partition groups, where the bound lies, that non-finite
values fail every check, and the fp16 spacing and fp32-tie helpers."""
import numpy as np
import pytest
import torch

import parity
from oracle import contract as C
from oracle.primsdf import local_grid
from test_gpu_dit_stages import _check_with_null_half

S, N, CH, DH = 2, 300, 12, 4
CLASS = torch.tensor([0] + [-1] * (N - 1))
# name -> (partition, its part sizes on ones [S, N, CH])
PARTS = {
    "sequence": (parity.sequence, [N * CH] * S),
    "row": (parity.row, [CH] * (S * N)),
    "channel": (parity.channel, [S * N] * CH),
    "block": (parity.block(128), [128 * CH, 128 * CH, 44 * CH] * S),
    "head": (parity.head(DH), [N * DH] * (S * CH // DH)),
    "class": (parity.tokens(CLASS), [CH] * S),
    "pooled": (parity.pooled(torch.arange(N) % 3), [S * N * CH // 3] * 3),
}


def _triple(seed, shape=(S, N, CH)):
    """(ours, policy, exact): exact away from zero, the policy 1e-3 off it, ours equal to the policy."""
    g = torch.Generator().manual_seed(seed)
    ref = (torch.rand(shape, generator=g, dtype=torch.float64) + 0.5) * torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    pol = ref * (1 + 1e-3 * torch.randn(shape, generator=g, dtype=torch.float64))
    return pol.clone(), pol, ref


@pytest.mark.parametrize("name", list(PARTS))
def test_partition_sizes(name):
    part, sizes = PARTS[name]
    assert part(torch.ones(S, N, CH, dtype=torch.float64)).tolist() == sizes


@pytest.mark.parametrize("name", list(PARTS))
def test_one_element_moves_one_partition(name):
    part, _ = PARTS[name]
    ours, pol, ref = _triple(1)
    o0, p0 = parity.ratios(ours, pol, ref, part)
    assert torch.equal(o0, p0)
    for s, n, c in ((0, 0, 0), (1, 0, 7), (1, 299, 11), (0, 200, 5)):
        if name == "class" and n != 0:
            continue
        bad = ours.clone()
        bad[s, n, c] *= 1.5
        o1, p1 = parity.ratios(bad, pol, ref, part)
        assert torch.equal(p1, p0) and int((o1 != o0).sum()) == 1, (s, n, c)


def test_voxel_classes():
    assert torch.bincount(parity.boundary_count(4)).tolist() == [8, 24, 24, 8]
    assert torch.bincount(parity.boundary_count(8)).tolist() == [216, 216, 72, 8]
    assert torch.bincount(parity.face_class(4)).tolist() == [8, 19, 19, 18]
    # voxel v = (z S + y) S + x: (0, 1, 2) is on the low face z = 0 only; (3, 3, 1) on the high faces only; (0, 3, 3) a corner
    assert [int(parity.face_class(4)[(z * 4 + y) * 4 + x]) for z, y, x in ((0, 1, 2), (3, 3, 1), (0, 3, 3), (1, 2, 1))] == [1, 2, 3, 0]
    assert [int(parity.boundary_count(4)[(z * 4 + y) * 4 + x]) for z, y, x in ((0, 1, 2), (3, 3, 1), (0, 3, 3), (1, 2, 1))] == [1, 2, 3, 0]


def test_channels_last_round_trip():
    x = torch.arange(2 * 3 * 4 ** 3).reshape(2, 3, 4, 4, 4)
    cl = parity.to_cl(x)
    assert cl.shape == (2, 64, 3) and int(cl[1, (2 * 4 + 1) * 4 + 3, 2]) == int(x[1, 2, 2, 1, 3])
    assert torch.equal(parity.to_ncdhw(cl), x)


@pytest.mark.parametrize("name", list(PARTS))
def test_bound_edge(name):
    """Every part at 0.99 x the bound passes, at 1.01 x fails; with the policy's error 1e-3 and with it zero (the floor)."""
    part = {name: PARTS[name][0]}
    ref = torch.ones(S, N, CH, dtype=torch.float64)
    for p in (1e-3, 0.0):
        pol = ref * (1 + p)
        for f, ok in ((0.99, True), (1.01, False)):
            ours = ref * (1 - f * parity.bound(p))
            assert parity.rejects(ours, pol, ref, part) is not ok, (p, f)
            if ok:
                assert abs(parity.check(name, ours, pol, ref, part)[name] - f) < 1e-9
            else:
                with pytest.raises(AssertionError, match="exceed the bound"):
                    parity.check(name, ours, pol, ref, part)


def test_shapes_must_match():
    ours, pol, ref = _triple(2)
    with pytest.raises(AssertionError, match="shapes differ"):
        parity.check("x", ours[:, :-1], pol, ref, {"sequence": parity.sequence})


NON_FINITE = [float("nan"), float("inf"), float("-inf")]


@pytest.mark.parametrize("value", NON_FINITE, ids=str)
@pytest.mark.parametrize("which", [0, 1, 2], ids=["ours", "policy", "exact"])
def test_non_finite_fails_check(which, value):
    t = list(_triple(3))
    parts = {h: PARTS[h][0] for h in PARTS}
    parity.check("finite", *t, parts)
    t[which] = t[which].clone()
    t[which][1, 137, 5] = value
    assert parity.rejects(*t, parts)
    with pytest.raises(AssertionError, match="non-finite"):
        parity.check("one non-finite element", *t, parts)


@pytest.mark.parametrize("value", NON_FINITE, ids=str)
@pytest.mark.parametrize("which", [0, 1, 2], ids=["ours", "want", "tol"])
def test_non_finite_fails_check_elementwise(which, value):
    g = torch.Generator().manual_seed(4)
    want = torch.randn(40, 7, generator=g).half().double()
    t = [want + 0.5 * parity.ulp16(want), want, parity.ulp16(want)]
    assert parity.check_elementwise("finite", *t) == (0.5, 280)
    t[which] = t[which].clone()
    t[which][17, 3] = value
    with pytest.raises(AssertionError, match="1 elements off"):
        parity.check_elementwise("one non-finite element", *t)


def _null_half_triple(B, seed):
    """DiT increments of B conditional sequences and B null-context ones (each channel constant over the tokens there)."""
    ours, pol, ref = _triple(seed, (2 * B, 160, 64))
    for t in (ours, pol, ref):
        t[B:] = t[B:, :1]
    return ours, pol, ref


@pytest.mark.parametrize("value", NON_FINITE, ids=str)
@pytest.mark.parametrize("which", [0, 1, 2], ids=["ours", "policy", "exact"])
@pytest.mark.parametrize("seq", [0, 1])
def test_non_finite_fails_the_null_half_check(seq, which, value):
    t = list(_null_half_triple(1, 5))
    _check_with_null_half(("host", "null half"), *t, 1)
    t[which] = t[which].clone()
    t[which][seq, 9, 3] = value
    with pytest.raises(AssertionError):
        _check_with_null_half(("host", "null half"), *t, 1)


def test_null_half_channel_mean():
    """One null-half channel of ours off the policy's by a few of its ulps fails the mean check; within one ulp passes."""
    ours, pol, ref = _null_half_triple(1, 6)
    ulp = parity.ulp16(pol[1, 0, 3])
    ours[1:, :, 3] += ulp
    _check_with_null_half(("host", "null mean"), ours, pol, ref, 1)
    ours[1:, :, 3] += 9 * ulp
    with pytest.raises(AssertionError, match="null-half channel means"):
        _check_with_null_half(("host", "null mean"), ours, pol, ref, 1)


def test_ulp16_matches_the_contract_on_every_finite_fp16_value():
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.float16)
    x = x[torch.isfinite(x)]
    assert x.numel() == 63488 and bool((x == 0).sum() == 2)
    got = parity.ulp16(x)
    assert got.dtype == torch.float64
    assert np.array_equal(got.numpy(), C.ulp16(x.double().numpy()))
    assert float(parity.ulp16(torch.tensor(1.0))) == 2.0 ** -10 and float(parity.ulp16(torch.tensor(-0.0))) == 2.0 ** -24


def test_is_fp32_tie():
    S = 8
    srt = torch.tensor([[0.1, -0.5, 0.0, 0.0], [0.1, 0.5, 0.0, 0.0]], dtype=torch.float64)
    assert parity.is_fp32_tie(torch.tensor([0.0, 0.3, -0.2], dtype=torch.float64), srt, S)         # equidistant primitives
    assert not parity.is_fp32_tie(torch.tensor([0.1, 0.3, 0.2], dtype=torch.float64), srt, S)
    one = srt[1:]
    g = one[0, 1:] + one[0, 0] * local_grid(S).double()
    assert parity.is_fp32_tie((g[0] + g[1]) / 2, one, S)                          # equidistant voxels
    assert not parity.is_fp32_tie(g[0] + 0.3 * (g[1] - g[0]), one, S)


def test_fp32_ties_is_is_fp32_tie_per_point():
    """The batched form agrees with is_fp32_tie point by point: random points, constructed primitive and voxel ties, a negative
    scale (the box and the voxel grid are mirrored, the candidates the same), and a single primitive."""
    S = 8
    g = torch.Generator().manual_seed(3)
    srt = torch.cat([0.05 + 0.1 * torch.rand(40, 1, generator=g), torch.rand(40, 3, generator=g) * 1.6 - 0.8], 1).double()
    srt[7, 0] *= -1
    srt[1, 1:] = srt[0, 1:] + torch.tensor([0.3, 0.0, 0.0], dtype=torch.float64)
    vox = srt[7, 1:] + srt[7, 0] * local_grid(S).double()
    p = torch.cat([torch.rand(300, 3, generator=g).double() * 2.4 - 1.2,
                   (srt[0, 1:] + torch.tensor([0.15, 0.02, -0.01], dtype=torch.float64))[None],     # equidistant from primitives 0 and 1
                   ((vox[9] + vox[10]) / 2)[None] + 1e-9])
    want = torch.tensor([parity.is_fp32_tie(q, srt, S) for q in p])
    assert bool(want[-2]) and torch.equal(parity.fp32_ties(p, srt, S, chunk=64), want)
    assert torch.equal(parity.fp32_ties(p, srt[:1], S), torch.tensor([parity.is_fp32_tie(q, srt[:1], S) for q in p]))


def test_same_mesh_compares_bytes():
    V = np.array([[0.0, 1.0, 2.0], [3.0, 4.0, 5.0], [6.0, 7.0, 8.0]], np.float32)
    F = np.array([[0, 1, 2]], np.int64)
    parity.same_mesh((torch.from_numpy(V.copy()), torch.from_numpy(F.copy())), (V, F), "equal")
    neg = V.copy()
    neg[0, 0] = -0.0
    with pytest.raises(AssertionError, match="vertex bytes differ"):
        parity.same_mesh((torch.from_numpy(neg), torch.from_numpy(F.copy())), (V, F), "signed zero")
    with pytest.raises(AssertionError, match="faces differ"):
        parity.same_mesh((torch.from_numpy(V.copy()), torch.from_numpy(F[:, ::-1].copy())), (V, F), "order")
