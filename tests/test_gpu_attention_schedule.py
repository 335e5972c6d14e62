"""GPU: the schedule of the wgmma attention kernel (two consumer warpgroups taking turns on the tensor cores, S_{j+1} = Q K_{j+1}^T
issued with P_j V_j so that a softmax runs under the other products) at the shapes it depends on: one key tile, a ragged last tile and
pipelines of one to three tiles; query counts that leave the second consumer of a CTA with no rows, which must still take every turn.
Against fp32 softmax attention, and bit for bit between two launches."""
import pytest
import torch

from tpxl_b200 import _lib
from gpu_util import rel_l2, st

pytestmark = pytest.mark.gpu

DHP = 80


def _inputs(B, H, Nq, Nk, Dh, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def mk(n):
        t = torch.zeros(B, H, n, DHP, dtype=torch.float16, device="cuda")
        t[..., :Dh] = torch.randn(B, H, n, Dh, generator=g, device="cuda").half()
        return t
    q, k, v = mk(Nq), mk(Nk), mk(Nk)
    NkPad = (Nk + 7) // 8 * 8
    vT = torch.zeros(B, H, DHP, NkPad, dtype=torch.float16, device="cuda")
    vT[..., :Nk] = v.transpose(-1, -2)
    return q, k, v, vT


def _attention_tc(q, k, vT, B, H, Nq, Nk, Dh):
    out = torch.full((B, Nq, H * Dh), 9.0, dtype=torch.float16, device="cuda")
    _lib.check(_lib.lib().tpx_attention_tc(q.data_ptr(), k.data_ptr(), vT.data_ptr(), out.data_ptr(), B, H, Nq, Nk, vT.shape[-1], Dh, Dh ** -0.5,
                                           st()), "tpx_attention_tc")
    return out


def _reference(q, k, v, B, Nq, H, Dh):
    s = torch.matmul(q.float(), k.float().transpose(-1, -2)) * Dh ** -0.5
    return torch.matmul(torch.softmax(s, -1), v.float())[..., :Dh].permute(0, 2, 1, 3).reshape(B, Nq, H * Dh)


@pytest.mark.parametrize("Dh", [72, 64])
@pytest.mark.parametrize("Nq", [1, 64, 65, 128, 129])
@pytest.mark.parametrize("Nk", [1, 8, 127, 128, 129, 255, 256, 257])
def test_tiles_and_idle_consumer(Nk, Nq, Dh):
    B, H = 2, 3
    q, k, v, vT = _inputs(B, H, Nq, Nk, Dh, seed=Nk * 1000 + Nq * 3 + Dh)
    out = _attention_tc(q, k, vT, B, H, Nq, Nk, Dh)
    ref = _reference(q, k, v, B, Nq, H, Dh)
    torch.cuda.synchronize()
    assert rel_l2(out.float(), ref) < 2e-3
    assert (out.float() - ref).abs().max() < 2e-2


@pytest.mark.parametrize("B,H,Nq,Nk,Dh", [(2, 16, 2048, 2048, 72), (1, 16, 2048, 1370, 72), (1, 12, 1374, 1374, 64)])
def test_two_launches_identical(B, H, Nq, Nk, Dh):
    """The DiT self / cross attention and the DINOv2 shape: the turn order does not change a bit of the output."""
    q, k, _, vT = _inputs(B, H, Nq, Nk, Dh, seed=5)
    a = _attention_tc(q, k, vT, B, H, Nq, Nk, Dh)
    b = _attention_tc(q, k, vT, B, H, Nq, Nk, Dh)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
