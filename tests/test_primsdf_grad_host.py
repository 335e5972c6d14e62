"""CPU: the PrimSDF gradient oracle and the host side of PrimSDF's backward.

tests/golden/primsdf_grad.npz holds what the REFERENCE's own models.primsdf.PrimSDF gives under CPU autograd (x, srt_param and
feat_param as leaves, a seeded upstream gradient over (sdf, tex, mat)), in training and eval mode, on the scene of primsdf.npz and
on a constructed dyadic scene with inf-norm ties, a point at a centre, points on voxel planes and uncovered points
(tests/golden/make_primsdf_grad_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import primsdf as po
from oracle import primsdf_grad as pg
from tpxl_b200 import _lib

GRADS = ("grad_x", "grad_srt", "grad_feat")


def scene(golden_dir, name):
    """(srt, feat, pts, S, G) of a fixture scene as fp32 tensors."""
    d = np.load(os.path.join(golden_dir, "primsdf_grad.npz"))
    if name == "base":
        b = np.load(os.path.join(golden_dir, "primsdf.npz"))
        srt, feat, pts, S = b["srt"], b["feat"], b["pts"], 8
    else:
        srt, feat, pts, S = d["cons_srt"], d["cons_feat"], d["cons_pts"], 5
    t = torch.from_numpy
    return t(srt), t(feat), t(pts), S, t(d[f"{name}_G"])


def want(golden_dir, name, mode):
    d = np.load(os.path.join(golden_dir, "primsdf_grad.npz"))
    return {k: torch.from_numpy(d[f"{name}_{mode}_{k}"]) for k in ("out",) + GRADS}


def autograd(x, srt, feat, G, S, inference):
    leaves = [t.clone().requires_grad_(True) for t in (x, srt, feat)]
    o = po.query(*leaves, S=S, inference=inference)
    out = torch.cat([o["sdf"], o["tex"], o["mat"]], 1)
    out.backward(G)
    return out.detach(), dict(zip(GRADS, [t.grad for t in leaves]))


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("name", ["base", "cons"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_oracle_autograd_reproduces_the_reference(golden_dir, name, mode):
    """oracle.primsdf.query under autograd against the reference module under autograd: the same operation sequence on the same
    CPU.  Bound 1e-6 relative L2 per gradient."""
    srt, feat, x, S, G = scene(golden_dir, name)
    ref = want(golden_dir, name, mode)
    out, got = autograd(x, srt, feat, G, S, mode == "eval")
    assert float((out - ref["out"]).abs().max()) <= 1e-6
    for k in GRADS:
        r = rel(got[k], ref[k])
        print(f"{name} {mode} {k}: rel-L2 {r:.2e}")
        assert r <= 1e-6, (k, r)


def random_scene(seed, K=12, S=4, n=300):
    g = torch.Generator().manual_seed(seed)
    srt = torch.cat([torch.rand(K, 1, generator=g) * 0.3 + 0.1, torch.rand(K, 3, generator=g) * 1.2 - 0.6], 1)
    feat = torch.randn(K, 6 * S ** 3, generator=g) * 0.7 + 0.3
    x = torch.rand(n, 3, generator=g) * 2 - 1
    return srt, feat, x, S, torch.randn(n, 6, generator=g)


@pytest.mark.parametrize("name", ["base", "cons", "random"])
@pytest.mark.parametrize("inference", [False, True])
def test_kernel_shaped_oracle_matches_fp64_autograd(golden_dir, name, inference):
    """query_backward (the kernel's passes, written out) against fp64 autograd through oracle.primsdf.query: the formulas are the
    derivative, ties included (the constructed scene has two- and three-axis inf-norm ties and a point at a centre)."""
    srt, feat, x, S, G = random_scene(3) if name == "random" else scene(golden_dir, name)
    srt, feat, x, G = (t.double() for t in (srt, feat, x, G))
    _, ref = autograd(x, srt, feat, G, S, inference)
    got = pg.query_backward(x, srt, feat, G, S=S, inference=inference)
    for k, g in zip(GRADS, got):
        r = rel(g, ref[k])
        print(f"{name} inference={inference} {k}: rel-L2 {r:.2e}")
        assert r <= 1e-10, (k, r)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__._load_build_module().build()
    return _lib.load_library()


P = 1 << 20     # non-null, 256-B aligned, never dereferenced


def _bwd(lib, **kw):
    a = dict(x=P, srt=P, feat=P, ws=P, n=8, K=2, S=8, dim_feat=6, grad=P, gx=P, gs=P, gf=P)
    a.update(kw)
    nbytes = lib.tpx_primsdf_grid_bytes(1024) if a["ws"] else 0
    return lib.tpx_primsdf_query_backward(a["x"], a["srt"], a["feat"], a["ws"], nbytes, a["n"], a["K"], a["S"], a["dim_feat"], 1, a["grad"], a["gx"],
                                          a["gs"], a["gf"], None)


def test_backward_entry_checks_arguments_then_the_device(lib):
    """Null inputs, negative n, dim_feat != 6, bad S / K, a grid with no primitives, misaligned srt: rejected before any CUDA call.
    Valid arguments (any of the three outputs may be null, and so may the grid) fail in the device guard without a GPU."""
    assert _bwd(lib, n=0, x=None) == 0                    # nothing to do
    bad = [dict(x=None), dict(srt=None), dict(feat=None), dict(grad=None), dict(n=-1), dict(dim_feat=4), dict(S=1), dict(S=33), dict(K=-1),
           dict(K=0), dict(srt=P + 4)]
    for kw in bad:
        assert _bwd(lib, **kw) in (-1, -3), kw            # TPX_ERR_ARG / TPX_ERR_SHAPE, never the device guard (-2)
        assert lib.tpx_last_error(), kw
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses must never reach a GPU")
    for kw in (dict(), dict(ws=None), dict(ws=None, K=0), dict(gx=None, gs=None), dict(gf=None), dict(gx=None, gs=None, gf=None)):
        rc = _bwd(lib, **kw)
        assert rc == -2 and b"cudaGetDevice" in lib.tpx_last_error(), (kw, rc, lib.tpx_last_error())


def test_module_stays_cuda_only_and_opt_in():
    """differentiable defaults to False; host tensors raise TpxError with and without it, grad enabled or not."""
    import tpxl_b200
    for diff in (False, True):
        m = tpxl_b200.PrimSDF(num_prims=4, prim_shape=4, differentiable=diff) if diff else tpxl_b200.PrimSDF(num_prims=4, prim_shape=4)
        assert m.differentiable is diff
        with pytest.raises(_lib.TpxError):
            m(torch.zeros(5, 3, requires_grad=True))
