"""CPU: the ray-march gradient oracle and the host side of RayMarcher's backward and subsampling.

tests/golden/raymarch_grad.npz holds what the REFERENCE's own pure-PyTorch ray-marcher (the block its gradcheck runs against the CUDA
backward, mvpraymarch.py:391-467) gives under autograd on two scenes, plus the pixel coordinates of its subsample_pixel_coords /
resize_pixel_coords (tests/golden/make_raymarch_grad_golden.py executed both from the reference on the CPU)."""
import os

import numpy as np
import pytest
import torch

from oracle import raymarch as rmo
from oracle import raymarch_grad as rmg
from tpxl_b200 import _lib, ray_marcher

GRADS = ("template_chlast", "primpos", "primrot", "primscale")


def _scene(golden_dir, name):
    d = np.load(os.path.join(golden_dir, "raymarch_grad.npz"))
    t = lambda k: torch.from_numpy(d[f"{name}_{k}"][0])  # noqa: E731
    args = [t("raypos"), t("raydir"), float(d[f"{name}_stepsize"]), t("tminmax")]
    params = [t("template_chlast"), t("primpos"), t("primrot"), t("primscale")]
    fade = (float(d[f"{name}_fadescale"]), float(d[f"{name}_fadeexp"]))
    want = {k: t(f"grad_{k}") for k in GRADS}
    return args, params, fade, t("rayrgba"), t("grad_rayrgba"), want


def _grads(fn, args, params, fade, G):
    leaves = [p.clone().requires_grad_(True) for p in params]
    out = fn(*args, *leaves, *fade)
    out.backward(G)
    return out.detach(), dict(zip(GRADS, [p.grad for p in leaves]))


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", ["sparse", "dense"])
def test_dense_oracle_gradients_match_the_reference_torch_marcher(golden_dir, name):
    """raymarch_dense under autograd against the reference block under autograd: the same operations on the same CPU, up to
    grid_sample's own trilinear arithmetic.  Measured: image 5.7e-7 max-abs (the sparse scene 2.4e-7, as the forward pin), gradients
    <= 7.1e-7 relative L2.  Bounds 1e-6 and 2e-6."""
    args, params, fade, rgba, G, want = _scene(golden_dir, name)
    out, got = _grads(rmo.raymarch_dense, args, params, fade, G)
    assert float((out - rgba).abs().max()) < 1e-6
    for k in GRADS:
        rel = _rel(got[k], want[k])
        print(f"{name} {k}: rel-L2 {rel:.2e}")
        assert rel < 2e-6, (k, rel)


@pytest.mark.parametrize("name", ["sparse", "dense"])
def test_kernel_shaped_oracle_gradients_match_the_dense_oracle_on_order_free_rays(golden_dir, name):
    """raymarch_grad (the CUDA kernel's structure: per-warp hit lists, first step before the first hit, stop at saturation, strictly
    inside test) against raymarch_dense under autograd.  The step positions are the same lattice t0 + i dt reached by a different sum,
    so they differ in the last bits; measured: gradients <= 1.3e-6 relative L2 on both scenes.  Bound 1e-5.

    The dense marcher visits primitives in ascending index, the kernel's structure in the "fixedorder" tree's leaf order (K = 6:
    2..5, 0, 1; K = 10: 6..9, 0..5).  With its visiting order set to ascending, raymarch_grad matches the dense marcher on the whole
    image and all gradients.  In the tree order the two differ only on rays whose saturating step is inside two or more primitives, so
    there the image is compared on the other rays and the upstream gradient is zero on those rays."""
    args, params, fade, rgba, G, want = _scene(golden_dir, name)
    out_d, dense = _grads(rmo.raymarch_dense, args, params, fade, G)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(rmo, "fixedorder_visit", lambda K: list(range(K)))
        out_a, asc = _grads(rmg.raymarch_grad, args, params, fade, G)
    assert float((out_a - out_d).abs().max()) < 1.3e-6
    for k in GRADS:
        rel = _rel(asc[k], dense[k])
        print(f"{name} ascending {k}: rel-L2 {rel:.2e}")
        assert rel < 1e-5, (k, rel)

    order_free = rmo.saturating_overlap(*args, *params, *fade) < 2
    out_k, kern = _grads(rmg.raymarch_grad, args, params, fade, G)
    err = (out_k - out_d).abs().amax(-1)
    print(f"{name}: order-dependent rays {int((~order_free).sum())} of {order_free.numel()}, image max-abs there {float(err[~order_free].amax()) if bool((~order_free).any()) else 0.0:.2e}")
    assert float(order_free.float().mean()) > 0.5
    assert float(err[order_free].max()) < 1.3e-6
    G = G * order_free[..., None]
    out_d, dense = _grads(rmo.raymarch_dense, args, params, fade, G)
    out_k, kern = _grads(rmg.raymarch_grad, args, params, fade, G)
    for k in GRADS:
        rel = _rel(kern[k], dense[k])
        print(f"{name} {k}: rel-L2 {rel:.2e}")
        assert rel < 1e-5, (k, rel)


def test_kernel_shaped_oracle_forward_is_raymarch():
    """raymarch_grad's image is raymarch's, bit for bit (only the autograd treatment of the discrete part differs)."""
    g = torch.Generator().manual_seed(4)
    K, S, H, W = 12, 4, 20, 13
    pos = (torch.rand(1, K, 3, generator=g) - 0.5) * 0.8
    scale = 1.0 / (0.15 + 0.1 * torch.rand(1, K, 1, generator=g)).repeat(1, 1, 3)
    rgba = torch.rand(1, K, S, S, S, 4, generator=g) * torch.tensor([255.0, 255.0, 255.0, 60.0])
    rot = torch.linalg.qr(torch.randn(1, K, 3, 3, generator=g))[0]
    RT = torch.tensor([[[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, 3.0]]])
    Kc = torch.tensor([[[2.4 * W, 0, W / 2], [0, 2.4 * W, H / 2], [0, 0, 1.0]]])
    cam = rmo.convert_camera_parameters(RT, Kc)
    focal = torch.diagonal(cam["focal"], dim1=1, dim2=2)
    raypos, raydir, tmm = rmo.compute_raydirs(cam["campos"], cam["camrot"], focal, cam["princpt"], H, W, 1.0)
    args = (raypos[0], raydir[0], 0.02, tmm[0], rgba[0], pos[0], rot[0], scale[0])
    assert torch.equal(rmg.raymarch_grad(*args), rmo.raymarch(*args))
    pix = _pixel_grid(H, W)
    assert all(torch.equal(a, b) for a, b in zip(rmg.compute_raydirs_at(cam["campos"], cam["camrot"], focal, cam["princpt"], pix, 1.0),
                                                 (raypos, raydir, tmm)))


def _pixel_grid(H, W):
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return torch.stack([xs, ys], -1)[None]


def test_host_offset_draw_reproduces_the_reference_pixel_coords(golden_dir):
    """subsample_offsets / offset_pixel_coords against the reference's subsample_pixel_coords (training: torch.randint(0, f - 1) for x0
    then y0, per image, on the default generator) and resize_pixel_coords (eval: f // 2), exactly, and with the same generator state
    afterwards."""
    d = np.load(os.path.join(golden_dir, "raymarch_grad.npz"))
    B, H, W = (int(v) for v in d["pix_hw"])
    base = ray_marcher.RayMarcher(H, W, 1.0).base_pixel_coords
    torch.manual_seed(int(d["pix_seed"]))
    for f in (2, 3, 4):
        offs = ray_marcher.subsample_offsets(B, f, True)
        assert all(0 <= x <= max(f - 2, 0) and 0 <= y <= max(f - 2, 0) for x, y in offs)
        assert np.array_equal(ray_marcher.offset_pixel_coords(base, offs, f).numpy(), d[f"pix_train_f{f}"]), f
        ev = ray_marcher.offset_pixel_coords(base, ray_marcher.subsample_offsets(B, f, False), f)
        assert np.array_equal(ev.numpy(), d[f"pix_eval_f{f}"]), f


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__._load_build_module().build()
    return _lib.load_library()


P = 1 << 20     # non-null, 256-B aligned, never dereferenced


def _fwd(lib, **kw):
    a = dict(tpl=P, N=1, K=2, S=8, H=8, W=8, stride=1, offsets=None, out=P, raysat=None)
    a.update(kw)
    return lib.tpx_raymarch_forward(a["tpl"], P, P, P, P, P, P, P, a["N"], a["K"], a["S"], a["H"], a["W"], 1.0, 0.01, 8.0, 8.0, a["stride"], a["offsets"],
                                    a["out"], a["raysat"], None)


def _bwd(lib, **kw):
    a = dict(tpl=P, N=1, K=2, S=8, H=8, W=8, stride=1, raysat=P, grad=P, gt=P, gp=P, gr=P, gs=P)
    a.update(kw)
    return lib.tpx_raymarch_backward(a["tpl"], P, P, P, P, P, P, P, a["N"], a["K"], a["S"], a["H"], a["W"], 1.0, 0.01, 8.0, 8.0, a["stride"], None,
                                     a["raysat"], a["grad"], a["gt"], a["gp"], a["gr"], a["gs"], None)


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_raymarch_entries_reject_bad_arguments(lib, call):
    """Null pointers, N > 65535, stride < 1, a stride that leaves no pixel, misaligned template / gradients: rejected before any CUDA
    call.  Valid arguments fail in the device guard (no GPU here), after the argument checks."""
    bad = [dict(tpl=None), dict(N=65536), dict(N=0), dict(stride=0), dict(stride=9), dict(H=4, stride=5), dict(tpl=P + 4)]
    bad += [dict(out=None), dict(out=P + 8)] if call is _fwd else [dict(raysat=None), dict(grad=None), dict(gt=None), dict(gp=None), dict(gr=None),
                                                                    dict(gs=None), dict(grad=P + 4), dict(gt=P + 8)]
    for kw in bad:
        assert call(lib, **kw) in (-1, -3), kw        # TPX_ERR_ARG / TPX_ERR_SHAPE, never the device guard (-2)
        assert lib.tpx_last_error(), kw
    if torch.cuda.is_available():
        pytest.skip("the dummy device addresses must never reach a GPU")
    for kw in (dict(), dict(stride=2), dict(stride=8)) + ((dict(offsets=P, raysat=P),) if call is _fwd else ()):
        rc = call(lib, **kw)
        assert rc == -2 and b"cudaGetDevice" in lib.tpx_last_error(), (kw, rc, lib.tpx_last_error())


def test_raymarcher_checks_before_the_device():
    """The mirror's host checks: blocksize, CPU tensors, and a subsample factor that leaves no pixel."""
    import tpxl_b200
    z = (torch.zeros(1, 2, 4, 4, 4, 4), torch.zeros(1, 2, 3), torch.eye(3).expand(1, 2, 3, 3), torch.ones(1, 2, 3), torch.eye(3)[None],
         torch.zeros(1, 3, 4))
    with pytest.raises(NotImplementedError):
        tpxl_b200.RayMarcher(8, 8, 1.0, blocksize=(16, 8))(*z)
    with pytest.raises(_lib.TpxError):
        tpxl_b200.RayMarcher(8, 8, 1.0, ray_subsample_factor=2)(*z)


def _heap_walk(K):
    """ray_subset_fixedbvh's traversal of build_accel(fixedorder=True)'s tree with every node box hit: an explicit stack seeded with
    the sentinel -1, node 0 first; node i >= K - 1 is the leaf of primitive i - (K - 1), appended when reached; an inner node goes to
    its left child 2i + 1 and pushes its right child 2i + 2."""
    out, stack, node = [], [-1], 0
    while node != -1:
        if node >= K - 1:
            out.append(node - (K - 1))
            node = stack.pop()
        else:
            stack.append(2 * node + 2)
            node = 2 * node + 1
    return out


def test_fixedorder_visit_is_the_reference_tree_walk():
    """The order the kernel and both oracles list primitives in (ascending rotated by 2^ceil(log2 K) - K) is the reference's depth-first
    walk of its fixed-order tree, for every K from 1 to 4096; ascending exactly when K is a power of two."""
    for K in range(1, 4097):
        walk = _heap_walk(K)
        assert rmo.fixedorder_visit(K) == walk, K
        assert (walk == list(range(K))) == (K & (K - 1) == 0), K
    assert _heap_walk(600)[:2] == [424, 425] and _heap_walk(3) == [1, 2, 0]
