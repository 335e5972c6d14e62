"""-m gpu: tpxl_b200.RayMarcher against THE REFERENCE'S OWN ray marcher, ``dva.ray_marcher.RayMarcher`` over its own CUDA extensions
(compute_raydirs from utilslib, mvpraymarch "fixedorder" and its backward from mvpraymarchlib), running on the same H100.

The reference's Python wrappers are byte-identical staged copies under ``oracle/_ref/`` and its extensions are compiled from the
reference's sources for sm_90a with their own flags (recipe: oracle/stage_ref.py; loader: oracle.refmods.load_raymarcher).  Both
modules get the same inputs and camera; each is called once per case with autograd on, and the image and, under one seeded upstream
gradient, the gradients of prim_rgba, prim_pos, prim_rot and prim_scale are compared.  The reference's backward is its CUDA backward
through its own autograd Function.

Tolerances.  Both sides are fp32 with fast exp / pow; the reference's mvpraymarch is also built with approximate division and sqrt
and flushes denormals to zero, and its hit list comes from a tree walk where ours comes from a cone cull plus the same exact slab
test, so a grazing ray can flip a slab test, an inside test or its start step.  Bounds (the largest figures measured on one H100 80GB
HBM3 at 700 W are in DESIGN.md §2):
    image       relative L2 <= 2e-5; at most PIX_SHARE of the pixels off by more than 1e-3 of the channel's value range, none by more
                than PIX_MAX of it;
    gradients   relative L2 <= 1e-4 and cosine >= 1 - 1e-6, per tensor.
"""
import pytest
import torch

import tpxl_b200
from oracle import raymarch as rmo
from oracle import refmods

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not refmods.raymarcher_available(),
                                                  reason="the reference's ray marcher is not built (python oracle/stage_ref.py where the reference checkout exists)")]

NAMES = ("prim_rgba", "prim_pos", "prim_rot", "prim_scale")
IMG_REL, PIX_SHARE, PIX_MAX = 2e-5, 1e-3, 2e-2
GRAD_REL, GRAD_COS = 1e-4, 1 - 1e-6


def _rotations(g, N, K):
    return torch.linalg.qr(torch.randn(N, K, 3, 3, generator=g))[0]


def _scene(K, S, seed, rot=False, N=1, alpha=60.0, ps=1.0, aniso=False):
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(N, K, 3, generator=g) - 0.5) * ps
    if aniso:
        scale = 1.0 / (0.06 + 0.2 * torch.rand(N, K, 3, generator=g))
    else:
        scale = 1.0 / (0.12 + 0.1 * torch.rand(N, K, 1, generator=g)).repeat(1, 1, 3)
    R = _rotations(g, N, K) if rot else torch.eye(3)[None, None].repeat(N, K, 1, 1)
    rgba = torch.rand(N, K, 4, S, S, S, generator=g)
    rgba[:, :, :3] *= 255.0
    rgba[:, :, 3] *= alpha
    return rgba, pos, R, scale


def _camera(H, W, z, N=1, f=2.4):
    """Looking down -z from (0, 0, z) (world units)."""
    RT = torch.tensor([[[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, z]]]).repeat(N, 1, 1)
    Kc = torch.tensor([[[f * W, 0, W / 2], [0, f * W, H / 2], [0, 0, 1.0]]]).repeat(N, 1, 1)
    return Kc, RT


VR = 100.0
# name: (K, S, H, W, rot, N, alpha, pos scale), the scenes of test_gpu_raymarch_grad.py; seed 5 K + H
BASE = {
    "small": (24, 4, 32, 24, False, 1, 60.0, 1.0),
    "rotated": (40, 8, 33, 21, True, 1, 60.0, 1.0),
    "over_cap": (600, 4, 16, 16, False, 1, 60.0, 0.2),
    "saturating": (48, 4, 24, 24, True, 1, 400.0, 0.6),
    "two_images": (30, 4, 20, 28, True, 2, 120.0, 1.0),
}


def _base(name, K=None):
    K0, S, H, W, rot, N, alpha, ps = BASE[name]
    rgba, pos, R, scale = _scene(K0 if K is None else K, S, 5 * K0 + H, rot, N, alpha, ps)
    Kc, RT = _camera(H, W, 3.0 * VR, N)
    return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=H, W=W, vr=VR)


def _shipped(N=1, H=518, W=518):
    """2048 primitives of 8^3 at volradius 1e4, dt 1 (configs/inference_dit.yml), seen by the preview camera."""
    K, S, vr = 2048, 8, 10000.0
    g = torch.Generator().manual_seed(3)
    d = torch.randn(N, K, 3, generator=g)
    pos = d / d.norm(dim=-1, keepdim=True) * 0.5
    scale = torch.full((N, K, 3), 1.0 / 0.05)
    rgba = torch.rand(N, K, 4, S, S, S, generator=g) * 255.0
    rgba[:, :, 3] = 255.0 * torch.exp(-(torch.rand(N, K, S, S, S, generator=g) * 0.02 / 0.005) ** 2)
    R = torch.eye(3)[None, None].repeat(N, K, 1, 1)
    RT = torch.tensor([[[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, 5 * vr]]]).repeat(N, 1, 1)
    Kc = torch.tensor([[[2084.9526697685183 * H / 1024, 0, 512.0 * H / 1024], [0, 2084.9526697685183 * W / 1024, 512.0 * W / 1024], [0, 0, 1.0]]]).repeat(N, 1, 1)
    return dict(rgba=rgba, pos=pos * vr, R=R, scale=scale, Kc=Kc, RT=RT, H=H, W=W, vr=vr)


def _custom(name):
    if name == "K1":
        return _base("small", K=1)
    if name == "K3":
        return _base("saturating", K=3)
    if name == "anisotropic":
        rgba, pos, R, scale = _scene(40, 8, 211, rot=True, alpha=200.0, aniso=True)
        Kc, RT = _camera(33, 21, 3.0 * VR)
        return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=33, W=21, vr=VR)
    if name == "camera_in_cube":
        rgba, pos, R, scale = _scene(40, 4, 223, rot=True, alpha=120.0)
        Kc, RT = _camera(24, 24, 0.8 * VR, f=0.6)
        return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=24, W=24, vr=VR)
    if name == "camera_in_primitive":
        rgba, pos, R, scale = _scene(20, 4, 227, rot=True, alpha=120.0)
        pos[0, 0] = torch.tensor([0.02, -0.03, 0.75])           # the camera (0, 0, 0.75) is inside primitive 0 (half-size >= 0.12)
        Kc, RT = _camera(24, 24, 0.75 * VR, f=0.6)
        return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=24, W=24, vr=VR)
    if name == "behind_camera":
        rgba, pos, R, scale = _scene(48, 4, 229, rot=True, alpha=120.0)
        Kc, RT = _camera(24, 24, 0.0, f=0.5)                     # at the centre of the cloud: half of it is behind the camera
        return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=24, W=24, vr=VR)
    if name == "past_cache":
        rgba, pos, R, scale = _scene(250, 4, 233, rot=False, alpha=20.0, ps=0.25)
        Kc, RT = _camera(16, 16, 3.0 * VR)
        return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=16, W=16, vr=VR)
    if name == "over_cap_2048":
        rgba, pos, R, scale = _scene(2048, 4, 239, rot=False, alpha=4.0, ps=0.3)
        Kc, RT = _camera(16, 16, 3.0 * VR)
        return dict(rgba=rgba, pos=pos * VR, R=R, scale=scale, Kc=Kc, RT=RT, H=16, W=16, vr=VR)
    raise KeyError(name)


def _listed_per_warp(sc):
    """Per-warp count of primitives whose box a ray of the warp meets (before the cap), from the oracle's slab test, batch element 0."""
    cam = rmo.convert_camera_parameters(sc["RT"], sc["Kc"])
    raypos, raydir, _ = rmo.compute_raydirs(cam["campos"], cam["camrot"], torch.diagonal(cam["focal"], dim1=1, dim2=2), cam["princpt"], sc["H"], sc["W"], sc["vr"])
    hit = rmo.slab_hits(raypos[0], raydir[0], sc["pos"][0] / sc["vr"], sc["R"][0], sc["scale"][0])[0]
    K = hit.shape[0]
    return rmo.hit_lists(hit, maxhitboxes=K)[1].sum(1)


def _run(module, sc, G, seed):
    leaves = [sc[k].cuda().contiguous().requires_grad_(True) for k in ("rgba", "pos", "R", "scale")]     # the reference asserts contiguity
    torch.manual_seed(seed)
    res = module(*leaves, sc["Kc"].cuda(), sc["RT"].cuda())
    out = res["rgba_image"]
    out.backward(G(out.shape).cuda())
    torch.cuda.synchronize()
    return out.detach(), res["pixel_coords"], [t.grad for t in leaves]


def _check(what, sc, f=1, training=False, seed=5):
    kw = dict(dt=1.0, ray_subsample_factor=f)
    ours = tpxl_b200.RayMarcher(sc["H"], sc["W"], sc["vr"], **kw).cuda().train(training)
    ref = refmods.load_raymarcher()(sc["H"], sc["W"], sc["vr"], **kw).cuda().train(training)
    G = lambda shape: torch.randn(shape, generator=torch.Generator().manual_seed(7))   # noqa: E731
    img, pix, grads = _run(ours, sc, G, seed)
    rimg, rpix, rgrads = _run(ref, sc, G, seed)
    assert torch.equal(pix.cpu(), rpix.cpu()), what

    rel = float((img - rimg).norm() / rimg.norm())
    rng = (rimg.amax(dim=(0, 2, 3)) - rimg.amin(dim=(0, 2, 3))).clamp(min=1e-6).view(1, 4, 1, 1)
    dev = ((img - rimg).abs() / rng).amax(1)
    share, worst = float((dev > 1e-3).float().mean()), float(dev.max())
    alpha = rimg[:, 3]
    print(f"{what}: image rel-L2 {rel:.2e}, pixels > 1e-3 of range {share:.2e}, worst {worst:.2e}; "
          f"covered {float((alpha > 0).float().mean()):.2f}, saturated {float((alpha >= 1 - 1e-6).float().mean()):.2f}")
    stats = [(n, float((a.double() - b.double()).norm() / b.double().norm()),
              float((a.double().flatten() @ b.double().flatten()) / (a.double().norm() * b.double().norm()))) for n, a, b in zip(NAMES, grads, rgrads)]
    for n, r, c in stats:
        print(f"{what} {n}: rel-L2 {r:.2e}, cosine {c:.9f}")
    assert float(alpha.max()) > 0.3 and float((alpha > 0).float().mean()) > 0.05, what      # the scene is actually rendered
    assert rel <= IMG_REL and share <= PIX_SHARE and worst <= PIX_MAX, (what, rel, share, worst)
    for n, r, c in stats:
        assert r <= GRAD_REL and c >= GRAD_COS, (what, n, r, c)


@pytest.mark.parametrize("name", list(BASE))
def test_scenes_match_the_reference(name):
    """The scenes the kernel-shaped oracle is compared on; K = 24, 40, 600, 48, 30 are not powers of two, so the list order is the
    tree's rotated one, and over_cap / saturating depend on it."""
    _check(name, _base(name))


@pytest.mark.parametrize("K", [32, 64, 512])
@pytest.mark.parametrize("name", ["small", "saturating", "over_cap"])
def test_power_of_two_scenes_match_the_reference(name, K):
    """The same seeds with K a power of two, where the tree order is ascending."""
    _check(f"{name} K={K}", _base(name, K=K))


@pytest.mark.parametrize("name", ["K1", "K3", "anisotropic", "camera_in_cube", "camera_in_primitive", "behind_camera"])
def test_edge_scenes_match_the_reference(name):
    """One and three primitives; per-axis scales with rotations (a permuted scale axis shows); the camera inside the unit cube (the
    tmin clamp at 0) and inside a primitive (the cone cull's distance <= radius branch); primitives behind the camera, whose boxes the
    slab test still meets along the ray's line."""
    sc = _custom(name)
    if name == "camera_in_primitive":
        y = rmo._local(torch.tensor([0.0, 0.0, 0.75]), sc["pos"][0, 0] / VR, sc["R"][0, 0], sc["scale"][0, 0])
        assert bool((y.abs() < 1).all())
    if name == "behind_camera":
        assert int((sc["pos"][0, :, 2] > 0).sum()) > 10
    _check(name, sc)


@pytest.mark.parametrize("name", ["past_cache", "over_cap_2048"])
def test_long_hit_lists_match_the_reference(name):
    """More than 96 listed primitives per warp (past the shared-memory cache of transforms); K = 2048 with more than 512 per warp, so
    the cap is checked where the order is ascending."""
    sc = _custom(name)
    n = _listed_per_warp(sc)
    print(f"{name}: listed per warp min {int(n.min())} max {int(n.max())}")
    if name == "past_cache":
        assert int(n.max()) > 96 and int(n.max()) <= 512
    else:
        assert int(n.max()) > 512
    _check(name, sc)


def test_shipped_preview_matches_the_reference():
    """The shipped preview: 2048 primitives of 8^3, 518 x 518, volradius 1e4, dt 1; image and gradients."""
    _check("shipped 518", _shipped())


def test_app_batch_matches_the_reference():
    """N = 4 at 256 x 256, as app.py renders."""
    _check("shipped N=4 256", _shipped(N=4, H=256, W=256))


@pytest.mark.parametrize("f", [2, 4])
@pytest.mark.parametrize("training", [False, True])
def test_subsampled_rays_match_the_reference(f, training):
    """ray_subsample_factor 2 and 4, eval (offset f // 2) and training (offsets drawn from the default generator, seeded before each
    call): both modules march the same pixel coordinates."""
    _check(f"f={f} training={training}", _base("two_images"), f=f, training=training)
