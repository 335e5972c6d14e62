"""-m gpu: the ray-march backward (tpx_raymarch_forward / tpx_raymarch_backward behind tpxl_b200.RayMarcher under autograd) and
subsampled rays, against oracle.raymarch_grad.ray_marcher_backward (autograd through the kernel-shaped restatement, itself held to the
reference's own pure-PyTorch marcher under autograd in tests/test_raymarch_grad_host.py).

Tolerances: fp32 throughout.  The kernel uses the fast-math exp / pow the reference is compiled with, fused multiply-adds and
floating-point atomics (summation order varies run to run), the oracle plain torch math; a grazing ray could enter a box one step
earlier or later in one of them.  Measured on one H100 80GB HBM3 (700 W): images <= 2.5e-6 relative L2, gradients <= 1.5e-5 relative
L2 per tensor (the K = 600 scene's template gradient; every other tensor <= 8e-6), cosine 1 to 8 digits.  Bounds: image 2e-5,
gradients relative L2 1e-4 and cosine >= 1 - 1e-6."""
import pytest
import torch

import oracle.raymarch_grad
import tpxl_b200
from tpxl_b200 import _lib

pytestmark = pytest.mark.gpu

NAMES = ("prim_rgba", "prim_pos", "prim_rot", "prim_scale")


def _scene(K, S, seed, rot=False, N=1, alpha=60.0):
    g = torch.Generator().manual_seed(seed)
    pos = (torch.rand(N, K, 3, generator=g) - 0.5) * 1.0
    scale = 1.0 / (0.12 + 0.1 * torch.rand(N, K, 1, generator=g)).repeat(1, 1, 3)
    if rot:
        R = torch.linalg.qr(torch.randn(N, K, 3, 3, generator=g))[0]
    else:
        R = torch.eye(3)[None, None].repeat(N, K, 1, 1)
    rgba = torch.rand(N, K, 4, S, S, S, generator=g)
    rgba[:, :, :3] *= 255.0
    rgba[:, :, 3] *= alpha
    return rgba, pos, R, scale


def _camera(H, W, volradius, N=1):
    RT = torch.tensor([[[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, 3.0 * volradius]]]).repeat(N, 1, 1)
    Kc = torch.tensor([[[2.4 * W, 0, W / 2], [0, 2.4 * W, H / 2], [0, 0, 1.0]]]).repeat(N, 1, 1)
    return Kc, RT


SCENES = {   # name: (K, S, H, W, rot, N, alpha, pos scale)
    "small": (24, 4, 32, 24, False, 1, 60.0, 1.0),
    "rotated": (40, 8, 33, 21, True, 1, 60.0, 1.0),
    "over_cap": (600, 4, 16, 16, False, 1, 60.0, 0.2),
    "saturating": (48, 4, 24, 24, True, 1, 400.0, 0.6),
    "two_images": (30, 4, 20, 28, True, 2, 120.0, 1.0),
}


def _make(name, volradius=100.0):
    K, S, H, W, rot, N, alpha, ps = SCENES[name]
    rgba, pos, R, scale = _scene(K, S, 5 * K + H, rot, N, alpha)
    Kc, RT = _camera(H, W, volradius, N)
    return rgba, pos * ps * volradius, R, scale, Kc, RT, H, W


def _compare(got, want, what):
    worst = []
    for n, a, b in zip(NAMES, got, want):
        a, b = a.detach().double().cpu().flatten(), b.double().flatten()
        cos = float(a @ b / (a.norm() * b.norm()))
        rel = float((a - b).norm() / b.norm())
        print(f"{what} {n}: cosine {cos:.8f}, rel-L2 {rel:.2e}")
        worst.append((n, cos, rel))
    for n, cos, rel in worst:
        assert cos >= 1 - 1e-6 and rel <= 1e-4, (what, n, cos, rel)


def _leaves(rgba, pos, R, scale):
    return [t.cuda().requires_grad_(True) for t in (rgba, pos, R, scale)]


def _prep(rgba, pos, R, scale, Kc, RT, volradius):
    """The arguments RayMarcher hands the C entries."""
    cam = tpxl_b200.ray_marcher.convert_camera_parameters(RT.cuda(), Kc.cuda())
    c = [cam["campos"], cam["camrot"], torch.diagonal(cam["focal"], dim1=1, dim2=2), cam["princpt"]]
    c = [t.float().contiguous() for t in c]
    tpl = rgba.cuda().float().permute(0, 1, 3, 4, 5, 2).contiguous()
    return tpl, (pos.cuda() / volradius).contiguous(), R.cuda().contiguous(), scale.cuda().contiguous(), c


@pytest.mark.parametrize("name", ["small", "rotated", "over_cap"])
def test_saving_forward_is_the_preview(name):
    """tpx_raymarch_forward with stride 1 and no offsets gives tpx_raymarch_preview's image bit for bit, with or without raysat;
    raysat is the saturating sample's colour (>= 0 here) exactly on the rays whose alpha reached 1, and -1 elsewhere."""
    rgba, pos, R, scale, Kc, RT, H, W = _make(name)
    volradius, dt = 100.0, 1.0
    tpl, p, r, s, c = _prep(rgba, pos, R, scale, Kc, RT, volradius)
    N, K, S = tpl.shape[0], tpl.shape[1], tpl.shape[2]
    L = _lib.lib()
    outs = []
    for fn, extra in (("tpx_raymarch_preview", None), ("tpx_raymarch_forward", False), ("tpx_raymarch_forward", True)):
        out = torch.full((N, H, W, 4), float("nan"), device="cuda")
        raysat = torch.full((N, H, W, 3), float("nan"), device="cuda")
        args = [tpl.data_ptr(), p.data_ptr(), r.data_ptr(), s.data_ptr(), *[t.data_ptr() for t in c], N, K, S, H, W, volradius, dt / volradius, 8.0, 8.0]
        if extra is None:
            _lib.check(getattr(L, fn)(*args, out.data_ptr(), _lib.stream_ptr()), fn)
        else:
            _lib.check(getattr(L, fn)(*args, 1, None, out.data_ptr(), raysat.data_ptr() if extra else None, _lib.stream_ptr()), fn)
        outs.append((out, raysat))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][0], outs[2][0])
    alpha, raysat = outs[2][0][..., 3], outs[2][1]
    sat = raysat[..., 0] >= 0
    assert bool(((raysat >= 0).all(-1) == sat).all()) and bool((raysat[~sat] == -1).all())
    assert bool((alpha[sat] >= 1 - 1e-6).all()) and bool((alpha[~sat] < 1).all())
    print(f"{name}: saturated rays {float(sat.float().mean()):.2f}")


@pytest.mark.parametrize("name", list(SCENES))
def test_gradients_match_the_oracle(name):
    """Image and the four gradients through RayMarcher against autograd through the kernel-shaped oracle, with a random upstream
    gradient.  Ragged sizes, rotations, K = 600 past the 512-entry hit-list cap, a scene where a large share of the rays saturates, and
    two images with different primitives."""
    rgba, pos, R, scale, Kc, RT, H, W = _make(name)
    volradius = 100.0
    G = torch.randn(rgba.shape[0], 4, H, W, generator=torch.Generator().manual_seed(7))
    rm = tpxl_b200.RayMarcher(H, W, volradius).cuda()
    leaves = _leaves(rgba, pos, R, scale)
    out = rm(*leaves, Kc.cuda(), RT.cuda())["rgba_image"]
    out.backward(G.cuda())
    ref, grads = oracle.raymarch_grad.ray_marcher_backward(rgba, pos, R, scale, Kc, RT, H, W, volradius, G)
    sat = float((ref[:, 3] >= 1 - 1e-6).float().mean())
    rel = float((out.detach().cpu() - ref).norm() / ref.norm())
    print(f"{name}: image rel-L2 {rel:.2e}, saturated {sat:.2f}, covered {float((ref[:, 3] > 0).float().mean()):.2f}")
    assert rel < 2e-5
    if name == "saturating":
        assert sat > 0.1
    _compare([t.grad for t in leaves], grads, name)


def test_rgb_gradient_is_exact_for_a_linear_direction():
    """Oracle-free: for fixed alpha the image is linear in the template's rgb, so a central difference of <G, image> along a random rgb
    direction equals <grad, direction> up to fp32 rounding."""
    rgba, pos, R, scale, Kc, RT, H, W = _make("saturating")
    volradius = 100.0
    g = torch.Generator().manual_seed(9)
    G = torch.randn(1, 4, H, W, generator=g)
    G[:, 3] = 0
    d = torch.zeros_like(rgba)
    d[:, :, :3] = torch.randn(rgba[:, :, :3].shape, generator=g) * 10.0
    rm = tpxl_b200.RayMarcher(H, W, volradius).cuda()
    leaves = _leaves(rgba, pos, R, scale)
    (rm(*leaves, Kc.cuda(), RT.cuda())["rgba_image"] * G.cuda()).sum().backward()
    with torch.no_grad():
        f = lambda x: float((rm(x.cuda(), pos.cuda(), R.cuda(), scale.cuda(), Kc.cuda(), RT.cuda())["rgba_image"].double() * G.cuda()).sum())  # noqa: E731
        fd = (f(rgba + d) - f(rgba - d)) / 2
    an = float((leaves[0].grad.double().cpu() * d).sum())
    print(f"central difference {fd:.6e}, <grad, d> {an:.6e}")
    assert abs(fd - an) <= 1e-4 * abs(an)


@pytest.mark.parametrize("f", [2, 4])
@pytest.mark.parametrize("training", [False, True])
def test_subsampled_rays_match_the_oracle(f, training):
    """ray_subsample_factor > 1: the offsets drawn as the reference's subsample_pixel_coords draws them (training) or f // 2 (eval);
    image and gradients against the oracle at the same pixel coordinates; with and without grad the same image."""
    rgba, pos, R, scale, Kc, RT, H, W = _make("two_images")
    volradius = 100.0
    rm = tpxl_b200.RayMarcher(H, W, volradius, ray_subsample_factor=f).cuda().train(training)
    torch.manual_seed(5)
    leaves = _leaves(rgba, pos, R, scale)
    res = rm(*leaves, Kc.cuda(), RT.cuda())
    out, pix = res["rgba_image"], res["pixel_coords"]
    assert out.shape == (2, 4, H // f, W // f) and pix.shape == (2, H // f, W // f, 2)
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(3))
    out.backward(G.cuda())
    torch.manual_seed(5)
    with torch.no_grad():
        res2 = rm(rgba.cuda(), pos.cuda(), R.cuda(), scale.cuda(), Kc.cuda(), RT.cuda())
    assert torch.equal(res2["pixel_coords"], pix) and torch.equal(res2["rgba_image"], out.detach())
    ref, grads = oracle.raymarch_grad.ray_marcher_backward(rgba, pos, R, scale, Kc, RT, H, W, volradius, G, pixelcoords=pix.cpu())
    rel = float((out.detach().cpu() - ref).norm() / ref.norm())
    print(f"f={f} training={training}: image rel-L2 {rel:.2e}")
    assert rel < 2e-5
    _compare([t.grad for t in leaves], grads, f"f={f} training={training}")


def test_subsampled_pixel_coords_match_the_reference_fixture(golden_dir):
    """The seeded training draw through RayMarcher gives the reference's subsample_pixel_coords output (tests/golden/raymarch_grad.npz)."""
    import os
    import numpy as np
    d = np.load(os.path.join(golden_dir, "raymarch_grad.npz"))
    B, H, W = (int(v) for v in d["pix_hw"])
    rgba, pos, R, scale = _scene(4, 4, 1, N=B)
    Kc, RT = _camera(H, W, 100.0, B)
    torch.manual_seed(int(d["pix_seed"]))
    for f in (2, 3, 4):
        rm = tpxl_b200.RayMarcher(H, W, 100.0, ray_subsample_factor=f).cuda().train()
        pix = rm(rgba.cuda(), (pos * 100).cuda(), R.cuda(), scale.cuda(), Kc.cuda(), RT.cuda())["pixel_coords"]
        assert np.array_equal(pix.cpu().numpy(), d[f"pix_train_f{f}"]), f
        pix = rm.eval()(rgba.cuda(), (pos * 100).cuda(), R.cuda(), scale.cuda(), Kc.cuda(), RT.cuda())["pixel_coords"]
        assert np.array_equal(pix.cpu().numpy(), d[f"pix_eval_f{f}"]), f


def test_raymarcher_autograd_contract():
    """Gradients reach every primitive input in the caller's layout, units and dtype (fp16 prim_rgba gets an fp16 gradient; prim_pos is
    in world units), the camera gets none, a primitive that no ray lists gets exactly zero, and under no_grad the output is the
    preview's bit for bit."""
    rgba, pos, R, scale, Kc, RT, H, W = _make("rotated")
    volradius = 100.0
    pos[0, 0] = torch.tensor([50.0, 50.0, 0.0]) * volradius     # far outside the view: never listed
    rm = tpxl_b200.RayMarcher(H, W, volradius).cuda()
    Kg, RTg = Kc.cuda().requires_grad_(True), RT.cuda().requires_grad_(True)
    leaves = _leaves(rgba, pos, R, scale)
    out = rm(*leaves, Kg, RTg)["rgba_image"]
    assert out.requires_grad
    loss = ((out[:, :3] - 100.0) ** 2).mean() + out[:, 3].abs().mean()
    loss.backward()
    assert Kg.grad is None and RTg.grad is None
    for n, t in zip(NAMES, leaves):
        assert t.grad is not None and t.grad.shape == t.shape and bool(torch.isfinite(t.grad).all()), n
        assert float(t.grad.abs().sum()) > 0, n
        assert float(t.grad[0, 0].abs().max()) == 0.0, n
    with torch.no_grad():
        prev = rm(*[t.detach() for t in leaves], Kc.cuda(), RT.cuda())["rgba_image"]
    assert torch.equal(prev, out.detach())
    # units: the same gradient through an explicit world -> volume scaling matches the mirror's
    pos_unit = (pos / volradius).cuda().requires_grad_(True)
    out2 = rm(leaves[0].detach(), pos_unit * volradius, leaves[2].detach(), leaves[3].detach(), Kc.cuda(), RT.cuda())["rgba_image"]
    (((out2[:, :3] - 100.0) ** 2).mean() + out2[:, 3].abs().mean()).backward()
    assert torch.allclose(pos_unit.grad / volradius, leaves[1].grad, rtol=1e-4, atol=1e-12 + 1e-6 * float(leaves[1].grad.abs().max()))
    # fp16 template in, fp16 gradient out, equal to the fp32 gradient on the same (fp16-representable) values up to fp16 rounding
    h = rgba.half().cuda().requires_grad_(True)
    f32 = rgba.half().float().cuda().requires_grad_(True)
    G = torch.randn(1, 4, H, W, generator=torch.Generator().manual_seed(2)).cuda()
    (rm(h, *[t.detach() for t in leaves[1:]], Kc.cuda(), RT.cuda())["rgba_image"] * G).sum().backward()
    (rm(f32, *[t.detach() for t in leaves[1:]], Kc.cuda(), RT.cuda())["rgba_image"] * G).sum().backward()
    assert h.grad.dtype == torch.float16
    assert float((h.grad.float() - f32.grad).norm() / f32.grad.norm()) < 2e-3


def _shipped(N=4, H=256, W=256):
    K, S, volradius = 2048, 8, 10000.0
    g = torch.Generator().manual_seed(3)
    d = torch.randn(N, K, 3, generator=g)
    pos = d / d.norm(dim=-1, keepdim=True) * 0.5
    scale = torch.full((N, K, 3), 1.0 / 0.05)
    rgba = torch.rand(N, K, 4, S, S, S, generator=g) * 255.0
    rgba[:, :, 3] = 255.0 * torch.exp(-(torch.rand(N, K, S, S, S, generator=g) * 0.02 / 0.005) ** 2)
    R = torch.eye(3)[None, None].repeat(N, K, 1, 1)
    RT = torch.tensor([[[1.0, 0, 0, 0], [0, -1.0, 0, 0], [0, 0, -1.0, 5 * volradius]]]).repeat(N, 1, 1)
    Kc = torch.tensor([[[2084.9526697685183 * H / 1024, 0, 512.0 * H / 1024], [0, 2084.9526697685183 * W / 1024, 512.0 * W / 1024], [0, 0, 1.0]]]).repeat(N, 1, 1)
    return rgba, pos * volradius, R, scale, Kc, RT, H, W, volradius


def test_shipped_size_gradients_are_finite_and_repeatable():
    """2048 primitives of 8^3, 256 x 256 as app.py renders, N = 4: finite gradients, and two runs agree to 1e-5 relative L2 per tensor
    (only the atomics' summation order differs)."""
    rgba, pos, R, scale, Kc, RT, H, W, volradius = _shipped()
    rm = tpxl_b200.RayMarcher(H, W, volradius).cuda()
    G = torch.randn(4, 4, H, W, generator=torch.Generator().manual_seed(1)).cuda()
    runs = []
    for _ in range(2):
        leaves = _leaves(rgba, pos, R, scale)
        (rm(*leaves, Kc.cuda(), RT.cuda())["rgba_image"] * G).sum().backward()
        runs.append([t.grad for t in leaves])
    for n, a, b in zip(NAMES, *runs):
        assert bool(torch.isfinite(a).all()), n
        rel = float((a - b).norm() / b.norm())
        print(f"shipped {n}: run-to-run rel-L2 {rel:.2e}, norm {float(b.norm()):.3e}")
        assert rel <= 1e-5 and float(b.norm()) > 0, n


def test_adam_refinement_lowers_the_image_loss():
    """A reference-style fitting loop (rgba_image -> rgb MSE + alpha MAE -> backward -> Adam step) on the template toward a target
    rendered from perturbed parameters: 20 steps, the loss falls at every step."""
    rgba, pos, R, scale, Kc, RT, H, W = _make("rotated")
    volradius = 100.0
    rm = tpxl_b200.RayMarcher(H, W, volradius).cuda()
    cam = (Kc.cuda(), RT.cuda())
    g = torch.Generator().manual_seed(12)
    target_rgba = rgba.clone()
    target_rgba[:, :, :3] = (target_rgba[:, :, :3] + 40.0 * torch.randn(rgba[:, :, :3].shape, generator=g)).clamp(0, 255)
    target_rgba[:, :, 3] = (target_rgba[:, :, 3] * (0.5 + torch.rand(rgba[:, :, 3].shape, generator=g))).clamp(min=0)
    geo = [t.cuda() for t in (pos, R, scale)]
    with torch.no_grad():
        target = rm(target_rgba.cuda(), *geo, *cam)["rgba_image"]
    param = rgba.cuda().requires_grad_(True)
    opt = torch.optim.Adam([param], lr=1.0)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        img = rm(param, *geo, *cam)["rgba_image"]
        loss = ((img[:, :3] - target[:, :3]) ** 2).mean() / 255.0 ** 2 + (img[:, 3] - target[:, 3]).abs().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    print("losses", " ".join(f"{v:.4e}" for v in losses))
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < 0.8 * losses[0]
