"""Oracle of the preview payloads (TEST INFRASTRUCTURE): torch restatements of dva/visualize.py's colour draw, box template, payload
and orbit cameras, and the loader of the STAGED reference ``dva.visualize`` (oracle/stage_visualize.py).

  * ``box_colors`` / ``box_template``: generate_colored_boxes (dva/ray_marcher.py:232-279) as whole-tensor torch ops, the reference's
    per-primitive loop folded into one broadcast (each element sees the same fp32 operations in the same order);
  * ``payload``: the prim_rgba statements of visualize_primvolume (visualize.py:217-234), channels-last, and the material variant
    (0, roughness, metallic) * 255 with the same alpha;
  * ``orbit_poses`` / ``intrinsics``: get_pose_on_orbit (visualize.py:9-22) per view, as visualize_video_primvolume calls it, and
    the 1024-pixel intrinsics scaled by H / 1024 (row 0) and W / 1024 (row 1).
``reference_visualize(over)`` imports the staged, unmodified ``dva/visualize.py`` over the reference's ``RayMarcher`` (over=
"reference", its compiled extensions) or over ``tpxl_b200.ray_marcher`` (over="ours", what ``tpxl_b200.install()`` binds), with a
frame-capturing stub as ``imageio``; on exit ``dva``, the extensions and ``imageio`` leave ``sys.modules`` again.
"""
from __future__ import annotations

import contextlib
import importlib
import sys
import types

import numpy as np
import torch

from . import stage_ref, stage_visualize


def box_colors(K: int, seed: int = 123456) -> torch.Tensor:
    """np.random.seed(seed), then per primitive three np.random.rand() * 255.0 draws, each assigned to an fp32 tensor -> [K, 3]."""
    np.random.seed(seed)
    return torch.tensor([[np.random.rand() * 255.0 for _ in range(3)] for _ in range(K)], dtype=torch.float64).float()


def box_template(N: int, K: int, S: int, colors: torch.Tensor, alpha: float = 10000.0, device="cpu") -> torch.Tensor:
    """-> [N, K, 4, S, S, S] fp32, the reference's layout."""
    lightdir = -3 * torch.ones([N, 3], dtype=torch.float32, device=device)
    lightdir = lightdir / torch.norm(lightdir, p=2, dim=1, keepdim=True)
    lin = torch.linspace(-1.0, 1.0, S, device=device)
    zz, yy, xx = torch.meshgrid(lin, lin, lin, indexing="ij")
    ax, ay, az = xx.abs(), yy.abs(), zz.abs()
    nx = torch.where((ax >= ay) & (ax >= az), torch.sign(xx) * torch.ones_like(xx), torch.zeros_like(xx))
    ny = torch.where((ay >= ax) & (ay >= az), torch.sign(yy) * torch.ones_like(xx), torch.zeros_like(xx))
    nz = torch.where((az >= ax) & (az >= ay), torch.sign(zz) * torch.ones_like(xx), torch.zeros_like(xx))
    n = torch.stack([nx, -ny, -nz], dim=-1)
    n = n / torch.sqrt(torch.sum(n ** 2, dim=-1, keepdim=True))
    mult = torch.sum(lightdir[:, None, None, None, :] * n[None], dim=-1)[:, None].clamp(min=0.2)       # [N, 1, S, S, S]
    out = torch.empty(N, K, 4, S, S, S, dtype=torch.float32, device=device)
    out[:, :, :3] = colors.to(device)[None, :, :, None, None, None]
    out[:, :, 3] = alpha
    out[:, :, :3] *= (1.4 * mult)[:, :, None]
    return out


def payload(recon: torch.Tensor, kind: str = "rgb") -> torch.Tensor:
    """recon_param [B, P, 4 + 6 S^3] -> channels-last template [B, P, S, S, S, 4]."""
    B, P, C = recon.shape
    S = int(np.round(((C - 4) / 6) ** (1 / 3)))
    S3 = S ** 3
    geo = recon[:, :, 4:4 + S3]
    alpha = torch.exp(-(geo / 0.005) ** 2).reshape(B, P, 1, S, S, S) * 255
    if kind == "rgb":
        rgb = recon[:, :, 4 + S3:4 + 4 * S3].reshape(B, P, 3, S, S, S) * 255
    else:
        mat = recon[:, :, 4 + 4 * S3:4 + 6 * S3].reshape(B, P, 2, S, S, S) * 255
        rgb = torch.cat([torch.zeros_like(mat[:, :, :1]), mat], dim=2)
    return torch.cat([rgb, alpha], dim=2).permute(0, 1, 3, 4, 5, 2).contiguous()


def orbit_poses(radius: float, view_angles: torch.Tensor, bs: int) -> torch.Tensor:
    """[V, bs, 3, 4]: get_pose_on_orbit(radius, 0, angle.repeat(bs)) per view angle, on the host."""
    world_up = torch.Tensor([0, 1, 0])
    out = []
    for a in view_angles:
        angles = a.repeat(bs,)
        x, h, z = radius * torch.cos(angles), torch.ones((bs,)) * 0, radius * torch.sin(angles)
        position = torch.stack([x, h, z], dim=-1)
        forward = position / torch.norm(position, p=2, dim=-1, keepdim=True)
        right = -torch.cross(world_up[None, ...], forward)        # no dim: torch's first axis of size 3, as the reference calls it
        right /= torch.norm(right, dim=-1, keepdim=True)
        up = torch.cross(forward, right)
        up /= torch.norm(up, p=2, dim=-1, keepdim=True)
        rot = torch.stack([right, up, forward], dim=1)
        out.append(torch.concat([rot, torch.Tensor([0, 0, radius])[None, :, None].repeat(bs, 1, 1)], dim=2))
    return torch.stack(out, 0)


def intrinsics(H: int, W: int, bs: int) -> torch.Tensor:
    K = torch.Tensor([[2084.9526697685183, 0.0, 512.0], [0.0, 2084.9526697685183, 512.0], [0.0, 0.0, 1.0]])[None].repeat(bs, 1, 1)
    K[:, 0:1, :] *= H / 1024.
    K[:, 1:2, :] *= W / 1024.
    return K


def available(over: str = "reference") -> bool:
    """The staged dva/visualize.py is there, and for over="reference" the reference's ray marcher extensions too."""
    if not stage_visualize.visualize_staged():
        return False
    return over == "ours" or stage_ref.raymarcher_staged()


def imageio_stub() -> types.ModuleType:
    """A stand-in ``imageio`` whose get_writer(path, **kw) returns a writer that keeps every appended frame: ``stub.frames[path]`` is
    the list of numpy frames, ``stub.closed`` the paths closed, in order."""
    stub = types.ModuleType("imageio")
    stub.frames, stub.closed, stub.kwargs = {}, [], {}

    class _Writer:
        def __init__(self, path, **kw):
            self.path = path
            stub.frames[path] = []
            stub.kwargs[path] = kw

        def append_data(self, frame):
            stub.frames[self.path].append(np.array(frame, copy=True))

        def close(self):
            stub.closed.append(self.path)

    stub.get_writer = lambda path, **kw: _Writer(path, **kw)
    return stub


@contextlib.contextmanager
def reference_visualize(over: str = "reference"):
    """Context: yields (the staged reference ``dva.visualize`` module, the imageio stub).  over="reference": its ``RayMarcher`` and
    ``generate_colored_boxes`` are the reference's (compiled extensions); over="ours": ``dva.ray_marcher`` is ``tpxl_b200.ray_marcher``,
    as after ``tpxl_b200.install()``.  Raises FileNotFoundError when the files are not staged."""
    if over not in ("reference", "ours"):
        raise ValueError(over)
    if not available(over):
        raise FileNotFoundError("dva/visualize.py is not staged: run `python oracle/stage_ref.py` and `python oracle/stage_visualize.py`")
    taken = ("dva", "mvpraymarchlib", "utilslib", "imageio")
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in taken}
    for k in saved:
        del sys.modules[k]
    stub = imageio_stub()
    sys.modules["imageio"] = stub
    sys.path.insert(0, stage_ref.DEST)
    try:
        dva = importlib.import_module("dva")
        if over == "ours":
            import tpxl_b200
            sys.modules["dva.ray_marcher"] = tpxl_b200.ray_marcher
            dva.ray_marcher = tpxl_b200.ray_marcher
        vis = importlib.import_module("dva.visualize")
        sys.path.remove(stage_ref.DEST)
        yield vis, stub
    finally:
        if stage_ref.DEST in sys.path:
            sys.path.remove(stage_ref.DEST)
        for k in [k for k in sys.modules if k.split(".")[0] in taken]:
            del sys.modules[k]
        sys.modules.update(saved)
