"""Drop-in for the reference's ``dva.visualize`` (the preview images and turntable videos of inference.py:349-350 and app.py:140), with
every per-pixel step on the device.

Same functions and signatures as the reference: ``get_pose_on_orbit``, ``render_mvp_boxes``, ``save_image_summary``,
``visualize_primvolume``, ``visualize_multiview_primvolume`` and ``visualize_video_primvolume``, writing the same files.  The core is
``render_views(prim_volume, rm, Rt, K, kinds)``, which does no file I/O:
  * the rgb and material templates come straight from ``recon_param`` in one launch each (tpx_primvolume_payload), channels-last as
    the march reads them, bit for bit the reference's slices, ``exp`` and ``concat``;
  * the coloured-box template is built once per call, not once per view (tpx_colored_boxes; the same numpy draws as the reference's
    ``generate_colored_boxes``, which reseeds numpy's global generator);
  * every view of one kind is one march launch over that one template (tpx_raymarch_preview_views), each image bit-identical to the
    reference's per-view ``RayMarcher`` call on this package's marcher.
Cameras are built on the host with the reference's torch statements (orbit poses; intrinsics scaled by H / 1024 in row 0 and W / 1024
in row 1) and converted on the device per view, exactly as the reference's per-view ``RayMarcher`` calls convert them.

One deliberate addition: ``visualize_video_primvolume`` also writes ``mat.mp4`` next to ``rgb.mp4`` and ``prim.mp4``, the material
render (colour (0, roughness, metallic), the R / G / B order of the ``roughness_metallic.jpg`` that extract_texmesh writes, glTF's
metallicRoughness convention) that app.py's "Material" panel shows.  Encoding stays on the host: ``imageio``, ``cv2`` and
``torchvision`` are imported only by the functions that write files.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib
from .ray_marcher import RayMarcher, box_colors, colored_boxes, generate_colored_boxes, march_camera, march_views  # noqa: F401

KINDS = ("rgb", "boxes", "mat")
_FOCAL, _PRINCPT = 2084.9526697685183, 512.0


def get_pose_on_orbit(radius, height, angles, world_up=torch.Tensor([0, 1, 0])):
    """dva/visualize.py:9-22: extrinsics [n, 3, 4] of cameras on a horizontal circle looking at the origin (host torch arithmetic)."""
    n = angles.shape[0]
    position = torch.stack([radius * torch.cos(angles), torch.ones((n,)) * height, radius * torch.sin(angles)], dim=-1)
    forward = position / torch.norm(position, p=2, dim=-1, keepdim=True)
    right = -torch.cross(world_up[None, ...], forward)
    right /= torch.norm(right, dim=-1, keepdim=True)
    up = torch.cross(forward, right)
    up /= torch.norm(up, p=2, dim=-1, keepdim=True)
    rotation = torch.stack([right, up, forward], dim=1)
    translation = torch.Tensor([0, 0, radius])[None, :, None].repeat(n, 1, 1)
    return torch.concat([rotation, translation], dim=2)


def preview_intrinsics(rm, bs: int) -> torch.Tensor:
    """The preview camera's K [bs, 3, 3] on the host: the 1024-pixel intrinsics with row 0 scaled by image_height / 1024 and row 1 by
    image_width / 1024, as the reference scales them."""
    K = torch.Tensor([[_FOCAL, 0.0, _PRINCPT], [0.0, _FOCAL, _PRINCPT], [0.0, 0.0, 1.0]])[None, ...].repeat(bs, 1, 1)
    K[:, 0:1, :] *= rm.image_height / 1024.
    K[:, 1:2, :] *= rm.image_width / 1024.
    return K


def front_extrinsics(rm, bs: int) -> torch.Tensor:
    """The single-image preview's Rt [bs, 3, 4]: 5 volume radii in front of the origin, y and z flipped."""
    vr = rm.volradius
    return torch.Tensor([[1.0, 0.0, 0.0, 0.0 * vr], [0.0, -1.0, 0.0, 0.0 * vr], [0.0, 0.0, -1.0, 5 * vr]])[None, ...].repeat(bs, 1, 1)


def orbit_extrinsics(rm, bs: int, view_angles: torch.Tensor) -> torch.Tensor:
    """[V, bs, 3, 4]: for each angle, the poses the reference's loop builds, ``get_pose_on_orbit(5 volradius, 0, angle.repeat(bs))``."""
    return torch.stack([get_pose_on_orbit(radius=5 * rm.volradius, height=0, angles=a.repeat(bs,)) for a in view_angles], 0)


def prim_shape_of(prim_volume: torch.Tensor) -> int:
    S = int(np.round(((prim_volume.shape[2] - 4) / 6) ** (1 / 3)))
    if prim_volume.dim() != 3 or prim_volume.shape[2] != 4 + 6 * S ** 3:
        raise ValueError(f"prim_volume must be [B, P, 4 + 6 S^3], got {tuple(prim_volume.shape)}")
    return S


def primvolume_payload(prim_volume: torch.Tensor, kind: str = "rgb") -> torch.Tensor:
    """tpx_primvolume_payload: recon_param [B, P, 4 + 6 S^3] fp32 on CUDA -> the channels-last march template [B, P, S, S, S, 4]:
    colour tex * 255 ("rgb") or (0, roughness, metallic) * 255 ("mat"), alpha exp(-(sdf / 0.005) ** 2) * 255."""
    S = prim_shape_of(prim_volume)
    if kind not in ("rgb", "mat"):
        raise ValueError(f"payload kind must be 'rgb' or 'mat', got {kind!r}")
    if prim_volume.dtype != torch.float32:
        raise ValueError(f"prim_volume must be fp32, got {prim_volume.dtype}")
    if not prim_volume.is_cuda:
        raise _lib.TpxError("the preview payload runs on CUDA only (no CPU path)")
    B, P = prim_volume.shape[:2]
    src = prim_volume.contiguous()
    out = torch.empty(B, P, S, S, S, 4, dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        _lib.check(_lib.lib().tpx_primvolume_payload(src.data_ptr(), B, P, S, _lib.PAYLOAD_MAT if kind == "mat" else _lib.PAYLOAD_RGB, out.data_ptr(),
                                                     _lib.stream_ptr()), "tpx_primvolume_payload")
    return out


@torch.no_grad()
def render_views(prim_volume: torch.Tensor, rm, Rt: torch.Tensor, K: torch.Tensor, kinds=KINDS, alpha: bool = False) -> dict:
    """Render V views of each of the B primitive volumes in `prim_volume` [B, P, 4 + 6 S^3] (fp32, CUDA) with the settings of `rm` (a
    RayMarcher: image size, volradius, dt, fade; no ray subsampling).  Rt: extrinsics [V, B, 3, 4] or [V, 3, 4] (one pose per view for
    every volume); K: intrinsics [B, 3, 3] or [3, 3], the same for every view.  Returns {kind: [V * B, H, W, 3]} for kind in `kinds`
    ("rgb": the asset, "boxes": every primitive as a lit box, "mat": the material render), frames view-major (view v, volume b at
    v * B + b), as the reference concatenates its per-view renders.  With `alpha` the frames keep the march's alpha: [V * B, H, W, 4]."""
    for k in kinds:
        if k not in KINDS:
            raise ValueError(f"unknown kind {k!r}; expected a subset of {KINDS}")
    if getattr(rm, "ray_subsample_factor", 1) != 1:
        raise NotImplementedError("render_views marches every pixel (ray_subsample_factor 1)")
    S = prim_shape_of(prim_volume)
    B, P = prim_volume.shape[:2]
    dev = prim_volume.device
    H, W = rm.image_height, rm.image_width
    if Rt.dim() == 3:
        Rt = Rt[:, None].expand(-1, B, -1, -1)
    if K.dim() == 2:
        K = K[None].expand(B, -1, -1).contiguous()
    V = Rt.shape[0]
    if tuple(Rt.shape[1:]) != (B, 3, 4) or tuple(K.shape) != (B, 3, 3):
        raise ValueError(f"Rt must be [V, {B}, 3, 4] or [V, 3, 4] and K [{B}, 3, 3] or [3, 3], got {tuple(Rt.shape)} and {tuple(K.shape)}")
    # the reference's statements (visualize.py:235-239), then RayMarcher.forward's hand-over to the march
    pos = prim_volume[:, :, 1:4].reshape(B, P, 3) * rm.volradius
    rot = torch.eye(3).to(pos)[None, None, ...].repeat(B, P, 1, 1)
    scale = 1 / prim_volume[:, :, 0:1].reshape(B, P, 1).repeat(1, 1, 3)
    pos, rot, scale = (pos / rm.volradius).float().contiguous(), rot.float().contiguous(), scale.float().contiguous()
    # per view, on a fresh [B] tensor, as each of the reference's per-view calls converts its batch["Rt"]; then set-major for the march
    per_view = [march_camera(Rt[v].clone(memory_format=torch.contiguous_format), K, dev) for v in range(V)]
    cam = tuple(torch.stack([c[i] for c in per_view], 1).reshape(B * V, *per_view[0][i].shape[1:]).contiguous() for i in range(4))
    geom = (H, W, float(rm.volradius), float(rm.dt / rm.volradius), float(rm.fadescale), float(rm.fadeexp))
    out = {}
    for kind in kinds:
        if kind == "boxes":
            tpl = colored_boxes(B, P, S, box_colors(P), 10000.0, True, dev)
        else:
            tpl = primvolume_payload(prim_volume.float(), kind)
        rgba = march_views(tpl, pos, rot, scale, cam, V, *geom)
        out[kind] = rgba.view(B, V, H, W, 4).transpose(0, 1).reshape(V * B, H, W, 4)[..., :4 if alpha else 3].contiguous()
    return out


def render_mvp_boxes(rm, batch, preds):
    """dva/visualize.py:24-39: the primitives of ``preds`` as lit boxes through `rm` -> [B, H, W, 3]."""
    with torch.no_grad():
        boxes_rgba = generate_colored_boxes(preds["prim_rgba"], preds["prim_rot"])
        preds_boxes = rm(prim_rgba=boxes_rgba, prim_pos=preds["prim_pos"], prim_scale=preds["prim_scale"], prim_rot=preds["prim_rot"],
                         RT=batch["Rt"], K=batch["K"])
    return preds_boxes["rgba_image"][:, :3].permute(0, 2, 3, 1)


def save_image_summary(path, batch, preds):
    """dva/visualize.py:42-62: the rgb frames above the box frames, one grid image at `path`; with ``folder`` / ``key`` in `batch` the
    box frames are captioned and the names written to ``<path stem>.txt``."""
    import cv2
    from torchvision.utils import make_grid, save_image
    rgb = preds["rgb"].detach().permute(0, 3, 1, 2)
    rgb_boxes = preds["rgb_boxes"].detach().permute(0, 3, 1, 2)
    if "folder" in batch and "key" in batch:
        names = []
        for i in range(rgb_boxes.shape[0]):
            img = np.ascontiguousarray(rgb_boxes[i].permute(1, 2, 0).to(torch.uint8).cpu().numpy())
            folder, key = batch["folder"][i], batch["key"][i]
            names.append("{}/{}\n".format(folder, key))
            cv2.putText(img, "{}".format(folder), (200, 200), cv2.FONT_HERSHEY_SIMPLEX, 2, (255, 0, 0), 2)
            cv2.putText(img, "{}".format(key), (200, 400), cv2.FONT_HERSHEY_SIMPLEX, 2, (255, 0, 0), 2)
            rgb_boxes[i] = torch.as_tensor(img).permute(2, 0, 1).float()
        with open(os.path.splitext(path)[0] + ".txt", "w") as f:
            f.writelines(names)
    save_image(make_grid(torch.cat([rgb, rgb_boxes], dim=2) / 255.0).clip(0.0, 1.0), path)


@torch.no_grad()
def visualize_primvolume(image_save_path, batch, prim_volume, rm: RayMarcher, device):
    """dva/visualize.py:214-293: the front view of each volume and its boxes, saved as one summary image.  Sets batch["Rt"] /
    batch["K"] as the reference does."""
    bs = prim_volume.shape[0]
    batch["Rt"] = front_extrinsics(rm, bs).to(device)
    batch["K"] = preview_intrinsics(rm, bs).to(device)
    frames = render_views(prim_volume, rm, batch["Rt"][None], batch["K"], kinds=("rgb", "boxes"))
    save_image_summary(image_save_path, batch, {"rgb": frames["rgb"], "rgb_boxes": frames["boxes"]})


@torch.no_grad()
def visualize_multiview_primvolume(image_save_path, batch, prim_volume, view_counts, rm: RayMarcher, device):
    """dva/visualize.py:295-367: `view_counts` views on the orbit from 0.5 pi to 2.5 pi (end excluded), saved as one summary image."""
    bs = prim_volume.shape[0]
    view_angles = (torch.linspace(0.5, 2.5, view_counts + 1) * torch.pi)[:-1]
    batch["K"] = preview_intrinsics(rm, bs).to(device)
    Rt = orbit_extrinsics(rm, bs, view_angles).to(prim_volume)
    batch["Rt"] = Rt[-1]
    frames = render_views(prim_volume, rm, Rt, batch["K"], kinds=("rgb", "boxes"))
    save_image_summary(image_save_path, batch, {"rgb": frames["rgb"], "rgb_boxes": frames["boxes"]})


@torch.no_grad()
def visualize_video_primvolume(video_save_folder, batch, prim_volume, view_counts, rm: RayMarcher, device):
    """dva/visualize.py:370-455: `view_counts` + 1 views on the orbit from 1.5 pi to 3.5 pi, written at 20 fps as rgb.mp4 (the asset),
    prim.mp4 (the boxes) and, in addition to the reference, mat.mp4 (the material render) in `video_save_folder`."""
    import imageio
    bs = prim_volume.shape[0]
    view_angles = torch.linspace(1.5, 3.5, view_counts + 1) * torch.pi
    batch["K"] = preview_intrinsics(rm, bs).to(device)
    Rt = orbit_extrinsics(rm, bs, view_angles).to(prim_volume)
    batch["Rt"] = Rt[-1]
    frames = render_views(prim_volume, rm, Rt, batch["K"], kinds=KINDS)
    videos = (("rgb.mp4", "rgb"), ("prim.mp4", "boxes"), ("mat.mp4", "mat"))
    writers = [imageio.get_writer(os.path.join(video_save_folder, name), fps=20) for name, _ in videos]
    data = [np.clip(frames[kind].detach().cpu().numpy(), 0, 255).astype(np.uint8) for _, kind in videos]
    for fidx in range(data[0].shape[0]):
        for w, d in zip(writers, data):
            w.append_data(d[fidx])
    for w in writers:
        w.close()
