#!/usr/bin/env python
"""Golden vectors for the preview payloads, produced by RUNNING THE REFERENCE'S OWN ``dva/visualize.py`` and ``generate_colored_boxes``
on the CPU.

Needs the staged reference (``python oracle/stage_ref.py`` and ``python oracle/stage_visualize.py`` where a reference checkout
exists; the staged ray-march extensions import without a GPU):

    python tests/golden/make_visualize_golden.py

  * ``generate_colored_boxes(zeros [B, K, 4, S, S, S], rot)`` for (K, S, B) in CASES, with numpy's global generator state after the
    call; at K = 2048 every primitive at voxel (0, 0, 0) and four primitives' templates are kept (the whole template is 16.8 MB);
  * ``visualize_primvolume`` and ``visualize_video_primvolume`` run with a stand-in ray marcher that records what it is handed and
    renders nothing: the payload (prim_rgba, prim_pos, prim_rot, prim_scale) of a seeded recon_param, and the per-view cameras
    (RT, K) at B = 1 and 2 for the 16-view app.py video at 256^2 and the 61-view inference.py video at 518^2.
Everything goes to tests/golden/visualize.npz; tests/test_visualize_host.py holds oracle.visualize and the package's host code to it.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import visualize as ov  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "visualize.npz")
BOX_CASES = [(6, 4, 1), (6, 5, 2), (6, 8, 1), (6, 8, 2), (2048, 8, 1)]
BIG_PRIMS = [0, 1, 1023, 2047]
PAYLOAD_CASES = [(1, 6, 4), (2, 6, 5), (1, 6, 8), (2, 6, 8)]             # (B, P, S)
VIDEO_CASES = [(1, 15, 256), (2, 15, 256), (1, 60, 518), (2, 60, 518)]    # (B, view_counts, H = W)
VOLRADIUS = 10000.0


class CaptureRM:
    """Stands in for RayMarcher: records each call's inputs and returns a black image."""

    def __init__(self, H, W):
        self.image_height, self.image_width, self.volradius = H, W, VOLRADIUS
        self.calls = []

    def __call__(self, prim_rgba, prim_pos, prim_rot, prim_scale, K, RT):
        self.calls.append({k: v.detach().clone() for k, v in dict(prim_rgba=prim_rgba, prim_pos=prim_pos, prim_rot=prim_rot, prim_scale=prim_scale,
                                                                  K=K, RT=RT).items()})
        return {"rgba_image": torch.zeros(prim_rgba.shape[0], 4, self.image_height, self.image_width)}


def recon_param(B, P, S, seed):
    """A recon_param of the layout LatentCodec.pack writes, with values like the decoder's: scale ~ 0.05, pos in the unit ball, sdf
    near 0, colours and material in [0, 1]."""
    g = torch.Generator().manual_seed(seed)
    S3 = S ** 3
    scale = 0.04 + 0.02 * torch.rand(B, P, 1, generator=g)
    pos = torch.rand(B, P, 3, generator=g) - 0.5
    sdf = (torch.rand(B, P, S3, generator=g) - 0.5) * 0.04
    rest = torch.rand(B, P, 5 * S3, generator=g)
    return torch.cat([scale, pos, sdf, rest], dim=-1)


def main():
    out = {}
    with ov.reference_visualize("reference") as (vis, stub), tempfile.TemporaryDirectory() as tmp:
        gcb = vis.generate_colored_boxes
        for K, S, B in BOX_CASES:
            tag = f"boxes_K{K}_S{S}_B{B}"
            np.random.seed(999)
            t = gcb(torch.zeros(B, K, 4, S, S, S), torch.eye(3)[None, None].repeat(B, K, 1, 1))
            st = np.random.get_state()
            out[tag + "_rng_keys"], out[tag + "_rng_pos"] = st[1].copy(), np.array(st[2])
            if K > 64:
                out[tag + "_prims"] = t[:, BIG_PRIMS].numpy()
                out[tag + "_corner"] = t[0, :, :, 0, 0, 0].numpy()          # every primitive at voxel (0, 0, 0)
            else:
                out[tag] = t.numpy()
        for B, P, S in PAYLOAD_CASES:
            tag = f"payload_B{B}_P{P}_S{S}"
            rm = CaptureRM(518, 518)
            recon = recon_param(B, P, S, 1000 + 10 * B + S)
            vis.visualize_primvolume(os.path.join(tmp, "x.jpg"), {}, recon, rm, "cpu")
            asset, boxes = rm.calls
            out[tag + "_recon"] = recon.numpy()
            for k in ("prim_rgba", "prim_pos", "prim_rot", "prim_scale", "RT", "K"):
                out[f"{tag}_{k}"] = asset[k].numpy()
            out[tag + "_boxes"] = boxes["prim_rgba"].numpy()
        for B, V, H in VIDEO_CASES:
            tag = f"video_B{B}_V{V + 1}_H{H}"
            rm = CaptureRM(H, H)
            vis.visualize_video_primvolume(tmp, {}, recon_param(B, 4, 4, 7), V, rm, "cpu")
            asset_calls = rm.calls[0::2]
            assert len(asset_calls) == V + 1 and len(stub.frames[os.path.join(tmp, "rgb.mp4")]) == (V + 1) * B
            out[tag + "_RT"] = torch.stack([c["RT"] for c in asset_calls], 0).numpy()
            out[tag + "_K"] = asset_calls[0]["K"].numpy()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
