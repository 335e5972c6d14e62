#!/usr/bin/env python
"""Recipe that stages the reference's UNMODIFIED ``dva/visualize.py`` under ``oracle/_ref/`` beside the ray marcher oracle/stage_ref.py
stages (TEST INFRASTRUCTURE; ``oracle/_ref/`` is git-ignored).

    python oracle/stage_visualize.py [SRC]      # SRC = a checkout of the reference (default /root/reference)

The file is copied byte for byte (sha256 in ``oracle/_ref/MANIFEST_visualize.json``).  Its list and its check are its own, so the
skip conditions of the ray-march suites (``stage_ref.raymarcher_staged``) do not depend on it.  Importing it also needs the staged
``dva/__init__.py`` and ``dva/ray_marcher.py`` (or ``tpxl_b200.ray_marcher`` in their place) and cv2 / torchvision; its ``imageio``
is replaced by oracle.visualize's frame-capturing stub.
"""
from __future__ import annotations

import json
import os
import shutil
import sys

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import stage_ref  # noqa: E402

DEST = stage_ref.DEST
DEFAULT_SRC = stage_ref.DEFAULT_SRC
VISUALIZE_FILES = ["dva/visualize.py"]


def stage(src: str = DEFAULT_SRC, dest: str = DEST) -> dict:
    if not os.path.isdir(src):
        raise FileNotFoundError(f"{src} not found: pass the path of a reference checkout")
    manifest = {"source": src, "files": {}}
    for rel in VISUALIZE_FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        manifest["files"][rel] = stage_ref._sha(d)
    with open(os.path.join(dest, "MANIFEST_visualize.json"), "w") as f:
        json.dump(manifest, f, indent=1, sort_keys=True)
    return manifest


def visualize_staged(dest: str = DEST) -> bool:
    return all(os.path.exists(os.path.join(dest, rel)) for rel in VISUALIZE_FILES)


if __name__ == "__main__":
    m = stage(sys.argv[1] if len(sys.argv) > 1 else DEFAULT_SRC)
    print(f"staged {len(m['files'])} reference file(s) under {DEST}")
