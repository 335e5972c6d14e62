#!/usr/bin/env python
"""Recipe that stages the UNMODIFIED reference modules of the hot path under ``oracle/_ref/`` (TEST INFRASTRUCTURE).

    python oracle/stage_ref.py [SRC]      # SRC = a checkout of the reference (default /root/reference)

``oracle/_ref/`` is git-ignored (no reference source ever enters the history); like the built ``.so`` it is a build
product of the tree.  The staged files let the ``-m gpu`` parity
tests and ``bench.py --impl reference`` execute the reference's own ``DiT`` / ``create_diffusion`` / ``VAE`` — on the
GPU under ``torch.autocast('cuda', fp16)`` (the contract north_star's tolerance is stated against,
models/dit_crossattn.py:197) and on the host cores in fp32 (the timing baseline).

What is staged (byte-identical copies, sha256 recorded in ``oracle/_ref/MANIFEST.json``):
    models/__init__.py, models/{dit_crossattn,attention,utils,vae3d_dib}.py, models/diffusion/*.py, utils/typing.py
Nothing else of the reference is needed on this path.  The one un-vendored dependency, ``xformers.ops``
(models/attention.py:17; unpinned, README.md:67), is NOT staged or copied from anywhere: ``oracle/refmods.py``
restates its contract with ``torch.nn.functional.scaled_dot_product_attention``.

The ray marcher's preview (``dva.ray_marcher.RayMarcher``) is staged too, so the ``-m gpu`` suite can run the reference's own CUDA
extensions as the oracle of csrc/raymarch.cu:
    dva/__init__.py, dva/ray_marcher.py, dva/mvp/extensions/{mvpraymarch/mvpraymarch.py, utils/utils.py}   (byte-identical)
and its two torch extensions are compiled FROM THE CHECKOUT (no source is copied) into oracle/_ref/build/, in parallel, with the
flags of their own setup.py except that ``-arch=sm_70`` becomes ``-gencode arch=compute_90a,code=sm_90a``; each ``.so`` is then
placed beside its wrapper, where ``from . import mvpraymarchlib`` / ``from . import utilslib`` find it.  The host compile gets
``-DNDEBUG``: utils.cpp:67 and :113 assert on a ``size()`` that ``std::optional`` does not have, and the reference's setup.py build
never compiles those asserts because setuptools passes Python's CFLAGS, which carry ``-DNDEBUG``.

The first and last stages of the image-to-SDF path are staged too (byte-identical), so the ``-m gpu`` suite can run them next to the
kernels: the image conditioner ``models/conditioner/image_dinov2.py`` with the ``dinov2/{hub,models,layers}`` files its import reaches
(CONDITIONER_FILES; torchvision is its one outside dependency), and ``models/primsdf.py`` (PRIMSDF_FILES; its ``trimesh`` import is unused
on the query path and stubbed by the loader).  ``oracle/refmods.py`` builds them.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
DEFAULT_SRC = "/root/reference"
FILES = [
    "models/__init__.py", "models/dit_crossattn.py", "models/attention.py", "models/utils.py", "models/vae3d_dib.py",
    "models/diffusion/__init__.py", "models/diffusion/diffusion_utils.py", "models/diffusion/gaussian_diffusion.py",
    "models/diffusion/respace.py", "models/diffusion/timestep_sampler.py", "utils/typing.py",
]
RAYMARCH_FILES = [
    "dva/__init__.py", "dva/ray_marcher.py", "dva/mvp/extensions/mvpraymarch/mvpraymarch.py", "dva/mvp/extensions/utils/utils.py",
]
CONDITIONER_FILES = [
    "models/conditioner/image_dinov2.py", "models/conditioner/dinov2/__init__.py",
    "models/conditioner/dinov2/hub/__init__.py", "models/conditioner/dinov2/hub/backbones.py", "models/conditioner/dinov2/hub/utils.py",
    "models/conditioner/dinov2/models/__init__.py", "models/conditioner/dinov2/models/vision_transformer.py",
    *[f"models/conditioner/dinov2/layers/{m}.py" for m in ("__init__", "attention", "block", "dino_head", "drop_path", "layer_scale", "mlp",
                                                           "patch_embed", "swiglu_ffn")],
]
PRIMSDF_FILES = ["models/primsdf.py"]
SM90A = ["-gencode", "arch=compute_90a,code=sm_90a"]
# name -> (directory under the checkout, sources, nvcc flags of its setup.py with the arch replaced)
EXTENSIONS = {
    "mvpraymarchlib": ("dva/mvp/extensions/mvpraymarch", ["mvpraymarch.cpp", "mvpraymarch_kernel.cu", "bvh.cu"],
                       ["-use_fast_math", *SM90A, "-std=c++17", "-lineinfo"]),
    "utilslib": ("dva/mvp/extensions/utils", ["utils.cpp", "utils_kernel.cu"], [*SM90A, "-std=c++14", "-lineinfo"]),
}
_BUILD = """
import sys
from torch.utils.cpp_extension import load
name, build_dir, flags, *sources = sys.argv[1:]
load(name=name, sources=sources, extra_cflags=["-DNDEBUG"], extra_cuda_cflags=flags.split(), build_directory=build_dir, verbose=False)
"""


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(src: str = DEFAULT_SRC, dest: str = DEST) -> dict:
    if not os.path.isdir(src):
        raise FileNotFoundError(f"{src} not found: pass the path of a reference checkout")
    manifest = {"source": src, "files": {}}
    for rel in FILES + RAYMARCH_FILES + CONDITIONER_FILES + PRIMSDF_FILES:
        s, d = os.path.join(src, rel), os.path.join(dest, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
        manifest["files"][rel] = _sha(d)
    manifest["extensions"] = build_raymarch_extensions(src, dest)
    with open(os.path.join(dest, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1, sort_keys=True)
    return manifest


def build_raymarch_extensions(src: str = DEFAULT_SRC, dest: str = DEST) -> dict:
    """Compile mvpraymarchlib and utilslib side by side (one process each) and place each .so beside its staged wrapper.
    Returns {placed .so (relative to dest): its nvcc flags}."""
    jobs = {}
    for name, (rel, sources, flags) in EXTENSIONS.items():
        build_dir = os.path.join(dest, "build", name)
        os.makedirs(build_dir, exist_ok=True)
        cmd = [sys.executable, "-c", _BUILD, name, build_dir, " ".join(flags), *[os.path.join(src, rel, s) for s in sources]]
        jobs[name] = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    placed = {}
    for name, p in jobs.items():
        log = p.communicate()[0]
        if p.returncode != 0:
            raise RuntimeError(f"building the reference's {name} failed:\n{log[-4000:]}")
        rel, _, flags = EXTENSIONS[name]
        so = os.path.join(rel, name + ".so")
        shutil.copyfile(os.path.join(dest, "build", name, name + ".so"), os.path.join(dest, so))
        placed[so] = " ".join(flags)
    return placed


def staged(dest: str = DEST) -> bool:
    return all(os.path.exists(os.path.join(dest, rel)) for rel in FILES)


def raymarcher_staged(dest: str = DEST) -> bool:
    sos = [os.path.join(rel, name + ".so") for name, (rel, _, _) in EXTENSIONS.items()]
    return all(os.path.exists(os.path.join(dest, rel)) for rel in RAYMARCH_FILES + sos)


def conditioner_staged(dest: str = DEST) -> bool:
    return all(os.path.exists(os.path.join(dest, rel)) for rel in CONDITIONER_FILES)


def primsdf_staged(dest: str = DEST) -> bool:
    return all(os.path.exists(os.path.join(dest, rel)) for rel in PRIMSDF_FILES)


if __name__ == "__main__":
    m = stage(sys.argv[1] if len(sys.argv) > 1 else DEFAULT_SRC)
    print(f"staged {len(m['files'])} reference files and built {len(m['extensions'])} extensions under {DEST}")
