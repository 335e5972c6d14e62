"""H100-native denoising hot path for 3DTopia-XL: DiT step (CFG x2) + DDIM/DDPM update + VAE decode.

Python host layer = the reference's own interfaces (``DiT``, ``create_diffusion``, ``VAE``) calling the
sm_90a kernels in ``lib/libtpx_b200.so`` through the C ABI of ``include/tpx.h``.  See DESIGN.md and
INTEGRATION.md.  There is no CPU or other-architecture fallback anywhere in this package.
"""
import sys
import types

from . import synth  # noqa: F401
from . import _lib  # noqa: F401
from . import bake, diffusion, dinov2, dit, mesh, pipeline, primsdf, ray_marcher, shard, unwrap, vae, visualize  # noqa: F401
from .diffusion import SpacedDiffusion, create_diffusion  # noqa: F401
from .dit import DiT  # noqa: F401
from .pipeline import LatentCodec, PrimXPipeline  # noqa: F401
from .primsdf import PrimSDF  # noqa: F401
from .ray_marcher import RayMarcher  # noqa: F401
from .vae import VAE  # noqa: F401

__version__ = "0.1.0"


def install(mcubes: bool = False, nvdiffrast: bool = False, uv_unwrap: bool = False, meshutils: bool = False) -> None:
    """Make the reference's import paths resolve to this implementation, so ``inference.py`` / ``app.py`` run
    unchanged:  ``models.dit_crossattn`` -> dit, ``models.vae3d_dib`` -> vae, ``models.diffusion`` -> diffusion,
    ``models.primsdf`` -> primsdf, ``models.conditioner.image_dinov2`` -> dinov2, ``dva.ray_marcher`` -> ray_marcher,
    ``dva.visualize`` -> visualize.
    (Equivalent to editing ``class_name`` in configs/inference_dit.yml:32,53; see INTEGRATION.md.)  If the reference's
    ``models`` package is importable it is imported first so its other members (conditioner, primsdf) keep working.
    ``mcubes=True`` also binds ``sys.modules["mcubes"]`` to a module whose ``marching_cubes`` is the GPU one of ``mesh``, so
    extract_texmesh (inference.py:119) runs without PyMCubes; by default ``mcubes`` is left alone.  ``nvdiffrast=True`` likewise binds
    ``sys.modules["nvdiffrast"]`` / ``["nvdiffrast.torch"]`` to the forward-only UV-space rasteriser of ``bake`` (inference.py:22,31,172-174).
    ``uv_unwrap=True`` binds ``sys.modules["utils.uv_unwrap"]`` (and the attribute of an importable ``utils`` package) to the GPU
    box-projection unwrap of ``unwrap`` (inference.py:142-143).  ``meshutils=True`` binds ``sys.modules["utils.meshutils"]`` (and the
    attribute) to ``clean_mesh`` / ``decimate_mesh`` of ``mesh`` (inference.py:126-129), so the export path needs no pymeshlab."""
    try:
        import models as ref_models  # the reference checkout, when it is on sys.path
    except Exception:
        ref_models = types.ModuleType("models")
        ref_models.__path__ = []
        sys.modules["models"] = ref_models
    for name, mod in (("dit_crossattn", dit), ("vae3d_dib", vae), ("diffusion", diffusion), ("primsdf", primsdf)):
        sys.modules["models." + name] = mod
        setattr(ref_models, name, mod)
    # the image conditioner's encoder (configs/inference_dit.yml:49, ``models.conditioner.image_dinov2.Dinov2Wrapper``): the mirror runs
    # on the wgmma GEMM / attention kernels with fp16 tensor-core inputs
    sys.modules["models.conditioner.image_dinov2"] = dinov2
    try:
        import models.conditioner as ref_cond
        setattr(ref_cond, "image_dinov2", dinov2)
    except Exception:
        pass
    # the preview renderer: ``from dva.ray_marcher import RayMarcher`` (inference.py:12) resolves here, so the reference's sm_70
    # ray-march extensions (dva/mvp/extensions/*) need not be built at all
    sys.modules["dva.ray_marcher"] = ray_marcher
    # and the preview renders: ``from dva.visualize import visualize_primvolume, visualize_video_primvolume`` (inference.py:15,
    # app.py:18) resolves to the device drop-in; the reference's own dva.visualize also imports over this ray_marcher, whose
    # generate_colored_boxes it needs
    sys.modules["dva.visualize"] = visualize
    try:
        import dva as ref_dva
        setattr(ref_dva, "ray_marcher", ray_marcher)
        setattr(ref_dva, "visualize", visualize)
    except Exception:
        pass
    if mcubes:
        sys.modules["mcubes"] = mesh.mcubes_module()
    if nvdiffrast:
        sys.modules["nvdiffrast"], sys.modules["nvdiffrast.torch"] = bake.nvdiffrast_modules()
    for flag, name, make in ((uv_unwrap, "uv_unwrap", unwrap.uv_unwrap_module), (meshutils, "meshutils", mesh.meshutils_module)):
        if flag:
            m = make()
            sys.modules["utils." + name] = m
            try:
                import utils as ref_utils
                setattr(ref_utils, name, m)
            except Exception:
                pass
