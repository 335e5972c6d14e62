"""Build libtpx_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python 3dtopia-xl_b200/build.py [--force]

Objects are rebuilt only when their sources (or shared headers) are newer; the .so lands in
3dtopia-xl_b200/lib/ (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libtpx_b200.so")
SOURCES = ["runtime.cu", "gemm_tc.cu", "elementwise.cu", "attention.cu", "attention_tc.cu", "vae_kernels.cu", "conv_halo.cu", "primsdf.cu", "marching_cubes.cu", "texture_bake.cu", "mesh_simplify.cu", "mesh_remesh.cu", "uv_unwrap.cu", "raymarch.cu", "visualize.cu", "conditioner.cu", "dit.cu", "vae.cu"]
HEADERS = ["tpx_common.cuh", "gemm_tc.cuh", "kernels.cuh", "mesh_common.cuh", "mc_tables.cuh", "bake_interp.cuh", os.path.join("..", "..", "include", "tpx.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr"]
# per-file extras: the decimation's and the remesher's fp64 and the unwrap's fp32 arithmetic follow their numpy oracles operation for operation, so no
# contraction into FMA
FILE_FLAGS = {"mesh_simplify.cu": ["-fmad=false"], "mesh_remesh.cu": ["-fmad=false"], "uv_unwrap.cu": ["-fmad=false"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _mtime(p: str) -> float:
    return os.path.getmtime(p) if os.path.exists(p) else 0.0


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdr_time = max(_mtime(os.path.join(CSRC, h)) for h in HEADERS)
    nvcc = _nvcc()
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        if force or _mtime(o) < max(_mtime(s), hdr_time):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [nvcc, *NVCC_FLAGS, *FILE_FLAGS.get(os.path.basename(s), []), "-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print("compiled", os.path.basename(s))

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(compile_one, jobs))
    objs = [os.path.join(OBJDIR, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _mtime(LIB) < max(_mtime(o) for o in objs):
        cmd = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
