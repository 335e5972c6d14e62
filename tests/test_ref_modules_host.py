"""Host: the staged reference conditioner and PrimSDF, as oracle/refmods.py builds them (build_dinov2, build_primsdf), reproduce the
fixtures tests/golden/make_golden.py wrote by importing the reference checkout directly.  The GPU suite that runs these modules next to
the kernels (tests/test_gpu_ref_chain.py) therefore runs the modules the fixtures came from.  Skipped where oracle/_ref is not staged."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import dinov2 as odn
from oracle import refmods
from pictures import golden_picture, small_picture

pytestmark = pytest.mark.skipif(not (refmods.conditioner_available() and refmods.primsdf_available()),
                                reason="the reference's conditioner / PrimSDF not staged (python oracle/stage_ref.py where the reference checkout exists)")
REL = 1e-6


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def _untouched():
    return {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("models", "utils", "xformers", "trimesh")}


def test_staged_conditioner_reproduces_the_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "dinov2.npz"))
    before = _untouched()
    enc = refmods.build_dinov2(odn.synth_weights(int(g["seed"])))
    assert _untouched() == before, "build_dinov2 left reference modules in sys.modules"
    assert not enc.training and all(not p.requires_grad for p in enc.parameters())
    img = golden_picture(int(g["img_seed"]))
    with torch.no_grad():
        out = enc(torch.from_numpy(img))
        out_small = enc(torch.from_numpy(small_picture(img)))
    assert tuple(out.shape) == (1, 1370, 768)
    r = (_rel(out[:, ::6], g["out"]), _rel(out_small[:, ::24], g["out_small"]))
    print(f"staged conditioner vs dinov2.npz: out {r[0]:.2e}, out_small {r[1]:.2e}")
    assert r[0] <= REL and r[1] <= REL, r


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_staged_primsdf_reproduces_the_fixture(golden_dir, mode):
    g = np.load(os.path.join(golden_dir, "primsdf.npz"))
    before = _untouched()
    m = refmods.build_primsdf(torch.from_numpy(g["srt"]), torch.from_numpy(g["feat"])).train(mode == "train")
    assert _untouched() == before, "build_primsdf left reference modules in sys.modules"
    with torch.no_grad():
        out = m(torch.from_numpy(g["pts"]))
    cov = torch.from_numpy(g["covered"])
    assert int(cov.sum()) not in (0, len(cov)), "the fixture has covered and uncovered points"
    for k in ("sdf", "tex", "mat"):
        want = torch.from_numpy(g[k])
        if mode == "train":             # no nearest-voxel fill for uncovered points: their sdf stays 0
            if k == "sdf":
                assert float(out[k][~cov].abs().max()) == 0.0
            got, want = out[k][cov], want[cov]
        else:
            got = out[k]
        assert _rel(got, want) <= REL, (k, _rel(got, want))
