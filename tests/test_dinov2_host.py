"""CPU: the host side of the DINOv2 encoder mirror (3dtopia-xl_b200/dinov2.py, SURVEY §8f-2) — state-dict contract, and the
algebra of its launch plan (Normalize folded into the patch embedding, (i, j, c) patch layout, LayerNorm affine expressed as
modulation, LayerScale expressed as the residual gate, token assembly) checked by emulating each kernel's documented contract in
torch and comparing the whole pipeline with the oracle."""
import importlib

import numpy as np
import pytest
import torch

import oracle
import tpxl_b200  # noqa: F401
from oracle import dinov2 as odn
from oracle.dit import Policy, r16

d = importlib.import_module("tpxl_b200.dinov2")
POLICY = Policy("fp16")      # the launch plan's rounding points (oracle/dinov2.py); on fp32 tensors an fp32 emulation of them


def test_state_dict_contract_and_errors():
    m = d.Dinov2Wrapper("dinov2_vitb14_reg", freeze=True)
    assert list(m.state_dict().keys()) == list(oracle.dinov2.shapes().keys())
    sd = oracle.dinov2.synth_weights(3)
    sd["model.mask_token"] = torch.zeros(1, 768)                 # present in hub checkpoints, dropped by the reference loader
    m.load_state_dict(sd)
    bare = {k[len("model."):]: v for k, v in sd.items()}           # dinov2_vitb14_reg4_pretrain.pth has no wrapper prefix
    m.load_state_dict(bare)
    assert torch.equal(m.state_dict()["model.norm.weight"], sd["model.norm.weight"])
    with pytest.raises(RuntimeError):
        m.load_state_dict({k: v for k, v in sd.items() if "ls1" not in k})
    with pytest.raises(NotImplementedError):
        d.Dinov2Wrapper("dinov2_vitl14_reg")
    with pytest.raises(tpxl_b200._lib.TpxError):
        m(torch.zeros(1, 518, 518, 3))


def test_launch_plan_matches_policy_oracle():
    """The wrapper's operands against the policy's definition (Normalize folded into the patch weights, (i, j, c) patch layout, token
    assembly, LayerNorm affine as modulation, LayerScale as the gate, the final norm's affine kept for the host), then the whole policy
    pipeline against the fp32 oracle."""
    torch.set_grad_enabled(False)
    try:
        sd = odn.synth_weights(105)
        m = d.Dinov2Wrapper()
        m.load_state_dict(sd)
        w = m._operands(torch.device("cpu"))
        rs = np.random.RandomState(7)
        img = torch.from_numpy(rs.uniform(0, 255, size=(1, 518, 518, 3)).astype(np.float32))
        n, g, np_, nt = 1, 37, 1369, 1374
        patches = torch.zeros(n * np_, d.KPAD, dtype=torch.float16)
        patches[:, :d.KPATCH] = (img / 255.0).reshape(n, g, 14, g, 14, 3).permute(0, 1, 3, 2, 4, 5).reshape(n * np_, d.KPATCH).half()
        tok = torch.empty(n, nt, 768)
        tok[:, 0], tok[:, 1:5], tok[:, 5:] = w["row0"], w["regs"], w["pos_patches"]
        tok[0, 5:] += r16(patches.float() @ w["patch_w"].float().t() + w["patch_b"].float())      # tpx_linear_gated, gate 1
        pe = odn.patch_embed(sd, img, POLICY)
        assert float((tok - pe).norm() / pe.norm()) < 1e-4          # accumulation order only: an fp16 rounding flip here and there
        for i in range(d.DEPTH):
            b = f"model.blocks.{i}."
            for nn_ in ("1", "2"):
                assert torch.equal(w[f"{i}.ln{nn_}.scale"].float(), r16(sd[b + f"norm{nn_}.weight"] - 1).view(1, -1))
                assert torch.equal(w[f"{i}.ln{nn_}.shift"].float(), r16(sd[b + f"norm{nn_}.bias"]).view(1, -1))
                assert torch.equal(w[f"{i}.ls{nn_}"].float(), r16(sd[b + f"ls{nn_}.gamma"]).view(1, -1))
        assert not w["zeros"].any()
        assert torch.equal(w["norm.weight"], sd["model.norm.weight"]) and torch.equal(w["norm.bias"], sd["model.norm.bias"])
        x = tok
        for i in range(d.DEPTH):
            x = odn.block(sd, i, x, POLICY)
        o = odn.final_norm(sd, x, POLICY)
        out = torch.cat([o[:, :1], o[:, 5:]], 1)
        ref = odn.forward(sd, img)
        rel = float((out - ref).norm() / ref.norm())
        assert rel < 3e-3, rel                                   # fp16-input contract against the fp32 oracle: ~1e-3
        worst = float(((out - ref).norm(dim=(0, 1)) / ref.norm(dim=(0, 1))).max())
        assert worst < 4e-3, worst                               # per channel (the final norm's affine in fp32: ~2e-3)
    finally:
        torch.set_grad_enabled(True)


def test_oracle_runs_in_the_image_dtype():
    """fp64 weights and an fp64 image run the exact encoder in fp64 (depth 1 to keep it short); the fp32 path is unchanged by it."""
    sd = odn.synth_weights(5, depth=1)
    img = torch.from_numpy(np.random.RandomState(3).uniform(0, 255, size=(1, 518, 518, 3)))
    with torch.no_grad():
        o64 = odn.forward({k: v.double() for k, v in sd.items()}, img, depth=1)
        o32 = odn.forward(sd, img.float(), depth=1)
    assert o64.dtype == torch.float64 and o32.dtype == torch.float32
    assert float((o32.double() - o64).norm() / o64.norm()) < 1e-5
