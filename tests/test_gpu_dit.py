"""GPU: DiT.forward / forward_with_cfg through the reference-facing classes (-> C ABI -> sm_90a kernels) against
(i) the fixture produced by the reference's own modules (fp32, config #1) and (ii) the oracle under the fp16 policy.

Tolerances (relative L2 over the whole output tensor):
  vs the fp16-policy oracle   : 3e-3  — same rounding points, different accumulation order (fp16 eps = 9.8e-4)
  vs the fp32 reference       : 1e-2  — the reference's own fp16 autocast path sits at the same distance (printed)
"""
import json
import os

import numpy as np
import pytest
import torch

import oracle
import tpxl_b200
from tpxl_b200 import synth
from gpu_util import rel_l2
import parity

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _model(cfg, sd):
    m = tpxl_b200.DiT(**cfg)
    m.load_state_dict(sd)
    return m.to(DEV).eval()


def test_config1_against_reference_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "dit_cfg1.npz"))
    cfg = json.loads(str(g["cfg"]))
    sd = synth.synth_state_dict(synth.dit_shapes(**cfg), int(g["seed"]))
    x, y = synth.synth_inputs(1, cfg["seq_length"], cfg["in_channels"], int(g["M"]), cfg["condition_channels"], int(g["seed"]) + 1000)
    t = torch.from_numpy(g["t"])
    m = _model(cfg, sd)
    with torch.no_grad():
        out = m.forward(x.to(DEV), t.to(DEV), y.to(DEV), torch.float16, True)
        out_cfg = m.forward_with_cfg(x.to(DEV), t.to(DEV), y.to(DEV), cfg_scale=6.0, precision_dtype=torch.float16, enable_amp=True)
        sdd = {k: v.to(DEV) for k, v in sd.items()}
        o16 = oracle.dit.forward(sdd, x.to(DEV), t.to(DEV), y.to(DEV), cfg["num_heads"], "fp16")
        o16_cfg = oracle.dit.forward_with_cfg(sdd, x.to(DEV), t.to(DEV), y.to(DEV), 6.0, cfg["num_heads"], "fp16")
    ref, ref_cfg = torch.from_numpy(g["forward"]).to(DEV), torch.from_numpy(g["forward_with_cfg"]).to(DEV)
    assert out.dtype == torch.float16 and out.shape == ref.shape
    r = dict(ours_vs_ref32=rel_l2(out.float(), ref), oracle16_vs_ref32=rel_l2(o16, ref), ours_vs_oracle16=rel_l2(out.float(), o16),
             cfg_ours_vs_ref32=rel_l2(out_cfg.float(), ref_cfg), cfg_oracle16_vs_ref32=rel_l2(o16_cfg, ref_cfg), cfg_ours_vs_oracle16=rel_l2(out_cfg.float(), o16_cfg))
    print(r)
    assert r["ours_vs_oracle16"] < 3e-3 and r["cfg_ours_vs_oracle16"] < 3e-3
    assert r["ours_vs_ref32"] < 1e-2 and r["cfg_ours_vs_ref32"] < 1e-2
    assert r["ours_vs_ref32"] < parity.bound(r["oracle16_vs_ref32"])


def test_null_branch_constant_equals_real_cross_attention():
    cfg = dict(seq_length=256, in_channels=68, condition_channels=768, hidden_size=384, depth=3, num_heads=16, attn_proj_bias=True, cond_drop_prob=0.1)
    sd = synth.synth_state_dict(synth.dit_shapes(**cfg), 21)
    x, y = synth.synth_inputs(2, 256, 68, 100, 768, 22)
    t = torch.tensor([960, 960])
    m = _model(cfg, sd)
    with torch.no_grad():
        a = m.forward_with_cfg(x.to(DEV), t.to(DEV), y.to(DEV), cfg_scale=6.0, enable_amp=True)
        m.collapse_null_branch = False
        b = m.forward_with_cfg(x.to(DEV), t.to(DEV), y.to(DEV), cfg_scale=6.0, enable_amp=True)
    assert rel_l2(a.float(), b.float()) < 1e-3


def test_residual_stream_and_batch_consistency():
    cfg = dict(seq_length=384, in_channels=68, condition_channels=768, hidden_size=256, depth=2, num_heads=8, attn_proj_bias=False, cond_drop_prob=0.1)
    sd = synth.synth_state_dict(synth.dit_shapes(**cfg), 23)
    x, y = synth.synth_inputs(3, 384, 68, 50, 768, 24)
    t = torch.tensor([40, 520, 960])
    m = _model(cfg, sd)
    with torch.no_grad():
        out = m.forward(x.to(DEV), t.to(DEV), y.to(DEV), torch.float16, True)
        res = m.debug_residual(3)
        sdd = {k: v.to(DEV) for k, v in sd.items()}
        ref, blocks = oracle.dit.forward(sdd, x.to(DEV), t.to(DEV), y.to(DEV), 8, "fp16", return_blocks=True)
        one = m.forward(x[1:2].to(DEV), t[1:2].to(DEV), y[1:2].to(DEV), torch.float16, True)
    assert rel_l2(res, blocks[-1]) < 2e-3
    assert rel_l2(out.float(), ref) < 3e-3
    assert rel_l2(one.float(), out[1:2].float()) < 1e-3      # per-sample independence (sharding contract, SURVEY §8e)
    assert m.forward(x.to(DEV), t.to(DEV), y.to(DEV)).dtype == torch.float32      # enable_amp=False returns fp32


def test_full_size_block_stack_against_oracle():
    """Shipped dimensions (N=2048, D=1152, 16 heads x 72, M=1370) with a shortened stack (4 blocks) so the fp32 oracle
    fits the time budget; full depth is covered by the sampler test below."""
    cfg = dict(synth.FULL_DIT, depth=4)
    sd = synth.device_state_dict(synth.dit_shapes(**cfg), 31, DEV, torch.float16)
    m = tpxl_b200.DiT(**cfg)
    m.load_state_dict(sd)
    m = m.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(32)
    x = torch.randn(1, 2048, 68, generator=g, device=DEV)
    y = torch.randn(1, 1370, 768, generator=g, device=DEV)
    t = torch.tensor([960], device=DEV)
    with torch.no_grad():
        out = m.forward_with_cfg(x, t, y, cfg_scale=6.0, enable_amp=True)
        sdf = {k: v.float() for k, v in sd.items()}
        o16 = oracle.dit.forward_with_cfg(sdf, x, t, y, 6.0, 16, "fp16")
        o32 = oracle.dit.forward_with_cfg(sdf, x, t, y, 6.0, 16, "fp32")
    r = dict(ours_vs_o16=rel_l2(out.float(), o16), ours_vs_o32=rel_l2(out.float(), o32), o16_vs_o32=rel_l2(o16, o32))
    print(r)
    assert r["ours_vs_o16"] < 3e-3
    assert r["ours_vs_o32"] < parity.bound(r["o16_vs_o32"])


def test_error_paths():
    cfg = dict(seq_length=128, in_channels=8, condition_channels=64, hidden_size=128, depth=1, num_heads=4, attn_proj_bias=True, cond_drop_prob=0.1)
    m = _model(cfg, synth.synth_state_dict(synth.dit_shapes(**cfg), 41))
    with pytest.raises(ValueError):
        m.forward(torch.zeros(1, 64, 8, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, 4, 64, device=DEV))
    with pytest.raises(ValueError):
        m.forward(torch.zeros(1, 128, 8, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(2, 4, 64, device=DEV))
    with pytest.raises(tpxl_b200._lib.TpxError):
        m.forward(torch.zeros(9, 128, 8, device=DEV), torch.zeros(9, dtype=torch.int64, device=DEV), torch.zeros(9, 4, 64, device=DEV))
    with pytest.raises(tpxl_b200._lib.TpxError):
        tpxl_b200.DiT(seq_length=8, in_channels=8, condition_channels=64, hidden_size=100, depth=1, num_heads=4).to(DEV)


def test_full_model_full_size_against_oracle_and_batch_of_four():
    """The shipped model end to end (28 blocks, 2048 tokens, 1370 context tokens): forward_with_cfg against the oracle
    (fp16 policy and fp32) for one sample, then a batch of four samples (config #5: 4 samples per GPU -> 8 sequences per
    forward) against the same samples run one at a time."""
    sd = synth.device_state_dict(synth.dit_shapes(**synth.FULL_DIT), 81, DEV, torch.float16)
    m = tpxl_b200.DiT(**synth.FULL_DIT)
    m.load_state_dict(sd)
    m = m.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(82)
    x = torch.randn(4, 2048, 68, generator=g, device=DEV)
    y = torch.randn(4, 1370, 768, generator=g, device=DEV)
    t = torch.tensor([960, 960, 480, 40], device=DEV)
    with torch.no_grad():
        one = m.forward_with_cfg(x[:1], t[:1], y[:1].contiguous(), cfg_scale=6.0, enable_amp=True)
        sdf = {k: v.float() for k, v in sd.items()}
        o16 = oracle.dit.forward_with_cfg(sdf, x[:1], t[:1], y[:1], 6.0, 16, "fp16")
        o32 = oracle.dit.forward_with_cfg(sdf, x[:1], t[:1], y[:1], 6.0, 16, "fp32")
        del sdf
        four = m.forward_with_cfg(x, t, y, cfg_scale=6.0, enable_amp=True)
        singles = torch.cat([m.forward_with_cfg(x[i:i + 1], t[i:i + 1], y[i:i + 1].contiguous(), cfg_scale=6.0, enable_amp=True) for i in range(4)])
    r = dict(ours_vs_o16=rel_l2(one.float(), o16), ours_vs_o32=rel_l2(one.float(), o32), o16_vs_o32=rel_l2(o16, o32), batch_vs_single=rel_l2(four.float(), singles.float()))
    print(r)
    assert torch.isfinite(four.float()).all()
    assert r["ours_vs_o16"] < 5e-3                      # 28 blocks deep, CFG 6: fp16 noise of both sides, amplified
    assert r["ours_vs_o32"] < parity.bound(r["o16_vs_o32"])
    assert r["batch_vs_single"] < 1e-3


def test_checkpoint_ingestion_from_file_without_retained_copy(tmp_path):
    """SURVEY §8f-4: an fp16 checkpoint file ({'ema': state_dict}, like model_sview_dit_fp16.pt) goes file -> packed device store with
    no retained copy; the result equals the load_state_dict path, and state_dict() still answers (read back from the device)."""
    cfg = dict(seq_length=128, in_channels=68, condition_channels=768, hidden_size=384, depth=2, num_heads=16, attn_proj_bias=True, cond_drop_prob=0.1)
    sd = synth.synth_state_dict(synth.dit_shapes(**cfg), 47)
    path = os.path.join(tmp_path, "dit_fp16.pt")
    torch.save({"ema": {k: v.half() for k, v in sd.items()}, "step": 1}, path)
    a = _model(cfg, sd)
    b = tpxl_b200.DiT(**cfg).to(DEV).eval()
    b.load_checkpoint(path)
    assert b._sd is None                                            # nothing but the packed store is kept
    x, y = synth.synth_inputs(1, 128, 68, 77, 768, 48)
    t = torch.tensor([480], device=DEV)
    with torch.no_grad():
        oa = a.forward_with_cfg(x.to(DEV), t, y.to(DEV), cfg_scale=6.0, enable_amp=True)
        ob = b.forward_with_cfg(x.to(DEV), t, y.to(DEV), cfg_scale=6.0, enable_amp=True)
    assert torch.equal(oa, ob)
    back = b.state_dict()
    assert list(back) == list(sd) and all(torch.equal(back[k].cpu(), sd[k].half()) for k in sd)
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad.pop("x_embedder.bias")
        b.load_state_dict(bad)
    v = tpxl_b200.VAE(**synth.FULL_VAE).to(DEV)
    vsd = synth.synth_state_dict(synth.vae_decoder_shapes(**synth.FULL_VAE), 49)
    vpath = os.path.join(tmp_path, "vae_fp16.pt")
    torch.save({"model_state_dict": dict({k: w.half() for k, w in vsd.items()}, **{"encoder.conv_in.weight": torch.zeros(4, 4)})}, vpath)
    v.load_checkpoint(vpath)
    w = tpxl_b200.VAE(**synth.FULL_VAE)
    w.load_state_dict(vsd)
    w = w.to(DEV)
    z = torch.randn(3, 1, 4, 4, 4, device=DEV)
    assert torch.equal(v.decode(z), w.decode(z))
