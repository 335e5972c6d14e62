"""GPU: the DINOv2 image encoder (tpxl_b200.dinov2, the ViT-B/14-reg that produces the context tokens) stage by stage against an fp64
oracle, and the kernels it runs at its own shapes.

* Taps.  ``Dinov2Wrapper._forward(image, taps)`` runs the launch plan as ``forward`` does and clones its buffers after the patch
  embedding, after every launch of every block and after the final norm.  With and without taps the output is bit-identical and the
  launch count is n + 12 x 8 + 1 for n images.
* Stage-local parity.  Each branch of the oracle (oracle/dinov2.py attn_branch / mlp_branch) runs on the kernel's own residual tap, in
  fp64, exactly ("exact") and with the encoder's documented rounding points ("policy", oracle.dit.Policy("fp16")), so errors do not
  compound.  What is compared is the branch's increment (tap after minus tap before), never the residual.  Bound, as relative L2
  against exact: ours <= 2.5 x policy + 1e-4 for every partition: per image, per (image, 128-token block) (block 0 holds the class
  and register rows, block 10 is the ragged 1280-1373), per channel, the class-token row of each image, and per (image, head) for
  q / k / v and the attention output.
* Elementwise stages.  Where the kernel and the policy see the same input and differ only in fp32 reduction order (norm1, norm2 and
  the final norm on the kernel's residual, the GELU on the kernel's fc1 output, the patch embedding onto the position rows), each
  element is within one fp16 ulp of the policy's value, plus the fp32 round-off the reduction may carry.
* End to end, the output of a full forward per channel against the exact fp64 encoder.
* Kernel unit tests at the encoder's shapes against fp64: tpx_gelu_erf over every finite fp16 value, tpx_ln_modulate at D = 768,
  tpx_attention_tc at Dh 64 with ragged key counts, tpx_linear_heads at Dh 64 with 1374-token sequences, tpx_linear_gated at K = 640
  and 3072 with subnormal LayerScale gates.
* The bound rejects a 1 % error on one head of one image, one 128-token block of the second image of a batch, one channel, or the
  class token alone (on real taps).
"""
import importlib
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dinov2 as odn
from oracle.dit import Policy, r16
from tpxl_b200 import _lib
from gpu_util import st
import parity

pytestmark = pytest.mark.gpu
d = importlib.import_module("tpxl_b200.dinov2")
DEV = "cuda:0"
EXACT, POLICY = Policy("fp32"), Policy("fp16")    # on fp64 tensors: the exact encoder, and the encoder's rounding points
NT, DIM, H, DH, DHP = 1374, 768, 12, 64, 80
LAUNCHES_PER_BLOCK = 8                            # ln1, qkv, attention, proj, ln2, fc1, gelu, fc2
DEPTH_LAUNCHES = 12 * LAUNCHES_PER_BLOCK
E2E_CHANNEL_BOUND = 6e-3                          # worst channel of the output against exact (fp16 contract; ~2e-3 expected)
HARD_CHANNELS = (17, 300, 641)                    # residual channels scaled x 50 in the hard draw (ViT high-norm channels)
T0 = time.time()
WORST = {}                                        # (case, stage) -> {partition: worst ratio to the bound}


# ---- weights, images, cases -------------------------------------------------------------------------------------------------------
def _hard_weights():
    """synth_weights(105) with LayerNorm gains log-uniform in [0.02, 3] (5 % negated), LayerScale log-uniform in [1e-5, 1] (fp16
    subnormal gates below 6.1e-5) and three residual channels x 50 from the token embedding on."""
    sd = odn.synth_weights(105)
    rs = np.random.RandomState(2718)
    for k, v in sd.items():
        if "norm" in k and k.endswith("weight"):
            g = np.exp(rs.uniform(np.log(0.02), np.log(3.0), v.shape))
            g[rs.uniform(size=v.shape) < 0.05] *= -1
            sd[k] = torch.from_numpy(g.astype(np.float32))
        elif k.endswith("gamma"):
            sd[k] = torch.from_numpy(np.exp(rs.uniform(np.log(1e-5), 0.0, v.shape)).astype(np.float32))
    ch = list(HARD_CHANNELS)
    for k in ("model.cls_token", "model.pos_embed", "model.register_tokens"):
        sd[k][..., ch] *= 50
    sd["model.patch_embed.proj.weight"][ch] *= 50
    sd["model.patch_embed.proj.bias"][ch] *= 50
    return sd


_MODEL = {}


def _model(name):
    """(Dinov2Wrapper on the GPU, fp64 state dict on the GPU)."""
    if name not in _MODEL:
        sd = odn.synth_weights(105) if name == "synth" else _hard_weights()
        for k, v in sd.items():
            assert torch.isfinite(v).all(), k
        m = d.Dinov2Wrapper()
        m.load_state_dict(sd)
        _MODEL[name] = (m.to(DEV).eval(), {k: v.to(DEV, torch.float64) for k, v in sd.items()})
    return _MODEL[name]


def _image(seed, size=518):
    """A smooth colour field with texture and noise, 0..255, [1, size, size, 3] fp32."""
    rs = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, size), np.linspace(0, 1, size), indexing="ij")
    f = rs.uniform(2, 9, 6)
    img = np.stack([127 + 100 * np.sin(f[0] * xx + f[1] * yy), 127 + 100 * np.cos(f[2] * yy - f[3] * xx), 255 * (xx * yy) ** (f[4] / 5)], -1)
    img = np.clip(img + 12 * rs.standard_normal((size, size, 3)), 0, 255).astype(np.float32)
    return torch.from_numpy(img[None]).to(DEV)


ALL = tuple(range(12))
# case -> (weights, image seeds (one per image of the batch), image size, blocks checked)
CASES = {
    "synth_b1": ("synth", (1,), 518, ALL),
    "hard_b1": ("hard", (2,), 518, ALL),
    "synth_b2": ("synth", (1, 3), 518, (0, 5, 11)),
    "hard_b3": ("hard", (4, 2, 5), 518, (0, 5, 11)),          # 4122 rows: 128-row tiles straddle both image boundaries
    "synth_224": ("synth", (6,), 224, (0, 5, 11)),            # the resize path
}


# ---- partitions and the bound -----------------------------------------------------------------------------------------------------
PARTS = {"image": parity.sequence, "block": parity.block(128), "channel": parity.channel,
         "class": parity.tokens(torch.tensor([0] + [-1] * (NT - 1))), "head": parity.head(DH)}


def _check(key, ours, pol, ref, parts):
    """ours / pol / ref fp64 [S, N, C] against the bound (tests/parity.py) per partition named in parts; the worst ratios go to WORST."""
    worst = WORST.setdefault(key, {})
    for how, r in parity.check(f"{key}", ours, pol, ref, {h: PARTS[h] for h in parts}).items():
        worst[how] = max(worst.get(how, 0.0), r)


def _check_elementwise(key, ours, pol, extra=0.0):
    """|ours - pol| <= 1 fp16 ulp of the policy's value + extra (the fp32 round-off the kernel's reduction may carry)."""
    r, off = parity.check_elementwise(f"{key}", ours, pol, parity.ulp16(pol) + extra)
    w = WORST.setdefault(key, {})
    w["element"] = max(w.get("element", 0.0), r)
    w["elements off"] = w.get("elements off", 0) + off


def _ln_extra(x, m):
    """fp32 round-off of a two-pass LayerNorm on the rows x [.., D] (fp64), times the gain m: the mean carries ~log2(D) + 24 roundings
    of mean |x| (the per-lane serial sums and the warp tree), (x - mean) * rstd * m a few of |x - mean|."""
    mu = x.mean(-1, keepdim=True)
    rstd = (x.var(-1, unbiased=False, keepdim=True) + 1e-6).rsqrt()
    return 2.0 ** -24 * (4 * (x - mu).abs() + 40 * x.abs().mean(-1, keepdim=True)) * rstd * m.abs()


def _mod_gain(w):
    return r16(1 + r16(w - 1))


# ---- one case ---------------------------------------------------------------------------------------------------------------------
def _heads(t, n):
    """[n, H, NT, >= 64] -> [n, NT, H * 64] (the head-major token layout of the attention output)."""
    return t[..., :DH].permute(0, 2, 1, 3).reshape(n, NT, H * DH).double()


_KEPT = {}


def _case(case):
    name, seeds, size, blocks = CASES[case]
    m, sd64 = _model(name)
    img = torch.cat([_image(s, size) for s in seeds])
    n = img.shape[0]
    lib = _lib.lib()
    taps = {}
    kept = {}
    with torch.no_grad():
        # ---- the forward with and without taps; every image against its own single-image run ----
        out = m(img)
        n0 = lib.tpx_launch_count()
        out_t = m._forward(img, taps)
        assert lib.tpx_launch_count() - n0 == n + DEPTH_LAUNCHES + 1
        assert torch.equal(out, out_t), "taps changed the output"
        assert torch.isfinite(out).all()
        for j in range(n if n > 1 else 0):
            one = m(img[j:j + 1])
            r = float((out[j] - one[0]).double().norm() / one.double().norm())
            assert r < 1e-4, (case, j, r)          # tile widths depend on the row count: not necessarily bit-identical
        if case == "synth_b1":
            n0 = lib.tpx_launch_count()
            assert m._forward(img, {}, stop=(0, "att")) is None
            assert lib.tpx_launch_count() - n0 == n + 3
        img64 = img.double()

        # ---- patch embedding onto the position rows, element by element ----
        pe = odn.patch_embed(sd64, img64, POLICY)
        tok = taps["embed"].double()
        pos = sd64["model.pos_embed"][0, 1:]
        Wn = sd64["model.patch_embed.proj.weight"] / torch.tensor(odn.STD, dtype=torch.float64, device=DEV).view(1, 3, 1, 1)
        x01 = img64.permute(0, 3, 1, 2)
        if size != odn.IMG:
            x01 = F.interpolate(x01, size=(odn.IMG, odn.IMG), mode="bicubic", align_corners=False, antialias=True)
        mag = F.conv2d(r16(x01 / 255.0).abs(), r16(Wn).abs(), stride=odn.PATCH).flatten(2).transpose(1, 2)
        extra = 588 * 2.0 ** -24 * mag + 2.0 ** -23 * tok[:, 5:].abs()      # fp32 accumulation of 588 products; the fp32 add onto pos
        _check_elementwise((case, "patch embed"), tok[:, 5:] - pos, pe[:, 5:] - pos, extra)
        assert torch.allclose(tok[:, :5], pe[:, :5], rtol=2.0 ** -23, atol=0), "class / register rows"

        # ---- blocks ----
        for i in blocks:
            xin = (taps["embed"] if i == 0 else taps[(i - 1, "res2")]).double()
            # attention branch
            tp = {"exact": {}, "policy": {}}
            inc_e = odn.attn_branch(sd64, i, xin, EXACT, tp["exact"])
            inc_p = odn.residual_add(xin, odn.attn_branch(sd64, i, xin, POLICY, tp["policy"]), POLICY) - xin
            p = f"model.blocks.{i}."
            _check_elementwise((case, "norm1"), taps[(i, "ln1")].view(n, NT, DIM), tp["policy"]["ln"],
                               _ln_extra(xin, _mod_gain(sd64[p + "norm1.weight"])))
            q, k, vT = taps[(i, "q")], taps[(i, "k")], taps[(i, "vT")]
            assert not q[..., DH:].any() and not k[..., DH:].any(), "q / k padding columns not zero"
            assert not vT[:, :, DH:].any() and not vT[..., NT:].any(), "vT padding not zero"
            for nm, ours in (("q", _heads(q, n)), ("k", _heads(k, n)), ("v", _heads(vT[..., :NT].transpose(-1, -2), n))):
                _check((case, nm), ours, _heads(tp["policy"][nm], n), _heads(tp["exact"][nm], n), ("head",))
            trip = (taps[(i, "att")].view(n, NT, DIM).double(), tp["policy"]["ao"], tp["exact"]["ao"])
            _check((case, "attention out"), *trip, ("head", "block"))
            if i == 0:
                kept["att"] = trip
            trip = ((taps[(i, "res1")].double() - xin), inc_p, inc_e)
            _check((case, "attn increment"), *trip, ("image", "block", "channel", "class"))
            if i == 0:
                kept["attn inc"] = trip
            # MLP branch
            xin = taps[(i, "res1")].double()
            tp = {"exact": {}, "policy": {}}
            inc_e = odn.mlp_branch(sd64, i, xin, EXACT, tp["exact"])
            inc_p = odn.residual_add(xin, odn.mlp_branch(sd64, i, xin, POLICY, tp["policy"]), POLICY) - xin
            _check_elementwise((case, "norm2"), taps[(i, "ln2")].view(n, NT, DIM), tp["policy"]["ln"],
                               _ln_extra(xin, _mod_gain(sd64[p + "norm2.weight"])))
            _check_elementwise((case, "gelu"), taps[(i, "hid")], r16(F.gelu(taps[(i, "fc1")].double())))
            _check((case, "mlp hidden"), taps[(i, "hid")].view(n, NT, 4 * DIM).double(), tp["policy"]["hid"], tp["exact"]["hid"],
                   ("image", "block", "channel"))
            trip = ((taps[(i, "res2")].double() - xin), inc_p, inc_e)
            _check((case, "mlp increment"), *trip, ("image", "block", "channel", "class"))
            if i == 0:
                kept["mlp inc"] = trip

        # ---- final norm on the kernel's last residual, and the output end to end against exact ----
        last = taps[(11, "res2")].double()
        _check_elementwise((case, "final norm"), taps["out16"].view(n, NT, DIM), r16(F.layer_norm(last, (DIM,), eps=1e-6)),
                           _ln_extra(last, torch.ones(DIM, dtype=torch.float64, device=DEV)))
        ref = odn.forward(sd64, img64)
        o = out.double()
        per_ch = ((o - ref).norm(dim=(0, 1)) / ref.norm(dim=(0, 1)))
        # the same residual through the modulation form of the final norm's affine, h(LN(x) h(1 + h(g - 1)) + h(b)) (the form the
        # encoder used before its affine moved after the fp16 boundary), for comparison
        wv = sd64["model.norm.weight"].float()
        o_mod = torch.empty(n * NT, DIM, dtype=torch.float16, device=DEV)
        sc = (wv - 1).half().view(1, DIM).contiguous()
        sh = sd64["model.norm.bias"].float().half().view(1, DIM).contiguous()
        _lib.check(lib.tpx_ln_modulate(taps[(11, "res2")].data_ptr(), n * NT, DIM, 1e-6, sh.data_ptr(), sc.data_ptr(), DIM, n * NT, 1,
                                       o_mod.data_ptr(), None, None, 0, st()))
        o_mod = o_mod.view(n, NT, DIM).double()
        o_mod = torch.cat([o_mod[:, :1], o_mod[:, 5:]], 1)
        per_ch_mod = ((o_mod - ref).norm(dim=(0, 1)) / ref.norm(dim=(0, 1)))
        whole = float((o - ref).norm() / ref.norm())
        print(f"{case:10s} end to end: whole {whole:.2e}, class token {float((o[:, 0] - ref[:, 0]).norm() / ref[:, 0].norm()):.2e}, "
              f"worst channel {float(per_ch.max()):.2e} (modulation-form affine: {float(per_ch_mod.max()):.2e}), bound {E2E_CHANNEL_BOUND:.0e}")
        assert float(per_ch.max()) < E2E_CHANNEL_BOUND, (int(per_ch.argmax()), float(per_ch.max()))
        WORST.setdefault((case, "end to end"), {})["channel"] = float(per_ch.max()) / E2E_CHANNEL_BOUND
    for key in [k for k in WORST if k[0] == case]:
        print(f"{case:10s} {key[1]:16s} worst / bound: " + ", ".join(f"{h} {v:.3f}" if isinstance(v, float) else f"{h} {v}"
                                                                   for h, v in WORST[key].items()))
    return kept



@pytest.mark.parametrize("case", list(CASES))
def test_stage_local_parity(case):
    kept = _case(case)
    if case in ("synth_b1", "synth_b2"):
        _KEPT[case] = kept


def test_bound_rejects_one_percent_errors():
    """On real block-0 taps, a 1 % error in ours on one head of one image (attention output), one 128-token block of the second image
    of a batch of two (attention increment), one channel (MLP increment) or the class token alone (attention increment) fails the
    bound, while the taps as they are pass it."""
    k1 = _KEPT.get("synth_b1") or _case("synth_b1")
    k2 = _KEPT.get("synth_b2") or _case("synth_b2")
    for what, kept, tap, how, region in (("head", k1, "att", "head", (0, slice(None), slice(5 * DH, 6 * DH))),
                                         ("128-token block of image 1", k2, "attn inc", "block", (1, slice(640, 768))),
                                         ("channel", k1, "mlp inc", "channel", (slice(None), slice(None), 517)),
                                         ("class token", k1, "attn inc", "class", (slice(None), 0))):
        ours, pol, ref = kept[tap]
        parts = {how: PARTS[how]}
        assert not parity.rejects(ours, pol, ref, parts)
        bad = ours.clone()
        bad[region] *= 1.01
        o, p = parity.ratios(bad, pol, ref, PARTS[how])
        print(f"1 % on one {what} ({tap}): worst {how} partition at {float((o / parity.bound(p)).max()):.1f} x the bound")
        assert parity.rejects(bad, pol, ref, parts), what


# ---- kernel unit tests at the encoder's shapes --------------------------------------------------------------------------------------
def _gelu_ref(x16):
    return r16(F.gelu(x16.double()))


def _gelu_run(x16, sentinel=-1234.0):
    n = x16.numel()
    buf = torch.full((n + 64,), sentinel, dtype=torch.float16, device=DEV)
    buf[:n] = x16
    _lib.check(_lib.lib().tpx_gelu_erf(buf.data_ptr(), n, st()), "tpx_gelu_erf")
    torch.cuda.synchronize()
    assert bool((buf[n:] == sentinel).all()), "tpx_gelu_erf wrote past n"
    return buf[:n]


def test_gelu_erf_every_finite_fp16_value():
    """tpx_gelu_erf (fp32 erf on the fp16 value, one rounding) within 1 ulp of h(gelu_fp64(x)) for all 63488 finite fp16 inputs; also
    n = 8 and an n past one sweep of the grid-stride loop."""
    allv = torch.from_numpy(np.arange(65536, dtype=np.uint16).view(np.float16).copy())
    x = allv[torch.isfinite(allv.float())].to(DEV)
    assert x.numel() == 63488
    ours, ref = _gelu_run(x), _gelu_ref(x)
    err = (ours.double() - ref).abs()
    assert bool((err <= parity.ulp16(ref)).all()), x[err > parity.ulp16(ref)][:8].tolist()
    print(f"gelu_erf: {int((err > 0).sum())} of {x.numel()} finite fp16 inputs one ulp off h(gelu_fp64(x)), the rest exact")
    g = torch.Generator(device=DEV).manual_seed(11)
    x8 = (torch.randn(8, generator=g, device=DEV) * 3).half()
    assert bool(((_gelu_run(x8).double() - _gelu_ref(x8)).abs() <= parity.ulp16(_gelu_ref(x8))).all())
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nbig = sms * 8 * 256 * 8 + 8 * 1001                # more than one grid-stride sweep: the loop wraps
    xb = (torch.randn(nbig, generator=g, device=DEV) * 3).half()
    assert bool(((_gelu_run(xb).double() - _gelu_ref(xb)).abs() <= parity.ulp16(_gelu_ref(xb))).all())


def test_ln_modulate_d768_offset_rows():
    """tpx_ln_modulate at D = 768 (the encoder's width) on rows with an offset of 300 and three outlier channels x 50, with
    LayerNorm-gain-like scales, against fp64 element by element."""
    g = torch.Generator(device=DEV).manual_seed(5)
    rows = 2 * NT + 7
    x = 300 + torch.randn(rows, DIM, generator=g, device=DEV)
    x[:, list(HARD_CHANNELS)] = 300 + 50 * torch.randn(rows, len(HARD_CHANNELS), generator=g, device=DEV)
    gain = torch.exp(torch.empty(DIM, device=DEV).uniform_(np.log(0.02), np.log(3.0), generator=g))
    gain[::19] *= -1
    scale = (gain - 1).half().view(1, DIM)
    shift = (0.1 * torch.randn(1, DIM, generator=g, device=DEV)).half()
    out = torch.full((rows + 1, DIM), 7.0, dtype=torch.float16, device=DEV)
    x_in = x.clone()
    _lib.check(_lib.lib().tpx_ln_modulate(x.data_ptr(), rows, DIM, 1e-6, shift.data_ptr(), scale.data_ptr(), DIM, rows, 1, out.data_ptr(),
                                          None, None, 0, st()), "tpx_ln_modulate")
    torch.cuda.synchronize()
    assert torch.equal(x, x_in) and bool((out[rows] == 7.0).all())
    x64 = x.double()
    m = r16(1 + scale.double())
    ref = r16(F.layer_norm(x64, (DIM,), eps=1e-6) * m + shift.double())
    _check_elementwise(("unit", "ln_modulate D768"), out[:rows], ref, _ln_extra(x64, m))


def _attn_inputs(B, Nq, Nk, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    NkPad = (Nk + 7) // 8 * 8
    q = torch.zeros(B, H, Nq, DHP, dtype=torch.float16, device=DEV)
    k = torch.zeros(B, H, Nk, DHP, dtype=torch.float16, device=DEV)
    vT = torch.zeros(B, H, DHP, NkPad, dtype=torch.float16, device=DEV)
    q[..., :DH] = (torch.randn(B, H, Nq, DH, generator=g, device=DEV) * 8).half()       # logits with a standard deviation of ~8
    tile = torch.arange(Nk, device=DEV) // 128
    k[..., :DH] = (torch.randn(B, H, Nk, DH, generator=g, device=DEV) * (1.0 + 0.5 * tile.float())[:, None]).half()
    vT[:, :, :DH, :Nk] = torch.randn(B, H, DH, Nk, generator=g, device=DEV).half()
    return q, k, vT, NkPad


def _attn_run(q, k, vT, B, Nq, Nk, NkPad):
    out = torch.full((B, Nq, H * DH), 9.0, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().tpx_attention_tc(q.data_ptr(), k.data_ptr(), vT.data_ptr(), out.data_ptr(), B, H, Nq, Nk, NkPad, DH, DH ** -0.5, st()),
               "tpx_attention_tc")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B,Nq,Nk", [(1, NT, NT), (3, NT, NT), (1, 200, 129), (2, 256, 191), (1, 130, 255)])
def test_attention_tc_dh64_ragged(B, Nq, Nk):
    """tpx_attention_tc at Dh 64 (the encoder's heads) with peaky logits, per (image, head) against fp64 softmax on the fp16 operands;
    key counts that leave a partial last 128-key tile.  V's padding (rows 64-79 and key columns >= Nk) only has to be finite: the
    output does not change when it holds 7.0 instead of 0."""
    q, k, vT, NkPad = _attn_inputs(B, Nq, Nk, 100 * B + Nk)
    out = _attn_run(q, k, vT, B, Nq, Nk, NkPad)
    s = torch.matmul(q[..., :DH].double(), k[..., :DH].double().transpose(-1, -2)) * DH ** -0.5
    ref = torch.matmul(torch.softmax(s, -1), vT[:, :, :DH, :Nk].double().transpose(-1, -2))          # [B, H, Nq, 64]
    ours = out.view(B, Nq, H, DH).permute(0, 2, 1, 3).double()
    assert torch.isfinite(ours).all()
    rel = ((ours - ref).norm(dim=(2, 3)) / ref.norm(dim=(2, 3)))
    print(f"attention_tc Dh 64 B {B} Nq {Nq} Nk {Nk}: worst (image, head) rel L2 {float(rel.max()):.2e}")
    assert float(rel.max()) < 3e-3, rel
    assert float((ours - ref).abs().max()) < 2e-2
    vP = vT.clone()
    vP[:, :, DH:] = 7.0
    vP[..., Nk:] = 7.0
    assert torch.equal(_attn_run(q, k, vP, B, Nq, Nk, NkPad), out), "V padding changed the output"


@pytest.mark.parametrize("tile", [0, 144, 192])
@pytest.mark.parametrize("nimg", [1, 2, 3])
def test_linear_heads_dh64(nimg, tile):
    """tpx_linear_heads at the encoder's qkv shape (N 2304, K 768, 12 heads x 64 padded to 80, 1374 tokens per image, V transposed
    to ld 1376): the per-thread head-split epilogue with 144- / 192-wide tiles that straddle heads and, across rows, images.  Each
    element within 1 ulp of h(A W^T + b); the pad columns zero; vT's columns >= 1374 untouched."""
    g = torch.Generator(device=DEV).manual_seed(31 * nimg + tile)
    M, N, K, ld = nimg * NT, 3 * DIM, DIM, 1376
    A = torch.randn(M, K, generator=g, device=DEV).half()
    W = (torch.randn(N, K, generator=g, device=DEV) * K ** -0.5).half()
    b = (0.02 * torch.randn(N, generator=g, device=DEV)).half()
    sent = 5.0
    q = torch.full((nimg, H, NT, DHP), sent, dtype=torch.float16, device=DEV)
    k = torch.full_like(q, sent)
    vT = torch.full((nimg, H, DHP, ld), sent, dtype=torch.float16, device=DEV)
    _lib.check(_lib.lib().tpx_linear_heads(A.data_ptr(), K, W.data_ptr(), b.data_ptr(), q.data_ptr(), k.data_ptr(), vT.data_ptr(), M, N, K, DIM,
                                           H, DH, DHP, NT, 1.0, tile, 2, ld, st()), "tpx_linear_heads")
    torch.cuda.synchronize()
    acc = A.double() @ W.double().t() + b.double()
    ref = r16(acc).view(nimg, NT, 3, H, DH).permute(2, 0, 3, 1, 4)                   # [3, nimg, H, NT, 64]
    extra = K * 2.0 ** -24 * (A.double().abs() @ W.double().abs().t() + b.double().abs())
    extra = extra.view(nimg, NT, 3, H, DH).permute(2, 0, 3, 1, 4)
    for w, ours in ((0, q[..., :DH]), (1, k[..., :DH]), (2, vT[:, :, :DH, :NT].transpose(-1, -2))):
        _check_elementwise(("unit", f"linear_heads tile {tile}"), ours, ref[w], extra[w])
    assert not q[..., DH:].any() and not k[..., DH:].any(), "q / k pad columns not zero"
    assert not vT[:, :, DH:, :NT].any(), "vT pad rows not zero"
    assert bool((vT[..., NT:] == sent).all()), "vT columns >= n_seq_tokens written"


@pytest.mark.parametrize("K,M", [(640, 1369), (3072, 2 * NT)])
def test_linear_gated_layerscale(K, M):
    """tpx_linear_gated at the patch embedding's K = 640 (M = 1369) and fc2's K = 3072 (M = 2 x 1374) with one per-channel gate (a
    LayerScale: log-uniform in [1e-7, 1], fp16 subnormals below 6.1e-5, some negative, one zero): xres(fp32) += h(h(gamma) h(A W^T + b))."""
    g = torch.Generator(device=DEV).manual_seed(K + M)
    A = torch.randn(M, K, generator=g, device=DEV).half()
    W = (torch.randn(DIM, K, generator=g, device=DEV) * K ** -0.5).half()
    b = (0.02 * torch.randn(DIM, generator=g, device=DEV)).half()
    gate = torch.exp(torch.empty(DIM, device=DEV).uniform_(np.log(1e-7), 0.0, generator=g))
    gate[::7] *= -1
    gate[3] = 0
    gate = gate.half().view(1, DIM)
    assert bool(((gate.abs() < 2.0 ** -14) & (gate != 0)).any())
    x0 = torch.randn(M, DIM, generator=g, device=DEV) * 3
    x = x0.clone()
    _lib.check(_lib.lib().tpx_linear_gated(A.data_ptr(), K, W.data_ptr(), b.data_ptr(), gate.data_ptr(), DIM, 1, M, x.data_ptr(), DIM, M, DIM, K, 0,
                                           st()), "tpx_linear_gated")
    torch.cuda.synchronize()
    acc = A.double() @ W.double().t() + b.double()
    inc = r16(gate.double() * r16(acc))
    # the fp32 accumulation may round h(acc + b) the other way where acc lies within its round-off of a rounding boundary; the gate
    # then multiplies a value one ulp away
    budget = K * 2.0 ** -24 * (A.double().abs() @ W.double().abs().t() + b.double().abs())
    near_tie = parity.ulp16(r16(acc)) / 2 - (acc - r16(acc)).abs() <= budget
    extra = (budget + near_tie * parity.ulp16(r16(acc))) * gate.double().abs() + 2.0 ** -23 * x.double().abs()
    _check_elementwise(("unit", f"linear_gated K {K}"), x.double() - x0.double(), inc, extra)


def test_wall_time():
    print(f"test_gpu_dinov2_stages: {time.time() - T0:.0f} s since the module was imported")
