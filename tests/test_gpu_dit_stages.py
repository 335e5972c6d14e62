"""GPU: the DiT forward stage by stage against an fp64 oracle.

* Stops.  ``DiT.debug_stage`` (tpx_dit_debug_stage) runs the forward's own schedule up to the token embedding or up to the gated GEMM
  of block i's cross-attention, self-attention or MLP branch; ``DiT.debug_tap`` (tpx_dit_debug_tap) reads the residual stream, the
  attention output, the modulation rows and the pre-guidance output from the workspace.
* Stage-local parity.  Each branch of the oracle (oracle/dit.py cross_branch / self_branch / mlp_branch / final_apply) runs on the
  kernel's own previous tap and the kernel's own modulation rows, so errors do not compound, twice in fp64: exactly ("exact") and with
  the fp16 policy's rounding points ("policy", the reference under autocast).  What is compared is a branch's increment to the residual
  stream, tap after minus tap before, never the residual itself: the residual is 20 to 500 times larger and dilutes a branch's error.
  Bound, as relative L2 against exact: ours <= 2.5 x policy + 1e-4 for every partition: per sequence (the cond and uncond halves
  separately), per (sequence, 128-token block) (the last block is ragged where N % 128 != 0: GEMM tile and attention tail errors
  land there), per channel (144- / 128-wide tiles and 24-column head groups), and per (sequence, head) of the attention output.
  Under CFG the null-context half of the cross and self increments holds one constant per channel, repeated over every token; its
  channels are checked by their means against the policy's instead (_check_with_null_half).
* The modulation rows are a stage of their own (per sample and D-wide chunk, and per row of the timestep table); the token embedding
  is checked element by element at fp32 round-off; the CFG combine bit for bit on the kernel's own pre-guidance output.
* The bound rejects a 1 % error on one head of one sequence, one 128-token block of one sequence, or one channel (checked on real
  taps): the class of error a whole-tensor comparison of the output misses.
"""
import time

import pytest
import torch
import torch.nn.functional as F

import parity
import tpxl_b200
from oracle import dit as od
from tpxl_b200 import _lib, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EXACT, POLICY = od.Policy("fp32"), od.Policy("fp16")     # "fp32" has no rounding point: on fp64 tensors it is the exact fp64 reference
CFG_SCALE = 6.0
T_VALUES = [999, 0, 480, 40, 960, 250, 700, 120]         # distinct per sample, 0 and 999 among them
T0 = time.time()
WORST = {}                                                # (case, stage) -> {partition: worst ratio to the bound}

# width, heads, depth, context length; N = sequence length
MODELS = {
    "shipped": dict(N=2048, D=1152, H=16, depth=3, M=1370),
    "max_batch": dict(N=2048, D=1152, H=16, depth=2, M=1370),
    "ragged": dict(N=1000, D=1152, H=16, depth=2, M=77),
    "full_depth": dict(N=2048, D=1152, H=16, depth=28, M=1370),
    "dh32": dict(N=384, D=256, H=8, depth=2, M=50),
    "dh24": dict(N=384, D=384, H=16, depth=2, M=77),
    "dh64": dict(N=384, D=512, H=8, depth=2, M=77),
}
# case -> (model, batch, use_cfg, blocks checked)
CASES = {
    "shipped_b1": ("shipped", 1, 1, [0, 1, 2]),
    "shipped_b4": ("shipped", 4, 1, [0, 1, 2]),
    "max_batch_b8": ("max_batch", 8, 1, [0, 1]),
    "ragged_cfg1": ("ragged", 3, 1, [0, 1]),
    "ragged_cfg2": ("ragged", 3, 2, [0, 1]),
    "dh32_b3": ("dh32", 3, 0, [0, 1]),
    "dh32_cfg_b2": ("dh32", 2, 1, [0, 1]),
    "dh24_b3": ("dh24", 3, 0, [0, 1]),
    "dh24_cfg_b2": ("dh24", 2, 1, [0, 1]),
    "dh64_b3": ("dh64", 3, 0, [0, 1]),
    "dh64_cfg_b2": ("dh64", 2, 1, [0, 1]),
    "full_depth": ("full_depth", 1, 1, [0, 13, 27]),       # last: the tests after it reuse the depth-28 model
}
# kernel launches of tpx_dit_forward (dit_forward_impl): 3 GEMV (timestep MLP, adaLN) + x_embed, 11 per block (cross: LN, q, attention,
# gated proj; self: LN, qkv, attention, gated proj; MLP: LN, fc1, gated fc2), final layer 2, CFG combine 1
LAUNCHES_BRANCH = {"cross": 4, "self": 8, "mlp": 11}


class _F64(dict):
    """The state dict, each tensor converted to fp64 on first use (full depth holds 905 M parameters; a stage needs one block's)."""

    def __init__(self, sd):
        super().__init__()
        self.src = sd

    def __missing__(self, k):
        v = self[k] = self.src[k].double()
        return v

    def get(self, k, default=None):
        return self[k] if k in self.src else default

    def __contains__(self, k):
        return k in self.src


_MODEL = {}


def _model(name):
    """One model alive at a time (the full-depth store is 1.8 GB): (DiT, fp64 state dict, config)."""
    if name not in _MODEL:
        _MODEL.clear()
        torch.cuda.empty_cache()
        c = MODELS[name]
        cfg = dict(seq_length=c["N"], in_channels=68, condition_channels=768, hidden_size=c["D"], depth=c["depth"], num_heads=c["H"],
                   attn_proj_bias=True, cond_drop_prob=0.1)
        sd = synth.device_state_dict(synth.dit_shapes(**cfg), 500 + list(MODELS).index(name), DEV, torch.float16)
        m = tpxl_b200.DiT(**cfg)
        m.load_state_dict(sd)
        _MODEL[name] = (m.to(DEV).eval(), _F64(sd), c)
    return _MODEL[name]


def _inputs(c, B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, c["N"], 68, generator=g, device=DEV)
    y = torch.randn(B, c["M"], 768, generator=g, device=DEV)
    return x, y, torch.tensor(T_VALUES[:B], device=DEV)


# ---- partitions and the bound ---------------------------------------------------------------------------------------------------------
PARTS = {"row": parity.row, "sequence": parity.sequence, "block": parity.block(128), "channel": parity.channel}


def _parts(names, Dh=None):
    """The partitions named: PARTS, and "head" for the attention output's Dh-wide heads."""
    return {h: parity.head(Dh) if h == "head" else PARTS[h] for h in names}


def _check(key, ours, pol, ref, parts, Dh=None):
    """ours / pol / ref fp64 [S, N, C] against the bound (tests/parity.py) per partition named in parts; the worst ratios go to WORST."""
    worst = WORST.setdefault(key, {})
    for how, r in parity.check(f"{key}", ours, pol, ref, _parts(parts, Dh)).items():
        worst[how] = max(worst.get(how, 0.0), r)


INC_PARTS = ("sequence", "block", "channel")


def _check_with_null_half(key, ours, pol, ref, B):
    """An increment whose sequences from B on attend to the null context.  Cross-attention over an all-null context is the same
    vector for every token, so there each channel holds one value repeated over all N tokens: one draw of each rounding, not a
    sample of them, and a per-channel rate cannot be compared with the policy's (a channel whose value cancels in its dot product
    can have a policy error near zero by chance while an accumulation-order flip upstream moves ours by a few of its ulps).  So
    channels are partitioned over the first B sequences; the null half is partitioned per sequence and per block (D independent
    roundings each), and each of its per-(sequence, channel) means over tokens must lie within 2 fp16 ulps (a near-tie at the last
    rounding point rounded the other way) + 2.5 x the policy's rms error over that sequence's channels (a flip upstream, amplified by
    cancellation) + 1e-4 of their rms of the policy's mean: a wrong or misplaced channel of the constant fails that."""
    _check(key, ours, pol, ref, ("sequence", "block"))
    _check(key, ours[:B], pol[:B], ref[:B], ("channel",))
    if ours.shape[0] == B:
        return
    m_o, m_p, m_e = (a[B:].mean(1) for a in (ours, pol, ref))
    tol = (2 * parity.ulp16(m_p) + parity.K_POLICY * (m_p - m_e).pow(2).mean(1, keepdim=True).sqrt()
           + parity.FLOOR * m_e.pow(2).mean(1, keepdim=True).sqrt())
    worst, _ = parity.check_elementwise(f"{key}: null-half channel means", m_o, m_p, tol)
    WORST.setdefault(key, {})["null-half channel mean"] = worst


# ---- oracle pieces on the kernel's taps ------------------------------------------------------------------------------------------------
def _t_emb(sd64, t, exact: bool):
    """The timestep embedding: exact in fp64, or the reference's (fp32 sinusoid, then fp32 Linears: no fp16 rounding point)."""
    return od.t_embedder(sd64, t, dtype=torch.float64 if exact else torch.float32)


def _mod_rows(sd64, t, L):
    """[B, 9 L D + 2 D] modulation rows, exact and policy."""
    out = []
    for exact, pol in ((True, EXACT), (False, POLICY)):
        te = _t_emb(sd64, t, exact)
        chunks = [c for i in range(L) for c in od.block_modulation(sd64, i, te, pol)] + list(od.final_modulation(sd64, te, pol))
        out.append(torch.cat(chunks, 1))
    return out


def _chunks(mod, b, i, D):
    """Block i's 9 modulation chunks of sample b, from the kernel's rows, as [1, D] fp64."""
    return [c[None] for c in mod[b, 9 * i * D:9 * (i + 1) * D].double().view(9, D)]


def _stop(m, x, t, y, stage, block, use_cfg):
    lib = _lib.lib()
    n0 = lib.tpx_launch_count()
    r = m.debug_stage(x, t, y, stage, block, use_cfg)
    n = lib.tpx_launch_count() - n0
    want = 4 if stage == "embed" else 4 + 11 * block + LAUNCHES_BRANCH[stage]
    assert n == want, (stage, block, n, want)
    return r


def _case(case):
    """Every check of one case.  Returns block 0's (ours, policy, exact) triples of the cross increment, the self-attention output and
    the MLP increment."""
    name, B, use_cfg, blocks = CASES[case]
    m, sd64, c = _model(name)
    N, D, H, L = c["N"], c["D"], c["H"], c["depth"]
    Dh = D // H
    S = 2 * B if use_cfg else B
    Sc = B if use_cfg == 1 else S
    x, y, t = _inputs(c, B, 1000 + list(CASES).index(case))
    null = sd64["null_cond_embedding"].expand(1, c["M"], -1)
    ctx = [y[s:s + 1].double() if s < B else null for s in range(S)]
    lib = _lib.lib()
    kept = {}
    with torch.no_grad():
        # ---- the full forward: its launches, determinism, modulation rows, final layer and CFG combine ----
        m._run(x, t, y, use_cfg, CFG_SCALE, True)             # conditioning store, first-launch attributes
        n0 = lib.tpx_launch_count()
        out = m._run(x, t, y, use_cfg, CFG_SCALE, True)
        assert lib.tpx_launch_count() - n0 == 4 + 11 * L + 2 + (1 if use_cfg else 0)
        assert torch.equal(out, m._run(x, t, y, use_cfg, CFG_SCALE, True))
        mod = m.debug_tap(S, "mod", B)
        last = m.debug_tap(S, "residual")
        pre = m.debug_tap(S, "pre_cfg") if use_cfg else out
        ref_mod, pol_mod = _mod_rows(sd64, t, L)
        nck = 9 * L + 2
        _check((case, "modulation"), mod.double().view(B, nck, D), pol_mod.view(B, nck, D), ref_mod.view(B, nck, D), ("row",))   # (sample, chunk)
        # final layer on the kernel's last residual and its own final modulation chunks
        fin_e, fin_p = [], []
        for s in range(S):
            b = s % B
            sh, sc = (mod[b, (9 * L + k) * D:(9 * L + k + 1) * D].double()[None] for k in (0, 1))
            fin_e.append(od.final_apply(sd64, last[s:s + 1].double(), sh, sc, EXACT))
            fin_p.append(od.final_apply(sd64, last[s:s + 1].double(), sh, sc, POLICY))
        _check((case, "final"), pre.double(), torch.cat(fin_p), torch.cat(fin_e), ("sequence", "channel"))
        if use_cfg:
            cond, unc = pre[:B].float(), pre[B:].float()
            d = (cond - unc).half().float()
            want = (unc + (d * CFG_SCALE).half().float()).half()
            assert torch.equal(out, want), "CFG combine differs from h(u + h(s h(c - u))) on the pre-guidance output"

        # ---- token embedding: fp32 accumulation of Cin + 1 terms against fp64 ----
        r_in = _stop(m, x, t, y, "embed", 0, use_cfg)
        xe = x.double()
        Wx, bx = sd64["x_embedder.weight"], sd64["x_embedder.bias"]
        ref = F.linear(xe, Wx, bx)
        budget = (Wx.shape[1] + 1) * 2.0 ** -24 * (xe.abs() @ Wx.abs().t() + bx.abs())
        err = (r_in[:B].double() - ref).abs()
        assert bool((err <= budget).all()), float((err / budget).max())
        WORST.setdefault((case, "embed"), {})["element"] = float((err / budget).max())
        if use_cfg:
            assert torch.equal(r_in[:B], r_in[B:])

        prev_block = -1
        for i in blocks:
            if i != prev_block + 1:
                r_in = _stop(m, x, t, y, "mlp", i - 1, use_cfg)
            prev_block = i
            # ---- cross-attention: sequences [0, Sc) attend to the context; under use_cfg 1 the null half is untouched here ----
            rc = _stop(m, x, t, y, "cross", i, use_cfg)
            ao_c = m.debug_tap(S, "ao", Sc)
            assert torch.equal(rc, m.debug_stage(x, t, y, "cross", i, use_cfg)), "two runs to the same stop differ"
            if Sc < S:
                assert torch.equal(rc[Sc:], r_in[Sc:]), "the null half changed before its collapsed cross-attention is added"
            inc = {"exact": [], "policy": []}
            ao = {"exact": [], "policy": []}
            for s in range(Sc):
                mc = _chunks(mod, s % B, i, D)
                for k, pol in (("exact", EXACT), ("policy", POLICY)):
                    tp = {}
                    inc[k].append(od.cross_branch(sd64, i, r_in[s:s + 1].double(), ctx[s], mc, H, pol, tp))
                    ao[k].append(tp["ao"])
            trip = ((rc - r_in)[:Sc].double(), torch.cat(inc["policy"]), torch.cat(inc["exact"]))
            _check_with_null_half((case, "cross"), *trip, B)
            _check((case, "cross ao"), ao_c.double(), torch.cat(ao["policy"]), torch.cat(ao["exact"]), ("head",), Dh)
            if i == 0:
                kept["cross"] = trip
            # ---- self-attention; the null half's increment includes its collapsed cross-attention, checked against real attention ----
            rs = _stop(m, x, t, y, "self", i, use_cfg)
            ao_s = m.debug_tap(S, "ao")
            inc = {"exact": [], "policy": []}
            ao = {"exact": [], "policy": []}
            for s in range(S):
                mc = _chunks(mod, s % B, i, D)
                for k, pol in (("exact", EXACT), ("policy", POLICY)):
                    tp = {}
                    if s < Sc:
                        inc[k].append(od.self_branch(sd64, i, rc[s:s + 1].double(), mc, H, pol, tp))
                    else:
                        xin = r_in[s:s + 1].double()
                        cross = od.cross_branch(sd64, i, xin, ctx[s], mc, H, pol)
                        inc[k].append(cross + od.self_branch(sd64, i, xin + cross, mc, H, pol, tp))
                    ao[k].append(tp["ao"])
            before = torch.cat([rc[:Sc], r_in[Sc:]])
            _check_with_null_half((case, "self"), (rs - before).double(), torch.cat(inc["policy"]), torch.cat(inc["exact"]), B)
            trip = (ao_s.double(), torch.cat(ao["policy"]), torch.cat(ao["exact"]))
            _check((case, "self ao"), *trip, ("head",), Dh)
            if i == 0:
                kept["self ao"] = trip
            # ---- MLP ----
            rm = _stop(m, x, t, y, "mlp", i, use_cfg)
            inc = {"exact": [], "policy": []}
            for s in range(S):
                mc = _chunks(mod, s % B, i, D)
                for k, pol in (("exact", EXACT), ("policy", POLICY)):
                    inc[k].append(od.mlp_branch(sd64, i, rs[s:s + 1].double(), mc, pol))
            trip = ((rm - rs).double(), torch.cat(inc["policy"]), torch.cat(inc["exact"]))
            _check((case, "mlp"), *trip, INC_PARTS)
            if i == 0:
                kept["mlp"] = trip
            r_in = rm
            if i == L - 1:
                assert torch.equal(rm, last), "the last block's MLP stop differs from the residual the full forward leaves"
    for key in [k for k in WORST if k[0] == case]:
        print(f"{case:14s} {key[1]:18s} worst / bound: " + ", ".join(f"{h} {v:.3f}" for h, v in WORST[key].items()))
    return kept


_KEPT = {}


@pytest.mark.parametrize("case", list(CASES))
def test_stage_local_parity(case):
    kept = _case(case)
    if case == "shipped_b1":
        _KEPT[case] = kept


def test_bound_rejects_one_percent_errors():
    """On the shipped model's real block-0 taps (B 1 with CFG), a 1 % error in ours at one head of one sequence (self-attention output),
    one 128-token block of one sequence (cross-attention increment) or one channel (MLP increment) fails the bound."""
    kept = _KEPT.get("shipped_b1") or _case("shipped_b1")
    Dh = 1152 // 16
    for what, tap, how, region in (("head", "self ao", "head", (1, slice(None), slice(5 * Dh, 6 * Dh))),
                                   ("128-token block", "cross", "block", (0, slice(640, 768))),
                                   ("channel", "mlp", "channel", (slice(None), slice(None), 517))):
        ours, pol, ref = kept[tap]
        parts = _parts((how,), Dh)
        assert not parity.rejects(ours, pol, ref, parts)
        bad = ours.clone()
        bad[region] *= 1.01
        o, p = parity.ratios(bad, pol, ref, parts[how])
        print(f"1 % on one {what} ({tap}): worst {how} partition at {float((o / parity.bound(p)).max()):.1f} x the bound")
        assert parity.rejects(bad, pol, ref, parts), what


def test_timestep_table_rows_against_fp64():
    """tpx_dit_set_timesteps at the shipped width and depth 28: the ddim25 map (passes of 8 + 8 + 8 + 1 timesteps) and the ddim100 map
    (12 x 8 + 4) against fp64, per (row, chunk): a row computed in the wrong slot of an 8-wide GEMV pass fails its chunks."""
    m, sd64, c = _model("full_depth")
    D, L = c["D"], c["depth"]
    nck = 9 * L + 2
    for spec in ("ddim25", "ddim100"):
        ts = list(tpxl_b200.create_diffusion(spec, "squaredcos_cap_v2", parameterization="v").timestep_map)
        m.set_timesteps(ts, force=True)
        table = m.debug_timestep_table().double()
        ref, pol = _mod_rows(sd64, torch.tensor(ts, device=DEV), L)
        _check(("timestep table", spec), table.view(len(ts), nck, D), pol.view(len(ts), nck, D), ref.view(len(ts), nck, D), ("row",))
        print(f"timestep table {spec:8s} worst / bound: " + ", ".join(f"{h} {v:.3f}" for h, v in WORST[("timestep table", spec)].items()))


def test_stop_arguments_and_wall_time():
    m, _, c = _model("full_depth")
    x, y, t = _inputs(c, 1, 7)
    with pytest.raises(_lib.TpxError, match="bad block"):
        m.debug_stage(x, t, y, "mlp", c["depth"], 1)
    with pytest.raises(_lib.TpxError, match="bad block"):
        m.debug_stage(x, t, y, "cross", -1, 1)
    with pytest.raises(ValueError):
        m.debug_stage(x, t, y, "final", 0, 1)
    print(f"test_gpu_dit_stages: {time.time() - T0:.0f} s since the module was imported")
