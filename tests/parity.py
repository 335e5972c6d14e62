"""The parity rule of the stage-by-stage suites (DESIGN §2), stated once, and the comparison helpers the GPU tests share.

Rule: per partition, the relative L2 of ours against exact fp64 is at most K_POLICY x the fp16 policy's + FLOOR.  A partition is
a function of a tensor t [S, N, C] (S sequences, images or primitives of N tokens or voxels with C channels) that returns the
1-D tensor of t's sums over each of its parts.  Every check accepts only what it can show is within its bound: a NaN or an
infinity anywhere fails it.

Torch only, on whatever device the tensors are on.
"""
import torch

from oracle.primsdf import local_grid

K_POLICY = 2.5      # ours may be this many times as far from exact as the fp16 policy is ...
FLOOR = 1e-4        # ... plus this, for partitions where the policy happens to be nearly exact


def bound(p):
    """The largest relative L2 error ours may have where the policy's is p."""
    return K_POLICY * p + FLOOR


# ---- partitions -------------------------------------------------------------------------------------------------------------------
def sequence(t):
    """Per sequence (image, primitive)."""
    return t.sum((1, 2))


def row(t):
    """Per (sequence, token)."""
    return t.sum(2).flatten()


def channel(t):
    """Per channel, over all sequences."""
    return t.sum((0, 1))


def head(Dh):
    """Per (sequence, head) of Dh consecutive channels."""
    def part(t):
        S, N, C = t.shape
        return t.reshape(S, N, C // Dh, Dh).sum((1, 3)).flatten()
    return part


def _by_label(t, labels, pool):
    labels = labels.to(t.device)
    keep = labels >= 0
    x = t.sum(2)[:, keep]
    if pool:
        x = x.sum(0, keepdim=True)
    return torch.zeros(x.shape[0], int(labels.max()) + 1, dtype=t.dtype, device=t.device).index_add_(1, labels[keep], x).flatten()


def tokens(labels):
    """Per (sequence, label): labels [N] give each token's part; a token labelled -1 is in none."""
    return lambda t: _by_label(t, labels, pool=False)


def pooled(labels):
    """Per label, over all sequences: labels [N] give each token's part; a token labelled -1 is in none."""
    return lambda t: _by_label(t, labels, pool=True)


def block(n):
    """Per (sequence, block of n consecutive tokens); the last block is ragged where N % n != 0."""
    return lambda t: _by_label(t, torch.arange(t.shape[1]) // n, pool=False)


def boundary_count(S):
    """[S^3] labels of an S^3 volume, voxel v = (z S + y) S + x: how many of its coordinates lie on the volume's boundary (0 interior,
    1 face, 2 edge, 3 corner).  Halo and zero-padding errors of a stride-1 convolution land on the boundary classes."""
    i = torch.arange(S)
    b = ((i == 0) | (i == S - 1)).long()
    return (b[:, None, None] + b[None, :, None] + b[None, None, :]).reshape(-1)


def face_class(S):
    """[S^3] labels of an S^3 volume: 0 interior, 1 on a low face only (some coordinate 0: the zero padding a stride-2 layer reads),
    2 on a high face only (some coordinate S - 1), 3 on both."""
    i = torch.arange(S)
    lo, hi = (i == 0).long(), (i == S - 1).long()
    any_lo = ((lo[:, None, None] + lo[None, :, None] + lo[None, None, :]) > 0).reshape(-1)
    any_hi = ((hi[:, None, None] + hi[None, :, None] + hi[None, None, :]) > 0).reshape(-1)
    return any_lo.long() + 2 * any_hi.long()


def to_ncdhw(tap):
    """[P, S^3, C] channels-last -> [P, C, S, S, S]."""
    P, S3, C = tap.shape
    S = round(S3 ** (1 / 3))
    return tap.reshape(P, S, S, S, C).permute(0, 4, 1, 2, 3)


def to_cl(x):
    """[P, C, S, S, S] -> [P, S^3, C] channels-last."""
    P, C = x.shape[:2]
    return x.permute(0, 2, 3, 4, 1).reshape(P, -1, C)


# ---- the rule ---------------------------------------------------------------------------------------------------------------------
def ratios(ours, pol, ref, part):
    """ours / pol / ref fp64 [S, N, C]: per part of the partition, the relative L2 of ours and of the policy against ref."""
    den = part(ref ** 2).sqrt().clamp_min(1e-30)
    return part((ours - ref) ** 2).sqrt() / den, part((pol - ref) ** 2).sqrt() / den


def _verdict(ours, pol, ref, parts):
    """(why the rule rejects ours, or None; {partition name: worst ratio to the bound} of the partitions that passed)."""
    if not ours.shape == pol.shape == ref.shape:
        return f"shapes differ: ours {tuple(ours.shape)}, policy {tuple(pol.shape)}, exact {tuple(ref.shape)}", {}
    for what, t in (("ours", ours), ("policy", pol), ("exact", ref)):
        bad = ~torch.isfinite(t)
        if bool(bad.any()):
            return f"{int(bad.sum())} non-finite elements in {what}, the first at {bad.nonzero()[0].tolist()}", {}
    worst = {}
    for how, part in parts.items():
        o, p = ratios(ours, pol, ref, part)
        ok = o <= bound(p)
        if not bool(ok.all()):
            bad = ~ok
            return (f"{how} partitions {bad.nonzero().flatten().tolist()[:8]} exceed the bound: ours {o[bad][:8].tolist()} vs policy "
                    f"{p[bad][:8].tolist()}"), worst
        worst[how] = float((o / bound(p)).max())
    return None, worst


def check(name, ours, pol, ref, parts):
    """Accept iff the shapes are equal, all three tensors are finite and every part of every partition in parts ({name: partition})
    is within the bound.  Returns {partition name: worst ratio to the bound}."""
    why, worst = _verdict(ours, pol, ref, parts)
    assert why is None, f"{name}: {why}"
    return worst


def rejects(ours, pol, ref, parts) -> bool:
    """Whether check would fail."""
    return _verdict(ours, pol, ref, parts)[0] is not None


def ulp16(x):
    """fp16 spacing at |x| (2^-24 in the subnormal range), in fp64."""
    return torch.exp2(torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -14))) - 10)


def check_elementwise(name, ours, want, tol):
    """Accept iff every element is finite and |ours - want| <= tol (broadcast).  Returns (worst |ours - want| / tol, the number of
    elements where ours differs from want)."""
    ours, want = torch.broadcast_tensors(ours.double(), want)
    err = (ours - want).abs()
    tol = tol + torch.zeros_like(err)
    bad = ~(torch.isfinite(err) & torch.isfinite(tol) & (err <= tol))
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())} elements off by more than their tolerance, e.g. at {bad.nonzero()[:4].tolist()}: "
                                 f"{ours[bad][:4].tolist()} vs {want[bad][:4].tolist()} (allowed {tol[bad][:4].tolist()})")
    return float((err / tol).max()), int((err > 0).sum())


# ---- PrimSDF and mesh comparisons -------------------------------------------------------------------------------------------------
def is_fp32_tie(p, srt, S):
    """True if, for the point p [3], the two nearest primitives of srt [K, 4] (scale, centre), or the two nearest voxels of the
    nearest one's S^3 grid, are the same distance away to within fp32 resolution: which one an fp32 argmin picks is rounding."""
    d = (p[None] - srt[:, 1:4]).norm(dim=1)
    order = d.argsort()
    if len(order) > 1 and float(d[order[1]] - d[order[0]]) < 4e-7 * float(d[order[0]]):
        return True
    k = int(order[0])
    cand = srt[k, 1:4][None] + srt[k, 0] * local_grid(S).to(srt)
    dv = (p[None] - cand).norm(dim=1).sort().values
    return float(dv[1] - dv[0]) < 4e-7 * float(dv[0])


def fp32_ties(p, srt, S, chunk=2048):
    """is_fp32_tie of every point of p [n, 3] at once, on p's device in p's dtype (pass fp64): [n] bool."""
    grid = local_grid(S).to(srt)
    out = []
    for c in p.split(chunk):
        d = (c[:, None] - srt[None, :, 1:4]).norm(dim=2)
        near = d.topk(min(2, d.shape[1]), dim=1, largest=False)
        tie = (near.values[:, 1] - near.values[:, 0] < 4e-7 * near.values[:, 0]) if d.shape[1] > 1 else torch.zeros_like(d[:, 0], dtype=torch.bool)
        k = near.indices[:, 0]
        cand = srt[k, 1:4][:, None] + srt[k, 0][:, None, None] * grid[None]
        dv = (c[:, None] - cand).norm(dim=2).topk(2, dim=1, largest=False).values
        out.append(tie | (dv[:, 1] - dv[:, 0] < 4e-7 * dv[:, 0]))
    return torch.cat(out) if out else torch.zeros(0, dtype=torch.bool, device=p.device)


def same_mesh(got, want, what=""):
    """got (vertices fp32, faces int64) tensors equal to want (vertices, faces) numpy arrays byte for byte."""
    v, f = got
    where = f"{what}: " if what else ""
    assert v.dtype == torch.float32 and f.dtype == torch.int64
    assert torch.equal(f.cpu(), torch.as_tensor(want[1])), f"{where}faces differ ({f.shape[0]} vs {len(want[1])})"
    assert torch.equal(v.cpu().view(torch.int32), torch.as_tensor(want[0]).view(torch.int32)), f"{where}vertex bytes differ"
