"""Oracle of the box-projection UV unwrap and the primitive noise filter (TEST INFRASTRUCTURE — see oracle/__init__.py).

A numpy restatement of DESIGN.md §1 f-8 (utils/uv_unwrap.py:65-685 and inference.py:90-103 of the reference), one function per stage,
each callable on any previous-stage input (the GPU tests feed it the kernels' own stage outputs).  fp32 arithmetic is spelled one
rounded numpy operation at a time in the kernels' order (csrc/uv_unwrap.cu is built without FMA contraction); per-vertex sums run in the
reference's scatter_add_ order; the two-dimensional triangle test is fp64.  Each decision comes with an ambiguity margin, the distance
of the quantity it was taken on from its threshold:
  * project: the gap between the two largest axis dots;
  * assign: per face and kind, the smallest |d - 3 r| over the pairs near the candidate threshold, |det - 1e-6| over the edge tests of
    its candidate pairs, |winding det| where flipping the winding would change a result, and |c_first - c_second| of the centroid order.
Candidates are found with a kd-tree per slice (radius slightly above 3 r) and filtered with the exact fp32 test, so the work stays
near-linear in the face count.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

f32 = np.float32
BIG = np.float64(np.inf)


def _normalize(x, eps):
    """F.normalize(x, dim=-1, eps): x / max(sqrt((x0^2 + x1^2) + x2^2), eps) in fp32."""
    x = x.astype(f32)
    n = np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])
    n = np.maximum(n, f32(eps))
    return (x / n[:, None]).astype(f32)


def _normalize_pm1(x):
    """F.normalize(x, -1) as utils/uv_unwrap.py:414-419 calls it: -1 is p, not dim, so x / max((sum_d |x_d|^-1)^-1, 1e-12) along dim 1
    (a zero component makes the divisor 1e-12)."""
    x = x.astype(f32)
    with np.errstate(divide="ignore"):
        inv = [f32(1) / np.abs(x[:, d]) for d in range(3)]
        n = f32(1) / ((inv[0] + inv[1]) + inv[2])
    return (x / np.maximum(n, f32(1e-12))[:, None]).astype(f32)


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1).astype(f32)


def _scatter_rows(V, f, rows):
    """sum over corners of rows[face] per vertex, in scatter_add_ order (corner 0 by ascending face, then corner 1, then 2)."""
    acc = np.zeros((V, 3), f32)
    for c in range(3):
        np.add.at(acc, f[:, c], rows)
    return acc


def vertex_normals(v, f):
    v, f = np.asarray(v, f32), np.asarray(f, np.int64)
    p = v[f]
    fn = _cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    s = _scatter_rows(len(v), f, fn)
    d = (s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2]
    s[~(d > f32(1e-20))] = (0, 0, 1)
    return _normalize(s, 1e-12)


def project(v, n, f):
    """_box_assign_vertex_to_cube_face: (slice int [F], face_uv fp32 [F,3,2], margin [F])."""
    v, n, f = np.asarray(v, f32), np.asarray(n, f32), np.asarray(f, np.int64)
    lo, hi = v.min(0), v.max(0)
    q = ((v - lo) / (hi - lo)).astype(f32) * f32(2) - f32(1)
    tri = q[f]                                                              # [F,3,3]
    fn = _normalize((n[f[:, 0]] + n[f[:, 1]]) + n[f[:, 2]], 1e-6)
    dots = np.stack([fn[:, 0], -fn[:, 0], fn[:, 1], -fn[:, 1], fn[:, 2], -fn[:, 2]], 1)
    s = dots.argmax(1)
    srt = np.sort(dots, 1)
    margin = (srt[:, -1].astype(np.float64) - srt[:, -2])
    ax = s // 2
    F = len(f)
    coord = tri[np.arange(F), :, ax]                                        # [F,3]
    div = np.abs(coord).max(0)                                              # per corner slot
    x, y, z = tri[..., 0], tri[..., 1], tri[..., 2]
    u = np.where((s <= 1)[:, None], y, x)
    vv = np.where((s <= 3)[:, None], -z, np.where((s == 4)[:, None], y, -y))
    uc = np.clip((u / div[None] + f32(1)) * f32(0.5), 0, 1).astype(f32)
    vc = np.clip((vv / div[None] + f32(1)) * f32(0.5), 0, 1).astype(f32)
    return s, np.stack([uc, vc], -1).astype(f32), margin


def rotate(v, n, f, face_uv, slc):
    """calculate_tangents + _rotate_uv_slices_consistent_space: (angle fp32 [6], rotated uv fp32 [F,3,2])."""
    v, n, f = np.asarray(v, f32), np.asarray(n, f32), np.asarray(f, np.int64)
    t = np.asarray(face_uv, f32)
    d1 = t[:, 1] - t[:, 0]
    d2 = t[:, 2] - t[:, 0]
    p = v[f]
    den = np.maximum(d1[:, 0] * d2[:, 1] - d1[:, 1] * d2[:, 0], f32(1e-6))
    tang = (((p[:, 1] - p[:, 0]) * d2[:, 1:2] - (p[:, 2] - p[:, 0]) * d1[:, 1:2]) / den[:, None]).astype(f32)
    s = _scatter_rows(len(v), f, tang)
    cnt = np.zeros(len(v), f32)
    for c in range(3):
        np.add.at(cnt, f[:, c], f32(1))
    with np.errstate(invalid="ignore", divide="ignore"):
        s = _normalize(s / cnt[:, None], 1e-12)
    dn = (s[:, 0] * n[:, 0] + s[:, 1] * n[:, 1]) + s[:, 2] * n[:, 2]
    vt = _normalize(s - dn[:, None] * n, 1e-12)
    ps = np.stack([-v[:, 1], v[:, 0], np.zeros(len(v), f32)], 1)
    ve = _normalize_pm1(_cross(n, _cross(ps, n)))
    angle = np.zeros(6, f32)
    out = np.empty_like(t)
    for i in range(6):
        m = slc == i
        if not m.any():
            continue
        a = (vt[f[m]].astype(np.float64).reshape(-1, 3).sum(0) / (3 * m.sum())).astype(f32)
        e = (ve[f[m]].astype(np.float64).reshape(-1, 3).sum(0) / (3 * m.sum())).astype(f32)
        ang = np.arctan2(a[0] * e[1] - a[1] * e[0], (a[0] * e[0] + a[1] * e[1]) + a[2] * e[2]).astype(f32)
        angle[i] = ang
        c, sn = np.cos(ang).astype(f32), np.sin(ang).astype(f32)
        uc = t[m] * f32(2) - f32(1)
        r = np.stack([c * uc[..., 0] + (-sn) * uc[..., 1], sn * uc[..., 0] + c * uc[..., 1]], -1).astype(f32)
        lo, hi = r.min(), r.max()
        out[m] = (r - lo) / (hi - lo)
    return angle, out


def _wound(t):
    """[N,3,2] fp32 -> fp64 triangles wound by the sign of their determinant, and that determinant."""
    t = t.astype(np.float64)
    det = (t[:, 1, 0] - t[:, 0, 0]) * (t[:, 2, 1] - t[:, 0, 1]) - (t[:, 1, 1] - t[:, 0, 1]) * (t[:, 2, 0] - t[:, 0, 0])
    w = t.copy()
    flip = det < 0
    w[flip, 1], w[flip, 2] = t[flip, 2], t[flip, 1]
    return w, det


_EDGES = ((0, 1), (2, 0), (1, 2))


def _edge_dets(a, b):
    """[N,3 edges,3 points] det of edge of a against the points of b."""
    out = np.empty((len(a), 3, 3))
    for k, (i, j) in enumerate(_EDGES):
        ex, ey = a[:, i, 0][:, None], a[:, i, 1][:, None]
        out[:, k] = (a[:, j, 0][:, None] - ex) * (b[:, :, 1] - ey) - (a[:, j, 1][:, None] - ey) * (b[:, :, 0] - ex)
    return out


def _intersect(ta, tb):
    """triangle_intersection_2d(eps=1e-6) in fp64 on wound triangles: (collide [N], min |det - 1e-6| [N])."""
    da, db = _edge_dets(ta, tb), _edge_dets(tb, ta)
    sep = (~(da > 1e-6)).all(2).any(1) | (~(db > 1e-6)).all(2).any(1)
    margin = np.minimum(np.abs(da - 1e-6).min((1, 2)), np.abs(db - 1e-6).min((1, 2)))
    return ~sep, margin


def assign(v, f, rot_uv, slc):
    """_assign_faces_uv_to_atlas_index, two passes: (assign int [F], margins {kind: [F]}) with kinds "radius" (|d - 3 r|), "edge"
    (|det - 1e-6|), "winding" (|det| where the winding matters) and "tie" (|c_first - c_second|; the tie rule is exact fp32 arithmetic on
    the input positions, so a tie is a decision, not an ambiguity)."""
    v, f = np.asarray(v, f32), np.asarray(f, np.int64)
    t = np.asarray(rot_uv, f32)
    F = len(f)
    cu = ((t[:, 0, 0] + t[:, 1, 0]) + t[:, 2, 0]) / f32(3)
    cv = ((t[:, 0, 1] + t[:, 1, 1]) + t[:, 2, 1]) / f32(3)
    du, dv = t[:, :, 0] - cu[:, None], t[:, :, 1] - cv[:, None]
    rad = np.sqrt(du * du + dv * dv).max(1)
    r3 = (rad * f32(3)).astype(f32)
    c3 = ((v[f[:, 0]] + v[f[:, 1]]) + v[f[:, 2]]) / f32(3)
    w, det = _wound(t)
    wflip = w[:, [0, 2, 1]]
    out = np.asarray(slc).astype(np.int64).copy()
    mk = {k: np.full(F, BIG) for k in ("radius", "edge", "winding", "tie")}
    for s in range(2):
        flag = np.zeros(F, bool)
        for i in range(6 * s, 6 * s + 6):
            ids = np.nonzero(out == i)[0]
            if len(ids) < 2:
                continue
            pts = np.stack([cu[ids], cv[ids]], 1).astype(np.float64)
            ok = np.isfinite(pts).all(1) & np.isfinite(r3[ids])
            tree = cKDTree(np.where(ok[:, None], pts, 1e9))
            near = tree.query_ball_point(np.where(ok[:, None], pts, 1e9), np.where(ok, r3[ids].astype(np.float64) * 1.001 + 1e-7, 0.0))
            la = np.repeat(np.arange(len(ids)), [len(x) for x in near])
            lb = np.concatenate([np.asarray(x, np.int64) for x in near]) if len(la) else np.zeros(0, np.int64)
            keep = la != lb
            a, b = ids[la[keep]], ids[lb[keep]]
            d = np.sqrt((cu[b] - cu[a]) * (cu[b] - cu[a]) + (cv[b] - cv[a]) * (cv[b] - cv[a])).astype(f32)
            gap = np.abs(d.astype(np.float64) - r3[a])
            np.minimum.at(mk["radius"], a, gap)
            np.minimum.at(mk["radius"], b, gap)
            cand = d <= r3[a]
            lo, hi = np.minimum(a[cand], b[cand]), np.maximum(a[cand], b[cand])
            pair = np.unique(np.stack([lo, hi], 1), axis=0)
            if not len(pair):
                continue
            lo, hi = pair[:, 0], pair[:, 1]
            hit, dm = _intersect(w[lo], w[hi])
            for x in (lo, hi):
                np.minimum.at(mk["edge"], x, dm)
            # a winding only matters where flipping it changes the result
            for x, other in ((lo, hi), (hi, lo)):
                near0 = np.abs(det[x]) < 1e-6
                if near0.any():
                    alt_a = np.where(near0[:, None, None], wflip[x], w[x])
                    h2, _ = _intersect(alt_a, w[other])
                    ch = h2 != hit
                    np.minimum.at(mk["winding"], x[ch], np.abs(det[x][ch]))
            ax = 0 if i < 2 else 1 if i < 4 else 2
            c_lo, c_hi = c3[lo, ax], c3[hi, ax]
            mark = (c_lo > c_hi) if i % 2 == 1 else (c_lo < c_hi)
            moved = np.where(mark, hi, lo)
            tie = np.abs(c_lo.astype(np.float64) - c_hi)
            np.minimum.at(mk["tie"], lo, tie)
            np.minimum.at(mk["tie"], hi, tie)
            flag[moved[hit]] = True
        out[flag] += 6
    return np.minimum(out, 12), mk


def ambiguous(mk, radius_tol=1e-9, edge_tol=1e-12, winding_tol=1e-6):
    """bool [F]: faces with a decision within the tolerance of its threshold.  An exact d == 3 r is a tie, not an ambiguity: d and r are
    a few correctly rounded fp32 operations on the same uv in every implementation (marching-cubes lattices make such ties common).
    The edge test is fp64 everywhere; the reference's fp32 LU determinant decides the winding."""
    return ((mk["radius"] > 0) & (mk["radius"] <= radius_tol)) | (mk["edge"] <= edge_tol) | (mk["winding"] <= winding_tol)


def place(rot_uv, asg, island_padding):
    """_find_slice_offset_and_scale + _distribute_individual_uvs_in_atlas: placed uv fp32 [F,3,2]."""
    t = np.asarray(rot_uv, f32).copy()
    asg = np.asarray(asg)
    p = float(island_padding)
    uc, vc = t[..., 0], t[..., 1]
    for i in range(6, 12):
        m = asg == i
        if m.any():
            for c in (uc, vc):
                lo = c[m].min()
                c[m] = (c[m] - lo) / np.maximum(c[m].max() - lo, f32(0.5))
    uc = np.clip(uc * f32(1 - 2 * p) + f32(p), 0, 1).astype(f32)
    vc = np.clip(vc * f32(1 - 2 * p) + f32(p), 0, 1).astype(f32)
    m12 = asg >= 12
    n12 = int(m12.sum())
    if n12:
        mult = np.sqrt(n12 / (0.5 * (1 / 3)))
        nw = int(np.ceil(0.5 * mult))
        nh = int(np.ceil(n12 / nw))
        width, height = 1 / nw, 1 / nh
        clip = f32(min(width, height) * 1.5)
        idx = np.arange(n12)
        for c, n, sz, cell in ((uc, nw, width, idx % nw), (vc, nh, height, idx // nw)):
            x = c[m12]
            lo = x.min(1, keepdims=True)
            x = (x - lo) / np.maximum(x.max(1, keepdims=True) - lo, clip)
            x = np.clip(x * f32(1 - p * n * 0.5) + f32(p * n * 0.25), 0, 1).astype(f32)
            x = x * f32(sz) + (cell.astype(f32) * f32(sz))[:, None]
            c[m12] = np.clip(x * f32(1 - 2 * p * 0.5) + f32(p * 0.5), 0, 1)
    m = asg % 6
    gx, gy = (m % 3).astype(np.float64), (m // 3).astype(np.float64)
    ox = np.where(asg < 6, 1 / 3 * gx, np.where(asg < 12, 1 / 6 * gx, 0.5)).astype(f32)
    oy = np.where(asg < 6, 1 / 3 * gy, np.where(asg < 12, 1 / 6 * gy + 1 / 3 * 2, 1 / 3 * 2)).astype(f32)
    dx = np.where(asg < 6, 3, np.where(asg < 12, 6, 2)).astype(f32)
    dy = np.where(asg < 6, 3, np.where(asg < 12, 6, 3)).astype(f32)
    return np.stack([uc / dx[:, None] + ox[:, None], vc / dy[:, None] + oy[:, None]], -1).astype(f32)


def unique(placed):
    """_get_unique_face_uv: (uv [U,2] sorted by (u, v), vtex_idx [F,3])."""
    rows = np.asarray(placed, f32).reshape(-1, 2)
    uv, inv = np.unique(rows, axis=0, return_inverse=True)
    return uv, inv.reshape(-1, 3)


def unwrap(v, n, f, island_padding=0.02):
    """All stages: a dict of every stage output and margin."""
    slc, fuv, pm = project(v, n, f)
    angle, ruv = rotate(v, n, f, fuv, slc)
    asg, am = assign(v, f, ruv, slc)
    placed = place(ruv, asg, island_padding)
    uv, vidx = unique(placed)
    return dict(slice=slc, face_uv=fuv, project_margin=pm, angle=angle, rot_uv=ruv, assign=asg, assign_margin=am, placed=placed, uv=uv, vidx=vidx)


def noise_filter(srt):
    """inference.py:90-103 in fp32: (keep bool [K], nn int [K])."""
    srt = np.asarray(srt, f32)
    p, s = srt[:, 1:4], srt[:, 0]
    d = p[:, None, :] - p[None, :, :]
    dist = np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    dist = dist + np.eye(len(p), dtype=f32)
    nn = dist.argmin(1)
    return dist[np.arange(len(p)), nn] < (s + s[nn]), nn


def residual_overlaps(rot_uv, asg):
    """Pairs of faces left in one slice 0..11 that the reference's candidate + intersection test would still flag (0 after assign)."""
    t = np.asarray(rot_uv, f32)
    asg = np.asarray(asg)
    cu = ((t[:, 0, 0] + t[:, 1, 0]) + t[:, 2, 0]) / f32(3)
    cv = ((t[:, 0, 1] + t[:, 1, 1]) + t[:, 2, 1]) / f32(3)
    du, dv = t[:, :, 0] - cu[:, None], t[:, :, 1] - cv[:, None]
    r3 = (np.sqrt(du * du + dv * dv).max(1) * f32(3)).astype(f32)
    w, _ = _wound(t)
    total = 0
    for i in range(12):
        ids = np.nonzero(asg == i)[0]
        if len(ids) < 2:
            continue
        pts = np.stack([cu[ids], cv[ids]], 1).astype(np.float64)
        near = cKDTree(pts).query_ball_point(pts, r3[ids].astype(np.float64) * 1.001 + 1e-7)
        la = np.repeat(np.arange(len(ids)), [len(x) for x in near])
        lb = np.concatenate([np.asarray(x, np.int64) for x in near])
        a, b = ids[la[la != lb]], ids[lb[la != lb]]
        d = np.sqrt((cu[b] - cu[a]) * (cu[b] - cu[a]) + (cv[b] - cv[a]) * (cv[b] - cv[a])).astype(f32)
        a, b = a[d <= r3[a]], b[d <= r3[a]]
        if len(a):
            total += int(_intersect(w[a], w[b])[0].sum())
    return total


def slot_cells(asg):
    """[F,4] (x0, y0, x1, y1) of each face's atlas cell."""
    asg = np.asarray(asg)
    m = asg % 6
    gx, gy = m % 3, m // 3
    x0 = np.where(asg < 6, gx / 3, np.where(asg < 12, gx / 6, 0.5))
    y0 = np.where(asg < 6, gy / 3, np.where(asg < 12, 2 / 3 + gy / 6, 2 / 3))
    w = np.where(asg < 6, 1 / 3, np.where(asg < 12, 1 / 6, 0.5))
    h = np.where(asg < 6, 1 / 3, np.where(asg < 12, 1 / 6, 1 / 3))
    return np.stack([x0, y0, x0 + w, y0 + h], 1)
