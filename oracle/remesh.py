"""Oracle isotropic remeshing (TEST INFRASTRUCTURE — see oracle/__init__.py).

numpy restatement of the contract of csrc/mesh_remesh.cu, the GPU stand-in for pymeshlab's
meshing_isotropic_explicit_remeshing(iterations=3, targetlen=PercentageValue(1)) that decimate_mesh(..., remesh=True) runs after the
quadric decimation (utils/meshutils.py:101-105, inference.py:128-129).  pymeshlab is not installed anywhere this package runs, so the
rules below are this project's reading of VCG's IsotropicRemeshing with pymeshlab's defaults (featuredeg 30; split, collapse, swap,
smooth and reproject on; not adaptive).  They are NOT verified against pymeshlab.  Slow (vectorised per round), exact: the kernels
must give the same bytes.  fp64 expressions are written in the order the kernels evaluate them; fp32 values round to nearest.

Input: verts fp32 [V,3], faces int64 [F,3] with the checks of decimate.check_mesh.  L = target_len; an edge is short below 4/5 L and
long above 4/3 L (lo = L * 0.8, hi = L * (4 / 3), compared as squared fp64 lengths of the fp32 ends, (dx² + dy²) + dz²).

Features.  At the start an edge with exactly two faces is a crease iff the angle between the faces' normals n1, n2 (fp64 cross
products of the fp32 corners) exceeds feature_deg: n1·n2 < cos(feature_deg) · (sqrt(|n1|²) · sqrt(|n2|²)).  Creases are kept as a
sorted list of (min, max) edge keys; a split crease is replaced by its two halves; no other phase can remove one (a crease is never
flipped, and a collapse never removes a vertex that ends one).  A vertex is a feature iff it is frozen by decimation's rule (boundary,
non-manifold or inconsistently oriented edge, more than one fan, or unreferenced; recomputed every round of every phase) or it ends a
crease.  Features never move and are never removed.

Each iteration, in VCG's order:
  1. split, one pass: every long edge (ascending (min, max) key) gets a new vertex at its fp32 midpoint fp32((pa + pb) * 0.5), ids
     V, V+1, ... in that order.  Each face, rotated so that its pattern is canonical, is replaced in place by its children:
     0 split: (v0, v1, v2); 1 split (edge v0v1): (v0, m0, v2), (m0, v1, v2); 2 splits (v0v1, v1v2): the corner (m0, v1, m1) and the quad
     v0 m0 m1 v2 cut by its shorter diagonal, m0v2 if |m0 - v2|² < |v0 - m1|² else v0m1, children in the order
     (v0, m0, v2), (m0, v1, m1), (m0, m1, v2) or (v0, m0, m1), (m0, v1, m1), (v0, m1, v2); 3 splits: (v0, m0, m2), (m0, v1, m1),
     (m2, m1, v2), (m0, m1, m2).  The rotation starts the face at its split edge (1 split) or after its unsplit edge (2 splits).
  2. collapse, in rounds until one accepts nothing: a candidate is a short edge whose ends are not both features.  The survivor s is
     the feature end if there is one (it stays put), otherwise min(a, b) at the fp32 midpoint x̄; r is the other end.  Valid iff
     N(r) ∩ N(s) = {c, d} (the vertices opposite the edge), deg(a) + deg(b) >= 7, deg(c) >= 4, deg(d) >= 4, every neighbour of r or s
     but r and s is closer than hi to x̄, and no face of the two stars but the two on the edge turns its normal by 90 degrees or more
     (decimation's test).  key = fp32(length²) bits << 32 | edge id; accepted with decimation's two-ring minimum rule.
  3. flip, in rounds until one accepts nothing: targets t = 4 at frozen vertices, 6 elsewhere.  A candidate is a non-crease edge with
     at least one end x not frozen (the smaller such end), other end y, faces (x, y, c) and (x, d, y) in x's fan, c != d and c–d not an
     edge.  Its gain, the drop of Σ (val - t)² over x, y, c, d, must be > 0.  Valid iff the new faces (x, d, c) and (d, y, c) have
     normals with a positive dot against both old normals and are not a crease pair by the test above.  key = (2³² - 1 - gain) << 32 |
     edge id; accepted iff it is the minimum key of every candidate touching x, y, c or d, so accepted quads share no vertex.  The face
     holding (x, y, c) becomes (x, d, c), the one holding (x, d, y) becomes (d, y, c).
  4. tangential smoothing, one Jacobi pass: a non-feature vertex p moves to p + (d - n (n·d)), d = c - p, with c the mean of its
     neighbours (fp64 sum in ascending neighbour id, divided by their count) and n the normalised sum of the cross products of its
     faces in ascending face id; the move is dropped when n is zero or any face of its star would turn by 90 degrees or more against
     the old positions.
  5. projection: every non-feature vertex goes to the closest point of the INPUT mesh (Ericson's closest point on a triangle in fp64,
     see ``closest_point``), smallest squared distance, ties to the smallest face id, rounded to fp32.  Faces with a zero cross
     product are skipped; a face whose barycentric denominator va + vb + vc is not positive gives its first corner.  A vertex keeps
     its position when every input face is skipped.

Output: the referenced vertices in ascending id, then the faces in slot order, remapped, winding kept.  iterations = 0 gives the
input, compacted.  Left out of VCG: CollapseCrosses, the surface-distance check of the collapse (checksurfdist / maxsurfdist) and
adaptive lengths.
"""
from __future__ import annotations

import math

import numpy as np

from .decimate import NONE, _corners, _cross, _star_ok, check_mesh, compact, vertex_state

M32 = np.int64(0xFFFFFFFF)


def params(target_len, feature_deg):
    L = float(target_len)
    lo, hi = L * 0.8, L * (4.0 / 3.0)
    return lo * lo, hi * hi, math.cos(math.radians(float(feature_deg)))


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _len2(pa, pb):
    d = pa.astype(np.float64) - pb.astype(np.float64)
    return d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]


def _is_crease(n1, n2, cosf):
    l1, l2 = _dot(n1, n1), _dot(n2, n2)
    return _dot(n1, n2) < cosf * (np.sqrt(l1) * np.sqrt(l2))


def _edges(T):
    a, b = T, np.roll(T, -1, axis=1)
    return np.unique((np.minimum(a, b) << 32 | np.maximum(a, b)).ravel())


def _find(sorted_keys, q):
    """index of q in sorted_keys, -1 where absent"""
    i = np.searchsorted(sorted_keys, q)
    i = np.minimum(i, max(len(sorted_keys) - 1, 0))
    hit = (sorted_keys[i] == q) if len(sorted_keys) else np.zeros(np.shape(q), bool)
    return np.where(hit, i, -1)


def initial_creases(P, T, cosf):
    F = len(T)
    if F == 0:
        return np.zeros(0, np.int64)
    a, b = T, np.roll(T, -1, axis=1)
    key = (np.minimum(a, b) << 32 | np.maximum(a, b)).ravel()
    fid = np.repeat(np.arange(F), 3)
    order = np.lexsort((fid, key))
    k, f = key[order], fid[order]
    start = np.flatnonzero(np.concatenate([[True], k[1:] != k[:-1]]))
    cnt = np.diff(np.concatenate([start, [len(k)]]))
    two = start[cnt == 2]
    p = P[T].astype(np.float64)
    n = np.stack(_cross(p[:, 0], p[:, 1], p[:, 2]), 1)              # [F,3]
    n1, n2 = n[f[two]].T, n[f[two + 1]].T
    return np.sort(k[two][_is_crease(n1, n2, cosf)])


def state(P, T, C):
    """corner lists, frozen, deg, feature flags"""
    V = len(P)
    FACE, OUT, IN, n, _ = _corners(T, V)
    frozen, deg = vertex_state(OUT, IN, n)
    feat = frozen.copy()
    feat[C >> 32] = True
    feat[C & M32] = True
    return FACE, OUT, IN, n, frozen, deg, feat


# ---------------------------------------------------------------------------------------------------------------- split
def split(P, T, C, hi2):
    V, F = len(P), len(T)
    E = _edges(T)
    ea, eb = E >> 32, E & M32
    long_ = _len2(P[ea], P[eb]) > hi2
    ns = int(long_.sum())
    if ns == 0:
        return P, T, C, 0
    nid = np.where(long_, V + np.cumsum(long_) - 1, -1)
    mid = ((P[ea[long_]].astype(np.float64) + P[eb[long_]].astype(np.float64)) * 0.5).astype(np.float32)
    P = np.concatenate([P, mid])
    a, b = T, np.roll(T, -1, axis=1)
    s = nid[_find(E, np.minimum(a, b) << 32 | np.maximum(a, b))]      # [F,3] split vertex of edge k (t[k], t[k+1]) or -1
    cnt = (s >= 0).sum(1)
    unsplit = np.argmax(s < 0, 1)
    r = np.where(cnt == 1, np.argmax(s >= 0, 1), np.where(cnt == 2, (unsplit + 1) % 3, 0))
    idx = (r[:, None] + np.arange(3)[None, :]) % 3
    rows = np.arange(F)[:, None]
    v, m = T[rows, idx], s[rows, idx]
    v0, v1, v2, m0, m1, m2 = v[:, 0], v[:, 1], v[:, 2], m[:, 0], m[:, 1], m[:, 2]
    kid = np.full((F, 4, 3), -1, np.int64)
    kid[:, 0] = np.stack([v0, v1, v2], 1)
    c1 = cnt == 1
    kid[c1, 0] = np.stack([v0, m0, v2], 1)[c1]
    kid[c1, 1] = np.stack([m0, v1, v2], 1)[c1]
    c2 = cnt == 2
    if c2.any():
        da = _len2(P[np.where(c2, m0, 0)], P[v2])
        db = _len2(P[v0], P[np.where(c2, m1, 0)])
        short = c2 & (da < db)
        other = c2 & ~short
        kid[short, 0] = np.stack([v0, m0, v2], 1)[short]
        kid[short, 2] = np.stack([m0, m1, v2], 1)[short]
        kid[other, 0] = np.stack([v0, m0, m1], 1)[other]
        kid[other, 2] = np.stack([v0, m1, v2], 1)[other]
        kid[c2, 1] = np.stack([m0, v1, m1], 1)[c2]
    c3 = cnt == 3
    kid[c3, 0] = np.stack([v0, m0, m2], 1)[c3]
    kid[c3, 1] = np.stack([m0, v1, m1], 1)[c3]
    kid[c3, 2] = np.stack([m2, m1, v2], 1)[c3]
    kid[c3, 3] = np.stack([m0, m1, m2], 1)[c3]
    keep = np.arange(4)[None, :] <= cnt[:, None]
    T = kid[keep]
    ci = _find(E, C)
    cm = nid[ci]
    halves = np.concatenate([(C >> 32)[cm >= 0] << 32 | cm[cm >= 0], (C & M32)[cm >= 0] << 32 | cm[cm >= 0]])
    C = np.sort(np.concatenate([C[cm < 0], halves]))
    return P, T, C, ns


# ---------------------------------------------------------------------------------------------------------------- collapse
def _in_rows(X, rows, q):
    """per row i: q[i] in X[rows[i]] (q >= 0)"""
    return (X[rows] == q[:, None]).any(1)


def collapse_round(P, T, C, lo2, hi2):
    V = len(P)
    FACE, OUT, IN, n, frozen, deg, feat = state(P, T, C)
    E = _edges(T)
    ea, eb = E >> 32, E & M32
    len2 = _len2(P[ea], P[eb])
    key = np.full(len(E), NONE, np.uint64)
    cand = np.flatnonzero((len2 < lo2) & ~(feat[ea] & feat[eb]))
    xbar = np.zeros((len(E), 3), np.float32)
    if len(cand):
        A, B = ea[cand], eb[cand]
        s = np.where(feat[A], A, np.where(feat[B], B, A))
        r = np.where(s == A, B, A)
        mid = ((P[A].astype(np.float64) + P[B].astype(np.float64)) * 0.5).astype(np.float32)
        x = np.where(feat[s][:, None], P[s], mid)
        c = IN[r, np.argmax(OUT[r] == s[:, None], 1)]
        d = OUT[r, np.argmax(IN[r] == s[:, None], 1)]
        D = OUT.shape[1]
        valid_r = np.arange(D)[None, :] < n[r][:, None]
        nr = np.where(valid_r, OUT[r], -1)                                    # r is not frozen: OUT lists every neighbour once
        ns_ = np.concatenate([OUT[s], IN[s]], 1)
        valid_s = np.concatenate([np.arange(D)[None, :] < n[s][:, None]] * 2, 1)
        ns_ = np.where(valid_s, ns_, -3)
        link = ((nr[:, :, None] == ns_[:, None, :]).any(2) & (nr >= 0)).sum(1)
        ok = (link == 2) & (c != d) & (deg[A] + deg[B] >= 7) & (deg[c] >= 4) & (deg[d] >= 4)
        nb = np.concatenate([nr, ns_], 1)
        nbv = (nb >= 0) & (nb != r[:, None]) & (nb != s[:, None])
        l2 = _len2(P[np.where(nbv, nb, 0)], x[:, None, :])
        ok &= (~nbv | (l2 < hi2)).all(1)
        ok &= _star_ok(P, T, FACE, n, r, s, x) & _star_ok(P, T, FACE, n, s, r, x)
        bits = len2[cand].astype(np.float32).view(np.uint32).astype(np.uint64)
        key[cand] = np.where(ok, bits << np.uint64(32) | cand.astype(np.uint64), NONE)
        xbar[cand] = x
    m1 = np.full(V, NONE, np.uint64)
    np.minimum.at(m1, ea, key)
    np.minimum.at(m1, eb, key)
    m2 = m1.copy()
    np.minimum.at(m2, ea, m1[eb])
    np.minimum.at(m2, eb, m1[ea])
    acc = np.flatnonzero((key != NONE) & (m2[ea] == key) & (m2[eb] == key))
    if len(acc) == 0:
        return P, T, 0
    A, B = ea[acc], eb[acc]
    s = np.where(feat[A], A, np.where(feat[B], B, A))
    r = np.where(s == A, B, A)
    P = P.copy()
    P[s] = xbar[acc]
    rep = np.arange(V)
    rep[r] = s
    T = rep[T]
    keep = (T[:, 0] != T[:, 1]) & (T[:, 1] != T[:, 2]) & (T[:, 2] != T[:, 0])
    return P, T[keep], len(acc)


# ---------------------------------------------------------------------------------------------------------------- flip
def valence_energy(T, V):
    _, OUT, IN, n, _ = _corners(T, V)
    frozen, deg = vertex_state(OUT, IN, n)
    used = n > 0
    t = np.where(frozen, 4, 6)
    return int(((deg - t) ** 2)[used].sum())


def flip_round(P, T, C, cosf):
    V = len(P)
    FACE, OUT, IN, n, frozen, deg, feat = state(P, T, C)
    E = _edges(T)
    ea, eb = E >> 32, E & M32
    tgt = np.where(frozen, 4, 6)
    crease = _find(C, E) >= 0
    cand = np.flatnonzero(~crease & (~frozen[ea] | ~frozen[eb]))
    key = np.full(len(E), NONE, np.uint64)
    if len(cand) == 0:
        return T, 0
    A, B = ea[cand], eb[cand]
    x = np.where(~frozen[A], A, B)
    y = np.where(x == A, B, A)
    j1 = np.argmax(OUT[x] == y[:, None], 1)
    j2 = np.argmax(IN[x] == y[:, None], 1)
    c, d = IN[x, j1], OUT[x, j2]
    f1, f2 = FACE[x, j1], FACE[x, j2]
    ok = c != d
    ok &= _find(E, np.minimum(c, d) << 32 | np.maximum(c, d)) < 0
    e = deg - tgt
    gain = (2 * e[x] - 1) + (2 * e[y] - 1) - (2 * e[c] + 1) - (2 * e[d] + 1)
    ok &= gain > 0
    p = lambda i: P[i].astype(np.float64)                                      # noqa: E731
    px, py, pc, pd = p(x), p(y), p(c), p(d)
    o1, o2 = _cross(px, py, pc), _cross(px, pd, py)
    n1, n2 = _cross(px, pd, pc), _cross(pd, py, pc)
    nz = lambda q: (q[0] != 0) | (q[1] != 0) | (q[2] != 0)                      # noqa: E731
    ok &= nz(n1) & nz(n2)
    ok &= (_dot(n1, o1) > 0) & (_dot(n1, o2) > 0) & (_dot(n2, o1) > 0) & (_dot(n2, o2) > 0)
    ok &= ~_is_crease(n1, n2, cosf)
    key[cand] = np.where(ok, (np.uint64(0xFFFFFFFF) - gain.astype(np.uint64)) << np.uint64(32) | cand.astype(np.uint64), NONE)
    kc = key[cand]
    m1 = np.full(V, NONE, np.uint64)
    for q in (x, y, c, d):
        np.minimum.at(m1, q, kc)
    acc = (kc != NONE) & (m1[x] == kc) & (m1[y] == kc) & (m1[c] == kc) & (m1[d] == kc)
    if not acc.any():
        return T, 0
    T = T.copy()
    T[f1[acc]] = np.stack([x, d, c], 1)[acc]
    T[f2[acc]] = np.stack([d, y, c], 1)[acc]
    return T, int(acc.sum())


# ---------------------------------------------------------------------------------------------------------------- smoothing
def smooth(P, T, C):
    V = len(P)
    FACE, OUT, IN, n, frozen, deg, feat = state(P, T, C)
    mov = np.flatnonzero(~feat)
    if len(mov) == 0:
        return P
    D = OUT.shape[1]
    valid = np.arange(D)[None, :] < n[mov][:, None]
    nb = np.sort(np.where(valid, OUT[mov], np.iinfo(np.int64).max), 1)
    acc = np.zeros((len(mov), 3))
    for j in range(D):
        vj = valid[:, j]
        acc = np.where(vj[:, None], acc + P[np.where(vj, nb[:, j], 0)].astype(np.float64), acc)
    c = acc / n[mov][:, None].astype(np.float64)
    nacc = np.zeros((len(mov), 3))
    for j in range(D):
        vj = valid[:, j]
        t = T[np.where(vj, FACE[mov, j], 0)]
        q = P[t].astype(np.float64)
        cr = np.stack(_cross(q[:, 0], q[:, 1], q[:, 2]), 1)
        nacc = np.where(vj[:, None], nacc + cr, nacc)
    ln = np.sqrt(nacc[:, 0] * nacc[:, 0] + nacc[:, 1] * nacc[:, 1] + nacc[:, 2] * nacc[:, 2])
    with np.errstate(all="ignore"):
        nn = nacc / ln[:, None]
    p = P[mov].astype(np.float64)
    dd = c - p
    t = nn[:, 0] * dd[:, 0] + nn[:, 1] * dd[:, 1] + nn[:, 2] * dd[:, 2]
    with np.errstate(all="ignore"):
        q = (p + (dd - nn * t[:, None])).astype(np.float32)
    ok = (ln != 0) & _star_ok(P, T, FACE, n, mov, np.full(len(mov), -1), q)
    out = P.copy()
    out[mov[ok]] = q[ok]
    return out


# ---------------------------------------------------------------------------------------------------------------- projection
def closest_point(p, a, b, c):
    """Ericson's closest point of p on triangle abc, fp64, broadcast over [..., 3] arrays, in the kernels' order; the region tests run
    in this order and the first that holds gives the point."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = _dot(ab.T, ap.T), _dot(ac.T, ap.T)
    bp = p - b
    d3, d4 = _dot(ab.T, bp.T), _dot(ac.T, bp.T)
    cp = p - c
    d5, d6 = _dot(ab.T, cp.T), _dot(ac.T, cp.T)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    with np.errstate(all="ignore"):
        tv = d1 / (d1 - d3)
        tw = d2 / (d2 - d6)
        tu = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        s = va + vb + vc
        iv, iw = vb / s, vc / s
    q_int = (a + ab * iv[:, None]) + ac * iw[:, None]
    conds = [((d1 <= 0) & (d2 <= 0), a),
             ((d3 >= 0) & (d4 <= d3), b),
             ((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + ab * tv[:, None]),
             ((d6 >= 0) & (d5 <= d6), c),
             ((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + ac * tw[:, None]),
             ((va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0), b + (c - b) * tu[:, None]),
             (~(s > 0), a)]
    q = q_int
    for cond, val in reversed(conds):
        q = np.where(cond[:, None], val, q)
    return q


def nearest(pts, P0, T0, chunk=64):
    """Closest point of the input (P0, T0) to each of pts fp32 [n,3] by brute force over every face: (fp32 [n,3], face id int64 [n]);
    smallest squared distance, then smallest face id; faces with a zero cross product skipped; a point with no face left keeps its
    position (face -1)."""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    out, fid = pts.copy(), np.full(len(pts), -1, np.int64)
    if len(T0) == 0:
        return out, fid
    tri = P0[T0].astype(np.float64)                                            # [F0,3,3]
    cr = np.stack(_cross(tri[:, 0], tri[:, 1], tri[:, 2]), 1)
    live = np.flatnonzero((cr != 0).any(1))
    if len(live) == 0:
        return out, fid
    tri = tri[live]
    for i in range(0, len(pts), chunk):
        p = pts[i:i + chunk].astype(np.float64)
        k, m = len(p), len(live)
        pp = np.repeat(p, m, 0)
        a, b, c = (np.tile(tri[:, j], (k, 1)) for j in range(3))
        q = closest_point(pp, a, b, c)
        dd = q - pp
        d2 = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1] + dd[:, 2] * dd[:, 2]).reshape(k, m)
        best = np.argmin(d2, 1)                                                 # first minimum: the smallest face id
        out[i:i + k] = q.reshape(k, m, 3)[np.arange(k), best].astype(np.float32)
        fid[i:i + k] = live[best]
    return out, fid


def project(P, T, C, P0, T0):
    """(P with every non-feature vertex at its closest input point, the ids moved)"""
    _, _, _, _, _, _, feat = state(P, T, C)
    mov = np.flatnonzero(~feat)
    out = P.copy()
    if len(mov):
        out[mov] = nearest(P[mov], P0, T0)[0]
    return out, mov


# ---------------------------------------------------------------------------------------------------------------- driver
def remesh(verts, faces, target_len, iterations=3, feature_deg=30.0, record=False):
    """(verts fp32, faces int64[, info]).  ``info`` lists per iteration dict(split=new vertices, collapse=[accepted per round],
    flip=[accepted per round], F=faces after each phase, energy=valence energy before / after the flips, projected=(vertex ids, their
    positions before and after the projection)))."""
    P, T = check_mesh(verts, faces)
    L, it = float(target_len), int(iterations)
    if not (math.isfinite(L) and L > 0) or it < 0 or not (0.0 <= float(feature_deg) <= 180.0):
        raise ValueError("target_len must be finite and > 0, iterations >= 0, feature_deg in [0, 180]")
    lo2, hi2, cosf = params(L, feature_deg)
    P0, T0 = P.copy(), T.copy()
    C = initial_creases(P, T, cosf)
    info = []
    for _ in range(it):
        rec = dict(collapse=[], flip=[], F=[])
        P, T, C, rec["split"] = split(P, T, C, hi2)
        rec["F"].append(len(T))
        while True:
            P, T, k = collapse_round(P, T, C, lo2, hi2)
            if k == 0:
                break
            rec["collapse"].append(k)
        rec["F"].append(len(T))
        e0 = valence_energy(T, len(P))
        while True:
            T, k = flip_round(P, T, C, cosf)
            if k == 0:
                break
            rec["flip"].append(k)
        rec["energy"] = (e0, valence_energy(T, len(P)))
        rec["F"].append(len(T))
        P = smooth(P, T, C)
        before = P
        P, mov = project(P, T, C, P0, T0)
        rec["projected"] = (mov, before[mov], P[mov])
        info.append(rec)
    v, f = compact(P, T)
    return (v, f, info) if record else (v, f)
