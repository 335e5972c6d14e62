"""Oracle mesh clean-up and decimation (TEST INFRASTRUCTURE — see oracle/__init__.py).

numpy restatement of the contract of csrc/mesh_simplify.cu, the GPU stand-in for the clean_mesh / decimate_mesh calls of
extract_texmesh (/root/reference/inference.py:126-129, utils/meshutils.py:63-193).  Slow (vectorised per round), exact: the
kernels must give the same bytes.  Every fp64 expression below is written in the order the kernels evaluate it (numpy evaluates
``a + b + c`` as ``(a + b) + c`` and never contracts a product into a sum); fp32 values are rounded to nearest.

Input: verts fp32 [V,3], faces int64 [F,3]; an index outside [0, V) or a face that repeats an index is a ValueError.
Output: the vertices some face uses, in ascending original id; the kept faces in their original order, remapped, with their
own cyclic vertex order.

Component filter: faces are adjacent iff they share an undirected edge.  A component is removed iff it has fewer than
``min_faces`` faces or its box diagonal is below ``min_diameter`` times the diagonal of the box of all referenced vertices.

Decimation, in rounds of independent edge collapses (see ``decimate``):
  * quadrics: fp64, 10 coefficients (a², ab, ac, ad, b², bc, bd, c², cd, d²) of the unit plane (a, b, c, d) of each face,
    normal from (v1 - v0) x (v2 - v0), weighted by the face's area; zero-area faces contribute nothing; Q_v is summed over the
    faces containing v in ascending face index, sequentially from 0; a survivor keeps Q_a + Q_b;
  * frozen: a vertex whose corners (out, in) = (next, previous vertex of each face containing it) do not list every neighbour
    exactly once as out and once as in (a boundary, non-manifold or inconsistently oriented edge), or do not form one cycle
    (more than one fan); recomputed every round;
  * edges: the current undirected edges in ascending (min id, max id) order; candidate iff neither end is frozen;
  * placement: Q = Q_a + Q_b; the 3 x 3 system solved by cofactors unless |det| <= 1e-10 tr³ or a component of the fp32
    result is not finite, in which case the cheapest of midpoint, a, b (that order on ties); cost = max(0, x̄ᵀQx̄) at the fp32 x̄;
  * valid iff link condition N(a) ∩ N(b) = {c, d}, deg(a) + deg(b) >= 7, deg(c) >= 4, deg(d) >= 4, and no face of the two stars
    (but the two removed) with a non-zero normal turns it by 90 degrees or more;
  * key = fp32(cost) bits << 32 | edge id (valid), else 2⁶⁴ - 1; accepted iff its key is the minimum of m1 (the least key at a
    vertex) over both ends and their neighbours; the last round keeps the ceil((F - target) / 2) smallest accepted keys;
  * collapse: min(a, b) takes x̄ and Q_a + Q_b, the other id is replaced by it in every face, the two faces on the edge go.
"""
from __future__ import annotations

import numpy as np

NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
SINGULAR_REL = 1e-10


def check_mesh(verts, faces):
    """(fp32 [V,3] copy, int64 [F,3] copy); ValueError for malformed input."""
    P = np.array(verts, dtype=np.float32).reshape(-1, 3) if np.size(verts) else np.zeros((0, 3), np.float32)
    T = np.array(faces, dtype=np.int64)
    if T.size == 0:
        T = T.reshape(0, 3)
    if T.ndim != 2 or T.shape[1] != 3:
        raise ValueError(f"faces must be [F,3], got {T.shape}")
    if len(T) and (T.min() < 0 or T.max() >= len(P)):
        raise ValueError("face index outside [0, V)")
    if len(T) and ((T[:, 0] == T[:, 1]) | (T[:, 1] == T[:, 2]) | (T[:, 2] == T[:, 0])).any():
        raise ValueError("a face repeats a vertex index")
    return P, T


def compact(P, T):
    """Referenced vertices in ascending id, faces remapped (order and cyclic order kept)."""
    used = np.zeros(len(P), bool)
    used[T.ravel()] = True
    newid = np.cumsum(used) - 1
    return P[used].copy(), newid[T].astype(np.int64).reshape(-1, 3)


# ---------------------------------------------------------------------------------------------------------------- components
def _ord(x):
    """fp32 -> int32 with the same order (the kernels' atomicMin / atomicMax key); its own inverse."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.int32)
    return np.where(b >= 0, b, b ^ np.int32(0x7FFFFFFF)).astype(np.int32)


def _unord(i):
    return _ord(np.asarray(i, np.int32).view(np.float32)).view(np.float32)


def _diag(lo_ord, hi_ord):
    lo, hi = _unord(lo_ord).astype(np.float64), _unord(hi_ord).astype(np.float64)
    d = hi - lo
    return np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2])


def component_labels(T):
    """Edge-connected components of the faces: label[f] = the smallest face id of f's component."""
    F = len(T)
    if F == 0:
        return np.zeros(0, np.int64)
    a, b = T, np.roll(T, -1, axis=1)
    key = (np.minimum(a, b) << 32 | np.maximum(a, b)).ravel()
    fid = np.repeat(np.arange(F), 3)
    order = np.lexsort((fid, key))
    k, f = key[order], fid[order]
    same = k[:-1] == k[1:]
    u, v = f[:-1][same], f[1:][same]
    label = np.arange(F)
    while True:
        m = np.minimum(label[u], label[v])
        new = label.copy()
        np.minimum.at(new, u, m)
        np.minimum.at(new, v, m)
        while True:
            j = new[new]
            if np.array_equal(j, new):
                break
            new = j
        if np.array_equal(new, label):
            return label
        label = new


def remove_small_components(verts, faces, min_faces=8, min_diameter=0.05, return_labels=False):
    """clean_mesh's remove_connected_component_by_face_number(min_f) and ..._by_diameter(PercentageValue(100 min_diameter))."""
    P, T = check_mesh(verts, faces)
    label = component_labels(T)
    keep = np.ones(len(T), bool)
    if len(T):
        O = _ord(P)
        fo = O[T]                                               # [F,3 verts,3 dims]
        gdiag = _diag(fo.reshape(-1, 3).min(0), fo.reshape(-1, 3).max(0))
        cmin = np.full((len(T), 3), np.iinfo(np.int32).max, np.int32)
        cmax = np.full((len(T), 3), np.iinfo(np.int32).min, np.int32)
        np.minimum.at(cmin, label, fo.min(1))
        np.maximum.at(cmax, label, fo.max(1))
        cnt = np.bincount(label, minlength=len(T))
        cdiag = _diag(cmin[label], cmax[label])
        keep = (cnt[label] >= min_faces) & ~(cdiag < np.float64(min_diameter) * gdiag)
    v, f = compact(P, T[keep])
    return (v, f, label) if return_labels else (v, f)


# ---------------------------------------------------------------------------------------------------------------- decimation
def face_quadrics(P, T):
    """[F,10] fp64 area-weighted plane quadrics."""
    p = P[T].astype(np.float64)                                 # [F,3,3]
    p0, p1, p2 = p[:, 0], p[:, 1], p[:, 2]
    cx, cy, cz = _cross(p0, p1, p2)
    ln = np.sqrt(cx * cx + cy * cy + cz * cz)
    with np.errstate(all="ignore"):
        area = 0.5 * ln
        nx, ny, nz = cx / ln, cy / ln, cz / ln
        d = -(nx * p0[:, 0] + ny * p0[:, 1] + nz * p0[:, 2])
        u = [nx, ny, nz, d]
        q = np.stack([area * (u[i] * u[j]) for i in range(4) for j in range(i, 4)], 1)
    q[ln == 0] = 0.0
    return q


def _cross(p0, p1, p2):
    e1, e2 = p1 - p0, p2 - p0
    return (e1[..., 1] * e2[..., 2] - e1[..., 2] * e2[..., 1], e1[..., 2] * e2[..., 0] - e1[..., 0] * e2[..., 2],
            e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0])


def _corners(T, V):
    """Per vertex, its corners in ascending face index, padded to the largest count D: FACE, OUT, IN [V,D] (pads -1, -1, -2), n [V]."""
    F = len(T)
    v = T.ravel()
    fid = np.repeat(np.arange(F), 3)
    k = np.tile(np.arange(3), F)
    out, inn = T[fid, (k + 1) % 3], T[fid, (k + 2) % 3]
    order = np.lexsort((fid, v))
    vs = v[order]
    n = np.bincount(v, minlength=V)
    start = np.concatenate([[0], np.cumsum(n)[:-1]])
    rank = np.arange(3 * F) - start[vs]
    D = max(int(n.max()) if V else 0, 1)
    FACE, OUT, IN = np.full((V, D), -1), np.full((V, D), -1), np.full((V, D), -2)
    FACE[vs, rank], OUT[vs, rank], IN[vs, rank] = fid[order], out[order], inn[order]
    return FACE, OUT, IN, n, (vs, fid[order], rank)


def init_quadrics(P, T):
    q = face_quadrics(P, T)
    _, _, _, _, (vs, fs, rank) = _corners(T, len(P))
    Q = np.zeros((len(P), 10))
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        s = rank == r
        Q[vs[s]] = Q[vs[s]] + q[fs[s]]
    return Q


def vertex_state(OUT, IN, n):
    """(frozen bool [V], deg int [V]) from the corner lists."""
    V, D = OUT.shape
    valid = np.arange(D)[None, :] < n[:, None]
    c_oo = (OUT[:, :, None] == OUT[:, None, :]).sum(2)
    c_oi = (OUT[:, :, None] == IN[:, None, :]).sum(2)
    ok = ((~valid) | ((c_oo == 1) & (c_oi == 1))).all(1) & (n > 0)
    rows = np.arange(V)
    cur, steps = IN[:, 0].copy(), np.ones(V, np.int64)
    done = ~ok | (cur == OUT[:, 0])
    for _ in range(D):
        act = ~done
        if not act.any():
            break
        j = np.argmax(OUT == cur[:, None], axis=1)
        cur = np.where(act, IN[rows, j], cur)
        steps += act
        done |= cur == OUT[:, 0]
    ok &= steps == n
    allv = np.where(np.concatenate([valid, valid], 1), np.concatenate([OUT, IN], 1), -1)
    s = np.sort(allv, 1)
    deg = ((s[:, 1:] != s[:, :-1]) & (s[:, 1:] >= 0)).sum(1) + (s[:, 0] >= 0)
    return ~ok, deg


def quadric_cost(q, x, y, z):
    r0 = q[:, 0] * x + q[:, 1] * y + q[:, 2] * z + q[:, 3]
    r1 = q[:, 1] * x + q[:, 4] * y + q[:, 5] * z + q[:, 6]
    r2 = q[:, 2] * x + q[:, 5] * y + q[:, 7] * z + q[:, 8]
    r3 = q[:, 3] * x + q[:, 6] * y + q[:, 8] * z + q[:, 9]
    c = r0 * x + r1 * y + r2 * z + r3
    return np.where(c > 0, c, 0.0)


def placement(q, pa, pb):
    """(x̄ fp32 [E,3], cost fp64 [E]) for summed quadrics q [E,10] and end positions pa, pb fp32 [E,3]."""
    c00, c01, c02 = q[:, 4] * q[:, 7] - q[:, 5] * q[:, 5], q[:, 2] * q[:, 5] - q[:, 1] * q[:, 7], q[:, 1] * q[:, 5] - q[:, 2] * q[:, 4]
    c11, c12, c22 = q[:, 0] * q[:, 7] - q[:, 2] * q[:, 2], q[:, 1] * q[:, 2] - q[:, 0] * q[:, 5], q[:, 0] * q[:, 4] - q[:, 1] * q[:, 1]
    det = q[:, 0] * c00 + q[:, 1] * c01 + q[:, 2] * c02
    tr = q[:, 0] + q[:, 4] + q[:, 7]
    b0, b1, b2 = -q[:, 3], -q[:, 6], -q[:, 8]
    with np.errstate(all="ignore"):
        x = np.stack([(c00 * b0 + c01 * b1 + c02 * b2) / det, (c01 * b0 + c11 * b1 + c12 * b2) / det,
                      (c02 * b0 + c12 * b1 + c22 * b2) / det], 1).astype(np.float32)
    solved = (np.abs(det) > SINGULAR_REL * (tr * tr * tr)) & np.isfinite(x).all(1)
    mid = ((pa.astype(np.float64) + pb.astype(np.float64)) * 0.5).astype(np.float32)

    def cost(p):
        p = p.astype(np.float64)
        return quadric_cost(q, p[:, 0], p[:, 1], p[:, 2])

    best, bc = mid, cost(mid)
    for alt in (pa, pb):
        ac = cost(alt)
        better = ac < bc
        best, bc = np.where(better[:, None], alt, best), np.where(better, ac, bc)
    xs = np.where(solved[:, None], x, best)
    return xs, np.where(solved, cost(x), bc)


def _star_ok(P, T, FACE, n, v, other, xbar):
    """Per edge: every face at v not containing `other`, with a non-zero old normal, keeps n_old . n_new > 0 with v at xbar."""
    fl = FACE[v]                                                # [E,D]
    valid = np.arange(FACE.shape[1])[None, :] < n[v][:, None]
    tv = T[np.where(valid, fl, 0)]                              # [E,D,3]
    valid &= ~(tv == other[:, None, None]).any(2)
    old = P[tv].astype(np.float64)                              # [E,D,3,3]
    new = np.where((tv == v[:, None, None])[..., None], xbar.astype(np.float64)[:, None, None, :], old)
    nx, ny, nz = _cross(old[:, :, 0], old[:, :, 1], old[:, :, 2])
    mx, my, mz = _cross(new[:, :, 0], new[:, :, 1], new[:, :, 2])
    nonzero = (nx != 0) | (ny != 0) | (nz != 0)
    good = (nx * mx + ny * my + nz * mz) > 0
    return (~valid | ~nonzero | good).all(1)


def decimation_round(P, T, Q, target):
    """One round on (P fp32 [V,3], T int64 [F,3], Q fp64 [V,10]), target > F assumed false.  Returns (P, T, Q, accepted [k,2])."""
    V, F = len(P), len(T)
    FACE, OUT, IN, n, _ = _corners(T, V)
    frozen, deg = vertex_state(OUT, IN, n)
    a, b = T, np.roll(T, -1, axis=1)
    ekey = np.unique((np.minimum(a, b) << 32 | np.maximum(a, b)).ravel())
    ea, eb = (ekey >> 32).astype(np.int64), (ekey & 0xFFFFFFFF).astype(np.int64)
    E = len(ekey)
    key = np.full(E, NONE, np.uint64)
    cand = np.flatnonzero(~frozen[ea] & ~frozen[eb])
    if len(cand):
        A, B = ea[cand], eb[cand]
        rows = np.arange(len(cand))
        c = IN[A, np.argmax(OUT[A] == B[:, None], 1)]
        d = OUT[A, np.argmax(IN[A] == B[:, None], 1)]
        oa, ob = OUT[A], OUT[B]
        link = ((oa[:, :, None] == ob[:, None, :]) & (oa[:, :, None] >= 0)).sum((1, 2))
        ok = (link == 2) & (c != d) & (deg[A] + deg[B] >= 7) & (deg[c] >= 4) & (deg[d] >= 4)
        q = Q[A] + Q[B]
        xbar, cost = placement(q, P[A], P[B])
        ok &= _star_ok(P, T, FACE, n, A, B, xbar) & _star_ok(P, T, FACE, n, B, A, xbar)
        bits = cost.astype(np.float32).view(np.uint32).astype(np.uint64)
        key[cand] = np.where(ok, bits << np.uint64(32) | cand.astype(np.uint64), NONE)
        del rows
    m1 = np.full(V, NONE, np.uint64)
    np.minimum.at(m1, ea, key)
    np.minimum.at(m1, eb, key)
    m2 = m1.copy()
    np.minimum.at(m2, ea, m1[eb])
    np.minimum.at(m2, eb, m1[ea])
    acc = (key != NONE) & (m2[ea] == key) & (m2[eb] == key)
    nacc = int(acc.sum())
    if nacc == 0:
        return P, T, Q, np.zeros((0, 2), np.int64)
    if F - 2 * nacc < target:
        k = (F - target + 1) // 2
        thr = np.sort(key[acc])[k - 1]
        acc &= key <= thr
    e = np.flatnonzero(acc)
    sel = np.searchsorted(cand, e)
    A, B = ea[e], eb[e]
    P, Q = P.copy(), Q.copy()
    P[A] = xbar[sel]
    Q[A] = Q[A] + Q[B]
    rep = np.arange(V)
    rep[B] = A
    T = rep[T]
    keep = (T[:, 0] != T[:, 1]) & (T[:, 1] != T[:, 2]) & (T[:, 2] != T[:, 0])
    return P, T[keep], Q, np.stack([A, B], 1)


def decimate(verts, faces, target, record=False):
    """Decimate to ``target`` faces: (verts fp32, faces int64[, rounds]).  Stops when F <= target (a reachable target ends at
    F in {target - 1, target}) or when a round accepts nothing (the mesh is then returned above target).  ``rounds`` lists, per
    round, dict(faces=the faces before it, accepted=[k,2] collapsed (survivor, removed) pairs, F=faces after it)."""
    P, T = check_mesh(verts, faces)
    target = int(target)
    rounds = []
    if len(T) > target:
        Q = init_quadrics(P, T)
        while len(T) > target:
            before = T
            P, T, Q, acc = decimation_round(P, T, Q, target)
            if len(acc) == 0:
                break
            if record:
                rounds.append(dict(faces=before, accepted=acc, F=len(T)))
    v, f = compact(P, T)
    return (v, f, rounds) if record else (v, f)
