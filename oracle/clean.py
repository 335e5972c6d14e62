"""Oracle mesh clean-up (TEST INFRASTRUCTURE — see oracle/__init__.py).

numpy restatement of the clean-up contract of csrc/mesh_simplify.cu (DESIGN.md §1 "clean-up contract"): this package's reading of
the VCG filters clean_mesh runs (/root/reference/utils/meshutils.py:118-193, called at inference.py:126).  pymeshlab is not run
anywhere here, so these rules are a reading, not a verified equivalence.  Exact: the kernels must give the same bytes.

  * weld (``weld``): unreferenced vertices dropped; r = frac x the fp64 diagonal of the fp32 box of the referenced vertices (the
    component filter's ``_diag``); in ascending id, a referenced vertex is a seed iff no earlier seed lies strictly within r
    (fp64 (dx² + dy²) + dz² < r² from the fp32 positions), otherwise it takes the id (and so the position) of the smallest-id seed
    within r.  Not a transitive closure.  frac = 0 (or r = 0) merges nothing.  Then faces onto the seeds; a face is kept iff its
    indices are distinct, no lower face id has the same index set, and its (v1 - v0) x (v2 - v0) (``decimate._cross``) is not
    exactly zero in all three components;
  * components: ``decimate.remove_small_components``;
  * repair (``repair``): the faces on an undirected edge with more than two faces, visited in ascending (|(v1 - v0) x (v2 - v0)|,
    face id), where |c| = sqrt((cx² + cy²) + cz²); a face is deleted iff one of its edges still has more than two faces.  Then the
    corners of every vertex are joined into fans through the edges (v, w) two faces share; the fan holding the vertex's smallest face
    id keeps it, every other fan gets a copy at the same position, appended in (vertex id, smallest face id of the fan) order.

Output: the vertices in use in ascending original id (then the copies), the kept faces in original order, remapped.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse
import scipy.sparse.csgraph

from . import decimate as od

_OFFSETS = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]


def _check_range(verts, faces):
    P = np.array(verts, dtype=np.float32).reshape(-1, 3) if np.size(verts) else np.zeros((0, 3), np.float32)
    T = np.array(faces, dtype=np.int64)
    if T.size == 0:
        T = T.reshape(0, 3)
    if T.ndim != 2 or T.shape[1] != 3:
        raise ValueError(f"faces must be [F,3], got {T.shape}")
    if len(T) and (T.min() < 0 or T.max() >= len(P)):
        raise ValueError("face index outside [0, V)")
    return P, T


def merge_radius(P, used, frac):
    """r (fp64) for the referenced vertices, or 0.0 when nothing can merge."""
    if not frac > 0 or not used.any():
        return 0.0
    O = od._ord(P[used])
    r = np.float64(frac) * od._diag(O.min(0), O.max(0))
    return float(r) if np.isfinite(r) and r * r > 0 else 0.0


def seeds(P, used, r):
    """rep [V]: each referenced vertex's seed (itself for a seed); the sequential greedy definition, with a grid of the seeds found
    so far (cells of side slightly above r) to gather candidates."""
    rep = np.arange(len(P))
    if r == 0.0:
        return rep
    r2 = r * r
    Pd = P.astype(np.float64)
    lo = Pd[used].min(0)
    cells = np.floor((Pd - lo) / (r * (1 + 1 / 1024))).astype(np.int64).tolist()
    pts = Pd.tolist()
    grid = {}
    for v in np.flatnonzero(used).tolist():
        cx, cy, cz = cells[v]
        px, py, pz = pts[v]
        best = -1
        for ox, oy, oz in _OFFSETS:
            for s in grid.get((cx + ox, cy + oy, cz + oz), ()):
                if best >= 0 and s > best:
                    break
                qx, qy, qz = pts[s]
                dx, dy, dz = qx - px, qy - py, qz - pz
                if dx * dx + dy * dy + dz * dz < r2:
                    best = s
                    break
        if best < 0:
            grid.setdefault((cx, cy, cz), []).append(v)
        else:
            rep[v] = best
    return rep


def weld(verts, faces, frac):
    """(verts fp32, faces int64) after the close-vertex merge and the duplicate / null face removal.  Faces may repeat an index."""
    P, T = _check_range(verts, faces)
    used = np.zeros(len(P), bool)
    used[T.ravel()] = True
    rep = seeds(P, used, merge_radius(P, used, frac))
    T = rep[T]
    keep = (T[:, 0] != T[:, 1]) & (T[:, 1] != T[:, 2]) & (T[:, 2] != T[:, 0])
    if keep.any():
        idx = np.flatnonzero(keep)
        _, first = np.unique(np.sort(T[idx], 1), axis=0, return_index=True)
        keep[:] = False
        keep[idx[first]] = True
        p = P[T].astype(np.float64)
        cx, cy, cz = od._cross(p[:, 0], p[:, 1], p[:, 2])
        keep &= (cx != 0) | (cy != 0) | (cz != 0)
    return od.compact(P, T[keep])


def _edge_ids(T):
    a, b = T, np.roll(T, -1, axis=1)
    key = (np.minimum(a, b) << 32 | np.maximum(a, b))
    _, eid = np.unique(key.ravel(), return_inverse=True)
    return eid.reshape(-1, 3)


def repair(verts, faces):
    """(verts fp32, faces int64) after the non-manifold edge removal and the non-manifold vertex split."""
    P, T = od.check_mesh(verts, faces)
    F = len(T)
    alive = np.ones(F, bool)
    if F:
        fe = _edge_ids(T)
        cnt = np.bincount(fe.ravel())
        cand = np.flatnonzero((cnt[fe] > 2).any(1))
        p = P[T[cand]].astype(np.float64)
        cx, cy, cz = od._cross(p[:, 0], p[:, 1], p[:, 2])
        area = np.sqrt(cx * cx + cy * cy + cz * cz)
        for f in cand[np.lexsort((cand, area))].tolist():
            e = fe[f]
            if (cnt[e] > 2).any():
                alive[f] = False
                cnt[e] -= 1
    fid = np.flatnonzero(alive)
    h = (3 * fid[:, None] + np.arange(3)).ravel()                       # corners of the kept faces
    v = T.ravel()[h]
    f_of = h // 3
    k = h % 3
    w1, w2 = T[f_of, (k + 1) % 3], T[f_of, (k + 2) % 3]
    key = np.concatenate([v << 32 | w1, v << 32 | w2])
    node = np.concatenate([h, h])
    o = np.argsort(key, kind="stable")
    same = key[o][1:] == key[o][:-1]
    g = scipy.sparse.coo_matrix((np.ones(int(same.sum())), (node[o][:-1][same], node[o][1:][same])), shape=(3 * F, 3 * F))
    _, lab = scipy.sparse.csgraph.connected_components(g, directed=False)
    big = np.iinfo(np.int64).max
    fanmin = np.full(3 * F, big)
    np.minimum.at(fanmin, lab[h], f_of)
    vmin = np.full(len(P), big)
    np.minimum.at(vmin, v, f_of)
    fm = fanmin[lab[h]]
    split = fm != vmin[v]
    used = np.zeros(len(P), bool)
    used[v] = True
    newid = np.cumsum(used) - 1
    Vs = int(used.sum())
    out = newid[v]
    if split.any():
        pairs, inv = np.unique(np.stack([v[split], fm[split]], 1), axis=0, return_inverse=True)
        out[split] = Vs + inv.ravel()
        Pout = np.concatenate([P[used], P[pairs[:, 0]]])
    else:
        Pout = P[used].copy()
    return Pout, out.reshape(-1, 3).astype(np.int64)


def clean_mesh(verts, faces, v_pct=1, min_f=64, min_d=20, repair_mesh=True):
    """clean_mesh(verts, faces, v_pct, min_f, min_d, repair, remesh=False) in the reference's order."""
    v, f = weld(verts, faces, float(v_pct) / 100.0)
    if min_f > 0 or min_d > 0:
        v, f = od.remove_small_components(v, f, int(min_f), float(min_d) / 100.0)
    if repair_mesh:
        v, f = repair(v, f)
    return v, f
