"""Oracle texture bake (TEST INFRASTRUCTURE — see oracle/__init__.py).

numpy float64 restatement of the contracts of csrc/texture_bake.cu, the GPU stand-ins for the nvdiffrast / scipy / scikit-learn calls
of extract_texmesh's texture block (/root/reference/inference.py:163-211):
  * ``rasterize_uv``: texel (row i, col j) sampled at its centre, row 0 at v = 0; coverage iff the three edge functions, oriented by
    the sign of the triangle's area, are >= 0 (edges inclusive, both windings, zero-area triangles and out-of-range indices skipped);
    an edge is evaluated with its endpoints ordered by (x, y), so both triangles sharing it see opposite values; the lowest
    covering triangle index wins; (u, v) weigh vertices 0 and 1.  Also returns, per texel, the smallest |min barycentric| over every
    triangle whose bounding box holds the centre: a coverage decision can only flip under rounding where that margin is tiny.
  * ``interpolate``: u a0 + v a1 + (1 - u - v) a2, zeros where rast[..., 3] == 0.
  * ``inpaint``: brute force from the definition of inference.py:200-211 — the region is the mask dilated ``pad`` times by the
    4-connected cross minus the mask; each of its texels takes the Euclidean-nearest mask texel (squared integer distances), the
    smallest (row, col) among equidistant ones.
"""
from __future__ import annotations

import numpy as np


def _edge(ax, ay, bx, by, cx, cy, W, H):
    """cross(a - p, b - p) in texel units with (a, b) ordered by (x, y); negated when that swapped them."""
    swap = (bx < ax) | ((bx == ax) & (by < ay))
    lx, ly, hx, hy = np.where(swap, bx, ax), np.where(swap, by, ay), np.where(swap, ax, bx), np.where(swap, ay, by)
    e = (lx * W - cx) * (hy * H - cy) - (ly * H - cy) * (hx * W - cx)
    return np.where(swap, -e, e)


def _oriented_edges(x, y, sign, i, j, W, H):
    cx, cy = j + 0.5, i + 0.5
    e0 = sign * _edge(x[:, 1], y[:, 1], x[:, 2], y[:, 2], cx, cy, W, H)
    e1 = sign * _edge(x[:, 2], y[:, 2], x[:, 0], y[:, 0], cx, cy, W, H)
    e2 = sign * _edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], cx, cy, W, H)
    return e0, e1, e2


def rasterize_uv(vt, ft, H: int, W: int, chunk: int = 1 << 22):
    """vt [Nt,2], ft [F,3] -> (rast float64 [H,W,4] = (u, v, 0, id + 1), tri int64 [H,W] (-1 = empty), margin float64 [H,W])."""
    vt = np.asarray(vt, dtype=np.float64).reshape(-1, 2)
    ft = np.asarray(ft, dtype=np.int64).reshape(-1, 3)
    ids = np.flatnonzero(((ft >= 0) & (ft < len(vt))).all(1))
    x, y = vt[ft[ids], 0], vt[ft[ids], 1]                                  # [n, 3]
    area = (x[:, 1] - x[:, 0]) * W * ((y[:, 2] - y[:, 0]) * H) - (y[:, 1] - y[:, 0]) * H * ((x[:, 2] - x[:, 0]) * W)
    keep = np.isfinite(area) & (area != 0)
    ids, x, y, area = ids[keep], x[keep], y[keep], area[keep]
    sign = np.sign(area)
    j0 = np.clip(np.floor(x.min(1) * W - 0.5) - 1, 0, W).astype(np.int64)
    j1 = np.clip(np.ceil(x.max(1) * W - 0.5) + 1, -1, W - 1).astype(np.int64)
    i0 = np.clip(np.floor(y.min(1) * H - 0.5) - 1, 0, H).astype(np.int64)
    i1 = np.clip(np.ceil(y.max(1) * H - 0.5) + 1, -1, H - 1).astype(np.int64)
    bw, bh = np.maximum(j1 - j0 + 1, 0), np.maximum(i1 - i0 + 1, 0)
    count = bw * bh
    winner = np.full(H * W, np.iinfo(np.int64).max, dtype=np.int64)
    margin = np.full(H * W, np.inf)
    start = 0
    while start < len(ids):
        stop, total = start, 0
        while stop < len(ids) and (stop == start or total + count[stop] <= chunk):
            total += count[stop]
            stop += 1
        n = count[start:stop]
        which = np.repeat(np.arange(start, stop), n)                        # triangle of each (triangle, texel) pair
        local = np.arange(total) - np.repeat(np.cumsum(n) - n, n)
        i, j = i0[which] + local // np.maximum(bw[which], 1), j0[which] + local % np.maximum(bw[which], 1)
        e0, e1, e2 = _oriented_edges(x[which], y[which], sign[which], i, j, W, H)
        low = np.minimum(np.minimum(e0, e1), e2)
        flat = i * W + j
        np.minimum.at(margin, flat, np.abs(low) / np.abs(area[which]))
        cov = low >= 0
        np.minimum.at(winner, flat[cov], ids[which[cov]])
        start = stop
    tri = np.where(winner == np.iinfo(np.int64).max, -1, winner).reshape(H, W)
    rast = np.zeros((H, W, 4))
    ci, cj = np.nonzero(tri >= 0)
    t = tri[ci, cj]
    ok = ((ft[t] >= 0) & (ft[t] < len(vt))).all(1)
    assert ok.all()
    tx, ty = vt[ft[t], 0], vt[ft[t], 1]
    ta = (tx[:, 1] - tx[:, 0]) * W * ((ty[:, 2] - ty[:, 0]) * H) - (ty[:, 1] - ty[:, 0]) * H * ((tx[:, 2] - tx[:, 0]) * W)
    e0, e1, e2 = _oriented_edges(tx, ty, np.sign(ta), ci, cj, W, H)
    s = e0 + e1 + e2
    rast[ci, cj, 0], rast[ci, cj, 1], rast[ci, cj, 3] = e0 / s, e1 / s, t + 1
    return rast, tri, margin.reshape(H, W)


def interpolate(attr, rast, tri):
    """attr [N,C], rast [H,W,4], tri [F,3] -> float64 [H,W,C]."""
    attr = np.asarray(attr, dtype=np.float64)
    tri = np.asarray(tri, dtype=np.int64)
    rast = np.asarray(rast, dtype=np.float64)
    out = np.zeros(rast.shape[:2] + (attr.shape[1],))
    ci, cj = np.nonzero(rast[..., 3] > 0)
    t = rast[ci, cj, 3].astype(np.int64) - 1
    u, v = rast[ci, cj, 0:1], rast[ci, cj, 1:2]
    out[ci, cj] = u * attr[tri[t, 0]] + v * attr[tri[t, 1]] + (1 - u - v) * attr[tri[t, 2]]
    return out


def dilate_cross(mask, iterations: int):
    """binary_dilation(mask, iterations=n) with scipy's default structuring element (the 4-connected cross)."""
    m = np.asarray(mask, dtype=bool).copy()
    for _ in range(iterations):
        g = m.copy()
        g[1:] |= m[:-1]
        g[:-1] |= m[1:]
        g[:, 1:] |= m[:, :-1]
        g[:, :-1] |= m[:, 1:]
        m = g
    return m


def inpaint(feats, mask, pad: int = 32):
    """feats [H,W,C], mask [H,W] -> (out, src int64 [H,W] flat source index or -1, d2 int64 [H,W] squared distance or -1)."""
    mask = np.asarray(mask, dtype=bool)
    H, W = mask.shape
    out = np.array(feats, copy=True)
    src = np.full((H, W), -1, dtype=np.int64)
    d2 = np.full((H, W), -1, dtype=np.int64)
    region = dilate_cross(mask, pad) & ~mask
    pi, pj = np.nonzero(region)
    # candidate offsets in the order the tie rule ranks them: squared distance, then row, then column
    r = np.arange(-pad, pad + 1)
    dy, dx = [a.ravel() for a in np.meshgrid(r, r, indexing="ij")]
    order = np.lexsort((dx, dy, dy * dy + dx * dx))
    for o in order:
        if len(pi) == 0:
            break
        if dy[o] * dy[o] + dx[o] * dx[o] > pad * pad:
            break                                      # a texel of the region has a mask texel within Euclidean distance pad
        si, sj = pi + dy[o], pj + dx[o]
        inside = (si >= 0) & (si < H) & (sj >= 0) & (sj < W)
        hit = np.zeros(len(pi), dtype=bool)
        hit[inside] = mask[si[inside], sj[inside]]
        if hit.any():
            src[pi[hit], pj[hit]] = si[hit] * W + sj[hit]
            d2[pi[hit], pj[hit]] = dy[o] * dy[o] + dx[o] * dx[o]
            pi, pj = pi[~hit], pj[~hit]
    assert len(pi) == 0, "a texel of the dilated region found no mask texel within the pad radius"
    wi, wj = np.nonzero(src >= 0)
    out[wi, wj] = np.asarray(feats)[src[wi, wj] // W, src[wi, wj] % W]
    return out, src, d2
