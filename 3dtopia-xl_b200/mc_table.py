"""Generator of the marching-cubes case table (csrc/mc_tables.cuh).  The table is derived, not typed in:

    python 3dtopia-xl_b200/mc_table.py          # rewrites csrc/mc_tables.cuh

Cube convention (the one csrc/marching_cubes.cu and the Python layer use):
  * corner n = (n & 1, (n >> 1) & 1, (n >> 2) & 1) along array axes (0, 1, 2); bit n of the case is set iff corner n is
    inside (value < iso);
  * the 12 edges are the corner pairs (a, b), a < b, that differ in one bit, in lexicographic order; edge e is owned by its
    lower corner a and runs along axis log2(a ^ b), so its vertex is the one the lattice point cell + corner(a) owns on that axis.

Rules, per case:
  1. on each of the 6 faces, the crossing points of the face's edges are joined into segments: 2 crossings give one segment,
     4 crossings (an ambiguous face) give two segments that cut off each inside corner separately.  The choice depends only on
     the face's four corner signs, so the two cells that share a face draw the same segments on it;
  2. every segment is directed so that the inside region lies on a fixed side relative to the face's outward normal; the
     segments then chain into closed loops (each crossing starts exactly one segment and ends exactly one);
  3. each loop is fan-triangulated from an apex chosen so that no fan chord joins two crossings on one cube face (such a
     chord would lie in the face and overlap the neighbour cell's triangles);
  4. triangles are wound so that (v1 - v0) x (v2 - v0) points toward increasing value (outward for an SDF that is negative inside).
"""
from __future__ import annotations

import os

import numpy as np

CORNERS = [(n & 1, (n >> 1) & 1, (n >> 2) & 1) for n in range(8)]
EDGES = [(a, b) for a in range(8) for b in range(a + 1, 8) if bin(a ^ b).count("1") == 1]
EDGE_AXIS = [(a ^ b).bit_length() - 1 for a, b in EDGES]
_EIDX = {e: i for i, e in enumerate(EDGES)}
MAX_TRIS = 5
HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "mc_tables.cuh")


def edge_id(a: int, b: int) -> int:
    return _EIDX[(min(a, b), max(a, b))]


def _faces():
    """The 6 cube faces as (axis, side, 4 corners in cyclic order)."""
    out = []
    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in (0, 1):
            cs = [n for n in range(8) if CORNERS[n][axis] == side]
            cyc = [(0, 0), (1, 0), (1, 1), (0, 1)]
            out.append((axis, side, sorted(cs, key=lambda n: cyc.index((CORNERS[n][u], CORNERS[n][v])))))
    return out


FACES = _faces()


def _on_one_face(e: int, g: int) -> bool:
    return any(set(EDGES[e]) <= set(f) and set(EDGES[g]) <= set(f) for _, _, f in FACES)


def face_segments(mask: int):
    """Directed segments (edge, edge) drawn on each face for case `mask` (rule 1 and 2)."""
    inside = [(mask >> n) & 1 for n in range(8)]
    corner = lambda n: np.array(CORNERS[n], float)  # noqa: E731
    mid = lambda e: (corner(EDGES[e][0]) + corner(EDGES[e][1])) / 2.0  # noqa: E731
    segs = []
    for axis, side, f in FACES:
        normal = np.zeros(3)
        normal[axis] = 1.0 if side else -1.0
        es = [edge_id(f[i], f[(i + 1) % 4]) for i in range(4)]
        cross = [i for i in range(4) if inside[f[i]] != inside[f[(i + 1) % 4]]]
        if len(cross) == 2:
            pairs = [(cross[0], cross[1])]
        elif len(cross) == 4:          # ambiguous face: cut off each inside corner on its own
            a = 0 if inside[f[0]] else 1
            pairs = [((a - 1) % 4, a), ((a + 1) % 4, (a + 2) % 4)]
        else:
            pairs = []
        for s, t in pairs:
            e0, e1 = es[s], es[t]
            shared = set(EDGES[e0]) & set(EDGES[e1])
            if shared:
                c = shared.pop()
                sgn = 1.0 if inside[c] else -1.0
            else:
                c = next(n for n in f if inside[n])
                sgn = 1.0
            d = mid(e1) - mid(e0)
            if sgn * (np.cross(d, corner(c) - mid(e0)) @ normal) < 0:
                e0, e1 = e1, e0
            segs.append((e0, e1))
    return segs


def case_triangles(mask: int):
    """Triangles (edge triples) of case `mask`, in table order."""
    nxt = {}
    for e0, e1 in face_segments(mask):
        assert e0 not in nxt, (mask, e0)
        nxt[e0] = e1
    seen, tris = set(), []
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, cur = [], start
        while cur not in seen:
            seen.add(cur)
            loop.append(cur)
            cur = nxt[cur]
        assert cur == start, (mask, loop)
        for r in range(len(loop)):      # rule 3: first rotation whose fan has no chord inside a cube face
            lp = loop[r:] + loop[:r]
            if not any(_on_one_face(lp[0], lp[i]) for i in range(2, len(lp) - 1)):
                break
        else:
            raise AssertionError(f"case {mask}: no fan apex for loop {loop}")
        # the segment direction of rule 2 runs the loops with the inside on their left: reverse them (rule 4)
        tris += [(lp[0], lp[i + 1], lp[i]) for i in range(1, len(lp) - 1)]
    return tris


def triangle_table():
    return [case_triangles(m) for m in range(256)]


def render() -> str:
    table = triangle_table()
    assert max(len(t) for t in table) <= MAX_TRIS
    counts = ", ".join(str(len(t)) for t in table)
    rows = []
    for m, t in enumerate(table):
        flat = [e for tri in t for e in tri] + [-1] * (3 * MAX_TRIS - 3 * len(t))
        rows.append("    {" + ", ".join(f"{e:2d}" for e in flat) + "},  // " + str(m))
    owner = ", ".join(str(a) for a, _ in EDGES)
    axis = ", ".join(str(a) for a in EDGE_AXIS)
    return f"""// GENERATED by 3dtopia-xl_b200/mc_table.py -- do not edit; rerun the generator instead.
// Marching-cubes case table.  Corner n = (n & 1, (n >> 1) & 1, (n >> 2) & 1) along array axes (0, 1, 2); bit n of a case is set
// iff corner n is inside (value < iso).  Edge e joins corners (kMcEdgeOwner[e], kMcEdgeOwner[e] | 1 << kMcEdgeAxis[e]).
// kMcTriEdges[case] lists kMcTriCount[case] triangles as edge triples, wound so that (v1 - v0) x (v2 - v0) points toward
// increasing value; unused slots are -1.
#pragma once
#include <stdint.h>

// included by one translation unit (marching_cubes.cu)
namespace tpx {{
constexpr int kMcMaxTris = {MAX_TRIS};
__constant__ int8_t kMcEdgeOwner[12] = {{{owner}}};
__constant__ int8_t kMcEdgeAxis[12] = {{{axis}}};
__constant__ int8_t kMcTriCount[256] = {{{counts}}};
__constant__ int8_t kMcTriEdges[256][3 * kMcMaxTris] = {{
{chr(10).join(rows)}
}};
}}  // namespace tpx
"""


if __name__ == "__main__":
    with open(HEADER, "w") as f:
        f.write(render())
    print("wrote", HEADER)
