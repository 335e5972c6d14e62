"""Oracle marching cubes (TEST INFRASTRUCTURE — see oracle/__init__.py).

Vectorised numpy float64 restatement of the contract of csrc/marching_cubes.cu, the GPU stand-in for the
``mcubes.marching_cubes(grid, 0.0)`` call of extract_texmesh (/root/reference/inference.py:119):
  * a corner is inside iff value < iso (strict);
  * one vertex per lattice edge whose ends classify differently; the edge p -> p + e_a is owned by p; ids ordered by the
    C-order linear index of p, then by axis a; position p + t e_a with t = (iso - f(p)) / (f(p + e_a) - f(p));
  * triangles ordered by the C-order linear index of the cell, then by table order within the cell's case; int64 faces.
The case table is read from the committed generated header (3dtopia-xl_b200/csrc/mc_tables.cuh); the property tests in
tests/test_mesh_host.py check it without using its own logic.
"""
from __future__ import annotations

import os

import numpy as np

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3dtopia-xl_b200", "csrc", "mc_tables.cuh")
CORNERS = np.array([(n & 1, (n >> 1) & 1, (n >> 2) & 1) for n in range(8)], dtype=np.int64)


def _array(text: str, name: str):
    body = text.split(name, 1)[1].split("=", 1)[1]
    body = body[:body.index("};")]
    body = "\n".join(line.split("//")[0] for line in body.split("\n"))
    return [int(v) for v in body.replace("{", " ").replace("}", " ").replace(",", " ").split()]


def load_table(path: str = HEADER):
    """(tri_edges int64 [256, MAX, 3] padded with -1, tri_count [256], edge_owner [12], edge_axis [12]) from the header."""
    text = open(path).read()
    count = np.array(_array(text, "kMcTriCount[256]"), dtype=np.int64)
    edges = np.array(_array(text, "kMcTriEdges[256]"), dtype=np.int64).reshape(256, -1, 3)
    owner = np.array(_array(text, "kMcEdgeOwner[12]"), dtype=np.int64)
    axis = np.array(_array(text, "kMcEdgeAxis[12]"), dtype=np.int64)
    assert count.shape == (256,) and owner.shape == (12,) and axis.shape == (12,)
    return edges, count, owner, axis


_TABLE = None


def cube_cases(vol: np.ndarray, iso: float = 0.0) -> np.ndarray:
    """Case byte of every cell [X-1, Y-1, Z-1]: bit n set iff corner n is inside."""
    inside = np.asarray(vol) < iso
    X, Y, Z = inside.shape
    c = np.zeros((X - 1, Y - 1, Z - 1), dtype=np.int64)
    for n, (a, b, d) in enumerate(CORNERS):
        c |= inside[a:X - 1 + a, b:Y - 1 + b, d:Z - 1 + d].astype(np.int64) << n
    return c


def marching_cubes(vol, iso: float = 0.0):
    """vol [X, Y, Z] -> (verts float64 [V, 3] in index units, faces int64 [F, 3])."""
    global _TABLE
    if _TABLE is None:
        _TABLE = load_table()
    tri_edges, tri_count, edge_owner, edge_axis = _TABLE
    f = np.ascontiguousarray(vol, dtype=np.float64)
    if f.ndim != 3:
        raise ValueError("volume must be 3-D")
    X, Y, Z = f.shape
    if min(X, Y, Z) < 2:
        return np.zeros((0, 3)), np.zeros((0, 3), dtype=np.int64)
    inside = f < iso
    strides = np.array([Y * Z, Z, 1], dtype=np.int64)
    cross = np.zeros((X, Y, Z, 3), dtype=bool)
    cross[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cross[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cross[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    slots = np.flatnonzero(cross.reshape(-1))            # (point * 3 + axis), ascending = vertex id order
    p, a = slots // 3, slots % 3
    f0, f1 = f.reshape(-1)[p], f.reshape(-1)[p + strides[a]]
    t = (iso - f0) / (f1 - f0)
    verts = np.stack(np.unravel_index(p, (X, Y, Z)), 1).astype(np.float64)
    verts[np.arange(len(p)), a] += t

    cases = cube_cases(f, iso).reshape(-1)
    cells = np.flatnonzero(tri_count[cases] > 0)
    cc = cases[cells]
    ci, cj, ck = np.unravel_index(cells, (X - 1, Y - 1, Z - 1))
    base = (ci * Y + cj) * Z + ck                       # the cell's lowest corner as a lattice point
    e = tri_edges[cc]                                   # [n, MAX, 3]
    valid = np.arange(tri_edges.shape[1])[None, :] < tri_count[cc][:, None]
    e = np.where(e < 0, 0, e)
    off = CORNERS[edge_owner[e]] @ strides               # owner corner offset, [n, MAX, 3]
    slot = (base[:, None, None] + off) * 3 + edge_axis[e]
    ids = np.searchsorted(slots, slot)
    faces = ids[valid].reshape(-1, 3).astype(np.int64)
    return verts, faces
