"""Float64 judge of the Delaunay adjacency (radfoam_b200.delaunay_adjacency / rfb_delaunay_count + _write), from the
definition in include/radfoam_b200.h and not from the kernels:

  {i, j} is an edge iff F_ij = { x in B : |x - p_i| = |x - p_j| <= |x - p_k| for all k } has positive area.

face_area(i, j) clips the bisector of (i, j) against the box and the bisectors of a SUPERSET of i's Voronoi
neighbours, with surface_model.face (the polygon of one CSR entry): Qhull's row of i for inputs in general position
(the Voronoi cell is the intersection over its Delaunay neighbours, whichever diagonals Qhull chose at ties), every
point for small sets (coplanar and collinear ones included, where Qhull fails).  A built graph may differ from Qhull's
only on edges whose face area is at most TAU |p_i - p_j|^2: faces outside B, and zero-area faces at ties.
"""
from __future__ import annotations

import numpy as np

import surface_model as sm

TAU = 1e-9


def edges(adjacency, offsets):
    """The set of directed (i, j) entries of a CSR."""
    rows = sm.rows_of(offsets)
    return set(zip(rows.tolist(), np.asarray(adjacency, np.int64).tolist()))


def codes(adjacency, offsets):
    """The directed entries of a CSR as sorted int64 codes i * 2^32 + j."""
    return np.sort((sm.rows_of(offsets).astype(np.int64) << 32) | np.asarray(adjacency, np.int64))


def polygon_area(v):
    if v.shape[0] < 3:
        return 0.0
    d = v[1:] - v[0]
    return 0.5 * float(np.linalg.norm(np.cross(d[:-1], d[1:]).sum(0)))


def face_area(points, i, j, superset, lo, hi):
    """Area of F_ij inside the box (lo, hi), with the cell of i cut by the bisectors of ``superset``."""
    ids = [i, j] + sorted(set(int(k) for k in superset) - {i, j})
    sub = np.asarray(points)[ids]
    m = len(ids) - 1
    v, _ = sm.face(sub, np.arange(1, m + 1, dtype=np.uint32), np.array([0, m], np.uint32), lo, hi, 0, 0)
    return polygon_area(v)


def judge(points, adjacency, offsets, ref_adjacency, ref_offsets, lo, hi, all_points=False):
    """Every entry where the graph differs from the reference graph (Qhull's), as (i, j, area / |p_i - p_j|^2, in
    the reference): the area from i's end, against Qhull's row of i plus j, or against every point."""
    ref = codes(ref_adjacency, ref_offsets)
    diff = np.setxor1d(codes(adjacency, offsets), ref, assume_unique=True)
    in_ref = np.isin(diff, ref, assume_unique=True)
    p = np.asarray(points, np.float64)
    n = p.shape[0]
    out = []
    for code, r in zip(diff.tolist(), in_ref.tolist()):
        i, j = code >> 32, code & 0xFFFFFFFF
        sup = range(n) if all_points else ref_adjacency[ref_offsets[i]:ref_offsets[i + 1]]
        a = face_area(points, i, j, sup, lo, hi)
        out.append((i, j, a / float(((p[i] - p[j]) ** 2).sum()), r))
    return out


def brute_graph(points, lo, hi):
    """The graph by definition, every pair against every point (small sets only): (adjacency, offsets)."""
    p = np.asarray(points, np.float64)
    n = p.shape[0]
    rows = []
    for i in range(n):
        rows.append([j for j in range(n) if j != i and
                     face_area(points, i, j, range(n), lo, hi) > TAU * float(((p[i] - p[j]) ** 2).sum())])
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum([len(r) for r in rows])
    adj = np.array([j for r in rows for j in r], np.uint32)
    return adj, off
