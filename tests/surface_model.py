"""Float64 model of surface extraction (Pipeline.extract_surface / rfb_surface_count + rfb_surface_write), written from
the definition in include/radfoam_b200.h and not from the kernels:

  for row i and every listed neighbour k with p_k != p_i:  H_k = { x : (p_k - p_i).x <= (p_k - p_i).(p_i + p_k)/2 },
  C_i = box ∩ (∩_k H_k),  F_e = C_i ∩ plane_e  for the CSR entry e = (i, j),
  emitted iff inside[i] and not inside[j], p_j != p_i and F_e has at least 3 vertices; CSR order; vertices
  counter-clockwise seen from j.

The kernels clip a polygon plane by plane; this model instead works in 2-D coordinates of plane_e: every other
constraint is a half-plane there, the polygon's vertices are the pairwise line intersections that satisfy all
constraints, and the cycle is their angular order about the centroid.  It also reports near-degenerate polygons:
a vertex where a third constraint passes within a tolerance (lattice ties), or two vertices within it -- there the
kernels may legitimately emit a different vertex list for the same point set.
"""
from __future__ import annotations

import dataclasses

import numpy as np

U32 = 2.0 ** -24


@dataclasses.dataclass
class Polygon:
    entry: int
    cells: tuple
    vertices: np.ndarray   # [m, 3] float64, counter-clockwise seen from j
    degenerate: bool


def rows_of(offsets: np.ndarray) -> np.ndarray:
    off = offsets.astype(np.int64)
    return np.repeat(np.arange(off.size - 1), np.diff(off))


def bounding_box(points: np.ndarray):
    p = points.astype(np.float32)
    return p.min(0).astype(np.float64), p.max(0).astype(np.float64)


def face(points, adjacency, offsets, lo, hi, i, e, tol=1e-10):
    """(vertices [m, 3] float64 CCW seen from j, degenerate flag) of F_e for entry e of row i; m = 0 when empty.
    ``tol`` is relative to the box diagonal."""
    p = points.astype(np.float64)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    scale = float(np.linalg.norm(hi - lo)) or 1.0
    j = int(adjacency[e])
    pi, pj = p[i], p[j]
    n = pj - pi
    m = 0.5 * (pi + pj)
    nn = n / np.linalg.norm(n)
    a = np.eye(3)[np.argmin(np.abs(nn))]
    u = np.cross(nn, a)
    u /= np.linalg.norm(u)
    v = np.cross(nn, u)  # u x v = nn
    # constraints A x <= b in 3-D: the box, then the neighbour planes (not p_i's own point, not plane_e itself)
    A = [np.eye(3)[c] for c in range(3)] + [-np.eye(3)[c] for c in range(3)]
    b = list(hi) + list(-lo)
    f32 = points.astype(np.float32)
    for k in range(int(offsets[i]), int(offsets[i + 1])):
        q = int(adjacency[k])
        if k == e or np.array_equal(f32[q], f32[i]) or np.array_equal(f32[q], f32[j]):
            continue
        nk = p[q] - pi
        A.append(nk)
        b.append(float(nk @ (0.5 * (pi + p[q]))))
    A, b = np.array(A), np.array(b)
    # in plane coordinates x = m + s u + t v:  (A u) s + (A v) t <= b - A m; normalise each line
    a2 = np.stack([A @ u, A @ v], 1)
    r = b - A @ m
    norm = np.linalg.norm(a2, axis=1)
    keep = norm > 0
    parallel_out = (~keep) & (r < 0)
    if parallel_out.any():
        return np.zeros((0, 3)), False
    a2, r = a2[keep] / norm[keep, None], r[keep] / norm[keep]
    L = a2.shape[0]
    ii, jj = np.triu_indices(L, 1)
    det = a2[ii, 0] * a2[jj, 1] - a2[ii, 1] * a2[jj, 0]
    ok = np.abs(det) > 1e-14
    ii, jj, det = ii[ok], jj[ok], det[ok]
    s = (r[ii] * a2[jj, 1] - r[jj] * a2[ii, 1]) / det
    t = (a2[ii, 0] * r[jj] - a2[jj, 0] * r[ii]) / det
    y = np.stack([s, t], 1)
    resid = y @ a2.T - r[None, :]                        # <= 0 inside
    feasible = (resid <= tol * scale).all(1)
    y, resid = y[feasible], resid[feasible]
    if y.shape[0] == 0:
        return np.zeros((0, 3)), False
    # merge coincident candidates (three or more lines through one vertex)
    order = np.lexsort((y[:, 1], y[:, 0]))
    y, resid = y[order], resid[order]
    uniq = []
    for k in range(y.shape[0]):
        if not any(np.linalg.norm(y[k] - y[w]) <= tol * scale for w in uniq):
            uniq.append(k)
    y, resid = y[uniq], resid[uniq]
    tight = (np.abs(resid) <= 1e3 * tol * scale).sum(1)
    degenerate = bool((tight > 2).any())
    if y.shape[0] >= 2:
        d = np.linalg.norm(y[:, None] - y[None], axis=-1) + np.eye(y.shape[0]) * 1e300
        degenerate |= bool(d.min() <= 1e3 * tol * scale)
    c = y.mean(0)
    ang = np.arctan2(y[:, 1] - c[1], y[:, 0] - c[0])
    y = y[np.argsort(ang, kind="stable")]
    if y.shape[0] < 3:
        return np.zeros((0, 3)), degenerate
    return m[None] + y[:, :1] * u[None] + y[:, 1:] * v[None], degenerate


def surface(points, adjacency, offsets, inside, bounds=None, entries=None, tol=1e-10):
    """The model's polygons, in CSR order (restricted to ``entries`` when given).  The box is float32, as the
    library takes it."""
    lo, hi = bounding_box(points) if bounds is None else (np.asarray(bounds[0], np.float32).astype(np.float64),
                                                          np.asarray(bounds[1], np.float32).astype(np.float64))
    rows = rows_of(offsets)
    f32 = points.astype(np.float32)
    inside = np.asarray(inside, bool)
    e_all = np.arange(adjacency.size) if entries is None else np.sort(np.asarray(entries, np.int64))
    out = []
    for e in e_all:
        i, j = int(rows[e]), int(adjacency[e])
        if not inside[i] or inside[j] or np.array_equal(f32[i], f32[j]):
            continue
        verts, deg = face(points, adjacency, offsets, lo, hi, i, int(e), tol)
        if verts.shape[0] >= 3:
            out.append(Polygon(int(e), (i, j), verts, deg))
    return out


def area_vector(v: np.ndarray) -> np.ndarray:
    """0.5 sum v_k x v_(k+1): the polygon's area times its right-hand unit normal."""
    v = np.asarray(v, np.float64)
    c = v.mean(0)
    w = v - c
    return 0.5 * np.cross(w, np.roll(w, -1, axis=0)).sum(0)


def enclosed_volume(polys) -> float:
    """Divergence theorem over outward-oriented polygons: (1/3) sum v_0 . area_vector."""
    return float(sum(np.asarray(v, np.float64)[0] @ area_vector(v) for v in polys) / 3.0)


def same_cycle(a: np.ndarray, b: np.ndarray, tol: float) -> bool:
    """``a`` and ``b`` list the same vertices in the same cyclic order (any starting vertex, same orientation)."""
    if a.shape != b.shape:
        return False
    k = int(np.argmin(np.linalg.norm(b - a[0], axis=1)))
    return bool(np.all(np.abs(np.roll(b, -k, axis=0) - a) <= tol))


def hausdorff(a: np.ndarray, b: np.ndarray) -> float:
    d = np.linalg.norm(np.asarray(a, np.float64)[:, None] - np.asarray(b, np.float64)[None], axis=-1)
    return float(max(d.min(1).max(), d.min(0).max()))


def vertex_bound(verts: np.ndarray, scale: float) -> np.ndarray:
    """Per-coordinate bound of a kernel vertex against the model: one fp32 rounding of the value, plus the fp64
    conditioning term of two plane solves (generous: 1e-9 of the scene scale)."""
    return U32 * np.abs(verts) + 1e-9 * scale
