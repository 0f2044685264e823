"""Stale scenes: a foam whose points have moved since its adjacency was built.

Training moves the points every optimizer step but rebuilds the Delaunay adjacency only every
``triangulation_update_period`` steps (a period that grows by 2 after each rebuild, up to 100), so most steps trace
points that have drifted away from the graph they are walked on.  On such a foam the walk skips cells with
t1 <= t0, re-enters a composited cell through a plane other than the previous composited cell's exit plane, and can
stop inside the scene at a cell without any face in front of the ray -- branches a fresh triangulation hardly runs.

``stale`` moves the points of a foam and keeps its adjacency, offsets and attributes; ``stale_case`` does the same to
a ``common.Case`` and recomputes the start cells on the moved points, as the start-point lookup of a training step
does.  ``stats`` reads, from a ``model64.trace`` result, how stale a case is, and ``assert_floors`` holds a case to
minimum staleness so that it cannot quietly become a fresh one.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.spatial import ConvexHull, cKDTree

import common
from radfoam_b200 import foam

KINDS = ("noise", "field")


def spacing(points: np.ndarray) -> np.ndarray:
    """Distance from every point to its nearest other point (float64)."""
    p = points.astype(np.float64)
    d, _ = cKDTree(p).query(p, k=2, workers=-1)
    return d[:, 1]


def displacement(points: np.ndarray, frac: float, kind: str, seed: int) -> np.ndarray:
    """float64 [N, 3] moves.  ``noise``: per point N(0, (frac * nearest-neighbour distance)^2) in each coordinate.
    ``field``: a smooth field (a sum of twelve random plane waves) of amplitude frac * the median spacing, nearly
    the same at neighbouring points, i.e. coherent drift."""
    rng = np.random.default_rng(seed)
    p = points.astype(np.float64)
    nn = spacing(points)
    if kind == "noise":
        return rng.normal(size=p.shape) * (frac * nn)[:, None]
    if kind == "field":
        h = float(np.median(nn))
        # wavelengths of about four median spacings: smooth from one point to the next, yet every cell's
        # neighbourhood is sheared, which is what invalidates an adjacency
        waves = rng.normal(size=(12, 3))
        waves *= (2 * np.pi / (4 * h)) / np.linalg.norm(waves, axis=1, keepdims=True)
        phase = rng.uniform(0, 2 * np.pi, size=12)
        direction = rng.normal(size=(12, 3))
        direction /= np.linalg.norm(direction, axis=1, keepdims=True)
        field = np.sin(p @ waves.T + phase) @ direction / np.sqrt(12 / 2)
        return field * frac * h
    raise ValueError(kind)


def stale(f: foam.Foam, frac: float, kind: str, seed: int) -> foam.Foam:
    """``f`` with its points moved by ``displacement`` and the unchanged adjacency, offsets and attributes."""
    moved = (f.points.astype(np.float64) + displacement(f.points, frac, kind, seed)).astype(np.float32)
    return foam.Foam(moved, f.attributes, f.adjacency, f.offsets, f.sh_degree)


def start_cells(points: np.ndarray, rays: np.ndarray) -> np.ndarray:
    """The nearest point of every ray's origin (float64 distances; the test cases keep clear of fp32 ties)."""
    o = rays[..., :3].reshape(-1, 3)
    uniq, inv = np.unique(o, axis=0, return_inverse=True)
    cells = np.array([foam.nearest_point(points, q) for q in uniq], dtype=np.uint32)
    return cells[inv.reshape(-1)].reshape(rays.shape[:-1])


def stale_case(case: common.Case, frac: float, kind: str, seed: int) -> common.Case:
    """The case's rays, quantiles and upstream gradients on the moved foam, with start cells recomputed."""
    f = stale(case.foam, frac, kind, seed)
    out = common.Case(f, case.rays, start_cells(f.points, case.rays), case.quantiles)
    out.grad_rgba, out.grad_depth = case.grad_rgba, case.grad_depth
    return out


@dataclasses.dataclass
class Stats:
    rays: int
    skipped: float      # share of rays that skip at least one cell (t1 <= t0)
    reentered: float    # share of composited cells not entered through the previous composited cell's exit plane
    stranded: int       # rays that stop for want of an exit face at a cell that is not on the hull

    def __str__(self):
        return (f"{self.rays} rays: {100 * self.skipped:.1f}% skip a cell, {100 * self.reentered:.2f}% of "
                f"composited cells re-entered, {self.stranded} stranded inside the hull")


def stats(m: dict, points: np.ndarray, rays=None) -> Stats:
    """Staleness of a traced case from ``model64.trace``'s walk statistics; ``rays`` (bool mask) restricts it."""
    sel = np.ones(m["skipped"].shape, dtype=bool) if rays is None else rays.reshape(m["skipped"].shape)
    hull = np.zeros(points.shape[0], dtype=bool)
    hull[ConvexHull(points.astype(np.float64)).vertices] = True
    stuck = m["stuck_cell"][sel]
    stuck = stuck[stuck >= 0]
    composited = int(m["composited"][sel].sum())
    return Stats(rays=int(sel.sum()), skipped=float(m["skipped"][sel].mean()),
                 reentered=float(m["reentered"][sel].sum() / max(composited, 1)),
                 stranded=int((~hull[stuck]).sum()))


def assert_floors(s: Stats, skipped: float, reentered: float, stranded: int = 0) -> None:
    assert s.skipped >= skipped, f"only {100 * s.skipped:.1f}% of the rays skip a cell (floor {100 * skipped:.1f}%)"
    assert s.reentered >= reentered, \
        f"only {100 * s.reentered:.2f}% of composited cells re-entered (floor {100 * reentered:.2f}%)"
    assert s.stranded >= stranded, f"only {s.stranded} rays stranded inside the hull (floor {stranded})"
