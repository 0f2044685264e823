"""The Delaunay adjacency of a point set, built on the GPU (rfb_delaunay_count / rfb_delaunay_write).

``delaunay_adjacency(points)`` gives the CSR graph the tracer walks, in the caller's point order.  ``Triangulation``
mirrors the part of ``radfoam.Triangulation`` (src/delaunay/delaunay.cu, ``rebuild``) that radfoam_model/scene.py
uses: ``permutation()``, ``rebuild(points, incremental)``, ``point_adjacency()`` and ``point_adjacency_offsets()``.
The graph is defined through Voronoi faces inside a box (include/radfoam_b200.h), so it is built cell by cell by
clipping, not by growing tetrahedra; the tet outputs are not provided.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib
from .pipeline import _ptr


class TriangulationFailedError(RuntimeError):
    """The points cannot be triangulated: two of them are equal, or one has a non-finite coordinate
    (``radfoam.TriangulationFailedError``; scene.py perturbs the points and retries on it)."""


_MASKS = ((32, 0x1F00000000FFFF), (16, 0x1F0000FF0000FF), (8, 0x100F00F00F00F00F), (4, 0x10C30C30C30C30C3),
          (2, 0x1249249249249249))


def morton_order(points: torch.Tensor) -> torch.Tensor:
    """A spatially coherent permutation of the points (``int64 [N]``): ascending 63-bit Morton codes inside the
    points' bounding box, ties in index order (``foam.morton_codes`` on the device)."""
    p = points.detach().to(torch.float64)
    if p.size(0) == 0:
        return torch.zeros((0,), dtype=torch.int64, device=p.device)
    lo, hi = p.amin(0), p.amax(0)
    q = ((p - lo) / torch.clamp(hi - lo, min=1e-30) * ((1 << 21) - 1)).to(torch.int64)
    code = torch.zeros(p.size(0), dtype=torch.int64, device=p.device)
    for c in range(3):
        v = q[:, c] & 0x1FFFFF
        for shift, mask in _MASKS:
            v = (v | (v << shift)) & mask
        code |= v << c
    return torch.argsort(code, stable=True)


def default_bounds(lo, hi):
    """The box used when none is given: a cube centred on the bounding box ``(lo, hi)``, with side 3 x its largest
    extent, rounded outward to float32."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    centre, half = 0.5 * (lo + hi), 1.5 * float((hi - lo).max())
    return (np.nextafter(np.float32(centre - half), np.float32(-np.inf)).astype(np.float32),
            np.nextafter(np.float32(centre + half), np.float32(np.inf)).astype(np.float32))


def delaunay_adjacency(points, bounds=None):
    """The Delaunay graph of ``points`` (float32 ``[N, 3]`` on a CUDA device) as ``(point_adjacency uint32[E],
    point_adjacency_offsets uint32[N+1])``: rows strictly ascending, no self entries, symmetric, in the caller's
    point order -- the layout ``foam.delaunay_adjacency`` returns.

    {i, j} is an edge iff the Voronoi face between p_i and p_j, inside the box B, has positive area.  For points in
    general position that is the Delaunay graph minus the edges whose Voronoi face lies wholly outside B; faces of
    zero area (co-spherical ties such as lattice diagonals) may be present or absent, from both ends alike.  B is
    ``default_bounds`` of the points' bounding box (a cube 3x its largest extent), grown to contain
    ``bounds = (lo[3], hi[3])`` when given -- pass a larger box to keep hull edges whose faces lie far out, e.g.
    for cameras far outside the scene.  Deterministic: two builds give identical bytes.

    Raises ``TriangulationFailedError`` on two equal points or a non-finite coordinate.  The call reads the bounding
    box and the build's totals back to the host, so it synchronises with the current stream."""
    return _build(points, bounds, None)


def _build(points, bounds, order):
    """The Delaunay adjacency of ``points`` in the locality order ``order`` (int64 [N], a permutation), or the Morton
    order when it is None."""
    if not isinstance(points, torch.Tensor) or points.device.type != "cuda":
        raise RuntimeError("points must be on CUDA device")
    if points.dtype != torch.float32:
        raise RuntimeError("points must have float32 dtype")
    if points.dim() != 2 or points.size(-1) != 3:
        raise RuntimeError("points must have shape [N, 3]")
    pts, dev, n = points.detach().contiguous(), points.device, points.size(0)
    if n >= 1 << 31:
        raise RuntimeError("delaunay_adjacency: at most 2^31 - 1 points")
    if n == 0:
        return (torch.zeros((0,), dtype=torch.uint32, device=dev), torch.zeros((1,), dtype=torch.uint32, device=dev))
    lo, hi = (np.asarray(x, np.float64) for x in torch.stack([pts.amin(0), pts.amax(0)]).cpu().tolist())
    if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
        raise TriangulationFailedError("a point has a non-finite coordinate")
    box_lo, box_hi = default_bounds(lo, hi)
    if bounds is not None:
        b = [torch.as_tensor(x, dtype=torch.float32).detach().cpu().reshape(-1).numpy() for x in bounds]
        if len(b) != 2 or b[0].shape != (3,) or b[1].shape != (3,) or not all(np.isfinite(x).all() for x in b):
            raise RuntimeError("bounds must be (lo[3], hi[3]), finite")
        box_lo, box_hi = np.minimum(box_lo, b[0]), np.maximum(box_hi, b[1])
    box = _lib.Box()
    box.lo[:], box.hi[:] = box_lo.tolist(), box_hi.tolist()
    order = (morton_order(pts) if order is None else order).to(torch.int32).view(torch.uint32)
    lib = _lib.load()
    pool = min(32 * n + 4096, 0xFFFFFFFF)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        while True:
            nbytes = int(lib.rfb_delaunay_scratch_bytes(n, pool))
            scratch = torch.empty((nbytes + 7) // 8, dtype=torch.int64, device=dev)
            _lib.check(lib.rfb_delaunay_count(_ptr(pts), n, _ptr(order), ctypes.byref(box), pool, _ptr(scratch),
                                              stream))
            _, edges, need, _, dup, nonfinite, over, bad_order = scratch[:8].cpu().tolist()
            if bad_order:
                raise RuntimeError("delaunay_adjacency: the locality order is not a permutation")
            if nonfinite:
                raise TriangulationFailedError("a point has a non-finite coordinate")
            if dup:
                raise TriangulationFailedError("two points are equal")
            if over:
                raise RuntimeError(f"delaunay_adjacency: {over} cells need more faces or vertices than the "
                                   "overflow kernel holds")
            if need <= pool:
                break
            pool = min(int(need), 0xFFFFFFFF)  # the face pool was too small: build again with the size it needs
        adjacency = torch.empty((edges,), dtype=torch.uint32, device=dev)
        offsets = torch.empty((n + 1,), dtype=torch.uint32, device=dev)
        rows = torch.empty((edges,), dtype=torch.uint32, device=dev)
        _lib.check(lib.rfb_delaunay_write(n, _ptr(order), pool, _ptr(scratch), _ptr(rows) if edges else None,
                                          _ptr(adjacency) if edges else None, _ptr(offsets), stream))
    return adjacency, offsets


class Triangulation:
    """``radfoam.Triangulation`` for the graph the tracer walks (src/delaunay/delaunay.cu ``rebuild``).

    ``Triangulation(points)`` builds at once.  ``rebuild(points, incremental=False)`` sorts the points into a
    spatially coherent order, returns True, and the graph then indexes ``points[permutation()]``.
    ``rebuild(points, incremental=True)`` with the same number of points keeps the given order and returns False
    (``permutation()`` is left as it was); with another number it behaves like the non-incremental rebuild.
    ``tets``, ``tet_adjacency`` and ``vert_to_tet`` are not provided: the graph is built from Voronoi cells, not
    tetrahedra, and neither scene.py nor the tracer reads them."""

    def __init__(self, points):
        self._num_points = -1
        self.rebuild(points, incremental=False)

    def rebuild(self, points, incremental=False) -> bool:
        if not isinstance(points, torch.Tensor) or points.size(-1) != 3:
            raise RuntimeError("points must have 3 as the last dimension")
        pts = points.detach().reshape(-1, 3)
        if incremental and pts.size(0) == self._num_points:
            self._adjacency, self._offsets = delaunay_adjacency(pts)
            return False
        perm = morton_order(pts)
        # the sorted points are their own locality order
        adjacency, offsets = _build(pts[perm], None, torch.arange(pts.size(0), device=pts.device))
        self._permutation = perm.to(torch.int32).view(torch.uint32)
        self._adjacency, self._offsets, self._num_points = adjacency, offsets, pts.size(0)
        return True

    def permutation(self) -> torch.Tensor:
        return self._permutation

    def point_adjacency(self) -> torch.Tensor:
        return self._adjacency

    def point_adjacency_offsets(self) -> torch.Tensor:
        return self._offsets

    def _no_tets(self, *args, **kwargs):
        raise RuntimeError("Triangulation builds the point adjacency only: tets, tet_adjacency and vert_to_tet are "
                           "not provided")

    tets = tet_adjacency = vert_to_tet = _no_tets
