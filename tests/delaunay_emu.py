"""rfb_delaunay_count / rfb_delaunay_write on the CPU kernel-logic emulator (tests/emu), driven as
radfoam_b200.delaunay.delaunay_adjacency drives them on the device, with numpy arrays for device memory."""
import ctypes
import os
import sys

import numpy as np

from radfoam_b200 import _lib as abi
from radfoam_b200 import foam
from radfoam_b200.delaunay import TriangulationFailedError, default_bounds

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402


def box_of(points, bounds=None):
    """The box the library uses: default_bounds of the bounding box, grown to contain ``bounds``."""
    p = np.asarray(points, np.float32)
    lo, hi = default_bounds(p.min(0), p.max(0))
    if bounds is not None:
        lo, hi = np.minimum(lo, np.float32(bounds[0])), np.maximum(hi, np.float32(bounds[1]))
    return lo.astype(np.float32), hi.astype(np.float32)


def build(points, bounds=None, order=None, pool=None):
    """(adjacency, offsets, totals) of the emulated build; ``order`` defaults to the Morton order."""
    lib = emu.load()
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    n = pts.shape[0]
    if n == 0:
        return np.zeros(0, np.uint32), np.zeros(1, np.uint32), np.zeros(8, np.uint64)
    if not np.isfinite(pts).all():
        raise TriangulationFailedError("a point has a non-finite coordinate")
    if order is None:
        order = np.argsort(foam.morton_codes(pts), kind="stable")
    order = np.ascontiguousarray(order, np.uint32)
    lo, hi = box_of(pts, bounds)
    box = abi.Box((ctypes.c_float * 3)(*map(float, lo)), (ctypes.c_float * 3)(*map(float, hi)))
    pool = 32 * n + 4096 if pool is None else pool
    while True:
        scratch = np.zeros((int(lib.rfb_delaunay_scratch_bytes(n, pool)) + 7) // 8, np.uint64)
        emu._check(lib.rfb_delaunay_count(emu._p(pts), n, emu._p(order), ctypes.byref(box), pool, emu._p(scratch),
                                          None))
        totals = scratch[:8].copy()
        if totals[5]:
            raise TriangulationFailedError("a point has a non-finite coordinate")
        if totals[4]:
            raise TriangulationFailedError("two points are equal")
        assert totals[6] == 0, "cells over the overflow kernel's capacity"
        if int(totals[2]) <= pool:
            break
        pool = int(totals[2])
    e = int(totals[1])
    adj, off, rows = np.full(e, 0xDEADBEEF, np.uint32), np.zeros(n + 1, np.uint32), np.zeros(e, np.uint32)
    emu._check(lib.rfb_delaunay_write(n, emu._p(order), pool, emu._p(scratch), emu._p(rows) if e else None,
                                      emu._p(adj) if e else None, emu._p(off), None))
    return adj, off, totals
