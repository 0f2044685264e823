"""ctypes binding of tests/vis_oracle.c, the CPU restatement of the reference's visualization kernel -- TEST
INFRASTRUCTURE ONLY.  The library is compiled on first use (gcc, the flags of oracle/Makefile) next to this file,
like the CPU kernel-logic emulator under tests/emu; the product never loads it."""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import c_float, c_int, c_uint32, c_void_p

import numpy as np

from oracle.oracle import _attr_dtype, _c, _p, sh_degree_of

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "vis_oracle.c")
BASE = os.path.join(os.path.dirname(HERE), "oracle", "radfoam_oracle.c")
LIB = os.path.join(HERE, "libvis_oracle.so")
_lib = None


def build() -> str:
    if os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in (SRC, BASE)):
        return LIB
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    tmp = f"{LIB}.{os.getpid()}.tmp"  # atomic replace: concurrent test processes may build at the same time
    subprocess.check_call([cc, "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-mfma",
                           "-mf16c", "-fno-fast-math", "-o", tmp, SRC, "-lm"])
    os.replace(tmp, LIB)
    return LIB


def load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build())
        P = c_void_p
        lib.rfo_trace_visualization.argtypes = [c_int, c_int, c_float, c_uint32, c_int, c_int, P, c_int, c_float,
                                                c_float, P, P, P, P, P, P, P, P, P, P, P, c_float, c_uint32,
                                                c_uint32, c_int, c_uint32, P, c_int]
        lib.rfo_trace_visualization.restype = c_int
        _lib = lib
    return _lib


VIS_MODES = {"rgb": 0, "depth": 1, "alpha": 2, "intersections": 3}
COLOR_MAPS = {"gray": 0, "viridis": 1, "inferno": 2, "turbo": 3}


def trace_visualization(points, attributes, adjacency, offsets, adjacent_diff, camera, start_index, tables=None,
                        mode="rgb", color_map="turbo", bg_color=(1.0, 1.0, 1.0), checker_bg=False, max_depth=10.0,
                        depth_quantile=0.5, weight_threshold=0.001, max_intersections=1024, num_threads=1):
    """The visualization kernel restated on the CPU -> uint32 [height, width] (bottom-up rows, as on the reference's
    surface).  ``tables``: four float32 [L, 3] arrays indexed by colour map (needed by depth / intersections)."""
    lib = load()
    adt, is_half = _attr_dtype(attributes)
    points = _c(points, np.float32)
    attributes = _c(attributes, adt)
    adjacency = _c(adjacency, np.uint32)
    offsets = _c(offsets, np.uint32)
    diff = _c(adjacent_diff, np.float16)
    w, h = int(camera["width"]), int(camera["height"])
    out = np.zeros((h, w), dtype=np.uint32)
    vec = {k: _c(np.asarray(camera[k]), np.float32) for k in ("position", "forward", "right", "up")}
    bg = _c(np.asarray(bg_color), np.float32)
    ptrs = sizes = arrs = None
    if tables is not None:
        arrs = [_c(t, np.float32) for t in tables]
        ptrs = np.array([a.ctypes.data for a in arrs], dtype=np.uint64)
        sizes = np.array([a.shape[0] for a in arrs], dtype=np.int32)
    rc = lib.rfo_trace_visualization(sh_degree_of(attributes.shape[-1]), is_half, weight_threshold,
                                     max_intersections, VIS_MODES[mode], COLOR_MAPS[color_map], _p(bg),
                                     int(bool(checker_bg)), float(max_depth), float(depth_quantile), _p(ptrs),
                                     _p(sizes), _p(points), _p(attributes), _p(adjacency), _p(offsets), _p(diff),
                                     _p(vec["position"]), _p(vec["forward"]), _p(vec["right"]), _p(vec["up"]),
                                     float(camera["fov"]), w, h, 0 if camera["model"] == "pinhole" else 1,
                                     int(start_index), _p(out), num_threads)
    if rc:
        raise RuntimeError(f"oracle trace_visualization failed ({rc})")
    return out
