"""ctypes wrapper of oracle/_ref/libradfoam_ref_vis.so (oracle/ref_vis_abi.cu, built by oracle/ref_vis.mk): the
reference's OWN visualization kernel, Pipeline::trace_visualization, rendering into a CUDA surface that is then copied
out -- TEST INFRASTRUCTURE ONLY.  /root/reference is not needed at run time, only the prebuilt libraries."""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_uint32, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libradfoam_ref_vis.so")
_lib = None

VIS_MODES = {"rgb": 0, "depth": 1, "alpha": 2, "intersections": 3}
COLOR_MAPS = {"gray": 0, "viridis": 1, "inferno": 2, "turbo": 3}


def available() -> bool:
    return os.path.exists(LIB_PATH)


def load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(LIB_PATH)
        P = c_void_p
        lib.rfrefvis_last_error.restype = c_char_p
        lib.rfrefvis_trace_visualization.argtypes = [c_int, c_int, c_float, c_uint32, c_int, c_int, P, c_int,
                                                     c_float, c_float, P, P, c_uint32, P, P, P, P, P, P, P, P, P,
                                                     c_float, c_uint32, c_uint32, c_int, c_uint32, P]
        _lib = lib
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _deg(attr_dim):
    return {4: 0, 13: 1, 28: 2, 49: 3}[attr_dim]


def trace_visualization(points, attributes, adjacency, offsets, adjacent_diff, camera, start_index, cmap_data,
                        cmap_sizes, output_rgba, mode="rgb", color_map="turbo", bg_color=(1.0, 1.0, 1.0),
                        checker_bg=False, max_depth=10.0, depth_quantile=0.5, weight_threshold=0.001,
                        max_intersections=1024):
    """The reference's visualization kernel on a surface it renders into, copied out to ``output_rgba``
    (uint32 [height, width], CUDA, bottom-up rows as on the surface).  ``cmap_data`` / ``cmap_sizes``: CUDA tensors
    holding the table's device pointers (int64 [4]) and lengths (int32 [4])."""
    lib = load()
    is_half = attributes.dtype == torch.float16
    vec = {k: (ctypes.c_float * 3)(*[float(v) for v in camera[k]])
           for k in ("position", "forward", "right", "up")}
    bg = (ctypes.c_float * 3)(*[float(v) for v in bg_color])
    rc = lib.rfrefvis_trace_visualization(
        _deg(attributes.size(-1)), int(is_half), weight_threshold, max_intersections, VIS_MODES[mode],
        COLOR_MAPS[color_map], ctypes.cast(bg, c_void_p), int(bool(checker_bg)), float(max_depth),
        float(depth_quantile), _ptr(cmap_data), _ptr(cmap_sizes), points.size(0), _ptr(points), _ptr(attributes),
        _ptr(adjacency), _ptr(offsets), _ptr(adjacent_diff),
        ctypes.cast(vec["position"], c_void_p), ctypes.cast(vec["forward"], c_void_p),
        ctypes.cast(vec["right"], c_void_p), ctypes.cast(vec["up"], c_void_p), float(camera["fov"]),
        int(camera["width"]), int(camera["height"]), 0 if camera["model"] == "pinhole" else 1, int(start_index),
        _ptr(output_rgba))
    if rc:
        raise RuntimeError(lib.rfrefvis_last_error().decode())
