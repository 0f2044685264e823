"""ctypes binding of the C ABI declared in include/radfoam_b200.h.

The library is built in-tree by ``__graft_entry__.build()`` (plain nvcc, sm_90a) as
radfoam_b200/libradfoam_b200.so.  There is no fallback: if it is missing or fails to
load, every tracing call raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_uint32, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_NAME = "libradfoam_b200.so"


def library_path() -> str:
    return os.path.join(_HERE, _LIB_NAME)


class TraceSettings(ctypes.Structure):  # rfb_trace_settings
    _fields_ = [("weight_threshold", c_float), ("max_intersections", c_uint32)]


class Camera(ctypes.Structure):  # rfb_camera
    _fields_ = [("position", c_float * 3), ("forward", c_float * 3), ("right", c_float * 3),
                ("up", c_float * 3), ("fov", c_float), ("width", c_uint32), ("height", c_uint32),
                ("model", c_int32)]


class SceneParams(ctypes.Structure):  # rfb_scene_params
    _fields_ = [("att_dc", c_void_p), ("att_sh", c_void_p), ("density", c_void_p), ("activation_scale", c_float)]


class Multicast(ctypes.Structure):  # rfb_multicast
    _fields_ = [("acc", c_void_p), ("attribute_grad", c_void_p), ("points_grad", c_void_p)]


class Box(ctypes.Structure):  # rfb_box
    _fields_ = [("lo", c_float * 3), ("hi", c_float * 3)]


class LaunchOpts(ctypes.Structure):  # rfb_launch_opts
    _fields_ = [("scene_version", c_uint64), ("image_width", c_uint32), ("flags", c_uint32)]


class VisualizationSettings(ctypes.Structure):  # rfb_visualization_settings
    _fields_ = [("mode", c_int32), ("color_map", c_int32), ("bg_color", c_float * 3), ("checker_bg", c_uint32),
                ("max_depth", c_float), ("depth_quantile", c_float)]


class CMapTable(ctypes.Structure):  # rfb_cmap_table (two device pointers)
    _fields_ = [("data", c_void_p), ("sizes", c_void_p)]


VIS_MODES = {"rgb": 0, "depth": 1, "alpha": 2, "intersections": 3}  # RFB_VIS_*
COLOR_MAPS = {"gray": 0, "viridis": 1, "inferno": 2, "turbo": 3}  # RFB_CMAP_*

FLAG_SCRUB_NONFINITE = 1
FLAG_RECORD_TAPE = 2
FLAG_USE_TAPE = 4
FLAG_RAY_GRAD = 8

# name -> (restype, argtypes); must list every symbol include/radfoam_b200.h declares
_P = c_void_p
SIGNATURES = {
    "rfb_last_error": (c_char_p, []),
    "rfb_abi_version": (c_int, []),
    "rfb_create_pipeline": (c_int, [c_int, c_int, POINTER(_P)]),
    "rfb_destroy_pipeline": (None, [_P]),
    "rfb_attribute_dim": (c_uint32, [_P]),
    "rfb_attribute_type": (c_int, [_P]),
    "rfb_prefetch_adjacent_diff": (c_int, [_P, c_uint32, c_uint32, _P, _P, _P, _P]),
    "rfb_nearest_point": (c_int, [_P, c_uint32, _P, c_uint32, _P, _P]),
    "rfb_start_points": (c_int, [_P, c_uint32, _P, c_uint32, _P, _P]),
    "rfb_farthest_neighbor": (c_int, [_P, c_uint32, _P, _P, _P, _P, _P]),
    "rfb_locate_points": (c_int, [_P, c_uint32, _P, _P, _P, c_uint32, _P, _P, _P]),
    "rfb_sample_field": (c_int, [_P, _P, c_uint32, _P, _P, _P, _P, c_uint32, _P, _P, _P, _P, _P, _P]),
    "rfb_sample_field_backward": (c_int, [_P, c_uint32, c_uint32, _P, _P, _P, _P, _P, _P, _P]),
    "rfb_surface_scratch_bytes": (c_uint64, [c_uint32]),
    "rfb_surface_count": (c_int, [_P, c_uint32, c_uint32, _P, _P, _P, POINTER(Box), _P, _P]),
    "rfb_surface_write": (c_int, [_P, _P, c_uint32, _P, c_uint32, _P, _P, _P, POINTER(Box), _P, _P, _P, _P, _P,
                                  _P]),
    "rfb_delaunay_scratch_bytes": (c_uint64, [c_uint32, c_uint32]),
    "rfb_delaunay_count": (c_int, [_P, c_uint32, _P, POINTER(Box), c_uint32, _P, _P]),
    "rfb_delaunay_write": (c_int, [c_uint32, _P, c_uint32, _P, _P, _P, _P, _P]),
    "rfb_trace_forward": (c_int, [_P, POINTER(TraceSettings), c_uint32, _P, _P, c_uint32, _P, _P,
                                  c_uint32, _P, _P, c_uint32, _P, _P, _P, _P, _P, _P,
                                  POINTER(LaunchOpts), _P]),
    "rfb_trace_backward": (c_int, [_P, POINTER(TraceSettings), c_uint32, _P, _P, c_uint32, _P, _P,
                                   c_uint32, _P, _P, c_uint32, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                   _P, POINTER(LaunchOpts), _P]),
    "rfb_trace_backward_accumulate": (c_int, [_P, POINTER(TraceSettings), c_uint32, _P, _P, c_uint32,
                                              _P, _P, c_uint32, _P, _P, c_uint32, _P, _P, _P, _P, _P,
                                              _P, _P, POINTER(LaunchOpts), _P]),
    "rfb_trace_backward_accumulate_rays": (c_int, [_P, POINTER(TraceSettings), c_uint32, _P, _P, c_uint32,
                                                   _P, _P, c_uint32, _P, _P, c_uint32, _P, _P, _P, _P, _P,
                                                   _P, _P, _P, POINTER(LaunchOpts), _P]),
    "rfb_grad_accumulator": (c_int, [_P, POINTER(_P), POINTER(c_uint64)]),
    "rfb_grad_row_floats": (c_uint32, [_P]),
    "rfb_trace_backward_finalize": (c_int, [_P, c_uint32, _P, _P, c_uint32, _P]),
    "rfb_bind_scene_params": (c_int, [_P, POINTER(SceneParams)]),
    "rfb_trace_backward_finalize_params": (c_int, [_P, c_uint32, _P, _P, _P, _P, c_uint32, _P]),
    "rfb_set_grad_accumulator": (c_int, [_P, _P, c_uint64]),
    "rfb_reduce_finalize_peers": (c_int, [_P, c_uint32, c_uint32, c_uint32, POINTER(_P), POINTER(_P), POINTER(_P),
                                          POINTER(Multicast), c_uint32, _P]),
    "rfb_trace_benchmark": (c_int, [_P, POINTER(TraceSettings), c_uint32, _P, _P, _P, _P, _P,
                                    POINTER(Camera), _P, _P, POINTER(LaunchOpts), _P]),
    "rfb_trace_visualization": (c_int, [_P, POINTER(TraceSettings), POINTER(VisualizationSettings),
                                        POINTER(Camera), POINTER(CMapTable), c_uint32, c_uint32, _P, _P, _P, _P,
                                        _P, c_uint32, c_uint64, POINTER(LaunchOpts), _P]),
    "rfb_trace_visualization_rgba8": (c_int, [_P, POINTER(TraceSettings), POINTER(VisualizationSettings),
                                              POINTER(Camera), POINTER(CMapTable), c_uint32, c_uint32, _P, _P, _P,
                                              _P, _P, c_uint32, _P, POINTER(LaunchOpts), _P]),
    "rfb_launch_count": (c_uint64, []),
    "rfb_reset_launch_count": (None, []),
    "rfb_device_alloc_counts": (None, [POINTER(c_uint64), POINTER(c_uint64)]),
    "rfb_invalidate_cache": (None, [_P]),
    "rfb_tape_status": (c_int, [_P, POINTER(c_uint32), POINTER(c_uint32), POINTER(c_uint32)]),
    "rfb_set_profiling": (None, [_P, c_int]),
    "rfb_last_kernel_ms": (c_int, [_P, c_int, POINTER(c_float)]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Load (once) and type the C ABI.  Raises if the CUDA library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"radfoam_b200: CUDA library {path} is missing -- run "
            "`python -c 'import __graft_entry__ as g; g.build()'` at the repo root. "
            "There is no CPU fallback.")
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so is stale
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.rfb_abi_version() != 1:
        raise RuntimeError("radfoam_b200: ABI version mismatch; rebuild the library")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().rfb_last_error()
        raise RuntimeError(msg.decode("utf-8", "replace") if msg else f"radfoam_b200 error {rc}")
