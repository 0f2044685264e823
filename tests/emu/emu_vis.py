"""trace_visualization on the CPU kernel-logic emulator (tests/emu) -- TEST INFRASTRUCTURE ONLY.

Both entry points: rfb_trace_visualization_rgba8 into a numpy buffer, and rfb_trace_visualization into the emulator's
emulator's surface (in an emulator build the cudaSurfaceObject_t is the address of an RfbEmuSurface,
radfoam_b200/csrc/foam_kernels.cuh), with a row pitch wider than the frame so
that a store to the wrong byte column or row would show."""
from __future__ import annotations

import ctypes

import numpy as np

import emu  # tests/emu on sys.path, as the emulator tests have it
from radfoam_b200 import _lib as product_abi


class EmuSurface(ctypes.Structure):  # RfbEmuSurface
    _fields_ = [("data", ctypes.c_void_p), ("pitch", ctypes.c_uint64), ("width_bytes", ctypes.c_uint32),
                ("height", ctypes.c_uint32)]


def _camera(camera):
    cam = product_abi.Camera()
    for key in ("position", "forward", "right", "up"):
        getattr(cam, key)[:] = [float(v) for v in np.asarray(camera[key]).reshape(-1)[:3]]
    cam.fov, cam.width, cam.height = float(camera["fov"]), int(camera["width"]), int(camera["height"])
    cam.model = 0 if camera["model"] == "pinhole" else 1
    return cam


def trace_visualization(pipe: emu.EmuPipeline, points, attributes, adjacency, offsets, adjacent_diff, camera,
                        start_index, tables=None, *, mode="rgb", color_map="turbo", bg_color=(1.0, 1.0, 1.0),
                        checker_bg=False, max_depth=10.0, depth_quantile=0.5, weight_threshold=None,
                        max_intersections=None, surface=False, scene_version=0):
    """-> uint32 [height, width] frame (bottom-up rows).  `tables`: four float32 [L, 3] arrays or None."""
    pts, att, adj, off = pipe._scene(points, attributes, adjacency, offsets)
    diff = emu._c(adjacent_diff, np.float16)
    cam = _camera(camera)
    keep = []
    table = None
    if tables is not None:
        arrs = [np.ascontiguousarray(t, dtype=np.float32) for t in tables]
        ptrs = np.array([a.ctypes.data for a in arrs], dtype=np.uint64)
        sizes = np.array([a.shape[0] for a in arrs], dtype=np.int32)
        keep += [arrs, ptrs, sizes]
        table = ctypes.byref(product_abi.CMapTable(ptrs.ctypes.data, sizes.ctypes.data))
    vis = product_abi.VisualizationSettings(product_abi.VIS_MODES[mode], product_abi.COLOR_MAPS[color_map],
                                            (ctypes.c_float * 3)(*[float(c) for c in bg_color]), int(bool(checker_bg)),
                                            float(max_depth), float(depth_quantile))
    settings = pipe._settings(weight_threshold, max_intersections)
    opts = product_abi.LaunchOpts(scene_version, 0, 0)
    args = (pipe.handle, ctypes.byref(settings), ctypes.byref(vis), ctypes.byref(cam), table, pts.shape[0], 0,
            emu._p(pts), emu._p(att), emu._p(adj), emu._p(off), emu._p(diff), int(start_index))
    if not surface:
        out = np.full((cam.height, cam.width), 0xDEADBEEF, dtype=np.uint32)
        emu._check(pipe.lib.rfb_trace_visualization_rgba8(*args, emu._p(out), ctypes.byref(opts), None))
        return out
    pad = 3  # texels of slack per row, left untouched
    buf = np.full((cam.height, cam.width + pad), 0xDEADBEEF, dtype=np.uint32)
    s = EmuSurface(buf.ctypes.data, buf.strides[0], 4 * cam.width, cam.height)
    emu._check(pipe.lib.rfb_trace_visualization(*args, ctypes.addressof(s), ctypes.byref(opts), None))
    assert np.all(buf[:, cam.width:] == 0xDEADBEEF), "a store landed outside the surface's width"
    return buf[:, :cam.width].copy()
