"""Ray gradients on the CPU kernel-logic emulator (tests/emu/emu.py) -- TEST INFRASTRUCTURE ONLY.

``EmuRayPipeline`` is an ``emu.EmuPipeline`` whose backward calls take ``ray_grad=False``: set, the call passes
RFB_FLAG_RAY_GRAD (``trace_backward``) or goes through rfb_trace_backward_accumulate_rays
(``trace_backward_accumulate``) and returns the ray gradient array."""
from __future__ import annotations

import ctypes

import numpy as np

import emu
from emu import _c, _check, _p, product_abi


class EmuRayPipeline(emu.EmuPipeline):
    def trace_backward(self, points, attributes, adjacency, offsets, rays, start, rgba, grad_rgba,
                       depth_quantiles=None, depth_indices=None, grad_depth=None, ray_error=None,
                       weight_threshold=None, max_intersections=None, scene_version=0, use_tape=False,
                       scrub_nonfinite=False, ray_grad=False, ray_grad_buffer=None):
        """``ray_grad``: set RFB_FLAG_RAY_GRAD and return the array as ``out["ray_grad"]``.  ``ray_grad_buffer``:
        the float32 array passed as ray_grad (default: a fresh zero array)."""
        if use_tape:  # same buffers as the recording forward, as the product's Python layer guarantees
            pts, att, adj, off, rays_c, start_c, dq = self._keep
        else:
            pts, att, adj, off = self._scene(points, attributes, adjacency, offsets)
            rays_c, start_c, dq = _c(rays, np.float32), _c(start, np.uint32), _c(depth_quantiles, np.float32)
        n, r = pts.shape[0], rays_c.size // 6
        q = 0 if dq is None else dq.shape[-1]
        rgba_c, g_c = _c(rgba, self.dtype), _c(grad_rgba, self.dtype)
        di, gd, err = _c(depth_indices, np.uint32), _c(grad_depth, np.float32), _c(ray_error, self.dtype)
        out = {"points_grad": np.empty((n, 3), np.float32), "attr_grad": np.empty((n, self.attr_dim), self.dtype)}
        if err is not None:
            out["point_error"] = np.zeros((n, 1), self.dtype)
        width = rays_c.shape[-2] if rays_c.ndim >= 3 else 0
        flags = (product_abi.FLAG_USE_TAPE if use_tape else 0) | (product_abi.FLAG_SCRUB_NONFINITE if scrub_nonfinite else 0)
        flags |= product_abi.FLAG_RAY_GRAD if ray_grad else 0
        opts = product_abi.LaunchOpts(scene_version, width, flags)
        settings = self._settings(weight_threshold, max_intersections)
        buf = np.zeros_like(rays_c) if ray_grad_buffer is None else ray_grad_buffer
        _check(self.lib.rfb_trace_backward(
            self.handle, ctypes.byref(settings), n, _p(pts), _p(att), adj.size, _p(adj), _p(off), r, _p(rays_c),
            _p(start_c), q, _p(dq), _p(di), _p(rgba_c), _p(g_c), _p(gd), _p(err), _p(buf),
            _p(out["points_grad"]), _p(out["attr_grad"]), _p(out.get("point_error")), ctypes.byref(opts), None))
        if ray_grad:
            out["ray_grad"] = buf
        return out

    def trace_backward_accumulate(self, points, attributes, adjacency, offsets, rays, start, rgba, grad_rgba,
                                  depth_quantiles=None, depth_indices=None, grad_depth=None,
                                  weight_threshold=None, max_intersections=None, ray_grad=False):
        """emu.EmuPipeline.trace_backward_accumulate; with ``ray_grad`` through rfb_trace_backward_accumulate_rays,
        returning (accumulator view, ray_grad)."""
        if not ray_grad:
            return super().trace_backward_accumulate(points, attributes, adjacency, offsets, rays, start, rgba,
                                                     grad_rgba, depth_quantiles, depth_indices, grad_depth,
                                                     weight_threshold, max_intersections)
        pts, att, adj, off = self._scene(points, attributes, adjacency, offsets)
        rays_c, start_c, dq = _c(rays, np.float32), _c(start, np.uint32), _c(depth_quantiles, np.float32)
        n, r = pts.shape[0], rays_c.size // 6
        q = 0 if dq is None else dq.shape[-1]
        rgba_c, g_c = _c(rgba, self.dtype), _c(grad_rgba, self.dtype)
        di, gd = _c(depth_indices, np.uint32), _c(grad_depth, np.float32)
        width = rays_c.shape[-2] if rays_c.ndim >= 3 else 0
        opts = product_abi.LaunchOpts(0, width, 0)
        settings = self._settings(weight_threshold, max_intersections)
        rg = np.zeros_like(rays_c)
        _check(self.lib.rfb_trace_backward_accumulate_rays(
            self.handle, ctypes.byref(settings), n, _p(pts), _p(att), adj.size, _p(adj), _p(off), r, _p(rays_c),
            _p(start_c), q, _p(dq), _p(di), _p(rgba_c), _p(g_c), _p(gd), None, None, _p(rg), ctypes.byref(opts), None))
        ptr, count = ctypes.c_void_p(), ctypes.c_uint64()
        _check(self.lib.rfb_grad_accumulator(self.handle, ctypes.byref(ptr), ctypes.byref(count)))
        row = int(self.lib.rfb_grad_row_floats(self.handle))
        acc = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), (count.value // row, row))
        return acc, rg
