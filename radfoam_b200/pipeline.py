"""Host-side mirror of radfoam's pipeline bindings for the tracing hot path.

Same names, keyword arguments, result-dict keys, dtypes, shapes and validation
errors as the pybind11 module the reference's Python code calls
(torch_bindings/pipeline_bindings.cpp:107-672), so
``radfoam_model/render.py::TraceRays`` runs unmodified against a ``Pipeline`` from
here.  PyTorch is used for device memory and streams only; the work happens in the
hand-written sm_90a kernels behind the C ABI (include/radfoam_b200.h), called
through ctypes with raw device pointers.  No CPU fallback exists.
"""
from __future__ import annotations

import ctypes
import weakref

import torch

from . import _lib

_DTYPES = {
    "float32": torch.float32, "float": torch.float32, torch.float32: torch.float32,
    "float16": torch.float16, "half": torch.float16, torch.float16: torch.float16,
}
_DTYPE_NAMES = {torch.float32: "float32", torch.float16: "float16", torch.float64: "float64",
                torch.uint32: "uint32", torch.int32: "int32", torch.int64: "int64"}


def _dtype_name(dt) -> str:
    return _DTYPE_NAMES.get(dt, str(dt).replace("torch.", ""))


def _ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


class Pipeline:
    """radfoam::Pipeline (src/tracing/pipeline.h:58-131) for one (sh_degree, dtype)."""

    def __init__(self, sh_degree: int, attr_dtype):
        if isinstance(attr_dtype, str) or isinstance(attr_dtype, torch.dtype):
            if attr_dtype not in _DTYPES:
                # dtype_to_scalar_type() accepts more names, create_pipeline() then rejects them
                raise RuntimeError("Unsupported attribute type")
            dt = _DTYPES[attr_dtype]
        else:
            raise RuntimeError("dtype must be a string or torch.dtype")
        self._lib = _lib.load()
        handle = ctypes.c_void_p()
        _lib.check(self._lib.rfb_create_pipeline(int(sh_degree), 1 if dt == torch.float16 else 0,
                                                 ctypes.byref(handle)))
        self._handle = handle
        self._dtype = dt
        self._sh_degree = int(sh_degree)
        self._attr_dim = int(self._lib.rfb_attribute_dim(handle))
        # scene-mirror cache bookkeeping: identity + torch version counters of the four
        # scene tensors last traced; a match means the device-side mirrors are current.
        self.cache_scene = True
        self._scene_refs = None
        self._scene_version = 0
        # walk tape: a forward whose scene inputs require grad records (cell, t1) per step so the
        # backward of the same step replays it instead of re-scanning faces
        self.record_tape = True
        self._tape_refs = None
        # set by the autograd ops around their forward: was autograd recording when the op was applied?
        # (inside Function.forward grad mode is always off; None = not called through such an op)
        self.autograd_recording = None
        self._external_acc = None  # keeps a caller-provided accumulator alive (set_grad_accumulator)
        self._params = None        # bound parameter-form scene (bind_scene_params)
        # unordered ray batches ([R, 6], the reference's training batches: train.py:61) are traced
        # in a coherent order -- sorted by (start cell, direction) -- and the per-ray outputs are
        # scattered back; results are unchanged, neighbouring lanes share cells again
        self.reorder_rays = True
        self.reorder_min_rays = 1 << 15
        self._reorder = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                self._lib.rfb_destroy_pipeline(self._handle)
                self._handle = None
        except Exception:
            pass

    # --- reference API -------------------------------------------------------------
    def attribute_dim(self) -> int:
        return self._attr_dim

    def attribute_type(self):
        return self._dtype

    @property
    def sh_degree(self) -> int:
        return self._sh_degree

    def grad_row_floats(self) -> int:
        return int(self._lib.rfb_grad_row_floats(self._handle))

    def set_profiling(self, enabled: bool) -> None:
        """Record CUDA events around the ray kernels (for roofline reporting)."""
        self._lib.rfb_set_profiling(self._handle, 1 if enabled else 0)

    def last_kernel_ms(self, which: str) -> float:
        ms = ctypes.c_float()
        _lib.check(self._lib.rfb_last_kernel_ms(self._handle, {"forward": 0, "backward": 1}[which],
                                                ctypes.byref(ms)))
        return float(ms.value)

    def tape_status(self) -> dict:
        """Walk-tape pool state after the last recording forward (synchronises on it)."""
        cap, used, over = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        _lib.check(self._lib.rfb_tape_status(self._handle, ctypes.byref(cap), ctypes.byref(used),
                                             ctypes.byref(over)))
        return {"capacity_chunks": cap.value, "used_chunks": used.value, "overflowed": bool(over.value),
                "bytes": used.value * 8192}

    def invalidate_cache(self) -> None:
        self._scene_refs = None
        self._lib.rfb_invalidate_cache(self._handle)

    # validate_scene_data(), pipeline_bindings.cpp:8-71
    def _validate_scene(self, points, attributes, point_adjacency, point_adjacency_offsets):
        if points.size(-1) != 3:
            raise RuntimeError(f"points had dimension {points.size(-1)} along axis -1, expected 3")
        if points.dtype != torch.float32:
            raise RuntimeError(f"points had dtype {_dtype_name(points.dtype)}, expected float32")
        if points.device.type != "cuda":
            raise RuntimeError("points must be on CUDA device")
        num_points = points.numel() // 3
        if attributes is None:
            if self._params is None:
                raise RuntimeError("attributes is None but no parameter-form scene is bound (bind_scene_params)")
        else:
            if self._params is not None:
                raise RuntimeError("a parameter-form scene is bound: pass attributes=None, or unbind it")
            if attributes.size(-1) != self._attr_dim:
                raise RuntimeError(f"attributes had dimension {attributes.size(-1)} along axis -1, "
                                   f"expected {self._attr_dim}")
            if attributes.numel() // self._attr_dim != num_points:
                raise RuntimeError("attributes must have the same number of rows as points")
            if attributes.dtype != self._dtype:
                raise RuntimeError(f"attributes had dtype {_dtype_name(attributes.dtype)}, "
                                   f"expected {_dtype_name(self._dtype)}")
            if attributes.device.type != "cuda":
                raise RuntimeError("attributes must be on CUDA device")
        if point_adjacency_offsets.dtype != torch.uint32:
            raise RuntimeError("point_adjacency_offsets must have uint32 dtype")
        if point_adjacency_offsets.device.type != "cuda":
            raise RuntimeError("point_adjacency_offsets must be on CUDA device")
        if point_adjacency_offsets.numel() != num_points + 1:
            raise RuntimeError("point_adjacency_offsets must have num_points + 1 elements")
        if point_adjacency.dtype != torch.uint32:
            raise RuntimeError("point_adjacency must have uint32 dtype")
        if point_adjacency.device.type != "cuda":
            raise RuntimeError("point_adjacency must be on CUDA device")

    @staticmethod
    def _validate_rays(rays, start_point, num_rays):
        if rays.size(-1) != 6:
            raise RuntimeError("rays must have 6 as the last dimension")
        if rays.dtype != torch.float32:
            raise RuntimeError("rays must have float32 dtype")
        if rays.device.type != "cuda":
            raise RuntimeError("rays must be on CUDA device")
        if start_point.numel() != num_rays:
            raise RuntimeError("start_point must have the same batch size as rays")
        if start_point.dtype != torch.uint32:
            raise RuntimeError("start_point must have uint32 dtype")
        if start_point.device.type != "cuda":
            raise RuntimeError("start_point must be on CUDA device")

    @staticmethod
    def _coherent_order(rays_c, start_c):
        """Permutation sorting rays by (start cell, Morton code of the direction on the octahedral
        map): rays of one camera with neighbouring directions become neighbours in the batch."""
        dirs = torch.nn.functional.normalize(rays_c[:, 3:6], dim=1)
        o = dirs[:, :2] / dirs.abs().sum(dim=1, keepdim=True).clamp_min(1e-30)
        o = torch.where(dirs[:, 2:3] < 0, (1 - o.flip(1).abs()) * torch.where(o < 0, -1.0, 1.0), o)
        uv = ((o * 0.5 + 0.5).clamp(0, 1) * 1023).to(torch.int64)

        def spread(v):
            v = (v | (v << 8)) & 0x00FF00FF
            v = (v | (v << 4)) & 0x0F0F0F0F
            v = (v | (v << 2)) & 0x33333333
            return (v | (v << 1)) & 0x55555555

        key = (start_c.to(torch.int64) << 20) | spread(uv[:, 0]) | (spread(uv[:, 1]) << 1)
        return torch.argsort(key)

    @staticmethod
    def _take(t, perm):
        """t[perm] along dim 0, also for uint32 tensors (indexing is not implemented for them)."""
        if t is None:
            return None
        if t.dtype == torch.uint32:
            return t.view(torch.int32)[perm].view(torch.uint32)
        return t[perm]

    @staticmethod
    def _untake(t_sorted, perm):
        """Inverse of _take: out[perm] = t_sorted."""
        if t_sorted is None:
            return None
        if t_sorted.dtype == torch.uint32:
            out = torch.empty_like(t_sorted).view(torch.int32)
            out[perm] = t_sorted.view(torch.int32)
            return out.view(torch.uint32)
        out = torch.empty_like(t_sorted)
        out[perm] = t_sorted
        return out

    def _tape_flag(self, rays_c, start_c, scene_version) -> int:
        """FLAG_USE_TAPE iff these are the very tensors (unmodified) of the last recording forward."""
        refs = self._tape_refs
        if not refs or refs[2] != scene_version or scene_version == 0:
            return 0
        same = all(r() is t and v == t._version for (r, v), t in zip(refs[:2], (rays_c, start_c)))
        return _lib.FLAG_USE_TAPE if same else 0

    def _backward_expected(self, trainable) -> bool:
        """Will a backward over this forward follow?  (Only then is the walk tape worth recording.)
        ``trainable`` = (points, attributes) or (points, att_dc, att_sh, density).
        nn.Parameters keep requires_grad under torch.no_grad(), so requires_grad alone is not enough."""
        points, rest = trainable[0], trainable[1:]
        if not any(t.requires_grad for t in trainable):
            return False
        if self.autograd_recording is not None:  # told by radfoam_b200's autograd ops
            return bool(self.autograd_recording)
        if torch.is_grad_enabled():  # direct call: the caller may run trace_backward by hand
            return True
        # Grad mode is off: either the caller is under torch.no_grad() (an eval render: no backward), or this
        # is the forward of somebody else's autograd.Function (radfoam_model/render.py), where it is always
        # off.  A non-leaf input that requires grad only exists while a graph is being recorded.  With leaves
        # only, the reference's eval path gives points (a Parameter) with attributes built under no_grad
        # (scene.py:202-217: requires_grad False); both being trainable leaves means a hand-made training step.
        if any(t.requires_grad and t.grad_fn is not None for t in trainable):
            return True
        return points.requires_grad and any(t.requires_grad for t in rest)

    def _settings(self, weight_threshold, max_intersections):
        s = _lib.TraceSettings(0.001, 1024)  # default_trace_settings(), pipeline.h:15-20
        if weight_threshold is not None:
            s.weight_threshold = float(weight_threshold)
        if max_intersections is not None:
            s.max_intersections = int(max_intersections)
        return s

    def _opts(self, scene, rays, flags=0):
        """Launch hints: scene-mirror reuse key and the image-tiling width."""
        version = 0
        if self.cache_scene:
            refs = self._scene_refs
            same = (refs is not None and all(r() is t and v == t._version
                                             for (r, v), t in zip(refs, scene)))
            if not same:
                self._scene_version += 1
                self._scene_refs = [(weakref.ref(t), t._version) for t in scene]
            version = self._scene_version
        width = int(rays.shape[-2]) if rays is not None and rays.dim() >= 3 else 0
        return _lib.LaunchOpts(version, width, flags)

    # trace_forward(), pipeline_bindings.cpp:107-265
    def trace_forward(self, points, attributes, point_adjacency, point_adjacency_offsets, rays,
                      start_point, depth_quantiles=None, weight_threshold=None,
                      max_intersections=None, return_contribution=False):
        (points_c, attributes_c, adj_c, off_c), scene_key = self._scene_tensors(
            points, attributes, point_adjacency, point_adjacency_offsets)
        rays_c = rays.contiguous()
        start_c = start_point.contiguous()

        return_depth = depth_quantiles is not None
        num_points = points_c.size(0)
        num_rays = rays_c.numel() // 6
        self._validate_rays(rays_c, start_c, num_rays)

        num_q = 0
        dq_c = None
        if return_depth:
            dq_c = depth_quantiles.contiguous()
            num_q = dq_c.size(-1)
            if dq_c.dtype != torch.float32:
                raise RuntimeError("depth_quantiles must have float32 dtype")
            if dq_c.device.type != "cuda":
                raise RuntimeError("depth_quantiles must be on CUDA device")
            if num_q == 0 or dq_c.numel() // num_q != num_rays:
                raise RuntimeError("depth_quantiles must have the same batch size as rays")

        settings = self._settings(weight_threshold, max_intersections)
        dev = rays_c.device
        perm = None
        self._reorder = None
        if self.reorder_rays and rays_c.dim() == 2 and num_rays >= self.reorder_min_rays:
            with torch.no_grad():
                perm = self._coherent_order(rays_c, start_c)
                sorted_in = (self._take(rays_c, perm), self._take(start_c, perm), self._take(dq_c, perm))
            self._reorder = ((weakref.ref(rays_c), rays_c._version), (weakref.ref(start_c), start_c._version),
                             perm, sorted_in)
            rays_c, start_c, dq_c = sorted_in
        batch = list(rays_c.shape[:-1])
        rgba = torch.empty(batch + [4], dtype=self._dtype, device=dev)
        num_intersections = torch.empty(batch + [1], dtype=torch.uint32, device=dev)
        contribution = None
        if return_contribution:
            contribution = torch.zeros((num_points, 1), dtype=self._dtype, device=dev)
        depth = depth_indices = None
        if return_depth:
            depth = torch.empty(batch + [num_q], dtype=torch.float32, device=dev)
            depth_indices = torch.empty(batch + [num_q], dtype=torch.uint32, device=dev)

        trainable = (points, attributes) if attributes is not None else (points,) + self._params[1]
        # through the autograd ops, rays that require grad expect a backward too (ray gradients)
        rays_grad = bool(self.autograd_recording) and rays.requires_grad
        record = self.record_tape and self.cache_scene and (self._backward_expected(trainable) or rays_grad)
        opts = self._opts(scene_key, rays_c, _lib.FLAG_RECORD_TAPE if record else 0)
        self._tape_refs = ([(weakref.ref(t), t._version) for t in (rays_c, start_c)]
                           + [opts.scene_version] if record else None)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_trace_forward(
                self._handle, ctypes.byref(settings), num_points, _ptr(points_c), _ptr(attributes_c),
                adj_c.numel(), _ptr(adj_c), _ptr(off_c), num_rays, _ptr(rays_c), _ptr(start_c),
                num_q, _ptr(dq_c), _ptr(rgba), _ptr(depth), _ptr(depth_indices),
                _ptr(num_intersections), _ptr(contribution), ctypes.byref(opts), stream))

        if perm is not None:  # back to the caller's ray order
            rgba, num_intersections = self._untake(rgba, perm), self._untake(num_intersections, perm)
            depth, depth_indices = self._untake(depth, perm), self._untake(depth_indices, perm)
        out = {"rgba": rgba}
        if return_depth:
            out["depth"] = depth
            out["depth_indices"] = depth_indices
        if return_contribution:
            out["contribution"] = contribution
        out["num_intersections"] = num_intersections
        return out

    def _sorted_backward_args(self, rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c):
        """If the last forward traced these very rays in a coherent order, hand the backward the
        same sorted tensors (so that the walk tape matches) and permute its per-ray inputs."""
        ro = self._reorder
        if ro is None:
            return rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c
        (r_ref, r_ver), (s_ref, s_ver), perm, (rays_k, start_k, dq_k) = ro
        if not (r_ref() is rays_c and r_ver == rays_c._version and s_ref() is start_c
                and s_ver == start_c._version):
            return rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c
        take = self._take
        del dq_k  # the backward's own quantiles are permuted, whatever the forward was given
        return (rays_k, start_k, take(rgb_c, perm), take(grad_c, perm), take(dq_c, perm),
                take(di_c, perm), take(dg_c, perm), take(err_c, perm))

    def _caller_order(self, ray_grad, rays_traced, rays_in):
        """A per-ray backward output in the caller's ray order: _sorted_backward_args may have handed the kernels
        the forward's coherently sorted copy of the rays instead of ``rays_in``."""
        if rays_traced is rays_in:
            return ray_grad
        with torch.no_grad():
            return self._untake(ray_grad, self._reorder[2]).view(rays_in.shape)

    def _backward_args(self, points, attributes, point_adjacency, point_adjacency_offsets, rays,
                       start_point, rgb_out, grad_in, depth_quantiles, depth_indices,
                       depth_grad_in, ray_error):
        """Shared validation of trace_backward (pipeline_bindings.cpp:267-439)."""
        (points_c, attributes_c, adj_c, off_c), scene_key = self._scene_tensors(
            points, attributes, point_adjacency, point_adjacency_offsets)
        rays_c = rays.contiguous()
        start_c = start_point.contiguous()
        num_rays = rays_c.numel() // 6
        self._validate_rays(rays_c, start_c, num_rays)

        grad_c = grad_in.contiguous()
        if grad_c.size(-1) != 4:
            raise RuntimeError("rgb_grad_in must have 4 as the last dimension")
        if grad_c.dtype != self._dtype:
            raise RuntimeError(f"rgb_grad_in had dtype {_dtype_name(grad_c.dtype)}, "
                               f"expected {_dtype_name(self._dtype)}")
        if grad_c.device.type != "cuda":
            raise RuntimeError("rgb_grad_in must be on CUDA device")
        if grad_c.numel() // 4 != num_rays:
            raise RuntimeError("rgb_grad_in must have the same batch size as rays")
        # the reference passes rgb_out.data_ptr() unchecked (pipeline_bindings.cpp:477); a
        # non-contiguous or wrong-dtype tensor would be read as garbage there, so reject it
        rgb_c = rgb_out.contiguous()
        if rgb_c.dtype != self._dtype or rgb_c.numel() != 4 * num_rays or rgb_c.device.type != "cuda":
            raise RuntimeError("rgb_out must be the [..., 4] rgba tensor trace_forward returned")

        num_q = 0
        dq_c = di_c = dg_c = None
        if depth_quantiles is not None:
            dq_c = depth_quantiles.contiguous()
            num_q = dq_c.size(-1)
            if dq_c.dtype != torch.float32:
                raise RuntimeError("depth_quantiles must have float32 dtype")
            if dq_c.device.type != "cuda":
                raise RuntimeError("depth_quantiles must be on CUDA device")
            if dq_c.numel() != num_rays * num_q:
                raise RuntimeError("depth_quantiles must have the same batch size as rays")
            if depth_grad_in is None:
                raise RuntimeError("depth_grad must be provided if depth_quantiles is provided")
            if depth_indices is None:
                raise RuntimeError("depth_indices must be provided if depth_quantiles is provided")
            di_c = depth_indices.contiguous()
            if di_c.dtype != torch.uint32:
                raise RuntimeError("depth_indices must have uint32 dtype")
            if di_c.device.type != "cuda":
                raise RuntimeError("depth_indices must be on CUDA device")
            if di_c.numel() != num_rays * num_q:
                raise RuntimeError("depth_indices must have the same batch size as rays")
            dg_c = depth_grad_in.contiguous()
            if dg_c.size(-1) != num_q:
                raise RuntimeError("depth_grad must have the same number of depth quantiles as "
                                   "depth_quantiles")
            if dg_c.dtype != torch.float32:
                raise RuntimeError(f"depth_grad had dtype {_dtype_name(dg_c.dtype)}, expected float32")
            if dg_c.device.type != "cuda":
                raise RuntimeError("depth_grad must be on CUDA device")
            if dg_c.numel() != num_rays * num_q:
                raise RuntimeError("depth_grad must have the same batch size as rays")

        err_c = None
        if ray_error is not None:
            err_c = ray_error.contiguous()
            if err_c.dtype != self._dtype:
                raise RuntimeError(f"ray_error had dtype {_dtype_name(err_c.dtype)}, "
                                   f"expected {_dtype_name(self._dtype)}")
            if err_c.device.type != "cuda":
                raise RuntimeError("ray_error must be on CUDA device")
            if err_c.numel() != num_rays:
                raise RuntimeError("ray_error must have the same batch size as rays")
        self._scene_key = scene_key
        return (points_c, attributes_c, adj_c, off_c, rays_c, start_c, rgb_c, grad_c, dq_c, di_c,
                dg_c, err_c, num_rays, num_q)

    # trace_backward(), pipeline_bindings.cpp:267-497
    def trace_backward(self, points, attributes, point_adjacency, point_adjacency_offsets, rays,
                       start_point, rgb_out, grad_in, depth_quantiles=None, depth_indices=None,
                       depth_grad_in=None, ray_error=None, weight_threshold=None,
                       max_intersections=None, scrub_nonfinite=False, return_ray_grad=False):
        """``scrub_nonfinite`` (extension, default off) zeroes non-finite gradient
        entries inside the kernel epilogue, saving the two masked passes
        radfoam_model/render.py:98-99 makes after this call.  ``return_ray_grad``
        (extension, default off) fills ``ray_grad`` with dL/d(origin, direction as passed
        in) for the walk's cell sequence held fixed; otherwise it is allocated and never
        written, as in the reference."""
        (points_c, attributes_c, adj_c, off_c, rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c,
         err_c, num_rays, num_q) = self._backward_args(
            points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point, rgb_out,
            grad_in, depth_quantiles, depth_indices, depth_grad_in, ray_error)
        rays_in = rays_c
        with torch.no_grad():
            rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c = self._sorted_backward_args(
                rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c)
        num_points = points_c.size(0)
        dev = rays_c.device
        settings = self._settings(weight_threshold, max_intersections)
        # fully overwritten by the kernels' epilogue: no zero-fill pass needed
        if attributes_c is None:
            raise RuntimeError("a parameter-form scene is bound: use trace_backward_params")
        attr_grad = torch.empty((num_points, self._attr_dim), dtype=self._dtype, device=dev)
        points_grad = torch.empty((num_points, 3), dtype=torch.float32, device=dev)
        # without return_ray_grad never written, like the reference (SURVEY A.5.4)
        ray_grad = torch.empty_like(rays_c)
        point_error = None
        if err_c is not None:
            point_error = torch.zeros((num_points, 1), dtype=self._dtype, device=dev)

        flags = (_lib.FLAG_SCRUB_NONFINITE if scrub_nonfinite else 0) | (_lib.FLAG_RAY_GRAD if return_ray_grad else 0)
        opts = self._opts(self._scene_key, rays_c, flags)
        opts.flags |= self._tape_flag(rays_c, start_c, opts.scene_version)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_trace_backward(
                self._handle, ctypes.byref(settings), num_points, _ptr(points_c), _ptr(attributes_c),
                adj_c.numel(), _ptr(adj_c), _ptr(off_c), num_rays, _ptr(rays_c), _ptr(start_c),
                num_q, _ptr(dq_c), _ptr(di_c), _ptr(rgb_c), _ptr(grad_c), _ptr(dg_c), _ptr(err_c),
                _ptr(ray_grad), _ptr(points_grad), _ptr(attr_grad), _ptr(point_error),
                ctypes.byref(opts), stream))
        if return_ray_grad:
            ray_grad = self._caller_order(ray_grad, rays_c, rays_in)

        out = {"points_grad": points_grad, "attr_grad": attr_grad, "ray_grad": ray_grad}
        if err_c is not None:
            out["point_error"] = point_error
        return out

    # ---- split backward (ray-sharded multi-GPU, SURVEY.md §8e) ---------------------
    def trace_backward_accumulate(self, points, attributes, point_adjacency,
                                  point_adjacency_offsets, rays, start_point, rgb_out, grad_in,
                                  depth_quantiles=None, depth_indices=None, depth_grad_in=None,
                                  ray_error=None, weight_threshold=None, max_intersections=None,
                                  return_ray_grad=False, scrub_nonfinite=False):
        """Backward into the pipeline's fp32 accumulator; returns it as a
        ``[N, grad_row_floats]`` tensor VIEW (valid until the next call) so a
        data-parallel caller can all-reduce it before ``trace_backward_finalize``.
        With ``return_ray_grad`` a third value is returned: ``ray_grad`` (see
        ``trace_backward``), whose non-finite entries ``scrub_nonfinite`` zeroes."""
        (points_c, attributes_c, adj_c, off_c, rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c,
         err_c, num_rays, num_q) = self._backward_args(
            points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point, rgb_out,
            grad_in, depth_quantiles, depth_indices, depth_grad_in, ray_error)
        rays_in = rays_c
        with torch.no_grad():
            rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c = self._sorted_backward_args(
                rays_c, start_c, rgb_c, grad_c, dq_c, di_c, dg_c, err_c)
        num_points = points_c.size(0)
        dev = rays_c.device
        settings = self._settings(weight_threshold, max_intersections)
        point_error = None
        if err_c is not None:
            point_error = torch.zeros((num_points, 1), dtype=self._dtype, device=dev)
        ray_grad = torch.empty_like(rays_c) if return_ray_grad else None
        opts = self._opts(self._scene_key, rays_c, _lib.FLAG_SCRUB_NONFINITE if scrub_nonfinite else 0)
        opts.flags |= self._tape_flag(rays_c, start_c, opts.scene_version)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_trace_backward_accumulate_rays(
                self._handle, ctypes.byref(settings), num_points, _ptr(points_c), _ptr(attributes_c),
                adj_c.numel(), _ptr(adj_c), _ptr(off_c), num_rays, _ptr(rays_c), _ptr(start_c),
                num_q, _ptr(dq_c), _ptr(di_c), _ptr(rgb_c), _ptr(grad_c), _ptr(dg_c), _ptr(err_c),
                _ptr(point_error), _ptr(ray_grad), ctypes.byref(opts), stream))
        if not return_ray_grad:
            return self.grad_accumulator(dev), point_error
        return self.grad_accumulator(dev), point_error, self._caller_order(ray_grad, rays_c, rays_in)

    def grad_accumulator(self, device):
        ptr = ctypes.c_void_p()
        count = ctypes.c_uint64()
        _lib.check(self._lib.rfb_grad_accumulator(self._handle, ctypes.byref(ptr), ctypes.byref(count)))
        row = self.grad_row_floats()
        n = count.value // row
        if n == 0:
            return torch.empty((0, row), dtype=torch.float32, device=device)
        return _wrap_device_memory(ptr.value, (n, row), device)

    # ---- parameter-form scene: get_trace_data (scene.py:202-217) fused into the re-layout / finalize kernels
    def bind_scene_params(self, att_dc, att_sh, density, activation_scale=1.0) -> None:
        """Trace the scene straight from the model's parameters: ``attributes = cat(att_dc, att_sh,
        activation_scale * softplus(density, beta=10)).to(attr_dtype)`` is evaluated inside the re-layout
        kernel instead of by torch ops.  While bound, pass ``attributes=None`` to the trace calls and use
        ``trace_backward_params``.  ``bind_scene_params(None, None, None)`` unbinds."""
        if att_dc is None:
            self._params = None
            _lib.check(self._lib.rfb_bind_scene_params(self._handle, None))
            return
        n = density.numel()
        if self._sh_degree == 0 and att_sh is None:
            att_sh = torch.empty((n, 0), dtype=torch.float32, device=density.device)
        for name, t, cols in (("att_dc", att_dc, 3), ("att_sh", att_sh, self._attr_dim - 4), ("density", density, 1)):
            if t.dtype != torch.float32:
                raise RuntimeError(f"{name} had dtype {_dtype_name(t.dtype)}, expected float32 (model parameters)")
            if t.device.type != "cuda":
                raise RuntimeError(f"{name} must be on CUDA device")
            if t.numel() != n * cols:
                raise RuntimeError(f"{name} must have {cols} columns and the same number of rows as density")
        if not all(t.is_contiguous() for t in (att_dc, att_sh, density)):
            raise RuntimeError("att_dc, att_sh and density must be contiguous (they are read in place)")
        tensors = tuple(t.detach() for t in (att_dc, att_sh, density))  # share storage and version counter
        self._params = (tensors, (att_dc, att_sh, density), float(activation_scale))
        sp = _lib.SceneParams(tensors[0].data_ptr(), tensors[1].data_ptr() if tensors[1].numel() else None,
                              tensors[2].data_ptr(), float(activation_scale))
        _lib.check(self._lib.rfb_bind_scene_params(self._handle, ctypes.byref(sp)))

    def trace_backward_params(self, points, point_adjacency, point_adjacency_offsets, rays, start_point, rgb_out,
                              grad_in, depth_quantiles=None, depth_indices=None, depth_grad_in=None, ray_error=None,
                              weight_threshold=None, max_intersections=None, scrub_nonfinite=True,
                              return_ray_grad=False):
        """Backward of a bound parameter-form scene: gradients of points, att_dc, att_sh and the raw density,
        and with ``return_ray_grad`` also ``ray_grad`` (see ``trace_backward``)."""
        if self._params is None:
            raise RuntimeError("no parameter-form scene is bound (bind_scene_params)")
        _, point_error, *ray_grad = self.trace_backward_accumulate(
            points, None, point_adjacency, point_adjacency_offsets, rays, start_point, rgb_out, grad_in,
            depth_quantiles, depth_indices, depth_grad_in, ray_error, weight_threshold, max_intersections,
            return_ray_grad=return_ray_grad, scrub_nonfinite=scrub_nonfinite)
        n, dev = points.shape[0], rays.device
        out = {"points_grad": torch.empty((n, 3), dtype=torch.float32, device=dev),
               "att_dc_grad": torch.empty((n, 3), dtype=torch.float32, device=dev),
               "att_sh_grad": torch.empty((n, self._attr_dim - 4), dtype=torch.float32, device=dev),
               "density_grad": torch.empty((n, 1), dtype=torch.float32, device=dev)}
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_trace_backward_finalize_params(
                self._handle, n, _ptr(out["points_grad"]), _ptr(out["att_dc_grad"]),
                _ptr(out["att_sh_grad"]) if out["att_sh_grad"].numel() else None, _ptr(out["density_grad"]),
                _lib.FLAG_SCRUB_NONFINITE if scrub_nonfinite else 0, stream))
        if point_error is not None:
            out["point_error"] = point_error
        if return_ray_grad:
            out["ray_grad"] = ray_grad[0]
        return out

    def _scene_tensors(self, points, attributes, point_adjacency, point_adjacency_offsets):
        """Validated, contiguous ``(points, attributes, adjacency, offsets)`` + the tensors whose identity and
        version key the mirror cache.  With a bound parameter-form scene ``attributes`` is None and the three
        parameter tensors take its place in the key."""
        self._validate_scene(points, attributes, point_adjacency, point_adjacency_offsets)
        scene = (points.contiguous(), None if attributes is None else attributes.contiguous(),
                 point_adjacency.contiguous(), point_adjacency_offsets.contiguous())
        if self._params is None:
            return scene, scene
        if self._params[0][2].numel() != points.numel() // 3:
            raise RuntimeError("the bound parameters must have the same number of rows as points")
        return scene, (scene[0],) + self._params[0] + scene[2:]

    def set_grad_accumulator(self, acc) -> None:
        """Scatter the backward into caller-provided memory (an ``[N, grad_row_floats]`` float32 CUDA tensor the
        caller keeps alive, e.g. symmetric memory the other GPUs can address); ``None`` = the pipeline's own."""
        if acc is None:
            self._external_acc = None
            _lib.check(self._lib.rfb_set_grad_accumulator(self._handle, None, 0))
            return
        if acc.dtype != torch.float32 or acc.device.type != "cuda" or not acc.is_contiguous():
            raise RuntimeError("the accumulator must be a contiguous float32 CUDA tensor")
        self._external_acc = acc
        _lib.check(self._lib.rfb_set_grad_accumulator(self._handle, acc.data_ptr(), acc.numel()))

    def reduce_finalize_peers(self, world, rank, num_points, peer_acc, peer_attr_grad, peer_points_grad, device,
                              scrub_nonfinite=False, multicast=None):
        """``rfb_reduce_finalize_peers``: the pointer tables are ctypes ``c_void_p`` arrays of ``world`` device
        addresses valid on this device; ``multicast`` = optional ``(acc, attr_grad, points_grad)`` NVSwitch
        multicast addresses.  The caller provides the cross-GPU barriers around it."""
        mc = None
        if multicast is not None:
            mc = ctypes.byref(_lib.Multicast(*[int(a) for a in multicast]))
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            _lib.check(self._lib.rfb_reduce_finalize_peers(
                self._handle, world, rank, num_points, peer_acc, peer_attr_grad, peer_points_grad, mc,
                _lib.FLAG_SCRUB_NONFINITE if scrub_nonfinite else 0, stream))

    def trace_backward_finalize(self, num_points, device, scrub_nonfinite=False):
        attr_grad = torch.empty((num_points, self._attr_dim), dtype=self._dtype, device=device)
        points_grad = torch.empty((num_points, 3), dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            _lib.check(self._lib.rfb_trace_backward_finalize(
                self._handle, num_points, _ptr(points_grad), _ptr(attr_grad),
                _lib.FLAG_SCRUB_NONFINITE if scrub_nonfinite else 0, stream))
        return points_grad, attr_grad

    # trace_benchmark(), pipeline_bindings.cpp:499-585
    def trace_benchmark(self, points, attributes, point_adjacency, point_adjacency_offsets,
                        adjacent_diff, camera, start_point, output_rgba, weight_threshold=None,
                        max_intersections=None):
        (points_c, attributes_c, adj_c, off_c), scene_key = self._scene_tensors(
            points, attributes, point_adjacency, point_adjacency_offsets)
        diff_c = adjacent_diff.contiguous()
        num_points = points_c.size(0)

        cam = _lib.Camera()
        for key in ("position", "forward", "up", "right"):
            vec = camera[key]
            vals = [float(v) for v in (vec.detach().cpu().reshape(-1).tolist()
                                       if isinstance(vec, torch.Tensor) else list(vec))]
            getattr(cam, key)[:] = vals[:3]
        cam.fov = float(camera["fov"])
        cam.width = int(camera["width"])
        cam.height = int(camera["height"])
        model = camera["model"]
        if model == "pinhole":
            cam.model = 0
        elif model == "fisheye":
            cam.model = 1
        else:
            raise RuntimeError("Invalid camera model")

        if start_point.numel() != 1:
            raise RuntimeError("start_point must have a single element")
        if start_point.dtype != torch.uint32:
            raise RuntimeError("start_point must have uint32 dtype")
        if start_point.device.type != "cuda":
            raise RuntimeError("start_point must be on CUDA device")
        if output_rgba.numel() != cam.width * cam.height:
            raise RuntimeError("output_rgba must have width * height elements")
        if output_rgba.dtype != torch.uint32:
            raise RuntimeError("output_rgba must have uint32 dtype")
        if output_rgba.device.type != "cuda":
            raise RuntimeError("output_rgba must be on CUDA device")
        if not output_rgba.is_contiguous():
            raise RuntimeError("output_rgba must be contiguous")
        if diff_c.numel() * diff_c.element_size() < 8 * adj_c.numel():
            raise RuntimeError("adjacent_diff must hold one half4 per adjacency entry")

        settings = self._settings(weight_threshold, max_intersections)
        dev = points_c.device
        opts = self._opts(scene_key, None)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_trace_benchmark(
                self._handle, ctypes.byref(settings), num_points, _ptr(points_c), _ptr(attributes_c),
                _ptr(adj_c), _ptr(off_c), _ptr(diff_c), ctypes.byref(cam), _ptr(start_point),
                _ptr(output_rgba), ctypes.byref(opts), stream))
        return None

    @staticmethod
    def _camera(camera):
        cam = _lib.Camera()
        for key in ("position", "forward", "up", "right"):
            vec = camera[key]
            vals = [float(v) for v in (vec.detach().cpu().reshape(-1).tolist()
                                       if isinstance(vec, torch.Tensor) else list(vec))]
            getattr(cam, key)[:] = vals[:3]
        cam.fov = float(camera["fov"])
        cam.width = int(camera["width"])
        cam.height = int(camera["height"])
        if camera["model"] not in ("pinhole", "fisheye"):
            raise RuntimeError("Invalid camera model")
        cam.model = 0 if camera["model"] == "pinhole" else 1
        return cam

    def _cmap_arrays(self, cmap_table, device):
        """Device arrays (pointer table, lengths) of a colour-map table: four float32 CUDA tensors [L_k, 3].
        Built once per table; the tensors are held so the pointers stay valid."""
        tables = tuple(cmap_table)
        if len(tables) != 4:
            raise RuntimeError("cmap_table must hold one [L, 3] table per colour map (gray, viridis, inferno, turbo)")
        for t in tables:
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != device:
                raise RuntimeError("cmap_table entries must be float32 tensors on the scene's CUDA device")
            if t.dim() != 2 or t.size(1) != 3 or t.size(0) < 1 or not t.is_contiguous():
                raise RuntimeError("cmap_table entries must be contiguous [L, 3] tensors with L >= 1")
        cached = getattr(self, "_cmap_cache", None)
        if cached is not None and len(cached[0]) == 4 and all(
                a is b and v == b._version for a, v, b in zip(cached[0], cached[1], tables)):
            return cached[2], cached[3]
        ptrs = torch.tensor([t.data_ptr() for t in tables], dtype=torch.int64).to(device)
        sizes = torch.tensor([t.size(0) for t in tables], dtype=torch.int32).to(device)
        self._cmap_cache = (tables, [t._version for t in tables], ptrs, sizes)
        return ptrs, sizes

    # Pipeline::trace_visualization (pipeline.h:102-115); the reference has no Python binding for it
    def trace_visualization(self, points, attributes, point_adjacency, point_adjacency_offsets, adjacent_diff,
                            camera, start_point, output_rgba=None, *, mode="rgb", color_map="turbo",
                            cmap_table=None, bg_color=(1.0, 1.0, 1.0), checker_bg=False, max_depth=10.0,
                            depth_quantile=0.5, weight_threshold=None, max_intersections=None):
        """Preview frame of the foam seen by ``camera`` (the dict ``trace_benchmark`` takes), as RGBA8 words in a
        uint32 ``[height, width]`` tensor whose rows are bottom-up, as on the reference's GL surface.

        mode: "rgb" (colour over ``bg_color``, or a grey checker), "depth" (colormap of the depth where the
        transmittance first falls below ``depth_quantile``, divided by ``max_depth``), "alpha" (1 - T), or
        "intersections" (colormap of cells entered - 1 over ``max_intersections``).  ``cmap_table``: four float32
        CUDA tensors ``[L_k, 3]`` indexed by colour map (gray, viridis, inferno, turbo); needed by "depth" and
        "intersections" only.  ``start_point``: the entry cell, an int or a one-element uint32 tensor."""
        if mode not in _lib.VIS_MODES:
            raise RuntimeError(f"unknown visualization mode {mode!r}; one of {sorted(_lib.VIS_MODES)}")
        if color_map not in _lib.COLOR_MAPS:
            raise RuntimeError(f"unknown color map {color_map!r}; one of {sorted(_lib.COLOR_MAPS)}")
        (points_c, attributes_c, adj_c, off_c), scene_key = self._scene_tensors(
            points, attributes, point_adjacency, point_adjacency_offsets)
        diff_c = adjacent_diff.contiguous()
        num_points = points_c.size(0)
        dev = points_c.device
        cam = self._camera(camera)
        if isinstance(start_point, torch.Tensor):
            if start_point.numel() != 1:
                raise RuntimeError("start_point must have a single element")
            if start_point.dtype != torch.uint32:
                raise RuntimeError("start_point must have uint32 dtype")
            start = int(start_point.reshape(-1).cpu().numpy()[0])
        else:
            start = int(start_point)
        if not 0 <= start < num_points:
            raise RuntimeError("start_point must be a point of the scene")
        if output_rgba is None:
            output_rgba = torch.empty((cam.height, cam.width), dtype=torch.uint32, device=dev)
        if output_rgba.numel() != cam.width * cam.height:
            raise RuntimeError("output_rgba must have width * height elements")
        if output_rgba.dtype != torch.uint32:
            raise RuntimeError("output_rgba must have uint32 dtype")
        if output_rgba.device != dev:
            raise RuntimeError("output_rgba must be on the scene's CUDA device")
        if not output_rgba.is_contiguous():
            raise RuntimeError("output_rgba must be contiguous")
        if diff_c.numel() * diff_c.element_size() < 8 * adj_c.numel():
            raise RuntimeError("adjacent_diff must hold one half4 per adjacency entry")
        table = _lib.CMapTable(None, None)
        if mode in ("depth", "intersections"):
            if cmap_table is None:
                raise RuntimeError(f"mode {mode!r} needs a cmap_table")
            ptrs, sizes = self._cmap_arrays(cmap_table, dev)
            table = _lib.CMapTable(ptrs.data_ptr(), sizes.data_ptr())
        vis = _lib.VisualizationSettings(_lib.VIS_MODES[mode], _lib.COLOR_MAPS[color_map],
                                         (ctypes.c_float * 3)(*[float(c) for c in bg_color]), int(bool(checker_bg)),
                                         float(max_depth), float(depth_quantile))
        settings = self._settings(weight_threshold, max_intersections)
        opts = self._opts(scene_key, None)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_trace_visualization_rgba8(
                self._handle, ctypes.byref(settings), ctypes.byref(vis), ctypes.byref(cam), ctypes.byref(table),
                num_points, 0, _ptr(points_c), _ptr(attributes_c), _ptr(adj_c), _ptr(off_c), _ptr(diff_c), start,
                _ptr(output_rgba), ctypes.byref(opts), stream))
        return output_rgba.view(cam.height, cam.width)

    # ---- the field at arbitrary points (rfb_sample_field): not part of the reference's Pipeline
    def sample_field(self, points, attributes, point_adjacency, point_adjacency_offsets, queries, directions=None,
                     hint=None):
        """The field at query points ``[..., 3]``: ``{"cell": uint32[...], "density": [...], "rgb": [..., 3]}`` --
        the cell of each query (as :func:`locate_points` finds it, ``hint`` likewise), its density (the attribute
        row's last column) and, when ``directions [..., 3]`` are given, the colour the tracer composites for that
        cell along a ray with that direction.  density and rgb are in the pipeline's attribute dtype; a query
        without a cell (a NaN coordinate) gets NaN.  Differentiable with respect to ``attributes`` through
        :class:`radfoam_b200.SampleField`."""
        self._validate_scene(points, attributes, point_adjacency, point_adjacency_offsets)
        if attributes is None:
            raise RuntimeError("sample_field needs the attributes (a bound parameter-form scene is not used here)")
        pts, attrs = points.detach().contiguous(), attributes.detach().contiguous()
        adj, off = point_adjacency.contiguous(), point_adjacency_offsets.contiguous()
        q, batch = _query_points(queries, pts.device)
        hints = _hints(hint, batch, pts.device)
        d = None
        if directions is not None:
            d = directions.detach()
            if d.dtype != torch.float32 or d.device != pts.device or tuple(d.shape) != batch + (3,):
                raise RuntimeError("directions must be float32 [..., 3] on the queries' device, one per query")
            d = d.contiguous()
        m = q.size(0)
        cell = torch.empty(batch, dtype=torch.uint32, device=pts.device)
        density = torch.empty(batch, dtype=self._dtype, device=pts.device)
        rgb = torch.empty(batch + (3,), dtype=self._dtype, device=pts.device) if d is not None else None
        with torch.cuda.device(pts.device):
            stream = torch.cuda.current_stream(pts.device).cuda_stream
            _lib.check(self._lib.rfb_sample_field(
                self._handle, _ptr(pts), pts.size(0), _ptr(attrs), _ptr(adj) if adj.numel() else None, _ptr(off),
                _ptr(q), m, _ptr(hints), _ptr(d), _ptr(cell), _ptr(density), _ptr(rgb), stream))
        out = {"cell": cell, "density": density}
        if rgb is not None:
            out["rgb"] = rgb
        return out

    def sample_field_backward(self, num_points, cell, directions=None, rgb=None, rgb_grad=None, density_grad=None):
        """Gradient of a :meth:`sample_field` call's outputs with respect to the attributes: ``[num_points, A]`` in
        the attribute dtype, summed in fp32 over the queries of each cell and rounded once.  ``rgb`` is the forward's
        colour output (its zeros mask the clamp); ``rgb_grad`` needs ``directions`` and ``rgb``.  The pipeline's
        own state (scene mirrors, walk tape, gradient accumulator) is not touched."""
        c = cell.detach().contiguous()
        if c.dtype != torch.uint32 or c.device.type != "cuda":
            raise RuntimeError("cell must be the uint32 CUDA tensor sample_field returned")
        batch, m = tuple(c.shape), c.numel()

        def per_query(name, t, cols, dtype):
            if t is None:
                return None
            t = t.detach()
            if t.dtype != dtype or t.device != c.device or tuple(t.shape) != batch + cols:
                raise RuntimeError(f"{name} must be {_dtype_name(dtype)} with shape {list(batch + cols)} "
                                   "on the cell's device")
            return t.contiguous()

        d = per_query("directions", directions, (3,), torch.float32)
        rgb_c = per_query("rgb", rgb, (3,), self._dtype)
        g_c = per_query("rgb_grad", rgb_grad, (3,), self._dtype)
        dg_c = per_query("density_grad", density_grad, (), self._dtype)
        if g_c is not None and (d is None or rgb_c is None):
            raise RuntimeError("rgb_grad needs the directions and the forward's rgb")
        attr_grad = torch.empty((int(num_points), self._attr_dim), dtype=self._dtype, device=c.device)
        with torch.cuda.device(c.device):
            stream = torch.cuda.current_stream(c.device).cuda_stream
            _lib.check(self._lib.rfb_sample_field_backward(
                self._handle, int(num_points), m, _ptr(c), _ptr(d), _ptr(rgb_c), _ptr(g_c), _ptr(dg_c),
                _ptr(attr_grad), stream))
        return attr_grad

    # ---- the density surface as Voronoi faces (rfb_surface_count / rfb_surface_write): not part of the reference
    def extract_surface(self, points, attributes, point_adjacency, point_adjacency_offsets, threshold=None,
                        inside=None, bounds=None):
        """The boundary between occupied and empty cells, as the exact Voronoi faces between them.

        Occupied cells are ``attributes[:, -1] > threshold`` or the bool ``[N]`` mask ``inside`` (pass exactly one).
        Every CSR entry ``(i, j)`` with ``i`` occupied, ``j`` empty and ``p_j != p_i`` gives the polygon where cell
        ``i`` -- clipped to ``bounds`` and to the bisector planes of its listed neighbours, the region the walk treats
        as cell ``i`` -- meets the bisector plane of ``(i, j)``, when it has at least 3 vertices.  Polygons come in
        CSR order, counter-clockwise seen from ``j`` (normals point out of the occupied cells), computed in float64
        and rounded once to float32; nothing is welded.  ``bounds = (lo[3], hi[3])`` defaults to the points'
        bounding box; the surface is open where occupied cells reach it.

        Returns ``{"vertices" f32[V, 3], "offsets" int64[P+1], "cells" uint32[P, 2], "rgb" [P, 3],
        "triangles" int64[V-2P, 3]}``: polygon ``k`` is ``vertices[offsets[k]:offsets[k+1]]`` between cells
        ``cells[k] = (i, j)``; ``rgb`` (attribute dtype) is cell ``i``'s colour along ``normalize(p_i - p_j)``, as
        :meth:`sample_field` gives it; ``triangles`` fan each polygon from its first vertex.

        The output sizes are read back from the device once (and, without ``bounds``, the bounding box), so the call
        synchronises with the current stream and cannot be captured in a CUDA graph.  Raises when a polygon needs more
        vertices than the kernels hold (32)."""
        self._validate_scene(points, attributes, point_adjacency, point_adjacency_offsets)
        if attributes is None:
            raise RuntimeError("extract_surface needs the attributes (a bound parameter-form scene is not used here)")
        if (threshold is None) == (inside is None):
            raise RuntimeError("extract_surface: pass exactly one of threshold and inside")
        pts, attrs = points.detach().contiguous(), attributes.detach().contiguous()
        if pts.dim() != 2:
            raise RuntimeError("points must have shape [N, 3]")
        adj, off = point_adjacency.contiguous(), point_adjacency_offsets.contiguous()
        dev, n = pts.device, pts.size(0)
        if adj.device != dev or off.device != dev or attrs.device != dev:
            raise RuntimeError("extract_surface: every tensor must be on the points' device")
        if inside is None:
            occupied = (attrs[:, -1] > float(threshold)).contiguous()
        else:
            if not isinstance(inside, torch.Tensor) or inside.dtype != torch.bool or inside.device != dev \
                    or tuple(inside.shape) != (n,):
                raise RuntimeError("inside must be a bool tensor [N] on the points' device")
            occupied = inside.detach().contiguous()
        box = _lib.Box()
        if bounds is None:
            if n:
                lo, hi = torch.stack([pts.amin(0), pts.amax(0)]).cpu().tolist()
            else:
                lo, hi = [0.0] * 3, [0.0] * 3
        else:
            lo, hi = (torch.as_tensor(b, dtype=torch.float32).detach().cpu().reshape(-1).tolist() for b in bounds)
            if len(lo) != 3 or len(hi) != 3:
                raise RuntimeError("bounds must be (lo[3], hi[3])")
        box.lo[:], box.hi[:] = lo, hi
        e = adj.numel()
        scratch = torch.empty((int(self._lib.rfb_surface_scratch_bytes(e)) + 7) // 8, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(self._lib.rfb_surface_count(
                _ptr(pts), n, e, _ptr(adj) if e else None, _ptr(off), _ptr(occupied), ctypes.byref(box),
                _ptr(scratch), stream))
            nv, npoly, over = (int(x) for x in scratch[:3].cpu().tolist())
            if over:
                raise RuntimeError(f"extract_surface: {over} polygons need more than 32 vertices; "
                                   "no surface was written")
            vertices = torch.empty((nv, 3), dtype=torch.float32, device=dev)
            offsets = torch.empty((npoly + 1,), dtype=torch.int64, device=dev)
            cells = torch.empty((npoly, 2), dtype=torch.uint32, device=dev)
            rgb = torch.empty((npoly, 3), dtype=self._dtype, device=dev)
            _lib.check(self._lib.rfb_surface_write(
                self._handle, _ptr(pts), n, _ptr(attrs), e, _ptr(adj) if e else None, _ptr(off), _ptr(occupied),
                ctypes.byref(box), _ptr(scratch), _ptr(vertices), _ptr(offsets), _ptr(cells), _ptr(rgb), stream))
        # fan triangulation: polygon k gives (o_k, o_k + t + 1, o_k + t + 2) for t < count_k - 2
        fan = torch.diff(offsets) - 2
        ntri = nv - 2 * npoly
        first = torch.repeat_interleave(offsets[:-1], fan, output_size=ntri)
        start = torch.repeat_interleave(torch.cumsum(fan, 0) - fan, fan, output_size=ntri)
        t = torch.arange(ntri, device=dev) - start
        triangles = torch.stack([first, first + t + 1, first + t + 2], -1)
        return {"vertices": vertices, "offsets": offsets, "cells": cells, "rgb": rgb, "triangles": triangles}

    # radfoam::prefetch_adjacent_diff (pipeline.h:50-56); handy for trace_benchmark callers
    def prefetch_adjacent_diff(self, points, point_adjacency, point_adjacency_offsets):
        points_c = points.contiguous()
        adj_c = point_adjacency.contiguous()
        off_c = point_adjacency_offsets.contiguous()
        out = torch.empty((adj_c.numel(), 4), dtype=torch.float16, device=points_c.device)
        with torch.cuda.device(points_c.device):
            stream = torch.cuda.current_stream(points_c.device).cuda_stream
            _lib.check(self._lib.rfb_prefetch_adjacent_diff(
                _ptr(points_c), points_c.size(0), adj_c.numel(), _ptr(adj_c), _ptr(off_c), _ptr(out),
                stream))
        return out


def _wrap_device_memory(ptr: int, shape, device) -> torch.Tensor:
    """Zero-copy float32 tensor over library-owned device memory."""

    class _Holder:
        pass

    h = _Holder()
    n = 1
    for s in shape:
        n *= int(s)
    h.__cuda_array_interface__ = {
        "shape": (n,), "typestr": "<f4", "data": (int(ptr), False), "version": 3,
    }
    t = torch.as_tensor(h, device=device)
    return t.view(*shape)


def nearest_point(points, queries):
    """Entry cells: index of the nearest point of each query, ``uint32[M]`` (exact, tiled brute force on
    the GPU; stands in for ``radfoam.nn(points, aabb_tree, queries)`` where the tracer needs it,
    radfoam_model/scene.py:224-234, benchmark.py:88-89)."""
    pts = points.detach().contiguous()
    q = queries.detach().reshape(-1, 3).to(torch.float32).contiguous()
    if pts.dtype != torch.float32 or pts.size(-1) != 3:
        raise RuntimeError("points must be float32 [N, 3]")
    if pts.device.type != "cuda" or q.device != pts.device:
        raise RuntimeError("points and queries must be on the same CUDA device")
    out = torch.empty((q.size(0),), dtype=torch.uint32, device=pts.device)
    with torch.cuda.device(pts.device):
        stream = torch.cuda.current_stream(pts.device).cuda_stream
        _lib.check(_lib.load().rfb_nearest_point(_ptr(pts), pts.size(0), _ptr(q), q.size(0), _ptr(out), stream))
    return out


def starting_points(rays, points):
    """Start cell of every ray (mirror of RadFoamScene.get_starting_point, scene.py:224-234): the nearest point
    of each ray's origin, in the rays' batch shape.  One library call -- device-side de-duplication of the
    origins (no ``torch.unique`` sort over the rays), one exact lookup per distinct origin, no host sync."""
    pts = points.detach().contiguous()
    r = rays.detach()
    if pts.dtype != torch.float32 or pts.size(-1) != 3:
        raise RuntimeError("points must be float32 [N, 3]")
    if r.size(-1) != 6 or r.dtype != torch.float32:
        raise RuntimeError("rays must be float32 [..., 6]")
    if pts.device.type != "cuda" or r.device != pts.device:
        raise RuntimeError("points and rays must be on the same CUDA device")
    r = r.contiguous()
    out = torch.empty(r.shape[:-1], dtype=torch.uint32, device=pts.device)
    with torch.cuda.device(pts.device):
        stream = torch.cuda.current_stream(pts.device).cuda_stream
        _lib.check(_lib.load().rfb_start_points(_ptr(pts), pts.size(0), _ptr(r), r.numel() // 6, _ptr(out), stream))
    return out


def _query_points(queries, device):
    """(contiguous float32 [M, 3] view, batch shape) of query points [..., 3]."""
    if queries.dtype != torch.float32 or queries.size(-1) != 3:
        raise RuntimeError("queries must be float32 [..., 3]")
    if queries.device != device:
        raise RuntimeError("queries must be on the same CUDA device as points")
    return queries.detach().contiguous().view(-1, 3), tuple(queries.shape[:-1])


def _hints(hint, batch, device):
    """uint32 [M] start cells of the walk from ``hint``: None, an int (one cell for every query) or a uint32 / int
    tensor of the queries' batch shape.  Values >= num_points leave the seed to the library."""
    if hint is None:
        return None
    if not isinstance(hint, torch.Tensor):
        h = int(hint)
        if h < 0:
            raise RuntimeError("hint must be a non-negative cell index")
        h = min(h, 0xFFFFFFFF)
        m = 1
        for s in batch:
            m *= s
        return torch.full((m,), h, dtype=torch.int64, device=device).to(torch.uint32)
    if tuple(hint.shape) != batch:
        raise RuntimeError(f"hint must have the queries' batch shape {list(batch)}")
    if hint.device != device:
        raise RuntimeError("hint must be on the same CUDA device as points")
    if hint.dtype == torch.uint32:
        return hint.detach().contiguous().view(-1)
    if hint.dtype in (torch.int32, torch.int64):
        return hint.detach().reshape(-1).clamp(0, 0xFFFFFFFF).to(torch.int64).to(torch.uint32)
    raise RuntimeError("hint must be an integer tensor (uint32, int32 or int64)")


def _csr(points, point_adjacency, point_adjacency_offsets):
    """Validated contiguous (points [N, 3], adjacency, offsets) of a foam, as farthest_neighbor takes them."""
    if points.device.type != "cuda":
        raise RuntimeError("points must be on CUDA device")
    pts = points.detach().contiguous()
    if pts.dtype != torch.float32:
        raise RuntimeError("points must have float32 dtype")
    if pts.dim() != 2 or pts.size(-1) != 3:
        raise RuntimeError("points must have shape [N, 3]")
    adj = point_adjacency.detach().contiguous()
    off = point_adjacency_offsets.detach().contiguous()
    for name, t in (("point_adjacency", adj), ("point_adjacency_offsets", off)):
        if t.dtype != torch.uint32:
            raise RuntimeError(f"{name} must have uint32 dtype")
        if t.device != pts.device:
            raise RuntimeError(f"{name} must be on the same device as points")
    if off.numel() != pts.size(0) + 1:
        raise RuntimeError("point_adjacency_offsets must have num_points + 1 elements")
    return pts, adj, off


def locate_points(points, point_adjacency, point_adjacency_offsets, queries, hint=None):
    """Cell of every query point ``[..., 3]`` (``uint32`` in the queries' batch shape) by a greedy walk over the
    adjacency graph: the nearest point, as :func:`nearest_point` defines it, when the adjacency is the Delaunay
    graph of ``points`` (up to fp32 near-ties); a local minimum of the distance over the graph when the points have
    moved since it was built.  ``hint``: a start cell per query (e.g. the ``depth_indices`` of the ray that reached
    it) or one int for all; a hint that is not a cell, or none, lets the library seed the walk.  A query with a NaN
    coordinate gets UINT32_MAX.  Costs a few row scans per query -- use it for many distinct queries, where
    :func:`nearest_point` costs N distances each."""
    pts, adj, off = _csr(points, point_adjacency, point_adjacency_offsets)
    q, batch = _query_points(queries, pts.device)
    hints = _hints(hint, batch, pts.device)
    out = torch.empty(batch, dtype=torch.uint32, device=pts.device)
    if q.size(0) == 0:
        return out
    if pts.size(0) == 0:
        raise RuntimeError("locate_points: empty point set")
    with torch.cuda.device(pts.device):
        stream = torch.cuda.current_stream(pts.device).cuda_stream
        _lib.check(_lib.load().rfb_locate_points(_ptr(pts), pts.size(0), _ptr(adj) if adj.numel() else None,
                                                 _ptr(off), _ptr(q), q.size(0), _ptr(hints), _ptr(out), stream))
    return out


def farthest_neighbor(points, point_adjacency, point_adjacency_offsets):
    """``radfoam.farthest_neighbor`` (torch_bindings/triangulation_bindings.cpp:184-216): returns
    ``(indices uint32[N], cell_radius float32[N])`` -- per point, the adjacent point farthest from it and half
    the mean neighbour distance; what ``prune_and_densify`` reads (radfoam_model/scene.py:434-461)."""
    if points.device.type != "cuda":
        raise RuntimeError("points must be on CUDA device")
    pts = points.detach().contiguous()
    if pts.dtype != torch.float32:
        raise RuntimeError("unsupported scalar type")  # triangulation_ops.cu:83-85
    if pts.dim() < 2 or pts.size(-1) != 3:
        raise RuntimeError("points must have shape [N, 3]")
    adj = point_adjacency.detach().contiguous()
    off = point_adjacency_offsets.detach().contiguous()
    for name, t in (("point_adjacency", adj), ("point_adjacency_offsets", off)):
        if t.dtype != torch.uint32:
            raise RuntimeError(f"{name} must have uint32 dtype")
        if t.device != pts.device:
            raise RuntimeError(f"{name} must be on the same device as points")
    num_points = pts.size(0)
    if off.numel() != num_points + 1:
        raise RuntimeError("point_adjacency_offsets must have num_points + 1 elements")
    shape = tuple(pts.shape[:-1])
    indices = torch.empty(shape, dtype=torch.uint32, device=pts.device)
    cell_radius = torch.empty(shape, dtype=torch.float32, device=pts.device)
    with torch.cuda.device(pts.device):
        stream = torch.cuda.current_stream(pts.device).cuda_stream
        _lib.check(_lib.load().rfb_farthest_neighbor(_ptr(pts), num_points, _ptr(adj), _ptr(off), _ptr(indices),
                                                     _ptr(cell_radius), stream))
    return indices, cell_radius


def create_pipeline(sh_degree, attr_dtype="float32") -> Pipeline:
    """radfoam.create_pipeline (pipeline_bindings.cpp:587-590, 669-672)."""
    if not isinstance(sh_degree, int) or sh_degree < 0 or sh_degree > 3:
        raise RuntimeError("Unsupported SH degree")
    return Pipeline(sh_degree, attr_dtype)


def launch_count() -> int:
    return int(_lib.load().rfb_launch_count())


def reset_launch_count() -> None:
    _lib.load().rfb_reset_launch_count()


def device_alloc_counts() -> tuple[int, int]:
    """(cudaMalloc, cudaFree) calls the native library has made so far (steady state: constant)."""
    a, f = ctypes.c_uint64(), ctypes.c_uint64()
    _lib.load().rfb_device_alloc_counts(ctypes.byref(a), ctypes.byref(f))
    return int(a.value), int(f.value)
