"""Autograd op over a :class:`radfoam_b200.Pipeline`.

Call contract = ``radfoam_model/render.py::TraceRays`` (lines 10-122): nine positional
arguments ``(pipeline, points, attributes, point_adjacency, point_adjacency_offsets, rays,
start_point, depth_quantiles, return_contribution)`` in, the 5-tuple ``(rgba, depth,
contribution, num_intersections, errbox)`` out, gradients for ``points`` and ``attributes`` (and, an
extension, for ``rays`` when they require grad: ``Pipeline.trace_backward(return_ray_grad=True)``), and
``errbox.ray_error`` (set by the caller between forward and backward) -> ``errbox.point_error``
(scene.py:497-548 uses that side channel for the densification error map).  The reference's own file
runs unmodified on a ``Pipeline`` too (tests/test_gpu_reference_op.py); this op is the native
counterpart, written for this library:

  * tensors go through ``save_for_backward`` (the forward's own ``rgba`` output included), so no
    tensor -> grad_fn -> ctx -> tensor reference cycle is left for Python's cyclic collector --
    the graph of a step is freed by reference counting the moment the loss goes out of scope;
  * ``apply`` notes whether autograd was recording when the op was called and tells the pipeline,
    which records the walk tape only when a backward can follow (inside ``Function.forward`` grad
    mode is always off, so the pipeline cannot see that by itself);
  * non-finite gradient entries are zeroed in the backward kernel's epilogue
    (``scrub_nonfinite=True``), not by two masked passes over the gradients afterwards.
"""
from __future__ import annotations

import torch


class ErrorBox:
    """Side channel of the op: ``ray_error`` in (per-ray weights), ``point_error`` out."""

    __slots__ = ("ray_error", "point_error")

    def __init__(self):
        self.ray_error = None
        self.point_error = None


class TraceRays(torch.autograd.Function):
    @classmethod
    def apply(cls, pipeline, *args):
        noted = hasattr(pipeline, "autograd_recording")
        if noted:
            before, pipeline.autograd_recording = pipeline.autograd_recording, torch.is_grad_enabled()
        try:
            return super().apply(pipeline, *args)
        finally:
            if noted:
                pipeline.autograd_recording = before

    @staticmethod
    def forward(ctx, pipeline, points, attributes, point_adjacency, point_adjacency_offsets, rays,
                start_point, depth_quantiles, return_contribution):
        out = pipeline.trace_forward(points, attributes, point_adjacency, point_adjacency_offsets, rays,
                                     start_point, depth_quantiles=depth_quantiles,
                                     return_contribution=return_contribution)
        rgba = out["rgba"]
        saved = [points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point, rgba]
        ctx.with_depth = depth_quantiles is not None
        if ctx.with_depth:
            saved += [depth_quantiles, out["depth_indices"]]
        ctx.save_for_backward(*saved)
        ctx.pipeline = pipeline
        ctx.errbox = box = ErrorBox()
        return rgba, out.get("depth"), out.get("contribution"), out["num_intersections"], box

    @staticmethod
    def backward(ctx, grad_rgba, grad_depth, _grad_contribution, _grad_num_intersections, _grad_box):
        saved = ctx.saved_tensors
        points, attributes, adjacency, offsets, rays, start_point, rgba = saved[:7]
        quantiles, depth_indices = (saved[7], saved[8]) if ctx.with_depth else (None, None)
        if ctx.with_depth and grad_depth is None:  # depth was returned but not used by the loss
            grad_depth = torch.zeros_like(quantiles)
        box = ctx.errbox
        want_rays = ctx.needs_input_grad[5]
        grads = ctx.pipeline.trace_backward(points, attributes, adjacency, offsets, rays, start_point, rgba,
                                            grad_rgba, quantiles, depth_indices, grad_depth, box.ray_error,
                                            scrub_nonfinite=True, return_ray_grad=want_rays)
        box.point_error = grads.get("point_error")
        ctx.pipeline = None
        return ((None, grads["points_grad"], grads["attr_grad"], None, None,
                 grads["ray_grad"] if want_rays else None) + (None,) * 3)


class SampleField(torch.autograd.Function):
    """The field at query points, differentiable with respect to the attributes:
    ``SampleField.apply(pipeline, points, attributes, point_adjacency, point_adjacency_offsets, queries, directions,
    hint)`` -> ``(density [...], rgb [..., 3] or None, cell uint32 [...])`` (see ``Pipeline.sample_field``).  The
    field is piecewise constant in space, so the gradient with respect to ``points`` is zero almost everywhere
    (returned as None); gradients with respect to ``queries`` and ``directions`` are not computed, and asking for
    them is an error."""

    @staticmethod
    def forward(ctx, pipeline, points, attributes, point_adjacency, point_adjacency_offsets, queries,
                directions=None, hint=None):
        for name, t in (("queries", queries), ("directions", directions)):
            if t is not None and t.requires_grad:
                raise RuntimeError(f"SampleField: gradients with respect to {name} are not computed; pass "
                                   f"{name}.detach()")
        out = pipeline.sample_field(points, attributes, point_adjacency, point_adjacency_offsets, queries,
                                    directions, hint)
        rgb = out.get("rgb")
        ctx.save_for_backward(out["cell"], directions, rgb)
        ctx.pipeline, ctx.num_points = pipeline, points.shape[0]
        ctx.mark_non_differentiable(out["cell"])
        return out["density"], rgb, out["cell"]

    @staticmethod
    def backward(ctx, grad_density, grad_rgb, _grad_cell):
        cell, directions, rgb = ctx.saved_tensors
        attr_grad = None
        if ctx.needs_input_grad[2]:
            attr_grad = ctx.pipeline.sample_field_backward(ctx.num_points, cell, directions, rgb,
                                                           None if rgb is None else grad_rgb, grad_density)
        ctx.pipeline = None
        return None, None, attr_grad, None, None, None, None, None


class TraceRaysParams(torch.autograd.Function):
    """The render op taken one step further out: ``RadFoamScene.forward`` = ``get_trace_data`` (a ``cat`` and a
    softplus, scene.py:202-217) followed by ``TraceRays`` (scene.py:236-261).  Here the model's PARAMETERS go in --
    ``(pipeline, points, att_dc, att_sh, density, activation_scale, point_adjacency, point_adjacency_offsets, rays,
    start_point, depth_quantiles, return_contribution)`` -- and their gradients come out; the attribute matrix and
    its gradient are never materialised (the re-layout and finalize kernels read / write the parameters directly).
    Same outputs as :class:`TraceRays`."""

    @classmethod
    def apply(cls, pipeline, *args):
        before, pipeline.autograd_recording = pipeline.autograd_recording, torch.is_grad_enabled()
        try:
            return super().apply(pipeline, *args)
        finally:
            pipeline.autograd_recording = before

    @staticmethod
    def forward(ctx, pipeline, points, att_dc, att_sh, density, activation_scale, point_adjacency,
                point_adjacency_offsets, rays, start_point, depth_quantiles, return_contribution):
        pipeline.bind_scene_params(att_dc, att_sh, density, activation_scale)
        try:
            out = pipeline.trace_forward(points, None, point_adjacency, point_adjacency_offsets, rays, start_point,
                                         depth_quantiles=depth_quantiles, return_contribution=return_contribution)
        finally:
            pipeline.bind_scene_params(None, None, None)
        rgba = out["rgba"]
        saved = [points, att_dc, att_sh, density, point_adjacency, point_adjacency_offsets, rays, start_point, rgba]
        ctx.with_depth = depth_quantiles is not None
        if ctx.with_depth:
            saved += [depth_quantiles, out["depth_indices"]]
        ctx.save_for_backward(*saved)
        ctx.pipeline, ctx.activation_scale = pipeline, activation_scale
        ctx.errbox = box = ErrorBox()
        return rgba, out.get("depth"), out.get("contribution"), out["num_intersections"], box

    @staticmethod
    def backward(ctx, grad_rgba, grad_depth, _grad_contribution, _grad_num_intersections, _grad_box):
        saved = ctx.saved_tensors
        points, att_dc, att_sh, density, adjacency, offsets, rays, start_point, rgba = saved[:9]
        quantiles, depth_indices = (saved[9], saved[10]) if ctx.with_depth else (None, None)
        pipeline, box = ctx.pipeline, ctx.errbox
        want_rays = ctx.needs_input_grad[8]
        pipeline.bind_scene_params(att_dc, att_sh, density, ctx.activation_scale)
        try:
            grads = pipeline.trace_backward_params(points, adjacency, offsets, rays, start_point, rgba, grad_rgba,
                                                   quantiles, depth_indices, grad_depth, box.ray_error,
                                                   scrub_nonfinite=True, return_ray_grad=want_rays)
        finally:
            pipeline.bind_scene_params(None, None, None)
        box.point_error = grads.get("point_error")
        ctx.pipeline = None
        return ((None, grads["points_grad"], grads["att_dc_grad"], grads["att_sh_grad"], grads["density_grad"])
                + (None,) * 3 + (grads.get("ray_grad"),) + (None,) * 3)
