"""Ray-sharded data parallelism over the GPUs of one box (SURVEY.md §8e).

The reference is single-GPU; this is the one thing the build adds around the hot path.
One process per GPU (torch.distributed, NCCL over NVLink/NVSwitch).  The scene buffers are
replicated on every rank; rays are dealt to ranks

  * image batches ``[H, W, 6]``: as interleaved bands of ``band`` (default 8) full-width
    pixel rows, band b going to rank ``b % world`` -- every rank samples the whole frame
    (load balance: sky and surface regions cost very different numbers of cells) and its
    shard is still a row-major image, so the kernels' 8x4 warp tiles stay coherent;
  * unordered batches ``[R, 6]``: as contiguous chunks.

Forward needs no collective (disjoint pixels).  Backward scatter-adds into an fp32
accumulator ``[N, grad_row]`` on each rank; ONE exchange step sums it over the ranks and writes
the reference-layout gradients (non-finite entries zeroed AFTER the sum, as
radfoam_model/render.py:98-99 does after its single-GPU kernel, SURVEY.md Appendix A.5 item 6):
a fused peer-memory kernel over NVLink where available, else an NCCL all-reduce + finalize.

The partition / reassembly helpers are pure index arithmetic on torch tensors and are
exercised on CPU with gloo (tests/test_sharded_gloo.py).
"""
from __future__ import annotations

import ctypes
import os

import torch
import torch.distributed as dist


def band_rows(height: int, rank: int, world: int, band: int = 8) -> torch.Tensor:
    """Row indices (ascending) of the image rows rank ``rank`` owns."""
    rows = torch.arange(height)
    return rows[(rows // band) % world == rank]


def shard_image(t: torch.Tensor, rank: int, world: int, band: int = 8) -> torch.Tensor:
    """``t`` is ``[H, W, ...]``; returns this rank's rows ``[h_r, W, ...]`` (a copy)."""
    if world == 1:
        return t
    idx = band_rows(t.shape[0], rank, world, band).to(t.device)
    return t.index_select(0, idx)


def shard_flat(t: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """``t`` is ``[R, ...]``; contiguous chunk ``rank`` of ``world`` (sizes differ by <= 1)."""
    if world == 1:
        return t
    n = t.shape[0]
    lo = (n * rank) // world
    hi = (n * (rank + 1)) // world
    return t[lo:hi]


def unshard_image(parts: list[torch.Tensor], height: int, band: int = 8) -> torch.Tensor:
    """Inverse of :func:`shard_image` given every rank's part in rank order."""
    world = len(parts)
    if world == 1:
        return parts[0]
    out = torch.empty((height,) + tuple(parts[0].shape[1:]), dtype=parts[0].dtype, device=parts[0].device)
    for r, p in enumerate(parts):
        out.index_copy_(0, band_rows(height, r, world, band).to(p.device), p)
    return out


class ShardedTracer:
    """Wraps a Pipeline (or any object with its trace_* methods) for ray-sharded use.

    ``trace_forward`` / ``trace_backward`` take THIS RANK'S shard of the rays (see
    :func:`shard_image` / :func:`shard_flat`) and the full, replicated scene; backward
    returns the full (reduced) gradients on every rank.

    The exchange step.  Default on NCCL/CUDA: ONE kernel per rank that sums the peers' accumulators over
    NVLink, finalizes and stores the result into every rank's output arrays
    (``rfb_reduce_finalize_peers``; the buffers live in torch symmetric memory, the two cross-GPU barriers
    are its signal-pad barriers).  Fallback (CPU/gloo, no peer access, ``fused_reduce=False`` or
    ``RFB_FUSED_REDUCE=0``): ``all_reduce`` of the accumulator, then the local finalize kernel.
    All ranks agree on the path (a MIN all-reduce of the set-up outcome).
    """

    def __init__(self, pipeline, group=None, band: int = 8, fused_reduce: bool | None = None):
        self.pipeline = pipeline
        self.group = group
        self.band = band
        if dist.is_available() and dist.is_initialized():
            self.rank = dist.get_rank(group)
            self.world = dist.get_world_size(group)
        else:
            self.rank, self.world = 0, 1
        if fused_reduce is None:
            fused_reduce = os.environ.get("RFB_FUSED_REDUCE", "1") != "0"
        self.fused_reduce = fused_reduce
        self._peer = None          # set-up state of the fused path; False = tried and unavailable
        self.profile_reduce = False  # record CUDA events around the parts of the fused exchange (bench.py)
        self.last_reduce_events = None
        self.fused_reduce_error = None

    # -- partition helpers bound to this rank
    def shard(self, t: torch.Tensor, image: bool) -> torch.Tensor:
        return (shard_image(t, self.rank, self.world, self.band) if image
                else shard_flat(t, self.rank, self.world))

    def gather_image(self, local: torch.Tensor, height: int) -> torch.Tensor:
        """All ranks receive the full ``[H, W, ...]`` image assembled from the shards."""
        if self.world == 1:
            return local
        sizes = [int(band_rows(height, r, self.world, self.band).numel()) for r in range(self.world)]
        rows = max(sizes)  # all_gather wants equal shapes: pad the short shards, trim after
        padded = local
        if local.shape[0] != rows:
            padded = torch.zeros((rows,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
            padded[:local.shape[0]] = local
        parts = [torch.empty_like(padded) for _ in range(self.world)]
        dist.all_gather(parts, padded.contiguous(), group=self.group)
        return unshard_image([p[:s] for p, s in zip(parts, sizes)], height, self.band)

    # -- the exchange step
    def reduction_name(self) -> str:
        if self.world == 1:
            return "no collective"
        if self._peer and self._peer["multicast"]:
            return ("one fused reduce+finalize kernel per rank over NVSwitch multicast (multimem.ld_reduce / "
                    "multimem.st on symmetric memory)")
        if self._peer:
            return "one fused peer-memory reduce+finalize kernel per rank (NVLink, symmetric memory)"
        return "one NCCL all-reduce"

    def last_reduce_ms(self):
        """Durations of the last fused exchange on this rank (after a synchronize): wait for the slowest rank's
        backward (barrier), the peer kernel, the closing barrier, the copies out of symmetric memory."""
        ev = self.last_reduce_events
        if not ev:
            return None
        names = ("barrier_all_accumulators_complete", "peer_reduce_finalize_kernel", "barrier_all_stores_landed",
                 "copy_out_of_symmetric_memory")
        return {n: round(float(ev[i].elapsed_time(ev[i + 1])), 4) for i, n in enumerate(names)}

    def _peer_setup(self, num_points: int, device):
        """Symmetric buffers [accumulator | attr_grad | points_grad] + peer pointer tables, once per size."""
        st = self._peer
        if st is False or (st and st["num_points"] == num_points):
            return st
        pipe = self.pipeline
        ok, err, st = True, None, None
        try:
            if not (self.fused_reduce and device.type == "cuda" and dist.get_backend(self.group) == "nccl"
                    and hasattr(pipe, "set_grad_accumulator")):
                raise RuntimeError("fused reduction needs CUDA + NCCL and a radfoam_b200.Pipeline")
            import torch.distributed._symmetric_memory as symm

            gr, adim = pipe.grad_row_floats(), pipe.attribute_dim()
            half = pipe.attribute_type() == torch.float16
            acc_f = num_points * gr
            attr_f = (num_points * adim * (2 if half else 4) + 15) // 16 * 4   # floats, 16-byte granules
            pts_f = (num_points * 3 + 3) // 4 * 4
            group = self.group if self.group is not None else dist.group.WORLD
            enable = getattr(symm, "enable_symm_mem_for_group", None)
            if enable is not None:
                try:
                    enable(group.group_name)
                except Exception:  # noqa: BLE001  (deprecated no-op in newer torch)
                    pass
            buf = symm.empty(acc_f + attr_f + pts_f, dtype=torch.float32, device=device)
            hdl = symm.rendezvous(buf, group)
            bases = [int(p) for p in hdl.buffer_ptrs]
            arr = lambda off: (ctypes.c_void_p * self.world)(*[b + 4 * off for b in bases])  # noqa: E731
            attr_view = buf[acc_f:acc_f + attr_f]
            attr_view = (attr_view.view(torch.float16) if half else attr_view)[:num_points * adim].view(num_points, adim)
            mc_base = int(getattr(hdl, "multicast_ptr", 0) or 0)
            multicast = None
            # NVSwitch multicast (NVLS) when available -- from 8 ranks on: per GPU and direction it moves
            # (1 + 1/W) accumulator sizes instead of 2 (W-1)/W, at less throughput per byte.
            want = os.environ.get("RFB_MULTICAST")
            if mc_base and (want == "1" or (want is None and self.world >= 8)):
                multicast = (mc_base, mc_base + 4 * acc_f, mc_base + 4 * (acc_f + attr_f))
            st = dict(num_points=num_points, buf=buf, hdl=hdl, multicast=multicast,
                      acc=buf[:acc_f].view(num_points, gr),
                      attr=attr_view, pts=buf[acc_f + attr_f:acc_f + attr_f + num_points * 3].view(num_points, 3),
                      peer_acc=arr(0), peer_attr=arr(acc_f), peer_pts=arr(acc_f + attr_f))
        except Exception as e:  # noqa: BLE001
            ok, err = False, repr(e)
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            self.fused_reduce_error = err or "another rank could not set up symmetric memory"
            if self._peer:
                self.pipeline.set_grad_accumulator(None)
            self._peer = False
            return False
        self._peer = st
        pipe.set_grad_accumulator(st["acc"])
        return st

    def reduce_and_finalize(self, num_points: int, device, scrub_nonfinite: bool = True, acc=None):
        """After ``trace_backward_accumulate`` on every rank (``acc`` = what it returned): ``(points_grad,
        attr_grad)`` summed over the ranks."""
        pipe = self.pipeline
        if self.world == 1:
            return pipe.trace_backward_finalize(num_points, device, scrub_nonfinite=scrub_nonfinite)
        st = self._peer
        if st:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)] if self.profile_reduce else None
            mark = (lambda i: ev[i].record()) if ev else (lambda i: None)
            mark(0)
            st["hdl"].barrier(channel=0)   # every rank's accumulator is complete
            mark(1)
            pipe.reduce_finalize_peers(self.world, self.rank, num_points, st["peer_acc"], st["peer_attr"],
                                       st["peer_pts"], device, scrub_nonfinite=scrub_nonfinite,
                                       multicast=st["multicast"])
            mark(2)
            st["hdl"].barrier(channel=1)   # every rank's stores have landed; accumulators may be reused
            mark(3)
            out = st["pts"].clone(), st["attr"].clone()
            mark(4)
            if ev:
                self.last_reduce_events = ev
            return out
        dist.all_reduce(acc if acc is not None else pipe.grad_accumulator(device), op=dist.ReduceOp.SUM,
                        group=self.group)
        return pipe.trace_backward_finalize(num_points, device, scrub_nonfinite=scrub_nonfinite)

    # -- the hot path
    def trace_forward(self, *args, **kwargs):
        return self.pipeline.trace_forward(*args, **kwargs)

    def trace_backward(self, points, attributes, point_adjacency, point_adjacency_offsets, rays,
                       start_point, rgb_out, grad_in, depth_quantiles=None, depth_indices=None,
                       depth_grad_in=None, ray_error=None, weight_threshold=None,
                       max_intersections=None, scrub_nonfinite=True):
        if self.world == 1:
            return self.pipeline.trace_backward(
                points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point,
                rgb_out, grad_in, depth_quantiles, depth_indices, depth_grad_in, ray_error,
                weight_threshold, max_intersections, scrub_nonfinite=scrub_nonfinite)
        if self._peer is None or (self._peer and self._peer["num_points"] != points.shape[0]):
            self._peer_setup(points.shape[0], rays.device)
        acc, point_error = self.pipeline.trace_backward_accumulate(
            points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point, rgb_out,
            grad_in, depth_quantiles, depth_indices, depth_grad_in, ray_error, weight_threshold,
            max_intersections)
        # the single exchange step of the path: per-point gradient sum over ranks
        points_grad, attr_grad = self.reduce_and_finalize(points.shape[0], rays.device, scrub_nonfinite, acc)
        if point_error is not None:
            dist.all_reduce(point_error, op=dist.ReduceOp.SUM, group=self.group)
        # ray gradients are not computed by the sharded path: ray_grad stays unwritten, as in the reference
        out = {"points_grad": points_grad, "attr_grad": attr_grad, "ray_grad": torch.empty_like(rays)}
        if point_error is not None:
            out["point_error"] = point_error
        return out


class ShardedTraceRays(torch.autograd.Function):
    """The render op (radfoam_b200/render.py) over a ShardedTracer: forward on the local ray shard,
    backward yields the all-reduced scene gradients on every rank.  Returns
    ``(rgba, depth, contribution, num_intersections)`` of the local shard.  Unlike ``TraceRays`` it does not
    compute ray gradients: the gradient for ``rays`` is always ``None``."""

    @classmethod
    def apply(cls, tracer, *args):
        pipe = tracer.pipeline
        noted = hasattr(pipe, "autograd_recording")
        if noted:
            before, pipe.autograd_recording = pipe.autograd_recording, torch.is_grad_enabled()
        try:
            return super().apply(tracer, *args)
        finally:
            if noted:
                pipe.autograd_recording = before

    @staticmethod
    def forward(ctx, tracer, points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point,
                depth_quantiles, return_contribution):
        out = tracer.trace_forward(points, attributes, point_adjacency, point_adjacency_offsets, rays,
                                   start_point, depth_quantiles=depth_quantiles,
                                   return_contribution=return_contribution)
        saved = [points, attributes, point_adjacency, point_adjacency_offsets, rays, start_point, out["rgba"]]
        ctx.with_depth = depth_quantiles is not None
        if ctx.with_depth:
            saved += [depth_quantiles, out["depth_indices"]]
        ctx.save_for_backward(*saved)  # no output tensor on ctx itself: that would be a reference cycle
        ctx.tracer = tracer
        return out["rgba"], out.get("depth"), out.get("contribution"), out["num_intersections"]

    @staticmethod
    def backward(ctx, grad_rgba, grad_depth, _grad_contribution, _grad_num_intersections):
        saved = ctx.saved_tensors
        pts, attrs, adj, off, rays, start, rgba = saved[:7]
        dq, didx = (saved[7], saved[8]) if ctx.with_depth else (None, None)
        res = ctx.tracer.trace_backward(pts, attrs, adj, off, rays, start, rgba, grad_rgba, dq, didx, grad_depth,
                                        scrub_nonfinite=True)
        ctx.tracer = None
        return (None, res["points_grad"], res["attr_grad"]) + (None,) * 6
