"""Per-entry checks of full-size backward launches against the float64 model (tests/model64.py), by masking the
upstream gradients to a chosen set S of rays.

The backward is linear in its upstream gradients ``grad_rgba``, ``grad_depth`` and ``ray_error``.  A full-frame
launch whose upstream is zero on every ray outside S has, in every entry of ``points_grad``, ``attr_grad`` and
``point_error``, the model's sum over S alone, so the model only has to trace S (as a flat batch).  The launch keeps
its full-size routing: the walk, the ``MATCH.ANY`` groups, the gradient cache, the bulk-versus-cache choice and
the tape replay do not depend on gradient values (a lane whose colour gradient is zero sends only its density
slot).  Every scene row is compared, rows that no ray of S touches must be exactly zero, and ``ray_grad`` must be
exactly zero on every ray outside S.

``contribution`` is a forward output summed over every ray and cannot be masked; it is not compared here.

The frame is an image: rays [H, W, 6], tiled by the kernels into 8x4-pixel warp tiles and 16x8-pixel CTA tiles
(radfoam_b200/csrc/foam_device.cuh).  Ray sets are flat indices y * W + x into it."""
from __future__ import annotations

import numpy as np

import model64 as M
import model64_rays as MR

WARP_W, WARP_H = 8, 4
CTA_W, CTA_H = 16, 8
FORWARD = ("rgba", "depth", "depth_indices", "num_intersections")
SCATTER = ("points_grad", "attr_grad", "point_error")


def cta_count(height: int, width: int) -> int:
    """CTAs of an image launch (one 16x8-pixel tile each)."""
    return -(-width // CTA_W) * -(-height // CTA_H)


# ---- ray sets ------------------------------------------------------------------------------------------
def block(height: int, width: int, x0: int, y0: int, w: int, h: int) -> np.ndarray:
    """The w x h pixels from (x0, y0)."""
    assert 0 <= x0 and x0 + w <= width and 0 <= y0 and y0 + h <= height
    ys, xs = np.mgrid[y0:y0 + h, x0:x0 + w]
    return (ys * width + xs).reshape(-1)


def one_lane_per_warp(height: int, width: int, count: int) -> np.ndarray:
    """One pixel in each of ``count`` warp tiles spread evenly over the frame: in the t-th chosen tile the pixel at
    offset (t mod 8, (t div 8) mod 4), so every lane position occurs."""
    tiles_x, tiles_y = width // WARP_W, height // WARP_H
    tiles = np.unique(np.linspace(0, tiles_x * tiles_y - 1, count).astype(np.int64))
    t = np.arange(tiles.size)
    x = (tiles % tiles_x) * WARP_W + t % WARP_W
    y = (tiles // tiles_x) * WARP_H + (t // WARP_W) % WARP_H
    return y * width + x


def longest(num_intersections: np.ndarray, count: int) -> np.ndarray:
    """The ``count`` rays with the most intersections (ties to the lower index)."""
    n = num_intersections.reshape(-1).astype(np.int64)
    return np.sort(np.lexsort((np.arange(n.size), -n))[:count])


def budget_exhausted(num_intersections: np.ndarray, max_intersections: int, count: int) -> np.ndarray:
    """``count`` of the rays that ran out of steps (n == max_intersections + 1), spread evenly over them."""
    hit = np.flatnonzero(num_intersections.reshape(-1) == max_intersections + 1)
    assert hit.size >= count, (hit.size, count)
    return hit[np.unique(np.linspace(0, hit.size - 1, count).astype(np.int64))]


# ---- the harness ---------------------------------------------------------------------------------------
class MaskedFrame:
    """A full frame (rays [H, W, 6], start [H, W], quantiles [H, W, Q] or None) and the set ``sel`` of flat ray
    indices whose upstream gradients are kept.  ``shift`` scatters S's upstream that many rays further along
    (a deliberately wrong harness, for showing that the check is not vacuous)."""

    def __init__(self, rays, start, quantiles, sel, shift: int = 0):
        self.rays, self.start, self.quantiles = rays, start, quantiles
        self.shape = rays.shape[:-1]
        self.size = int(np.prod(self.shape))
        self.sel = np.unique(np.asarray(sel, dtype=np.int64))
        self.shift = shift
        assert self.sel[0] >= 0 and self.sel[-1] + shift < self.size and self.sel[0] + shift >= 0

    def batch(self, a):
        """S's rows of a per-ray frame array, as a flat batch."""
        return None if a is None else a.reshape((self.size,) + a.shape[len(self.shape):])[self.sel]

    def scatter(self, a):
        """A flat batch of S's per-ray values -> a frame array, zero outside S (shifted by ``shift``)."""
        if a is None:
            return None
        out = np.zeros((self.size,) + a.shape[1:], dtype=a.dtype)
        out[self.sel + self.shift] = a
        return out.reshape(self.shape + a.shape[1:])

    def gather(self, full: dict) -> dict:
        """S's per-ray outputs and the whole scene outputs of a full-frame run; ``ray_grad`` must be exactly zero
        outside S and finite on S."""
        got = {k: self.batch(full[k]) for k in FORWARD if k in full}
        got.update({k: full[k] for k in SCATTER if k in full})
        if "ray_grad" in full:
            rg = full["ray_grad"].reshape(self.size, 6)
            outside = np.ones(self.size, dtype=bool)
            outside[self.sel] = False
            if (rg[outside] != 0).any():
                raise M.Mismatch(f"ray_grad: {int((rg[outside] != 0).any(1).sum())} rays outside S are not zero")
            if not np.isfinite(rg[self.sel]).all():
                raise M.Mismatch("ray_grad: non-finite on S")
            got["ray_grad"] = rg[self.sel]
        return got


def check_paths(scene, frame: MaskedFrame, grad_rgba, grad_depth, ray_error, runs: dict, weight_threshold=0.001,
                max_intersections=1024, half_atomics=False) -> dict:
    """Hold every full-frame run in ``runs`` to one model result for S.

    ``scene`` = (points, attributes, adjacency, offsets); ``grad_rgba``, ``grad_depth``, ``ray_error`` are S's
    upstream as a flat batch (``frame.batch`` of a frame array).  ``runs`` maps a name to
    ``run(grad_rgba, grad_depth, ray_error)``, which traces the whole frame forward and backward with these
    frame-shaped upstream arrays and returns its numpy outputs (with ``ray_grad`` when that path computes it).

    As in ``model64.check_implementation``, S's ambiguous rays get zero upstream.  The model (with ray gradients)
    runs once, on the first run's rgba and depth indices; every later run's forward outputs on S must be
    bit-identical to the first's.  Returns {name: model64 report}."""
    rays, start, dq = frame.batch(frame.rays), frame.batch(frame.start), frame.batch(frame.quantiles)
    settings = (weight_threshold, max_intersections)
    amb = MR.trace(*scene, rays, start, dq, *settings, backward=False)["ambiguous"]
    g = np.where(amb[:, None], 0, grad_rgba).astype(grad_rgba.dtype)
    gd = None if grad_depth is None else np.where(amb[:, None], 0, grad_depth).astype(grad_depth.dtype)
    err = None if ray_error is None else np.where(amb, 0, ray_error).astype(ray_error.dtype)
    upstream = (frame.scatter(g), frame.scatter(gd), frame.scatter(err))
    first, m, reports = None, None, {}
    for name, run in runs.items():
        got = frame.gather(run(*upstream))
        if first is None:
            first = got
            m = MR.trace(*scene, rays, start, dq, *settings, rgba=got["rgba"], grad_rgba=g, grad_depth=gd,
                         depth_indices=got.get("depth_indices"), ray_error=err, ray_grad=True)
            assert np.array_equal(m["ambiguous"], amb)
        else:
            for k in FORWARD:
                if k in first:
                    assert np.array_equal(got[k].view(np.uint8), first[k].view(np.uint8)), (name, k)
        report = MR.compare(got, m, half_atomics=half_atomics)
        report["ambiguous"] = int(amb.sum())
        reports[name] = report
    return reports
