"""References for the kernels around the tracer core: the parameter-form activation and the gradient epilogues.

Written from the operations' specification, importing no product code:

* ``softplus_beta10`` / ``softplus_beta10_backward``: ``F.softplus(x, beta=10)`` and its derivative with torch's
  threshold (the linear branch from ``x * 10 > 20`` on), in float64 with a first-order bound in the ``EV`` style of
  ``model64.py`` (``expf`` 2 ulp, ``log1pf`` 1 ulp: the CUDA Programming Guide's maxima).  The branch is taken from
  ``xb = float32(x) * float32(10)`` evaluated in numpy fp32 -- the same IEEE product the kernels and torch form,
  so the ``> 20`` decision is exact, and ``xb`` is an exact input of the rest.
* ``finalize`` / ``finalize_params`` / ``peer_sum``: the epilogues from an fp32 accumulator ``[N, grad_row]`` to the
  gradients the optimizer reads.  Rounding to fp16 is numpy's ``astype`` (round to nearest even, overflow to inf),
  the scrub zeroes non-finite values AFTER that rounding.
* ``crafted_accumulator`` and ``EDGE_RAW``: inputs at the places these kernels can go wrong.
"""
from __future__ import annotations

import numpy as np

from model64 import EV, TINY, U

LOG1PF_ULP = 1
THRESHOLD = 20.0


def sh_dim(deg: int) -> int:
    return (deg + 1) ** 2


def attr_dim(deg: int) -> int:
    return 1 + 3 * sh_dim(deg)


def sh_row(deg: int) -> int:
    """Accumulator slot of the density gradient: the SH colour gradients padded to whole float4."""
    return (3 * sh_dim(deg) + 3) // 4 * 4


def grad_row(deg: int) -> int:
    """Floats per accumulator row: [SH colour (padded)][density, gx, gy, gz]."""
    return sh_row(deg) + 4


def _xb(raw) -> np.ndarray:
    with np.errstate(all="ignore"):
        return np.asarray(raw, dtype=np.float32) * np.float32(10.0)


def _log1p(x: EV) -> EV:
    z = np.log1p(x.v)
    return EV(z, x.e / np.abs(1.0 + x.v) + 2 * LOG1PF_ULP * U * np.abs(z) + TINY)


def softplus_beta10(raw) -> EV:
    """softplus(raw, beta=10) = raw where raw*10 > 20, else log1p(exp(raw*10)) / 10."""
    xb = _xb(raw)
    lin = xb > np.float32(THRESHOLD)
    with np.errstate(all="ignore"):
        soft = _log1p(EV(np.where(lin, 0.0, xb.astype(np.float64))).exp()) / 10.0
    return EV(np.where(lin, np.asarray(raw, np.float64), soft.v), np.where(lin, 0.0, soft.e))


def softplus_beta10_backward(grad: EV, raw) -> EV:
    """d softplus(raw, beta=10) applied to an upstream gradient ``grad`` carrying its own bound: grad where
    raw*10 > 20, else (grad * z) / (z + 1) with z = exp(raw*10), in that evaluation order.  Beyond grad's bound,
    the rules add 4u|z| (expf) and one rounding each for grad*z, z+1 and the division: with grad = g*scale
    formed in fp32 (one more rounding), the total is |chain|*bound(g) + 8u|value| + subnormal terms."""
    grad = EV.of(grad)
    xb = _xb(raw)
    lin = xb > np.float32(THRESHOLD)
    with np.errstate(all="ignore"):
        z = EV(np.where(lin, 0.0, xb.astype(np.float64))).exp()
        soft = (grad * z) / (z + 1.0)
    return EV(np.where(lin, grad.v, soft.v), np.where(lin, np.broadcast_to(grad.e, lin.shape), soft.e))


def chain(raw, scale) -> np.ndarray:
    """d(scale * softplus(raw, beta=10)) / d raw in float64."""
    xb = _xb(raw)
    with np.errstate(all="ignore"):
        z = np.exp(np.where(xb > np.float32(THRESHOLD), 0.0, xb.astype(np.float64)))
        return float(np.float32(scale)) * np.where(xb > np.float32(THRESHOLD), 1.0, z / (z + 1.0))


# ---- the gradient epilogues --------------------------------------------------------------------------------
def _round_scrub(x: np.ndarray, dtype, scrub: bool) -> np.ndarray:
    with np.errstate(all="ignore"):
        o = np.asarray(x, np.float32).astype(dtype)
    if scrub:
        o = np.where(np.isfinite(o), o, np.zeros((), dtype)).astype(dtype)
    return o


def finalize(acc: np.ndarray, deg: int, dtype, scrub: bool):
    """acc [N, grad_row] fp32 -> (points_grad [N,3] fp32, attr_grad [N,A] dtype): attribute columns 0..A-2 from
    acc[:, :A-1], the density column from slot SR, the position from SR+1..SR+3; rounded once, then scrubbed."""
    a, sr = attr_dim(deg), sh_row(deg)
    acc = np.asarray(acc, np.float32)
    attr = np.concatenate([acc[:, :a - 1], acc[:, sr:sr + 1]], axis=1)
    return _round_scrub(acc[:, sr + 1:sr + 4], np.float32, scrub), _round_scrub(attr, dtype, scrub)


def finalize_params(acc: np.ndarray, raw, scale, deg: int, dtype, scrub: bool):
    """The parameter-form epilogue: dict of points_grad, att_dc_grad, att_sh_grad (fp32 arrays, exact) and
    density_grad (an EV: value and bound; the kernel's expf is not numpy's).  The attribute gradient is rounded
    to ``dtype`` and scrubbed exactly like ``finalize``; density then chains through torch's order:
    g * scale first (fp32), then softplus_backward."""
    pts, attr = finalize(acc, deg, dtype, scrub)
    g = attr.astype(np.float32)
    a = attr_dim(deg)
    with np.errstate(all="ignore"):
        gs = g[:, a - 1:a] * np.float32(scale)
    return {"points_grad": pts, "att_dc_grad": g[:, :3].copy(), "att_sh_grad": g[:, 3:a - 1].copy(),
            "density_grad": softplus_beta10_backward(EV(gs.astype(np.float64)), np.asarray(raw).reshape(-1, 1)),
            "density_column": g[:, a - 1:a].copy()}


def peer_sum(accs) -> np.ndarray:
    """((a0 + a1) + a2) + ... in fp32: the rank-order sum the peer reduction promises."""
    total = np.array(accs[0], dtype=np.float32, copy=True)
    with np.errstate(all="ignore"):
        for a in accs[1:]:
            total = total + np.asarray(a, np.float32)
    return total


# ---- inputs ---------------------------------------------------------------------------------------------------
F16_MIN_SUB = 2.0 ** -24
SPECIALS = np.array([
    65504.0, float(np.float32(65519.996)), 65520.0,           # fp16 max, just below / at its overflow point
    1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 2048.0 + 1.0,     # fp16 round-half-even ties (down, up, at 2^11)
    0.5 * F16_MIN_SUB, 1.5 * F16_MIN_SUB, 2.5 * F16_MIN_SUB,  # fp16 subnormal ties (to 0, up, down)
    F16_MIN_SUB, 37 * F16_MIN_SUB, 2.0 ** -14 - F16_MIN_SUB,  # fp16 subnormals, the largest one
    1e-8,                                                     # below half the smallest fp16 subnormal
    np.nan, np.inf, -np.inf, -0.0, float(np.finfo(np.float32).max),
], dtype=np.float32)


def crafted_accumulator(n: int, deg: int, seed: int, special_share: float = 0.25) -> np.ndarray:
    """A seeded [n, grad_row] fp32 accumulator: ordinary values over many magnitudes mixed with SPECIALS (random
    sign) in about ``special_share`` of the entries, every special in every column class when n allows."""
    rng = np.random.default_rng(seed)
    gr = grad_row(deg)
    acc = (rng.normal(size=(n, gr)) * 10.0 ** rng.integers(-6, 4, size=(n, gr))).astype(np.float32)
    pick = rng.random((n, gr)) < special_share
    sign = np.where(rng.random((n, gr)) < 0.5, -1.0, 1.0).astype(np.float32)
    vals = SPECIALS[rng.integers(0, SPECIALS.size, size=(n, gr))] * sign
    acc[pick] = vals[pick]
    # deterministic coverage of the first rows: every special in the density slot, a position slot and column 0
    sr = sh_row(deg)
    k = min(n, SPECIALS.size)
    for col in (0, sr, sr + 1):
        acc[:k, col] = SPECIALS[:k]
    return acc


# raw (pre-activation) densities at softplus' edges
_TWO = np.float32(2.0)
EDGE_RAW = np.array([
    _TWO, np.nextafter(_TWO, np.float32(np.inf)), np.nextafter(_TWO, np.float32(-np.inf)),   # the x*10 > 20 switch
    1.6, 1.9,                                   # log1p branch, just below the switch
    2.5, 50.0,                                  # linear branch
    0.0,
    -3.0, -8.7,                                 # tail: expf near the smallest normal at -8.7
    -9.0,                                       # subnormal expf
    -10.4,                                      # expf flushes to 0
    -30.0,
], dtype=np.float32)
EDGE_RAW_NONFINITE = np.array([np.nan, np.inf, -np.inf], dtype=np.float32)   # crafted epilogue cases only
