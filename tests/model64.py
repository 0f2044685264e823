"""The tracer's operation in float64, with a first-order rounding-error bound on every value it computes.

Written from the behavioural specification (SURVEY.md Appendix A.3-A.6, DESIGN.md §2), not from any
implementation: it imports neither the CPU oracle nor the kernel emulator.  Every quantity is carried as
a pair (value, bound on |fp32 evaluation - value|) with the rules

    add       e = ex + ey + u|z|
    multiply  e = |y| ex + |x| ey + u|z|
    divide    e = (ex + |z| ey) / |y| + u|z|
    expf/logf their maximum ulp error from the CUDA Programming Guide (2 and 1 ulp)

and u = 2^-24; the inputs (fp32 points and rays, fp16 or fp32 attributes widened exactly) are exact.
Dot products and sums are bounded in the order-free form gamma_n * sum|terms|, so a bound holds for any
association and any fused multiply-add; nothing here encodes the instruction order of a particular build.

Scatter outputs (gradients, contribution, point_error) are kept as per-entry sums of terms: value, the
sum of the terms' own bounds, sum |term| and the number of terms n.  The per-entry bound
sum e(term) + (n - 1) u sum|term| holds for any atomic order, warp aggregation or cross-rank sum.

A ray is *ambiguous* when one of the decisions on its walk -- winning face vs runner-up, dp > 0,
t1 > t0, T > threshold, T' < quantile, the ReLU's rgb == 0 -- has a margin within twice the sum of the
two sides' bounds: an fp32 evaluation may then take the other branch, so that ray's outputs are not
comparable with the model's.

``quirks=True`` is the reference's backward (SURVEY.md A.5, each quirk a commented branch below);
``quirks=False`` is the true derivative of the forward for a fixed cell sequence.  ``planes="exact"``
uses the unrounded offsets q - p instead of the operation's fp16 ones, which makes the forward a smooth
function of the points between walk changes, so finite differences can check the true derivative.
"""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24           # unit roundoff of fp32
TINY = 2.0 ** -149       # absolute error of an fp32 result in the subnormal range
HALF_U = 2.0 ** -11      # unit roundoff of fp16
HALF_TINY = 2.0 ** -25   # half the smallest fp16 subnormal
HALF_OVERFLOW = 65520.0  # the smallest magnitude that rounds to inf in fp16
EXPF_ULP, LOGF_ULP = 2, 1
NONE = 0xFFFFFFFF
STAB = float(np.float32(1e-6))   # the backward's stabiliser (A.5.5), as an fp32 constant


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


class EV:
    """A value and a bound on the error of its fp32 evaluation; numpy arrays broadcast as usual."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, dtype=np.float64)
        self.e = np.asarray(e, dtype=np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, EV) else EV(x)

    def __add__(self, o):
        o = EV.of(o)
        z = self.v + o.v
        return EV(z, self.e + o.e + U * np.abs(z))

    __radd__ = __add__

    def __sub__(self, o):
        o = EV.of(o)
        z = self.v - o.v
        return EV(z, self.e + o.e + U * np.abs(z))

    def __rsub__(self, o):
        return EV.of(o) - self

    def __neg__(self):
        return EV(-self.v, self.e)

    def __mul__(self, o):
        o = EV.of(o)
        z = self.v * o.v
        return EV(z, np.abs(o.v) * self.e + np.abs(self.v) * o.e + U * np.abs(z) + TINY * (z != 0))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = EV.of(o)
        z = self.v / o.v
        return EV(z, (self.e + np.abs(z) * o.e) / np.abs(o.v) + U * np.abs(z) + TINY * (z != 0))

    def __rtruediv__(self, o):
        return EV.of(o) / self

    def __getitem__(self, k):
        return EV(self.v[k], np.broadcast_to(self.e, self.v.shape)[k])

    def exp(self):
        z = np.exp(self.v)
        return EV(z, z * self.e + 2 * EXPF_ULP * U * z + TINY)

    def log(self):
        z = np.log(self.v)
        return EV(z, self.e / np.abs(self.v) + 2 * LOGF_ULP * U * np.abs(z) + TINY)


def where(mask, a: EV, b: EV) -> EV:
    a, b = EV.of(a), EV.of(b)
    return EV(np.where(mask, a.v, b.v), np.where(mask, a.e, b.e))


def close(x: EV, y, e_y=0.0):
    """The decision x > y (or x < y) may go either way in fp32: margin within 2 * (e_x + e_y)."""
    e = x.e + e_y
    return (np.abs(x.v - y) <= 2.0 * e) & (e > 0)


# ---- spherical harmonics ------------------------------------------------------------------------------
# Real SH basis in the usual graphics order and sign convention; each function is a list of
# monomials (coefficient, powers of x, y, z).  Constants are the fp32 values the kernels use.
_C0 = 0.28209479177387814
_C1 = 0.4886025119029199
_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
       -0.4570457994644658, 1.445305721320277, -0.5900435899266435)
_SH = [
    [(_C0, 0, 0, 0)],
    [(-_C1, 0, 1, 0)], [(_C1, 0, 0, 1)], [(-_C1, 1, 0, 0)],
    [(_C2[0], 1, 1, 0)], [(_C2[1], 0, 1, 1)],
    [(2 * _C2[2], 0, 0, 2), (-_C2[2], 2, 0, 0), (-_C2[2], 0, 2, 0)],
    [(_C2[3], 1, 0, 1)], [(_C2[4], 2, 0, 0), (-_C2[4], 0, 2, 0)],
    [(3 * _C3[0], 2, 1, 0), (-_C3[0], 0, 3, 0)],
    [(_C3[1], 1, 1, 1)],
    [(4 * _C3[2], 0, 1, 2), (-_C3[2], 2, 1, 0), (-_C3[2], 0, 3, 0)],
    [(2 * _C3[3], 0, 0, 3), (-3 * _C3[3], 2, 0, 1), (-3 * _C3[3], 0, 2, 1)],
    [(4 * _C3[4], 1, 0, 2), (-_C3[4], 3, 0, 0), (-_C3[4], 1, 2, 0)],
    [(_C3[5], 2, 0, 1), (-_C3[5], 0, 2, 1)],
    [(_C3[6], 3, 0, 0), (-3 * _C3[6], 1, 2, 0)],
]


def sh_basis(d: np.ndarray, e_rel_d: float, sh_degree: int) -> EV:
    """Y_k(d) for k < (deg+1)^2 with bounds, d [R,3] float64 whose components carry a relative error
    of at most e_rel_d.  A monomial of order m picks up m * e_rel_d; evaluating the polynomial in fp32
    (constant, products, at most three terms) adds at most 8u of the absolute-value polynomial."""
    k = (sh_degree + 1) ** 2
    v = np.zeros(d.shape[:-1] + (k,))
    a = np.zeros_like(v)
    order = np.zeros(k)
    for j, terms in enumerate(_SH[:k]):
        for c, px, py, pz in terms:
            c = float(np.float32(c))
            mono = d[..., 0] ** px * d[..., 1] ** py * d[..., 2] ** pz
            v[..., j] += c * mono
            a[..., j] += abs(c) * np.abs(mono)
            order[j] = px + py + pz
    return EV(v, (order * e_rel_d + 8 * U) * a)


# ---- scatter outputs ----------------------------------------------------------------------------------
class Scatter:
    """Per-entry sums of terms for an [N, C] output: value, sum of the terms' bounds, sum |term| and the
    number of terms per row (every column of a row receives the same number of terms here)."""

    def __init__(self, n: int, c: int):
        self.n, self.c = n, c
        self.value = np.zeros((n, c))
        self.err = np.zeros((n, c))
        self.abs = np.zeros((n, c))
        self.count = np.zeros(n, dtype=np.int64)
        self._rows, self._v, self._e, self._k = [], [], [], []

    def add(self, rows, cols, t: EV):
        """Terms t [r, len(cols)] into rows [r], one term per (row, column)."""
        if len(rows) == 0:
            return
        v = np.zeros((len(rows), self.c))
        e = np.zeros((len(rows), self.c))
        v[:, cols] = t.v
        e[:, cols] = np.broadcast_to(t.e, t.v.shape)
        self._rows.append(np.asarray(rows, dtype=np.int64))
        self._v.append(v)
        self._e.append(e)
        self._k.append(np.ones(len(rows), dtype=np.int64))

    def flush(self):
        if not self._rows:
            return
        rows = np.concatenate(self._rows)
        v, e = np.concatenate(self._v), np.concatenate(self._e)
        k = np.concatenate(self._k)
        self._rows, self._v, self._e, self._k = [], [], [], []
        order = np.argsort(rows, kind="stable")
        rows, v, e, k = rows[order], v[order], e[order], k[order]
        starts = np.flatnonzero(np.r_[True, rows[1:] != rows[:-1]])
        u = rows[starts]
        self.value[u] += np.add.reduceat(v, starts, axis=0)
        self.err[u] += np.add.reduceat(e, starts, axis=0)
        self.abs[u] += np.add.reduceat(np.abs(v), starts, axis=0)
        self.count[u] += np.add.reduceat(k, starts)

    def bound(self, form: str = "fp32") -> np.ndarray:
        """Per-entry bound on |device sum - value|.
        fp32:       accumulated in fp32 in any order.
        fp32_half:  accumulated in fp32 in any order, rounded to fp16 once.
        half:       every add a half-precision atomic (each term rounded to fp16, then each partial sum)."""
        n = self.count[:, None].astype(np.float64)
        if form == "half":
            return self.err + (n + 1) * HALF_U * self.abs + 2 * n * HALF_TINY
        b = self.err + np.maximum(n - 1, 0) * U * self.abs
        if form == "fp32_half":
            b = b + HALF_U * (np.abs(self.value) + b) + HALF_TINY
        return b


# ---- the operation -------------------------------------------------------------------------------------
def face_offsets(points, adjacency, offsets, planes="fp16"):
    """Per CSR entry, the offset q - p of the face plane: RN-to-half of the fp32 difference (the
    operation's planes, SURVEY.md A.1) or the unrounded difference."""
    rows = np.repeat(np.arange(points.shape[0]), np.diff(offsets.astype(np.int64)))
    q, p = points[adjacency.astype(np.int64)], points[rows]
    if planes == "fp16":
        with np.errstate(over="ignore"):
            return (q - p).astype(np.float16).astype(np.float64)
    if planes == "exact":
        return q.astype(np.float64) - p.astype(np.float64)
    raise ValueError(planes)


def isect_grad(p: EV, q: EV, o: np.ndarray, d: EV) -> EV:
    """dt/dp for the bisector plane of fp32 points p and q (SURVEY.md A.4, cell_intersection_grad):
    (num d + dp (o - p)) / dp^2 with num = ((p + q)/2 - o).(q - p), dp = (q - p).d.  Arrays [r, 3]."""
    diff = q - p
    a_v = 0.5 * (p.v + q.v) - o
    a = EV(a_v, 3 * U * (np.abs(p.v) + np.abs(q.v) + np.abs(o)))
    num = _dot(a, diff, 3)
    dp = _dot(diff, d, 3)
    op = EV(o) - p
    n_vec = num[:, None] * d + dp[:, None] * op
    n_vec = EV(n_vec.v, n_vec.e + U * np.abs(n_vec.v))            # the add may fuse either way
    return n_vec / (dp * dp)[:, None]


def _dot(x: EV, y: EV, n: int) -> EV:
    """sum_i x_i y_i over the last axis, bounded for any association and contraction."""
    xv, yv = np.broadcast_arrays(x.v, y.v)
    prod = xv * yv
    z = prod.sum(-1)
    e = (np.abs(yv) * x.e + np.abs(xv) * y.e).sum(-1) + gamma(n) * np.abs(prod).sum(-1)
    return EV(z, e + TINY * n * (np.abs(prod).sum(-1) > 0))


def trace(points, attributes, adjacency, offsets, rays, start, quantiles=None, weight_threshold=0.001,
          max_intersections=1024, rgba=None, grad_rgba=None, grad_depth=None, depth_indices=None,
          ray_error=None, quirks=True, planes="fp16", backward=True, chunk=4096):
    """Forward (and backward) of the operation with bounds.

    The backward is defined on the forward's saved ``rgba`` -- pass the output of the implementation
    under test; ``None`` uses the model's own (what a finite-difference check needs).  ``depth_indices``
    likewise (``None``: the model's).  Returns a dict: per-ray outputs ``rgba``, ``depth`` (each with an
    ``*_err`` bound), ``depth_indices``, ``num_intersections``, ``ambiguous``; ``Scatter`` objects
    ``contribution``, ``points_grad``, ``attr_grad`` and (with ``ray_error``) ``point_error``."""
    if backward and (rgba is None or depth_indices is None):
        fwd = trace(points, attributes, adjacency, offsets, rays, start, quantiles, weight_threshold,
                    max_intersections, planes=planes, backward=False, chunk=chunk)
        rgba = fwd["rgba"] if rgba is None else rgba
        depth_indices = fwd.get("depth_indices") if depth_indices is None else depth_indices
    batch = rays.shape[:-1]
    r_all = int(np.prod(batch))
    rays64 = rays.reshape(r_all, 6).astype(np.float64)
    start = start.reshape(r_all).astype(np.int64)
    q_n = 0 if quantiles is None else quantiles.shape[-1]
    tau = None if q_n == 0 else quantiles.reshape(r_all, q_n).astype(np.float64)
    pts = points.astype(np.float64)
    attr = attributes.astype(np.float64)
    n_pts, a_dim = attr.shape
    sh_degree = int(round(((a_dim - 1) // 3) ** 0.5)) - 1
    k_sh = (sh_degree + 1) ** 2
    sh_rows = attr[:, :3 * k_sh].reshape(n_pts, k_sh, 3)
    sigma_all = attr[:, a_dim - 1]
    off = offsets.astype(np.int64)
    adj = adjacency.astype(np.int64)
    faces = face_offsets(points, adjacency, offsets, planes)
    thr = float(np.float32(weight_threshold))

    out = dict(rgba=np.zeros((r_all, 4)), rgba_err=np.zeros((r_all, 4)),
               num_intersections=np.zeros(r_all, dtype=np.uint32), ambiguous=np.zeros(r_all, dtype=bool),
               first_cell=np.full(r_all, -1), last_cell=np.full(r_all, -1), last_next=np.full(r_all, -1),
               skipped=np.zeros(r_all, dtype=bool))
    if q_n:
        out.update(depth=np.full((r_all, q_n), -1.0), depth_err=np.zeros((r_all, q_n)),
                   depth_indices=np.full((r_all, q_n), NONE, dtype=np.uint32))
    contribution = Scatter(n_pts, 1)
    if backward:
        g_all = grad_rgba.reshape(r_all, 4).astype(np.float64)
        gd_all = None if q_n == 0 else grad_depth.reshape(r_all, q_n).astype(np.float64)
        di_all = None if q_n == 0 else depth_indices.reshape(r_all, q_n).astype(np.int64)
        saved = rgba.reshape(r_all, 4).astype(np.float64)
        err_all = None if ray_error is None else ray_error.reshape(r_all).astype(np.float64)
        points_grad, attr_grad = Scatter(n_pts, 3), Scatter(n_pts, a_dim)
        point_error = Scatter(n_pts, 1) if ray_error is not None else None
    sh_cols = np.arange(3 * k_sh)

    for s0 in range(0, r_all, chunk):
        sl = slice(s0, min(s0 + chunk, r_all))
        rc = sl.stop - sl.start
        o = rays64[sl, :3]
        d_in = rays64[sl, 3:]
        # the ray direction is renormalised in fp32 (A.3): |d| with gamma_3 / 2 + u, then a division
        d = EV(d_in / np.linalg.norm(d_in, axis=1, keepdims=True))
        d = EV(d.v, 4 * U * np.abs(d.v))
        Y = sh_basis(d.v, 4 * U, sh_degree)
        cur = start[sl].copy()
        P = pts[cur]
        t0 = EV(np.zeros(rc), np.zeros(rc))
        T = EV(np.ones(rc), np.zeros(rc))
        C = EV(np.zeros((rc, 3)), np.zeros((rc, 3)))
        n = np.zeros(rc, dtype=np.int64)
        qi = np.zeros(rc, dtype=np.int64)
        amb = np.zeros(rc, dtype=bool)
        first_cell, last_cell, last_next = np.full(rc, -1), np.full(rc, -1), np.full(rc, -1)
        skipped = np.zeros(rc, dtype=bool)
        active = np.ones(rc, dtype=bool)
        depth = np.full((rc, q_n), -1.0)
        depth_e = np.zeros((rc, q_n))
        didx = np.full((rc, q_n), NONE, dtype=np.uint32)
        if backward:
            g = g_all[sl]
            saved_c = saved[sl]
            if q_n:
                gd = gd_all[sl]
                di = di_all[sl]
                valid = di != NONE
                terms = np.where(valid, gd / np.where(valid, sigma_all[np.where(valid, di, 0)], 1.0), 0.0)
                cdg = EV(terms.sum(1), gamma(q_n + 1) * np.abs(terms).sum(1))
            # state of the point-gradient bookkeeping
            has_prev = np.zeros(rc, dtype=bool)
            prev_idx = np.zeros(rc, dtype=np.int64)
            prev_P = np.zeros((rc, 3))
            pend_v = np.zeros((rc, 3, 3))     # quirks: up to three pending terms for row prev_idx
            pend_e = np.zeros((rc, 3, 3))
            pend_n = np.zeros(rc, dtype=np.int64)
            carry_v = np.zeros((rc, 3))        # quirks: the term for the successor of the last cell
            carry_e = np.zeros((rc, 3))
            plane_a = np.zeros(rc, dtype=np.int64)   # true derivative: the plane t0 was set on
            plane_b = np.zeros(rc, dtype=np.int64)

        while True:
            a = np.flatnonzero(active)
            if a.size == 0:
                break
            n[a] += 1
            over = n[a] > max_intersections
            active[a[over]] = False
            a = a[~over]
            if a.size == 0:
                break
            c_cur = cur[a]
            b = off[c_cur]
            nf = off[c_cur + 1] - b
            F = int(nf.max())
            if F == 0:
                active[a] = False
                break
            cols = b[:, None] + np.arange(F)
            fm = np.arange(F) < nf[:, None]
            cols = np.where(fm, cols, 0)
            D = faces[cols]                                   # [r, F, 3]
            Pa, oa, da = P[a][:, None, :], o[a][:, None, :], d.v[a][:, None, :]
            ea_d = d.e[a][:, None, :]
            av = Pa + 0.5 * D - oa
            e_av = 2 * U * (np.abs(Pa) + 0.5 * np.abs(D) + np.abs(oa))
            num = (av * D).sum(-1)
            e_num = (np.abs(D) * e_av).sum(-1) + gamma(3) * np.abs(av * D).sum(-1)
            dp = (D * da).sum(-1)
            s_dp = np.abs(D * da).sum(-1)
            e_dp = (np.abs(D) * ea_d).sum(-1) + gamma(3) * s_dp + 3 * TINY * (s_dp > 0)
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                t = num / dp
                e_t = (e_num + np.abs(t) * e_dp) / np.abs(dp) + U * np.abs(t) + TINY
            e_t = np.where(np.isfinite(e_t), e_t, np.inf)
            valid = fm & (dp > 0)
            tv = np.where(valid, t, np.inf)
            win = np.argmin(tv, axis=1)
            found = valid.any(1)
            ri = np.arange(a.size)
            t1v, t1e = tv[ri, win], e_t[ri, win]
            # decisions dp > 0 and winner vs runner-up
            unsure_dp = fm & (np.abs(dp) <= 2 * e_dp) & (e_dp > 0)
            cand = fm & ((dp > 0) | unsure_dp)
            notwin = np.ones_like(fm)
            notwin[ri, win] = False
            with np.errstate(invalid="ignore"):
                rival = cand & notwin & ~(t > t1v[:, None] + 2 * (e_t + t1e[:, None]))
            amb_step = np.where(found, rival.any(1) | unsure_dp[ri, win], cand.any(1))
            amb[a] |= amb_step
            active[a[~found]] = False
            a, win, t1v, t1e = a[found], win[found], t1v[found], t1e[found]
            if a.size == 0:
                continue
            nxt = adj[cols[found][np.arange(a.size), win]]
            t1 = EV(t1v, t1e)
            t0a = t0[a]
            amb[a] |= close(t1, t0a.v, t0a.e)
            comp = t1v > t0a.v
            cidx = a[comp]
            skipped[a[~comp]] = True
            if cidx.size:
                first_cell[cidx] = np.where(first_cell[cidx] < 0, cur[cidx], first_cell[cidx])
                last_cell[cidx], last_next[cidx] = cur[cidx], nxt[comp]
                cont = _cell(locals())
                active[cidx[~cont]] = False
            # t0 = max(t0, t1), cur = next
            upd = t1v > t0a.v
            t0.v[a] = np.where(upd, t1v, t0a.v)
            t0.e[a] = np.where(upd, t1e, t0a.e)
            cur[a] = nxt
            P[a] = pts[nxt]

        sel = np.arange(sl.start, sl.stop)
        out["rgba"][sel, :3] = C.v
        out["rgba_err"][sel, :3] = C.e
        alpha = 1.0 - T
        out["rgba"][sel, 3] = alpha.v
        out["rgba_err"][sel, 3] = alpha.e
        out["num_intersections"][sel] = n
        out["ambiguous"][sel] = amb
        out["first_cell"][sel], out["last_cell"][sel], out["last_next"][sel] = first_cell, last_cell, last_next
        out["skipped"][sel] = skipped
        if q_n:
            out["depth"][sel] = depth
            out["depth_err"][sel] = depth_e
            out["depth_indices"][sel] = didx
        contribution.flush()
        if backward:
            points_grad.flush()
            attr_grad.flush()
            if point_error is not None:
                point_error.flush()

    res = {k: v.reshape(batch + v.shape[1:]) for k, v in out.items()}
    res["num_intersections"] = res["num_intersections"].reshape(batch + (1,))
    for k in ("ambiguous", "first_cell", "last_cell", "last_next", "skipped"):
        res[k] = out[k].reshape(batch)
    res["contribution"] = contribution
    if backward:
        res["points_grad"], res["attr_grad"] = points_grad, attr_grad
        if point_error is not None:
            res["point_error"] = point_error
    return res


def _cell(f):
    """Composite the cells of rays ``cidx`` (chunk-local) and, with ``backward``, scatter their gradient
    terms.  ``f`` is the walk's local namespace.  Returns, per ray, whether the walk continues."""
    cidx, comp = f["cidx"], f["comp"]
    T, C, t0, t1, qi, amb = f["T"], f["C"], f["t0"][cidx], f["t1"][comp], f["qi"], f["amb"]
    cc = f["cur"][cidx]
    nxt = f["nxt"][comp]
    sigma = f["sigma_all"][cc]
    q_n, tau, depth, depth_e, didx = f["q_n"], f["tau"], f["depth"], f["depth_e"], f["didx"]
    backward, quirks = f["backward"], f["quirks"]
    s0 = f["sl"].start
    Y = f["Y"][cidx]                                                 # [r, K]
    coef = f["sh_rows"][cc]                                          # [r, K, 3]
    k_sh = coef.shape[1]

    # rgb = max(0, 0.5 + sum_k Y_k a_k) behind the density gate sigma > 1e-6 (A.3)
    gate = sigma > 1e-6
    pre_v = 0.5 + (Y.v[:, :, None] * coef).sum(1)
    pre_e = (np.abs(coef) * Y.e[:, :, None]).sum(1) + gamma(k_sh + 1) * (
        0.5 + np.abs(Y.v[:, :, None] * coef).sum(1))
    lit = gate[:, None] & (pre_v > 0)
    amb[cidx] |= (gate[:, None] & (np.abs(pre_v) <= 2 * pre_e)).any(1)
    rgb = EV(np.where(lit, pre_v, 0.0), np.where(lit, pre_e, 0.0))

    Tb = T[cidx]
    delta = t1 - t0
    x = EV(sigma) * delta
    alpha = 1.0 - (-x).exp()
    w = Tb * alpha
    f["contribution"].add(cc, [0], EV(w.v[:, None], w.e[:, None]))
    Cb = C[cidx]
    Cn = Cb + EV(w.v[:, None], w.e[:, None]) * rgb
    C.v[cidx], C.e[cidx] = Cn.v, Cn.e
    oma = 1.0 - alpha
    Tn = Tb * oma

    if backward:
        g = f["g"][cidx]
        saved = f["saved_c"][cidx]
        gv = EV(g)
        # A.5.5: the ReLU mask is the exact compare rgb == 0 (it also covers the density gate)
        mask = rgb.v != 0 if quirks else lit
        d_rgb = where(mask, EV(g[:, :3]) * EV(w.v[:, None], w.e[:, None]), EV(0.0))
        # A.5.5: 1e-6 stabilisers in `rest` and in dL/dalpha; the true derivative has none
        den1 = oma + EV(STAB, U * STAB) if quirks else oma
        rest = (EV(saved[:, :3]) - Cn) / (Tb * den1)[:, None]
        diff = rgb - rest
        dot_v = (diff.v * g[:, :3]).sum(1)
        dot_e = (np.abs(g[:, :3]) * diff.e).sum(1) + gamma(4) * np.abs(diff.v * g[:, :3]).sum(1)
        d_alpha = Tb * EV(dot_v, dot_e) + (1.0 - EV(saved[:, 3])) * gv[:, 3] / den1
        if not quirks:
            # an opaque cell (1 - alpha == 0 in float64) hides everything behind it: dalpha/dsigma and
            # dalpha/ddelta are zero there, and the ratios above are 0/0
            d_alpha = where(oma.v == 0, EV(0.0), d_alpha)
        d_sigma = d_alpha * (delta * oma)
        d_delta = d_alpha * (EV(sigma) * oma)
        d_t0 = EV(np.zeros(cidx.size))
    # depth quantiles: while T' < tau_q, depth = t0 + log(T / tau_q) / sigma (A.3)
    for _ in range(q_n):
        live = qi[cidx] < q_n
        if not live.any():
            break
        qk = np.minimum(qi[cidx], q_n - 1)
        tq = tau[s0 + cidx, qk]
        amb[cidx] |= live & close(Tn, tq)
        fire = live & (Tn.v < tq)
        if not fire.any():
            break
        with np.errstate(divide="ignore", invalid="ignore"):
            lg = (Tb / EV(tq)).log()
            dep = t0 + lg / EV(sigma)
        ri = cidx[fire]
        depth[ri, qk[fire]] = dep.v[fire]
        depth_e[ri, qk[fire]] = dep.e[fire]
        didx[ri, qk[fire]] = cc[fire]
        if backward:
            gd_q = EV(f["gd"][cidx, qk])
            gq = where(fire, gd_q / EV(sigma), EV(0.0))
            # SURVEY.md A.4 gives dL/dt0 += gd_q / sigma for depth = t0 + log(T / tau) / sigma, whose
            # derivative in t0 is 1; the reference's stored gradients agree with the former, so it is a
            # quirk of the reference's backward (not listed in A.5)
            d_t0 = d_t0 + (gq if quirks else where(fire, gd_q, EV(0.0)))
            with np.errstate(invalid="ignore"):
                d_sigma = where(fire, d_sigma - gq * lg / EV(sigma), d_sigma)
            cdg = f["cdg"]
            new = cdg[cidx] - gq
            cdg.v[cidx] = np.where(fire, new.v, cdg.v[cidx])
            cdg.e[cidx] = np.where(fire, new.e, cdg.e[cidx])
        qi[cidx] += fire
    if backward and q_n:
        cd = f["cdg"][cidx]
        remain = qi[cidx] < q_n
        d_sigma = where(remain, d_sigma - delta * cd, d_sigma)
        d_delta = where(remain, d_delta - EV(sigma) * cd, d_delta)
    T.v[cidx], T.e[cidx] = Tn.v, Tn.e
    cont = Tn.v > f["thr"]
    amb[cidx] |= close(Tn, f["thr"])

    if backward:
        _scatter_grads(f, cidx, cc, nxt, Y, d_rgb, d_sigma, d_delta, d_t0, w)
    return cont


def _scatter_grads(f, cidx, cc, nxt, Y, d_rgb, d_sigma, d_delta, d_t0, w):
    quirks = f["quirks"]
    k_sh = Y.v.shape[1]
    a_dim = f["a_dim"]
    # SH: attr_grad[cur, 3k+c] += Y_k dL/drgb_c; density: attr_grad[cur, A-1] += dL/dsigma (A.4)
    sh = EV(Y.v[:, :, None] * d_rgb.v[:, None, :],
            np.abs(Y.v[:, :, None]) * d_rgb.e[:, None, :] + Y.e[:, :, None] * np.abs(d_rgb.v[:, None, :]))
    sh = EV(sh.v.reshape(len(cc), -1), sh.e.reshape(len(cc), -1) + U * np.abs(sh.v.reshape(len(cc), -1)))
    f["attr_grad"].add(cc, np.r_[f["sh_cols"], a_dim - 1],
                       EV(np.c_[sh.v, d_sigma.v], np.c_[sh.e, np.broadcast_to(d_sigma.e, d_sigma.v.shape)]))
    if f["point_error"] is not None:
        err = EV(f["err_all"][f["sl"].start + cidx])
        f["point_error"].add(cc, [0], EV((err * w).v[:, None], (err * w).e[:, None]))

    d_t0 = d_t0 - d_delta
    d_t1 = d_delta
    pts, o, d = f["pts"], f["o"][cidx], f["d"][cidx]
    Pc, Pn = EV(pts[cc]), EV(pts[nxt])
    pg = f["points_grad"]
    has_prev = f["has_prev"][cidx]
    if quirks:
        # A.5.2: for the first composited cell the previous point is (0,0,0), and dt0/dcurrent taken on the
        # plane between the current point and the origin is still added with weight dL/dt0
        # A.5.3: "previous" is the last composited cell, not the geometric predecessor
        prevP = EV(np.where(has_prev[:, None], f["prev_P"][cidx], 0.0))
        g_prev = isect_grad(prevP, Pc, o, d)
        g_cur0 = isect_grad(Pc, prevP, o, d)
        g_cur1 = isect_grad(Pc, Pn, o, d)
        g_next = isect_grad(Pn, Pc, o, d)
        t_prev = d_t0[:, None] * g_prev
        own0 = d_t0[:, None] * g_cur0
        own1 = d_t1[:, None] * g_cur1
        carry = d_t1[:, None] * g_next
        # A.5.1: point gradients are flushed one composited cell late: the previous cell's row receives its
        # pending terms plus this cell's dt0/dprevious term now; this cell's own terms and the term for its
        # successor wait for the next composited cell ...
        hp = np.flatnonzero(has_prev)
        if hp.size:
            ci = cidx[hp]
            pend_v, pend_e, pend_n = f["pend_v"][ci], f["pend_e"][ci], f["pend_n"][ci]
            for j in range(3):
                use = np.flatnonzero(pend_n > j)
                pg.add(f["prev_idx"][ci[use]], [0, 1, 2], EV(pend_v[use, j], pend_e[use, j]))
            pg.add(f["prev_idx"][ci], [0, 1, 2], t_prev[hp])
        # ... and the two accumulators left at the end of the walk (the last composited cell's and its
        # successor's) are never written: pending terms are simply dropped when the walk ends
        carried_v = np.where(has_prev[:, None], f["carry_v"][cidx], 0.0)
        carried_e = np.where(has_prev[:, None], f["carry_e"][cidx], 0.0)
        f["pend_v"][cidx] = np.stack([carried_v, own0.v, own1.v], 1)
        f["pend_e"][cidx] = np.stack([carried_e, own0.e, own1.e], 1)
        f["pend_n"][cidx] = 3
        f["carry_v"][cidx] = carry.v
        f["carry_e"][cidx] = carry.e
    else:
        # true derivative: t1 lies on the plane (cur, next); t0 on the plane t0 was last set on, and is the
        # constant 0 for the first composited cell
        g_cur1 = isect_grad(Pc, Pn, o, d)
        g_next = isect_grad(Pn, Pc, o, d)
        pg.add(cc, [0, 1, 2], d_t1[:, None] * g_cur1)
        pg.add(nxt, [0, 1, 2], d_t1[:, None] * g_next)
        hp = np.flatnonzero(has_prev)
        if hp.size:
            ci = cidx[hp]
            pa, pb = f["plane_a"][ci], f["plane_b"][ci]
            A, B = EV(pts[pa]), EV(pts[pb])
            oo, dd = o[hp], d[hp]
            pg.add(pa, [0, 1, 2], d_t0[hp][:, None] * isect_grad(A, B, oo, dd))
            pg.add(pb, [0, 1, 2], d_t0[hp][:, None] * isect_grad(B, A, oo, dd))
        f["plane_a"][cidx] = cc
        f["plane_b"][cidx] = nxt
    f["has_prev"][cidx] = True
    f["prev_idx"][cidx] = cc
    f["prev_P"][cidx] = pts[cc]


# ---- the comparator ------------------------------------------------------------------------------------
SCATTER = ("contribution", "points_grad", "attr_grad", "point_error")


class Mismatch(AssertionError):
    pass


def compare(got: dict, m: dict, half_atomics: bool = False, skip_rows=None, per_ray: bool = True) -> dict:
    """Hold an implementation's outputs ``got`` (numpy) to the model's ``m`` (from ``trace``):
    integers exact and floats within their bounds on unambiguous rays; every compared scatter entry within
    its per-entry bound, exactly zero where the model has no term, and finite wherever the bound is.
    fp16 scatter outputs use the half-atomic bound for ``contribution`` / ``point_error`` always and for the
    gradients when ``half_atomics`` (the reference); otherwise "accumulated in fp32, rounded once".
    ``skip_rows`` (bool [N]) excludes rows from the scatter comparison.  Returns a tightness report."""
    ok = ~m["ambiguous"]
    report = {"rays": int(ok.size), "rays_compared": int(ok.sum())}
    if per_ray:
        for k in ("num_intersections", "depth_indices"):
            if k in got and k in m:
                bad = (got[k] != m[k])[ok]
                if bad.any():
                    raise Mismatch(f"{k}: {int(bad.sum())} entries differ on unambiguous rays")
        for k in ("rgba", "depth"):
            if k not in got or k not in m:
                continue
            g = got[k].astype(np.float64)
            b = m[k + "_err"]
            if got[k].dtype == np.float16:
                b = b + HALF_U * (np.abs(m[k]) + b) + HALF_TINY
            _within(k, g[ok], m[k][ok], b[ok])
    for k in SCATTER:
        if k not in got or k not in m:
            continue
        s = m[k]
        g = got[k].astype(np.float64).reshape(s.value.shape)
        if got[k].dtype == np.float16:
            form = "half" if (half_atomics or k in ("contribution", "point_error")) else "fp32_half"
        else:
            form = "fp32"
        b = s.bound(form)
        if got[k].dtype == np.float16:
            # rounding to fp16 gives +-inf from |x| >= 65520 on: accepted where the bound reaches that far
            over = np.isinf(g) & (np.abs(s.value) + b >= HALF_OVERFLOW) & (np.sign(g) == np.sign(s.value))
            g = np.where(over, s.value, g)
        rows = np.ones(s.n, dtype=bool) if skip_rows is None else ~skip_rows
        zero = rows & (s.count == 0)
        if (g[zero] != 0).any():
            raise Mismatch(f"{k}: {int((g[zero] != 0).any(1).sum())} rows without any term are nonzero")
        sel = rows & (s.count > 0)
        _within(k, g[sel], s.value[sel], b[sel])
        live = s.abs[sel] > 0
        rel = b[sel][live] / s.abs[sel][live]
        scale = np.abs(s.value[sel]).max() if sel.any() else 0.0
        report[k] = dict(entries=int(s.value.size), compared=int(sel.sum() * s.c),
                         median_bound_over_abs=float(np.median(rel)) if rel.size else 0.0,
                         tighter_than_1e5_max=float((b[sel] < 1e-5 * scale).mean()) if sel.any() else 1.0)
    return report


def _within(name, got, value, bound):
    fin = np.isfinite(bound) & np.isfinite(value)
    if not np.isfinite(got[fin]).all():
        raise Mismatch(f"{name}: {int((~np.isfinite(got[fin])).sum())} non-finite where the model is finite")
    diff = np.abs(got[fin] - value[fin])
    bad = diff > bound[fin]
    if bad.any():
        i = np.flatnonzero(bad)[np.argmax((diff / np.maximum(bound[fin], 1e-300))[bad])]
        raise Mismatch(f"{name}: {int(bad.sum())} of {bad.size} entries outside their bound; worst "
                       f"got {got[fin][i]!r} model {value[fin][i]!r} bound {bound[fin][i]:.3e}")


def rows_reachable(m: dict, offsets, adjacency, points, attributes, rays, start, quantiles, weight_threshold,
                   max_intersections) -> np.ndarray:
    """Rows an ambiguous ray may scatter into: those its model walk touches, and their neighbours (an
    implementation that took the other branch at a near-tie enters a neighbouring cell).  For comparing
    with outputs made with every ray's upstream gradient -- the stored reference outputs."""
    amb = m["ambiguous"].reshape(-1)
    n = points.shape[0]
    rows = np.zeros(n, dtype=bool)
    if not amb.any():
        return rows
    r = rays.reshape(-1, 6)[amb]
    st = start.reshape(-1)[amb]
    q = None if quantiles is None else quantiles.reshape(-1, quantiles.shape[-1])[amb]
    t = trace(points, attributes, adjacency, offsets, r, st, q, weight_threshold, max_intersections,
              backward=False)
    rows |= t["contribution"].count > 0
    rows[st] = True
    off = offsets.astype(np.int64)
    nb = np.zeros(n, dtype=bool)
    for i in np.flatnonzero(rows):
        nb[adjacency[off[i]:off[i + 1]].astype(np.int64)] = True
    return rows | nb


def check_implementation(impl, points, attributes, adjacency, offsets, rays, start, quantiles, grad_rgba,
                         grad_depth, ray_error=None, weight_threshold=0.001, max_intersections=1024,
                         contribution=True, half_atomics=False) -> dict:
    """Trace a case with an implementation and hold every output to the model.

    ``impl(rays, start, quantiles, grad_rgba, grad_depth, ray_error, backward)`` returns numpy outputs of
    the forward (with contribution) and, with ``backward``, of the backward on its own saved rgba and depth
    indices.  Ambiguous rays get zero upstream gradients and ray error in both the model and the
    implementation, so the image and its layout stay as given; where any exist, ``contribution`` (a
    forward output) is compared on a flat batch of the unambiguous rays instead."""
    settings = (weight_threshold, max_intersections)
    scene = (points, attributes, adjacency, offsets)
    m0 = trace(*scene, rays, start, quantiles, *settings, backward=False)
    amb = m0["ambiguous"]
    g = np.where(amb[..., None], 0, grad_rgba).astype(grad_rgba.dtype)
    gd = None if grad_depth is None else np.where(amb[..., None], 0, grad_depth).astype(grad_depth.dtype)
    err = None if ray_error is None else np.where(amb.reshape(ray_error.shape), 0, ray_error).astype(ray_error.dtype)
    got = impl(rays, start, quantiles, g, gd, err, True)
    m = trace(*scene, rays, start, quantiles, *settings, rgba=got["rgba"], grad_rgba=g, grad_depth=gd,
              depth_indices=got.get("depth_indices"), ray_error=err)
    assert np.array_equal(m["ambiguous"], amb)
    if amb.any() or not contribution:
        got = {k: v for k, v in got.items() if k != "contribution"}
    report = compare(got, m, half_atomics=half_atomics)
    report["ambiguous"] = int(amb.sum())
    if contribution and amb.any():
        keep = ~amb.reshape(-1)
        r = rays.reshape(-1, 6)[keep]
        s = start.reshape(-1)[keep]
        q = None if quantiles is None else quantiles.reshape(-1, quantiles.shape[-1])[keep]
        flat = impl(r, s, q, None, None, None, False)
        mf = trace(*scene, r, s, q, *settings, backward=False)
        report["contribution"] = compare({"contribution": flat["contribution"]}, mf, per_ray=False)["contribution"]
    return report


def format_report(name: str, report: dict) -> str:
    """One line of the tightness table: rays compared, and per scatter output the share of entries compared,
    the median bound relative to sum|term| and the share of bounds tighter than 1e-5 of the largest entry."""
    parts = [f"{name}: rays {report['rays_compared']}/{report['rays']}"]
    for k in SCATTER:
        if k in report:
            r = report[k]
            parts.append(f"{k} {r['compared']}/{r['entries']} med {r['median_bound_over_abs']:.1e} "
                         f"<1e-5max {100 * r['tighter_than_1e5_max']:.0f}%")
    return " | ".join(parts)
