"""The float64 model of tests/model64.py with ray gradients: ``trace(..., ray_grad=True)`` adds each ray's
dL/d(origin, direction as passed in) and a bound on its fp32 evaluation.

The walk, the compositing and the scene gradients are model64's, restated here because the ray terms need the
per-cell quantities of its backward (dL/dalpha, dL/ddelta, dL/drgb, the fired quantiles); everything else --
the bound arithmetic (EV), the SH basis, the scatter sums, the scene-gradient scatter and the comparator -- is
imported from model64.  With ``ray_grad=False`` ``trace`` computes exactly what ``model64.trace`` does.

The ray gradient is defined for the walk's cell sequence held fixed.  Each t a ray term differentiates lies on
the bisector plane of the fp32 points (p, q) -- the plane of the points' own gradient, not the fp16 face
offsets -- with n = q - p, dp = n.d, num = ((p + q)/2 - o).n:  dt/do = -n/dp,  dt/dd = -(num/dp) n/dp
(d the unit direction).  A composited cell's t1 lies on its exit plane (cur, next); its t0 on the exit plane of
the previous composited cell (the constant 0 before the first one).  dL/dt1 = dL/ddelta and dL/dt0 = the sum of
the depth gradients of the quantiles the cell fires - dL/ddelta (the depth t0 + log(T/tau)/sigma has
t0-derivative 1 in both modes: the gd/sigma quirk of the points' gradient is not carried over).  The colour adds
sum over (cell, k, c) of dL/drgb_c a[cell, 3k+c] dY_k/dd, and the unit direction's gradient g is taken back
through d = d_in/|d_in| as (g - d (d.g)) / |d_in|.  Each ray's six sums are bounded as one sum over all their
terms, sum e(term) + (n - 1) u sum|term|; the renormalisation by the add / multiply / divide rules."""
from __future__ import annotations

import numpy as np

import model64 as M
from model64 import (EV, NONE, STAB, TINY, U, _SH, Scatter, _dot, _scatter_grads, close, face_offsets, gamma,
                     sh_basis, where)


def sh_basis_grad(d: np.ndarray, e_rel_d: float, sh_degree: int) -> EV:
    """dY_k/dd_i [R, K, 3] with bounds: the monomials of _SH differentiated, bounded by sh_basis's rule (a
    monomial of order m - 1 picks up (m - 1) e_rel_d, the fp32 evaluation 8u of the absolute polynomial)."""
    k = (sh_degree + 1) ** 2
    v = np.zeros(d.shape[:-1] + (k, 3))
    a = np.zeros_like(v)
    order = np.zeros((k, 3))
    for j, terms in enumerate(_SH[:k]):
        for c, *pw in terms:
            c = float(np.float32(c))
            for i in range(3):
                if pw[i] == 0:
                    continue
                q = list(pw)
                q[i] -= 1
                mono = pw[i] * c * d[..., 0] ** q[0] * d[..., 1] ** q[1] * d[..., 2] ** q[2]
                v[..., j, i] += mono
                a[..., j, i] += np.abs(mono)
                order[j, i] = sum(q)
    return EV(v, (order * e_rel_d + 8 * U) * a)


class RaySum:
    """Per-ray sums of terms for ray_grad [R, 6] (dL/do, then dL/dd for the unit direction before the
    renormalisation): value, sum of the terms' bounds, sum |term| and the number of terms per entry."""

    def __init__(self, r: int):
        self.value, self.err, self.abs = np.zeros((r, 6)), np.zeros((r, 6)), np.zeros((r, 6))
        self.count = np.zeros((r, 6))

    def add(self, rows, cols, t: EV, abs_=None, n=1):
        """One term t [r, len(cols)] per entry of rays ``rows`` (distinct), or -- with ``abs_`` and ``n`` -- the
        sum of n terms: t.v their sum, t.e the sum of their bounds, abs_ the sum of their absolute values."""
        self.value[rows[:, None], cols] += t.v
        self.err[rows[:, None], cols] += np.broadcast_to(t.e, t.v.shape)
        self.abs[rows[:, None], cols] += np.abs(t.v) if abs_ is None else abs_
        self.count[rows[:, None], cols] += n

    def bound(self) -> np.ndarray:
        return self.err + np.maximum(self.count - 1, 0) * U * self.abs


def trace(points, attributes, adjacency, offsets, rays, start, quantiles=None, weight_threshold=0.001,
          max_intersections=1024, rgba=None, grad_rgba=None, grad_depth=None, depth_indices=None,
          ray_error=None, quirks=True, planes="fp16", backward=True, chunk=4096, ray_grad=False):
    """Forward (and backward) of the operation with bounds.

    The backward is defined on the forward's saved ``rgba`` -- pass the output of the implementation
    under test; ``None`` uses the model's own (what a finite-difference check needs).  ``depth_indices``
    likewise (``None``: the model's).  Returns a dict: per-ray outputs ``rgba``, ``depth`` (each with an
    ``*_err`` bound), ``depth_indices``, ``num_intersections``, ``ambiguous``; ``Scatter`` objects
    ``contribution``, ``points_grad``, ``attr_grad`` and (with ``ray_error``) ``point_error``.

    ``ray_grad`` (with ``backward``) adds ``ray_grad`` [..., 6] = dL/d(origin, direction as passed in) and its
    bound ``ray_grad_err``: the walk's cell sequence held fixed, each t on the bisector plane of the fp32 points
    (t1 on the cell's exit plane, t0 on the previous composited cell's, the constant 0 before the first), with
    dt/do = -n/dp and dt/dd = -(num/dp) n/dp; dL/dt1 = dL/ddelta, dL/dt0 = sum of the fired quantiles' depth
    gradients - dL/ddelta (d depth/dt0 = 1 in both modes); the colour's direction term
    sum_(cell,k,c) dL/drgb_c a[cell,3k+c] grad Y_k; then dL/dd_in = (g - d (d.g)) / |d_in|.  Each ray's sum
    over all its terms is bounded as sum e(term) + (n - 1) u sum|term|."""
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
    if backward and ray_grad:
        out.update(ray_grad=np.zeros((r_all, 6)), ray_grad_err=np.zeros((r_all, 6)))
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
            if ray_grad:
                rsum = RaySum(rc)
                dY = sh_basis_grad(d.v, 4 * U, sh_degree)
                jo_v, jo_e = np.zeros((rc, 3)), np.zeros((rc, 3))   # previous exit plane: -n/dp ...
                jt_v, jt_e = np.zeros(rc), np.zeros(rc)             # ... and num/dp

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
        if backward and ray_grad:
            _ray_finish(out, sel, rsum, d, d_in)
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
        r_t0 = EV(np.zeros(cidx.size))       # the ray gradient's sum of fired depth gradients
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
            r_t0 = r_t0 + where(fire, gd_q, EV(0.0))
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
        if f["ray_grad"]:
            _ray_terms(f, cidx, cc, nxt, coef, d_rgb, d_delta, r_t0)
        _scatter_grads(f, cidx, cc, nxt, Y, d_rgb, d_sigma, d_delta, d_t0, w)
    return cont


def _ray_terms(f, cidx, cc, nxt, coef, d_rgb, d_delta, r_t0):
    """The ray-gradient terms of one composited cell (see ``trace``); reads has_prev before _scatter_grads
    sets it."""
    rs, pts, o, d = f["rsum"], f["pts"], f["o"][cidx], f["d"][cidx]
    P, Q = EV(pts[cc]), EV(pts[nxt])
    diff = Q - P
    a = EV(0.5 * (P.v + Q.v) - o, 3 * U * (np.abs(P.v) + np.abs(Q.v) + np.abs(o)))
    num, dp = _dot(a, diff, 3), _dot(diff, d, 3)
    jo, jt = -diff / dp[:, None], num / dp
    oc, dc = np.arange(3), np.arange(3, 6)
    hp = np.flatnonzero(f["has_prev"][cidx])
    if hp.size:   # t0 on the previous composited cell's exit plane
        dt0 = r_t0[hp] - d_delta[hp]
        pjo, pjt = EV(f["jo_v"][cidx[hp]], f["jo_e"][cidx[hp]]), EV(f["jt_v"][cidx[hp]], f["jt_e"][cidx[hp]])
        rs.add(cidx[hp], oc, dt0[:, None] * pjo)
        rs.add(cidx[hp], dc, (dt0 * pjt)[:, None] * pjo)
    rs.add(cidx, oc, d_delta[:, None] * jo)                  # t1 on this cell's exit plane
    rs.add(cidx, dc, (d_delta * jt)[:, None] * jo)
    f["jo_v"][cidx], f["jo_e"][cidx] = jo.v, jo.e
    f["jt_v"][cidx], f["jt_e"][cidx] = jt.v, jt.e
    # colour: dL/drgb_c a[3k+c] dY_k/dd_i, one term per (k, c); a is exact
    dY = f["dY"][cidx]                                         # [r, K, 3]
    t_v = d_rgb.v[:, None, :, None] * coef[:, :, :, None] * dY.v[:, :, None, :]   # [r, K, c, i]
    t_e = (np.abs(coef)[:, :, :, None] * (np.abs(dY.v[:, :, None, :]) * d_rgb.e[:, None, :, None]
                                         + np.abs(d_rgb.v[:, None, :, None]) * dY.e[:, :, None, :])
           + 2 * U * np.abs(t_v))
    k_terms = t_v.shape[1] * t_v.shape[2]
    rs.add(cidx, dc, EV(t_v.sum((1, 2)), t_e.sum((1, 2))), abs_=np.abs(t_v).sum((1, 2)), n=k_terms)


def _ray_finish(out, sel, rs, d: EV, d_in):
    """ray_grad of a chunk's rays: the sums' bounds, then the unit direction's gradient taken back through
    d = d_in / |d_in| (|d_in| in fp32: gamma_3 / 2 + u relative)."""
    b = rs.bound()
    g = EV(rs.value[:, 3:], b[:, 3:])
    dg = _dot(d, g, 3)
    norm_v = np.linalg.norm(d_in, axis=1)
    norm = EV(norm_v, (gamma(3) / 2 + U) * norm_v)
    gd = (g - d * dg[:, None]) / norm[:, None]
    out["ray_grad"][sel, :3] = rs.value[:, :3]
    out["ray_grad_err"][sel, :3] = b[:, :3]
    out["ray_grad"][sel, 3:] = gd.v
    out["ray_grad_err"][sel, 3:] = gd.e


def compare(got: dict, m: dict, **kw) -> dict:
    """model64.compare, and ``ray_grad`` within its bound on the unambiguous rays when both sides carry it."""
    report = M.compare({k: v for k, v in got.items() if k != "ray_grad"}, m, **kw)
    if "ray_grad" in got and "ray_grad" in m:
        ok = ~m["ambiguous"]
        M._within("ray_grad", got["ray_grad"].astype(np.float64)[ok], m["ray_grad"][ok], m["ray_grad_err"][ok])
    return report


def check_implementation(impl, points, attributes, adjacency, offsets, rays, start, quantiles, grad_rgba,
                         grad_depth, ray_error=None, weight_threshold=0.001, max_intersections=1024,
                         contribution=True, half_atomics=False, ray_grad=False) -> dict:
    """Trace a case with an implementation and hold every output to the model.

    ``impl(rays, start, quantiles, grad_rgba, grad_depth, ray_error, backward)`` returns numpy outputs of
    the forward (with contribution) and, with ``backward``, of the backward on its own saved rgba and depth
    indices.  Ambiguous rays get zero upstream gradients and ray error in both the model and the
    implementation, so the image and its layout stay as given; where any exist, ``contribution`` (a
    forward output) is compared on a flat batch of the unambiguous rays instead.  With ``ray_grad`` the model
    carries ray gradients, and the implementation's ``ray_grad`` output is held to them."""
    settings = (weight_threshold, max_intersections)
    scene = (points, attributes, adjacency, offsets)
    m0 = trace(*scene, rays, start, quantiles, *settings, backward=False)
    amb = m0["ambiguous"]
    g = np.where(amb[..., None], 0, grad_rgba).astype(grad_rgba.dtype)
    gd = None if grad_depth is None else np.where(amb[..., None], 0, grad_depth).astype(grad_depth.dtype)
    err = None if ray_error is None else np.where(amb.reshape(ray_error.shape), 0, ray_error).astype(ray_error.dtype)
    got = impl(rays, start, quantiles, g, gd, err, True)
    m = trace(*scene, rays, start, quantiles, *settings, rgba=got["rgba"], grad_rgba=g, grad_depth=gd,
              depth_indices=got.get("depth_indices"), ray_error=err, ray_grad=ray_grad)
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
