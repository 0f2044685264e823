"""Independent torch restatement of point location and field sampling (rfb_locate_points / rfb_sample_field /
rfb_sample_field_backward), for the tests and tests/tools/locate_bench.py.  Runs on CPU or CUDA tensors.

* keys(): the kernels' (d2, index) order, d2 = fma(dx,dx, fma(dy,dy, dz*dz)) in fp32 recomputed EXACTLY: every fma
  is formed in float64 (the product of two floats is exact there), its error recovered with TwoSum, and the sum
  rounded to odd before the final rounding to fp32 (53 >= 24 + 2 bits, so that double rounding is innocuous).
* local_min(): is a result a local minimum of that order over the CSR graph?
* walk(): the greedy walk from given seeds, with the number of moves per query; sample_seeds(): the library's seeds.
* field64() / field_grad64(): float64 models of the sampled density / colour and of the attribute gradient, with
  per-entry error bounds.
"""
from __future__ import annotations

import numpy as np
import torch

NONE = 0xFFFFFFFF
INF_BITS = 0x7F800000
U32 = 2.0 ** -24  # unit roundoff of fp32


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c) of float32 tensors."""
    a64, b64, c64 = a.double(), b.double(), c.double()
    p = a64 * b64
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)  # s + err == a*b + c exactly
    inexact = (err != 0) & torch.isfinite(s)
    over = inexact & ((err < 0) == (s > 0))  # |exact| < |s|: truncating toward zero steps down one ulp
    t = torch.where(over, torch.nextafter(s, torch.zeros_like(s)), s)
    t = torch.where(inexact, (t.view(torch.int64) | 1).view(torch.float64), t)
    return t.float()


def d2_32(px, py, pz, qx, qy, qz):
    dx, dy, dz = px - qx, py - qy, pz - qz  # fp32 subtractions, round to nearest
    return fma32(dx, dx, fma32(dy, dy, dz * dz))


def keys(points, idx, q):
    """int64 keys (d2 bits << 32 | index) of points[idx] for queries q (broadcasting); NaN counts as +inf."""
    p = points[idx]
    d2 = d2_32(p[..., 0], p[..., 1], p[..., 2], q[..., 0], q[..., 1], q[..., 2])
    bits = d2.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    bits = torch.where(torch.isnan(d2), torch.full_like(bits, INF_BITS), bits)
    return (bits << 32) | idx.to(torch.int64)


def _row_min(points, adj, off, cur, q):
    """Smallest neighbour key of row cur[i] for query q[i] (int64 max for an empty row)."""
    begin, end = off[cur], off[cur + 1]
    counts = end - begin
    owner = torch.repeat_interleave(torch.arange(cur.numel(), device=cur.device), counts)
    first = torch.cumsum(counts, 0) - counts
    pos = begin[owner] + torch.arange(owner.numel(), device=cur.device) - first[owner]
    k = keys(points, adj[pos], q[owner])
    out = torch.full((cur.numel(),), torch.iinfo(torch.int64).max, dtype=torch.int64, device=cur.device)
    return out.scatter_reduce(0, owner, k, reduce="amin")


def as_long(t):
    return t.view(torch.int32).to(torch.int64) & 0xFFFFFFFF if t.dtype == torch.uint32 else t.to(torch.int64)


def csr(adjacency, offsets, device):
    adj = torch.as_tensor(np.asarray(adjacency, dtype=np.int64), device=device)
    off = torch.as_tensor(np.asarray(offsets, dtype=np.int64), device=device)
    return adj, off


def local_min(points, adj, off, queries, result, chunk=1 << 20):
    """Bool per query: result[i] is a local minimum of (d2, index) over the graph (queries without a cell: True
    when the result is UINT32_MAX and the query has a NaN coordinate)."""
    result = as_long(result)
    nan = torch.isnan(queries).any(-1)
    ok = torch.empty(result.numel(), dtype=torch.bool, device=result.device)
    for s in range(0, result.numel(), chunk):
        r, q, n = result[s:s + chunk], queries[s:s + chunk], nan[s:s + chunk]
        good = torch.zeros_like(r, dtype=torch.bool)
        valid = (r != NONE) & ~n
        if valid.any():
            rv, qv = r[valid], q[valid]
            good[valid] = keys(points, rv, qv) <= _row_min(points, adj, off, rv, qv)
        good |= n & (r == NONE)
        ok[s:s + chunk] = good
    return ok


def sample_seeds(points, queries, sample):
    """The library's seed: the nearest of points[k * stride], k < sample, in (d2, index) order (point 0 when no
    sample point is at a finite distance)."""
    n = points.shape[0]
    sample = min(sample, n)
    chunk = max(256, (1 << 22) // sample)
    cand = torch.arange(sample, device=points.device, dtype=torch.int64) * (n // sample)
    out = torch.empty(queries.shape[0], dtype=torch.int64, device=points.device)
    for s in range(0, queries.shape[0], chunk):
        q = queries[s:s + chunk]
        k = keys(points, cand[None, :].expand(q.shape[0], -1), q[:, None, :]).amin(1)
        out[s:s + chunk] = torch.where((k >> 32) >= INF_BITS, torch.zeros_like(k), k & 0xFFFFFFFF)
    return out


def walk(points, adj, off, queries, seeds):
    """(cells, moves) of the greedy walk from `seeds`; NaN queries -> (UINT32_MAX, 0)."""
    cur = as_long(seeds).clone()
    key = keys(points, cur, queries)
    moves = torch.zeros_like(cur)
    active = torch.nonzero(~torch.isnan(queries).any(-1)).flatten()
    while active.numel():
        best = _row_min(points, adj, off, cur[active], queries[active])
        move = best < key[active]
        idx = active[move]
        key[idx] = best[move]
        cur[idx] = best[move] & 0xFFFFFFFF
        moves[idx] += 1
        active = idx
    cells = torch.where((key >> 32) >= INF_BITS, torch.full_like(cur, NONE), cur)
    cells = torch.where(torch.isnan(queries).any(-1), torch.full_like(cur, NONE), cells)
    return cells, moves


# ---- the field, float64 -----------------------------------------------------------------------------------------
def sh_basis64(d, deg):
    """Real SH basis (sh_utils.cuh:34-70) of unit directions d [M, 3], float64."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    out = [np.full_like(x, 0.28209479177387814)]
    if deg > 0:
        c1 = 0.4886025119029199
        out += [-c1 * y, c1 * z, -c1 * x]
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        out += [1.0925484305920792 * x * y, -1.0925484305920792 * y * z, 0.31539156525252005 * (2 * zz - xx - yy),
                -1.0925484305920792 * x * z, 0.5462742152960396 * (xx - yy)]
    if deg > 2:
        out += [-0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * y * z,
                -0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
                -0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
                -0.5900435899266435 * x * (xx - 3 * yy)]
    return np.stack(out, axis=1)


def out_rounding(ref, dtype):
    """Half an ulp of the output dtype at |ref| (rounding the fp32 result once more to fp16)."""
    if np.dtype(dtype) == np.float16:
        return np.maximum(np.abs(ref), 6.1e-5) * 2.0 ** -11 + 2.0 ** -25
    return np.zeros_like(ref)


def field64(attributes, cells, directions, deg, dtype):
    """(density, rgb, rgb_bound) in float64 for cells [M] (all valid) and directions [M, 3] (or None)."""
    a = attributes.astype(np.float64)
    rows = a[cells.astype(np.int64)]
    density = rows[:, -1]
    if directions is None:
        return density, None, None
    d = directions.astype(np.float64)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    y = sh_basis64(d, deg)
    coef = rows[:, :-1].reshape(-1, (deg + 1) ** 2, 3)
    terms = y[:, :, None] * coef
    raw = 0.5 + terms.sum(1)
    rgb = np.maximum(raw, 0.0)
    # the FFMA chain of up to 16 terms plus the fp32 basis (direction renormalisation, products): a few dozen ulps
    # of the sum of magnitudes
    bound = 64 * U32 * (0.5 + np.abs(terms).sum(1)) + 32 * U32 * np.abs(coef).sum(1) + out_rounding(rgb, dtype)
    return density, rgb, bound


def field_grad64(num_points, deg, cells, directions, rgb, rgb_grad, density_grad, dtype):
    """(attr_grad [N, A], bound [N, A]) in float64: the scatter of rfb_sample_field_backward."""
    a_dim = 1 + 3 * (deg + 1) ** 2
    c = cells.astype(np.int64)
    valid = c < num_points
    c = c[valid]
    contrib = np.zeros((c.size, a_dim))
    gmag = np.zeros((c.size, a_dim))
    if rgb_grad is not None:
        d = directions[valid].astype(np.float64)
        d = d / np.linalg.norm(d, axis=1, keepdims=True)
        y = sh_basis64(d, deg)
        g = np.where(rgb[valid].astype(np.float64) == 0.0, 0.0, rgb_grad[valid].astype(np.float64))
        contrib[:, :-1] = (y[:, :, None] * g[:, None, :]).reshape(c.size, -1)
        gmag[:, :-1] = np.tile(np.abs(g), (deg + 1) ** 2)
    if density_grad is not None:
        contrib[:, -1] = density_grad[valid].astype(np.float64)
    grad = np.zeros((num_points, a_dim))
    mag = np.zeros((num_points, a_dim))
    count = np.zeros(num_points)
    np.add.at(grad, c, contrib)
    gsum = np.zeros((num_points, a_dim))
    np.add.at(mag, c, np.abs(contrib))
    np.add.at(gsum, c, gmag)
    np.add.at(count, c, 1.0)
    # per term: the fp32 basis, whose polynomials cancel (absolute error a few ulps of the O(1) monomials: 32u |g|)
    # and the product; then a sum of `count` terms in some order
    bound = (count[:, None] + 16) * 2 * U32 * mag + 32 * U32 * gsum + out_rounding(grad, dtype)
    return grad, bound
