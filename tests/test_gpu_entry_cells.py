"""Entry cells held to their contract: ``nearest_point`` (smallest fp32 distance, ties to the lowest index, UINT32_MAX
for a NaN query), ``starting_points`` (``nearest_point`` of every ray's origin, through the device-side de-duplication
of the origins) and ``locate_points`` on a stale foam (a local minimum of the distance over the graph).  A training
step recomputes start cells on the moved points, so these run on fresh and on moved foams."""
import numpy as np
import pytest

import common
import locate_model as lm
import stale_cases as S

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF
GAP = 8 * lm.U32  # fp32 d2 keeps the order of squared distances further apart than GAP * (d1^2 + d2^2)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def exact_nearest(torch, points, queries):
    """The contract restated: per query the smallest (fp32 d2 in the kernels' fma order, index) key over all points,
    computed exactly (tests/locate_model.py); UINT32_MAX for a query with a NaN coordinate.  int64 numpy."""
    p, q = dev(torch, points), dev(torch, queries)
    n = p.shape[0]
    idx = torch.arange(n, device="cuda")
    out = torch.empty(q.shape[0], dtype=torch.int64, device="cuda")
    step = max(1, (1 << 22) // n)
    for s in range(0, q.shape[0], step):
        k = lm.keys(p, idx[None, :], q[s:s + step, None, :]).amin(1)
        out[s:s + step] = k & 0xFFFFFFFF
    out[torch.isnan(q).any(1)] = NONE
    return out.cpu().numpy()


def check_nearest(torch, points, queries, got):
    """``got`` (uint32 numpy, nearest_point's result for ``queries``) against the contract: equal to the exact
    restatement on every query; equal to cKDTree's float64 nearest wherever its best and second-best squared
    distances are further apart than the fp32 rounding of d2 can bridge, and within that gap everywhere else."""
    from scipy.spatial import cKDTree

    got = got.astype(np.int64)
    want = exact_nearest(torch, points, queries)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} queries differ from the exact rule, e.g. query {bad[:4]}: {got[bad[:4]]} " \
                          f"vs {want[bad[:4]]}"
    fin = np.isfinite(queries).all(1)
    p64, q64 = points.astype(np.float64), queries[fin].astype(np.float64)
    d, i = cKDTree(p64).query(q64, k=2, workers=-1)
    d1, d2 = d[:, 0] ** 2, d[:, 1] ** 2
    clear = d2 - d1 > GAP * (d1 + d2)
    assert np.array_equal(got[fin][clear], i[clear, 0])
    dg = ((p64[got[fin]] - q64) ** 2).sum(1)
    assert np.all(dg - d1 <= GAP * (dg + d1))
    return int(clear.sum()), int((~clear).sum())


@pytest.fixture(scope="module")
def foams():
    f = common.scene_case(num_points=60000, width=320, height=200).foam
    return {"fresh": f.points, "moved": S.stale(f, 0.2, "noise", seed=6).points}


def tie_points(points, count=48, seed=8):
    """A copy of ``points`` with ``count`` crafted exact ties and their queries: the query q lies on a 2^-10 grid,
    the two points at q + v and q - v (or at q + v and q + a permutation of v) with v a small multiple of 2^-12, so
    every difference and every square is exact and both d2 are equal.  The pair sits in different tiles of the
    kernel's point stream, the lower index alternately first and second.  Returns (points, queries, lower index)."""
    rng = np.random.default_rng(seed)
    pts = points.copy()
    n = pts.shape[0]
    q = np.round(rng.uniform(-1.4, 1.4, size=(count, 3)) * 1024) / 1024
    v = rng.integers(1, 6, size=(count, 3)) * 2.0 ** -12
    lo = rng.choice(np.arange(0, n // 2), size=count, replace=False)
    hi = rng.choice(np.arange(n // 2, n), size=count, replace=False)
    for k in range(count):
        a = q[k] + v[k]
        b = q[k] - v[k] if k % 3 else q[k] + v[k][[1, 2, 0]]
        first, second = (a, b) if k % 2 else (b, a)
        pts[lo[k]], pts[hi[k]] = first.astype(np.float32), second.astype(np.float32)
    # coincident points: the same position at two indices, queried from a nearby offset
    dup_lo = rng.choice(np.setdiff1d(np.arange(n // 2), lo), size=16, replace=False)
    dup_hi = rng.choice(np.setdiff1d(np.arange(n // 2, n), hi), size=16, replace=False)
    pts[dup_hi] = pts[dup_lo]
    dq = pts[dup_lo] + np.float32(1e-4)
    queries = np.concatenate([q.astype(np.float32), dq])
    return pts, queries, np.concatenate([lo, dup_lo])


@pytest.mark.parametrize("which", ["fresh", "moved"])
def test_nearest_point_contract(torch_cuda, foams, which):
    """4,096 queries around and inside the shell, NaN queries, the points themselves and crafted exact ties."""
    import radfoam_b200

    torch = torch_cuda
    pts = foams[which]
    rng = np.random.default_rng(2)
    n = pts.shape[0]
    own = rng.choice(n, size=64, replace=False)
    queries = np.concatenate([rng.normal(0, 1.2, size=(3000, 3)), rng.uniform(-1.6, 1.6, size=(960, 3)),
                              pts[own].astype(np.float64)]).astype(np.float32)
    nan = np.array([[np.nan, 0, 0], [0, np.nan, 0], [0, 0, np.nan], [np.nan] * 3], dtype=np.float32)
    queries = np.concatenate([queries, np.resize(nan, (4096 - queries.shape[0], 3))])
    got = radfoam_b200.nearest_point(dev(torch, pts), dev(torch, queries)).cpu().numpy()
    assert got.dtype == np.uint32
    clear, close = check_nearest(torch, pts, queries, got)
    assert np.array_equal(got[3960:4024], own.astype(np.uint32))          # a point is its own nearest point
    assert (got[np.isnan(queries).any(1)] == NONE).all()
    tp, tq, lower = tie_points(pts)
    tgot = radfoam_b200.nearest_point(dev(torch, tp), dev(torch, tq)).cpu().numpy()
    assert np.array_equal(exact_nearest(torch, tp, tq), lower)             # the crafted ties are the nearest pairs
    assert np.array_equal(tgot, lower.astype(np.uint32)), np.flatnonzero(tgot != lower)
    print(f"\n{which}: {clear} clear queries equal cKDTree, {close} within the fp32 gap, {lower.size} ties to the "
          f"lower index")


def start_rays(origins, repeat, seed):
    rng = np.random.default_rng(seed)
    o = np.repeat(origins, repeat, axis=0)
    perm = rng.permutation(o.shape[0])
    d = rng.normal(size=o.shape)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.concatenate([o[perm], d], axis=1).astype(np.float32), perm


@pytest.mark.parametrize("which", ["fresh", "moved"])
def test_starting_points_contract(torch_cuda, foams, which):
    """4,096 distinct origins, each on several rays in random order, some differing only in the sign of a zero
    component, one NaN: every ray's start cell is nearest_point of its origin, bit for bit.  Then a 2 M-ray frame from
    one origin."""
    import radfoam_b200

    torch = torch_cuda
    pts = foams[which]
    rng = np.random.default_rng(3)
    origins = rng.normal(0, 1.5, size=(4096, 3)).astype(np.float32)
    origins[:256, 0] = 0.0
    origins[256:512] = origins[:256]
    origins[256:512, 0] = -0.0                   # same value, different bits: a distinct origin to the hash
    origins[512:520, 1:] = 0.0
    origins[520:528] = origins[512:520] * np.float32(-1.0)
    origins[4095] = np.nan
    assert np.unique(origins.view(np.uint32), axis=0).shape[0] == 4096
    rays, perm = start_rays(origins, 5, seed=4)
    pts_d = dev(torch, pts)
    got = radfoam_b200.starting_points(dev(torch, rays), pts_d).cpu().numpy()
    per_origin = radfoam_b200.nearest_point(pts_d, dev(torch, origins)).cpu().numpy()
    check_nearest(torch, pts, origins, per_origin)
    want = np.repeat(per_origin, 5)[perm]
    assert np.array_equal(got, want), f"{int((got != want).sum())} rays differ"
    assert per_origin[4095] == NONE and np.array_equal(per_origin[:256], per_origin[256:512])
    # one camera: 1920 x 1080 rays from a single origin
    from radfoam_b200 import foam

    frame = foam.pinhole_rays(1920, 1080, (2.5, 2.5, 2.5), fov=0.9)
    sp = radfoam_b200.starting_points(dev(torch, frame), pts_d)
    one = radfoam_b200.nearest_point(pts_d, dev(torch, frame[0, 0, :3][None])).cpu().numpy()[0]
    assert sp.shape == (1080, 1920) and bool((lm.as_long(sp) == int(one)).all())
    assert one == exact_nearest(torch, pts, frame[0, 0, :3][None])[0]


def test_locate_points_stale_config4(torch_cuda):
    """locate_points with hints on config 4's foam with its points moved (f = 0.2): 2 M queries, the frame's median-depth
    points and nudged copies, each the cell the trace reported there as its hint.  Every result is a local minimum of
    (d2, index) over the graph; on a moved foam that is all the contract promises."""
    import bench
    import radfoam_b200

    torch = torch_cuda
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    moved = S.stale(f, 0.2, "noise", seed=4)
    fr = bench.make_frame(moved, 1920, 1080)
    pts, attrs, adj, off = (dev(torch, x) for x in (moved.points, moved.attributes, moved.adjacency, moved.offsets))
    pipe = radfoam_b200.create_pipeline(3)
    dq = torch.full((1080, 1920, 1), 0.5, device="cuda")
    out = pipe.trace_forward(pts, attrs, adj, off, dev(torch, fr["rays"]), dev(torch, fr["start"]), depth_quantiles=dq)
    rays = dev(torch, fr["rays"])
    depth, idx = out["depth"][..., 0], lm.as_long(out["depth_indices"][..., 0])
    hit = torch.isfinite(depth) & (idx != NONE)
    o = (rays[..., :3] + depth[..., None] * rays[..., 3:])[hit]
    hint = idx[hit]
    m = 2 * 1024 * 1024
    g = torch.Generator(device="cuda").manual_seed(0)
    pick = torch.randint(0, o.shape[0], (m - o.shape[0],), device="cuda", generator=g)
    q = torch.cat([o, o[pick] + 1e-3 * torch.randn((pick.shape[0], 3), device="cuda", generator=g)]).contiguous()
    hint = torch.cat([hint, hint[pick]]).to(torch.uint32)
    got = radfoam_b200.locate_points(pts, adj, off, q, hint=hint)
    ok = lm.local_min(pts, lm.as_long(adj), lm.as_long(off), q, got)
    assert bool(ok.all()), f"{int((~ok).sum())} of {q.shape[0]} results are not local minima"
    nearest = radfoam_b200.nearest_point(pts, q[:4096])
    moved_away = int((lm.as_long(nearest) != lm.as_long(got[:4096])).sum())
    print(f"\nstale config4: {q.shape[0]} queries, all local minima; {moved_away} of the first 4,096 are not the "
          f"global nearest point")
