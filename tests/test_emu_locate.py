"""Point location (rfb_locate_points) and field sampling (rfb_sample_field / rfb_sample_field_backward) on the CPU
kernel-logic emulator (tests/emu), against an independent torch restatement (tests/locate_model.py) and float64
references: scipy's cKDTree for the nearest point, float64 models with per-entry bounds for the sampled field and
its attribute gradient."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import fuzz_cases
import locate_model as lm
from radfoam_b200 import foam

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
import emu  # noqa: E402

NONE = 0xFFFFFFFF
# fp32 d2 = fma(dx,dx, fma(dy,dy, dz*dz)) with rounded differences: |d2_32 - d2| <= 6u d2 (u = 2^-24); two such
# distances keep their order when they differ by more than GAP * (d1 + d2).
GAP = 8 * lm.U32


def locate(points, adjacency, offsets, queries, hints=None):
    pts = np.ascontiguousarray(points, np.float32)
    adj, off = np.ascontiguousarray(adjacency, np.uint32), np.ascontiguousarray(offsets, np.uint32)
    q = np.ascontiguousarray(queries, np.float32).reshape(-1, 3)
    h = None if hints is None else np.ascontiguousarray(hints, np.uint32)
    out = np.full(q.shape[0], 12345, np.uint32)
    emu._check(emu.load().rfb_locate_points(emu._p(pts), pts.shape[0], emu._p(adj) if adj.size else None,
                                            emu._p(off), emu._p(q), q.shape[0], emu._p(h), emu._p(out), None))
    return out


def check_local_min(points, adjacency, offsets, queries, got):
    adj, off = lm.csr(adjacency, offsets, "cpu")
    ok = lm.local_min(torch.from_numpy(np.asarray(points, np.float32)), adj, off,
                      torch.from_numpy(np.asarray(queries, np.float32)), torch.from_numpy(got.astype(np.int64)))
    assert ok.all(), f"{int((~ok).sum())} results are not local minima, e.g. query {int(np.flatnonzero(~ok.numpy())[0])}"


def check_nearest(points, queries, got):
    """The cKDTree rule: equal to the float64 nearest point wherever the best / second-best gap exceeds the fp32
    rounding bound, and within that bound of the best distance everywhere."""
    p64, q64 = points.astype(np.float64), queries.astype(np.float64)
    d, i = cKDTree(p64).query(q64, k=2)
    d1, d2 = d[:, 0] ** 2, d[:, 1] ** 2
    clear = d2 - d1 > GAP * (d1 + d2)
    assert np.array_equal(got[clear], i[clear, 0].astype(np.uint32)), \
        f"{int((got[clear] != i[clear, 0]).sum())} clear-cut queries off the nearest point"
    dg = ((p64[got.astype(np.int64)] - q64) ** 2).sum(1)
    assert np.all(dg - d1 <= GAP * (dg + d1)), "a result farther than rounding from the nearest point"
    return int((~clear).sum())


def queries_for(f, rng, m):
    """Uniform points of the bounding box, the sites themselves, midpoints of Delaunay edges (on bisectors), and
    sites nudged by tiny offsets."""
    lo, hi = f.points.min(0), f.points.max(0)
    pick = rng.integers(0, f.num_points, m)
    rows = np.repeat(np.arange(f.num_points), np.diff(f.offsets.astype(np.int64)))
    e = rng.integers(0, f.adjacency.size, m)
    mid = 0.5 * (f.points[rows[e]].astype(np.float64) + f.points[f.adjacency[e]].astype(np.float64))
    return np.concatenate([rng.uniform(lo, hi, size=(m, 3)), f.points[pick].astype(np.float64), mid,
                           f.points[pick] + rng.normal(0, 1e-6, size=(m, 3)) * (hi - lo)]).astype(np.float32)


@pytest.mark.parametrize("sample", [None, "1", "7"])
@pytest.mark.parametrize("make", ["small", "scene"])
def test_walk_finds_the_nearest_point_on_a_delaunay_graph(make, sample, monkeypatch):
    """A seed sample of 1 or 7 points forces long walks on these small foams (the default sample covers them)."""
    if sample:
        monkeypatch.setenv("RFB_LOCATE_SAMPLE", sample)
    f = foam.small_foam(256, seed=3) if make == "small" else foam.scene_foam(3000, sh_degree=0, seed=5)
    q = queries_for(f, np.random.default_rng(1), 300)
    got = locate(f.points, f.adjacency, f.offsets, q)
    check_local_min(f.points, f.adjacency, f.offsets, q, got)
    check_nearest(f.points, q, got)


@pytest.mark.parametrize("seed", range(10))
def test_tie_heavy_scenes(seed, monkeypatch):
    """Lattices (exact and jittered), BCC, clusters, scaled scenes from tests/fuzz_cases.py, queried on sites, on
    bisectors and at random."""
    monkeypatch.setenv("RFB_LOCATE_SAMPLE", "5")
    rng = np.random.default_rng(1000 + seed)
    kind = fuzz_cases.SCENE_KINDS[seed % len(fuzz_cases.SCENE_KINDS)]
    f = fuzz_cases.make_scene(rng, kind, int(rng.integers(60, 400)), 0)
    q = queries_for(f, rng, 150)
    got = locate(f.points, f.adjacency, f.offsets, q)
    check_local_min(f.points, f.adjacency, f.offsets, q, got)
    check_nearest(f.points, q, got)


def test_stale_adjacency_gives_local_minima(monkeypatch):
    """Points moved after the triangulation: only the local-minimum property is promised."""
    monkeypatch.setenv("RFB_LOCATE_SAMPLE", "3")
    f = foam.small_foam(400, seed=8)
    rng = np.random.default_rng(2)
    moved = (f.points + rng.normal(0, 0.08, size=f.points.shape)).astype(np.float32)
    q = queries_for(f, rng, 200)
    got = locate(moved, f.adjacency, f.offsets, q)
    check_local_min(moved, f.adjacency, f.offsets, q, got)
    # the walk is the model's walk from the library's seeds
    adj, off = lm.csr(f.adjacency, f.offsets, "cpu")
    pts_t, q_t = torch.from_numpy(moved), torch.from_numpy(q)
    want, _ = lm.walk(pts_t, adj, off, q_t, lm.sample_seeds(pts_t, q_t, 3))
    assert np.array_equal(got.astype(np.int64), want.numpy())


def test_hints_in_range_out_of_range_and_null():
    f = foam.scene_foam(2000, sh_degree=0, seed=9)
    rng = np.random.default_rng(3)
    q = queries_for(f, rng, 100)
    m = q.shape[0]
    base = locate(f.points, f.adjacency, f.offsets, q)
    hints = rng.integers(0, f.num_points, m).astype(np.uint32)
    with_hints = locate(f.points, f.adjacency, f.offsets, q, hints)
    check_local_min(f.points, f.adjacency, f.offsets, q, with_hints)
    check_nearest(f.points, q, with_hints)
    adj, off = lm.csr(f.adjacency, f.offsets, "cpu")
    want, _ = lm.walk(torch.from_numpy(f.points), adj, off, torch.from_numpy(q), torch.from_numpy(hints.astype(np.int64)))
    assert np.array_equal(with_hints.astype(np.int64), want.numpy()), "hints are the walk's seeds"
    # hints that are not cells fall back to the library's seed: the same result as no hints at all
    bad = rng.choice(np.array([f.num_points, f.num_points + 7, NONE], dtype=np.uint32), m)
    assert np.array_equal(locate(f.points, f.adjacency, f.offsets, q, bad), base)
    mixed = np.where(rng.random(m) < 0.5, hints, bad).astype(np.uint32)
    check_nearest(f.points, q, locate(f.points, f.adjacency, f.offsets, q, mixed))


def test_nan_queries_empty_rows_and_no_queries():
    f = foam.small_foam(200, seed=4)
    rng = np.random.default_rng(5)
    q = queries_for(f, rng, 20)
    q[3, 0] = np.nan
    q[10, 2] = np.nan
    got = locate(f.points, f.adjacency, f.offsets, q)
    assert got[3] == NONE and got[10] == NONE
    check_local_min(f.points, f.adjacency, f.offsets, q, got)
    # an empty row: the walk stops there (hinted at it, the query stays in it)
    counts = np.diff(f.offsets.astype(np.int64))
    rows = [f.adjacency[f.offsets[i]:f.offsets[i + 1]] for i in range(f.num_points)]
    rows[17] = np.zeros(0, np.uint32)
    adj = np.concatenate(rows).astype(np.uint32)
    off = np.zeros(f.num_points + 1, np.uint32)
    off[1:] = np.cumsum([r.size for r in rows])
    assert counts[17] > 0
    got = locate(f.points, adj, off, q, np.full(q.shape[0], 17, np.uint32))
    assert np.all(got[~np.isnan(q).any(1)] == 17)
    check_local_min(f.points, adj, off, q, got)
    # no adjacency at all (one point, or every row empty)
    one = locate(f.points[:1], np.zeros(0, np.uint32), np.zeros(2, np.uint32), q)
    assert np.all(one[~np.isnan(q).any(1)] == 0)
    assert locate(f.points, f.adjacency, f.offsets, np.zeros((0, 3), np.float32)).size == 0


def test_shuffled_lane_schedule():
    """The seed search shares a shared-memory tile between the CTA's threads: under the emulator's shuffled resume
    order (RFB_EMU_SHUFFLE) a missing barrier gives wrong seeds.  Runs in a subprocess: the order is fixed at load."""
    code = f"""
import sys
sys.path[:0] = [{HERE!r}, {os.path.dirname(HERE)!r}]
import test_emu_locate as t
t._shuffled_body()
print("ok")
"""
    env = dict(os.environ, RFB_EMU_SHUFFLE="7", RFB_LOCATE_SAMPLE="1500")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stderr[-2000:]


def _shuffled_body():
    f = foam.scene_foam(3000, sh_degree=1, seed=6)
    rng = np.random.default_rng(6)
    q = queries_for(f, rng, 150)
    got = locate(f.points, f.adjacency, f.offsets, q)
    check_nearest(f.points, q, got)
    pts_t, q_t = torch.from_numpy(f.points), torch.from_numpy(q)
    seeds = lm.sample_seeds(pts_t, q_t, 1500)
    adj, off = lm.csr(f.adjacency, f.offsets, "cpu")
    want, _ = lm.walk(pts_t, adj, off, q_t, seeds)
    assert np.array_equal(got.astype(np.int64), want.numpy())
    pipe = emu.EmuPipeline(1)
    _check_sample_and_grad(pipe, f, q, rng, 1, np.float32)


# ---- field sampling ------------------------------------------------------------------------------------------------
def sample_field(pipe, f, attrs, q, dirs, hints=None):
    m = q.shape[0]
    pts, att = np.ascontiguousarray(f.points, np.float32), np.ascontiguousarray(attrs, pipe.dtype)
    adj, off = np.ascontiguousarray(f.adjacency, np.uint32), np.ascontiguousarray(f.offsets, np.uint32)
    q = np.ascontiguousarray(q, np.float32)
    d = None if dirs is None else np.ascontiguousarray(dirs, np.float32)
    h = None if hints is None else np.ascontiguousarray(hints, np.uint32)
    cells = np.empty(m, np.uint32)
    density = np.empty(m, pipe.dtype)
    rgb = None if d is None else np.empty((m, 3), pipe.dtype)
    emu._check(pipe.lib.rfb_sample_field(pipe.handle, emu._p(pts), pts.shape[0], emu._p(att), emu._p(adj),
                                         emu._p(off), emu._p(q), m, emu._p(h), emu._p(d), emu._p(cells),
                                         emu._p(density), emu._p(rgb), None))
    return cells, density, rgb


def sample_field_backward(pipe, n, cells, dirs, rgb, rgb_grad, density_grad):
    out = np.full((n, pipe.attr_dim), 7, pipe.dtype)  # fully overwritten
    c = np.ascontiguousarray(cells, np.uint32)
    args = [None if a is None else np.ascontiguousarray(a, t) for a, t in
            ((dirs, np.float32), (rgb, pipe.dtype), (rgb_grad, pipe.dtype), (density_grad, pipe.dtype))]
    emu._check(pipe.lib.rfb_sample_field_backward(pipe.handle, n, c.size, emu._p(c), *[emu._p(a) for a in args],
                                                  emu._p(out), None))
    return out


def _check_sample_and_grad(pipe, f, q, rng, deg, dtype):
    m = q.shape[0]
    attrs = f.attributes.astype(dtype)
    # make some colours clamp: a large negative DC term on a third of the cells
    attrs[rng.random(f.num_points) < 0.3, 0:3] = -4.0
    dirs = rng.normal(size=(m, 3)).astype(np.float32) * rng.choice([1e-3, 1.0, 1e3], size=(m, 1)).astype(np.float32)
    cells, density, rgb = sample_field(pipe, f, attrs, q, dirs)
    assert np.array_equal(cells, locate(f.points, f.adjacency, f.offsets, q))
    ok = cells != NONE
    want_d, want_rgb, bound = lm.field64(attrs, cells[ok], dirs[ok], deg, dtype)
    assert np.array_equal(density[ok].astype(np.float64), want_d), "density is the row's last column"
    err = np.abs(rgb[ok].astype(np.float64) - want_rgb)
    assert np.all(err <= bound), f"rgb off the float64 model by {float((err / bound).max()):.3g} bounds"
    assert np.isnan(density[~ok].astype(np.float32)).all() and np.isnan(rgb[~ok].astype(np.float32)).all()
    assert (rgb[ok] == 0).any(), "the clamp is exercised"
    # no directions: density only
    cells2, density2, rgb2 = sample_field(pipe, f, attrs, q, None)
    assert rgb2 is None and np.array_equal(cells2, cells) and np.array_equal(density2, density, equal_nan=True)
    # backward, many queries per cell
    g = rng.normal(size=(m, 3)).astype(dtype)
    dg = rng.normal(size=m).astype(dtype)
    for rgb_grad, density_grad in ((g, dg), (g, None), (None, dg)):
        got = sample_field_backward(pipe, f.num_points, cells, dirs, rgb, rgb_grad, density_grad)
        want, gb = lm.field_grad64(f.num_points, deg, cells, dirs, rgb, rgb_grad, density_grad, dtype)
        err = np.abs(got.astype(np.float64) - want)
        assert np.all(err <= gb), f"attr_grad off the float64 model by {float((err / np.maximum(gb, 1e-300)).max()):.3g} bounds"


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_sample_field_and_backward_vs_float64(deg, dtype):
    rng = np.random.default_rng(20 + deg)
    f = foam.small_foam(120, sh_degree=deg, seed=deg)
    # grid sampling (dozens of queries per cell) plus random points and a NaN query
    g = np.linspace(-0.9, 0.9, 9)
    grid = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    q = np.concatenate([grid, rng.uniform(-1, 1, size=(100, 3))]).astype(np.float32)
    q[5] = np.nan
    pipe = emu.EmuPipeline(deg, dtype)
    _check_sample_and_grad(pipe, f, q, rng, deg, dtype)


def test_sample_field_argument_checks():
    pipe = emu.EmuPipeline(1)
    f = foam.small_foam(50, sh_degree=1, seed=1)
    q = np.zeros((4, 3), np.float32)
    d = np.ones((4, 3), np.float32)
    with pytest.raises(RuntimeError, match="both"):
        pts = np.ascontiguousarray(f.points)
        emu._check(pipe.lib.rfb_sample_field(pipe.handle, emu._p(pts), 50, emu._p(f.attributes), emu._p(f.adjacency),
                                             emu._p(f.offsets), emu._p(q), 4, None, emu._p(d), emu._p(np.empty(4, np.uint32)),
                                             emu._p(np.empty(4, np.float32)), None, None))
    with pytest.raises(RuntimeError, match="rgb_grad needs"):
        sample_field_backward(pipe, 50, np.zeros(4, np.uint32), None, None, np.ones((4, 3), np.float32), None)
    # no queries: the gradient is all zeros
    assert not sample_field_backward(pipe, 50, np.zeros(0, np.uint32), None, None, None, None).any()
    # cells that are not points contribute nothing
    out = sample_field_backward(pipe, 50, np.array([NONE, 60, 2, 2], np.uint32), d, np.ones((4, 3), np.float32),
                                np.ones((4, 3), np.float32), np.ones(4, np.float32))
    assert out[2, -1] == 2.0 and np.count_nonzero(out[np.arange(50) != 2]) == 0
