"""CPU tests of the ray gradient dL/d(origin, direction): the float64 model's definition
(tests/model64_rays.py, ``trace(..., ray_grad=True)``) against finite differences and exact invariances, and
the product's kernel sources, run on the CPU emulator (tests/emu/emu_rays.py), against the model's per-ray
bounds."""
import os
import sys
import warnings

import numpy as np
import pytest

import common
import model64 as M
import model64_rays as MR
from test_model64 import fd_case

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def upstream(batch, q, loss, seed=17):
    rng = np.random.default_rng(seed)
    g = rng.normal(size=batch + (4,))
    g[..., :3] *= loss == "rgb"
    g[..., 3] *= loss == "alpha"
    gd = None if q == 0 else rng.normal(size=batch + (q,)) * (loss == "depth")
    return g, gd


# ------------------------------------------------------------------ the model's definition
@pytest.mark.parametrize("quirks", [True, False])
@pytest.mark.parametrize("deg,q", [(3, 2), (1, 3), (0, 0)])
def test_ray_model_restates_model64(deg, q, quirks):
    """model64_rays.trace restates model64.trace's walk to reach the per-cell quantities: with or without ray
    gradients it computes exactly model64's outputs, bounds and ambiguity."""
    case = common.config1(deg, q, fixed_quantiles=False)
    f = case.foam
    err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1])
    args = (f.points, f.attributes, f.adjacency, f.offsets, case.rays, case.start, case.quantiles)
    kw = dict(grad_rgba=case.grad_rgba, grad_depth=case.grad_depth, ray_error=err, quirks=quirks)
    ref = M.trace(*args, **kw)
    for ray_grad in (False, True):
        got = MR.trace(*args, ray_grad=ray_grad, **kw)
        assert ("ray_grad" in got) == ray_grad
        for k, v in ref.items():
            if isinstance(v, M.Scatter):
                for a in ("value", "err", "abs", "count"):
                    assert np.array_equal(getattr(v, a), getattr(got[k], a)), (k, a)
            else:
                assert np.array_equal(v, got[k]), k


@pytest.mark.parametrize("loss", ["rgb", "alpha", "depth"])
@pytest.mark.parametrize("kind,deg,q", [("config1", 0, 1), ("config1", 1, 3), ("config1", 2, 0),
                                        ("config1", 3, 2), ("small_foam", 0, 3), ("small_foam", 3, 1)])
def test_ray_grad_matches_finite_differences(kind, deg, q, loss):
    """True derivative, exact planes: ray_grad against central differences of the model's forward in each
    origin and direction component, on rays whose walk does not change under the step."""
    if loss == "depth" and q == 0:
        pytest.skip("no depth quantiles")
    f, rays, start, dq = fd_case(kind, deg, q)
    rays = rays.astype(np.float64)
    batch = rays.shape[:-1]
    g, gd = upstream(batch, q, loss)
    kw = dict(planes="exact", weight_threshold=0.0 if loss == "depth" else 0.001)
    scene = (f.points.astype(np.float64), f.attributes.astype(np.float64), f.adjacency, f.offsets)
    base = M.trace(*scene, rays, start, dq, backward=False, **kw)
    m = MR.trace(*scene, rays, start, dq, rgba=base["rgba"], grad_rgba=g, grad_depth=gd,
                depth_indices=base.get("depth_indices"), quirks=False, ray_grad=True, **kw)
    rg = m["ray_grad"].reshape(-1, 6)
    scale = np.abs(rg).max()
    flat_rays, flat_start = rays.reshape(-1, 6), start.reshape(-1)
    flat_dq = None if dq is None else dq.reshape(-1, q)
    flat_g, flat_gd = g.reshape(-1, 4), None if gd is None else gd.reshape(-1, q)
    nint = base["num_intersections"].reshape(-1)

    def value(ray_row, i):
        one = lambda a: None if a is None else a[i:i + 1]      # noqa: E731
        out = M.trace(*scene, ray_row[None], flat_start[i:i + 1], one(flat_dq), backward=False, **kw)
        v = (flat_g[i] * out["rgba"][0]).sum()
        if flat_gd is not None:
            v += (flat_gd[i] * np.where(out["depth_indices"][0] == M.NONE, 0.0, out["depth"][0])).sum()
        return v, int(out["num_intersections"].reshape(-1)[0])

    rng = np.random.default_rng(5)
    h = 1e-6
    checked = 0
    for col in range(6):
        rows = np.flatnonzero(np.abs(rg[:, col]) > 1e-4 * scale)
        for i in rng.permutation(rows)[:3]:
            plus, minus = flat_rays[i].copy(), flat_rays[i].copy()
            plus[col] += h
            minus[col] -= h
            vp, np_ = value(plus, i)
            vm, nm = value(minus, i)
            if np_ != nint[i] or nm != nint[i]:
                continue                                      # the walk changed: not differentiable here
            fd = (vp - vm) / (2 * h)
            assert abs(fd - rg[i, col]) <= 1e-5 * (abs(rg[i, col]) + 1e-3 * scale), (i, col, fd, rg[i, col])
            checked += 1
    assert checked >= 6


@pytest.mark.parametrize("deg,q", [(3, 2), (1, 3), (0, 0)])
def test_ray_grad_invariances(deg, q):
    """True derivative, exact planes.  Translating every point and origin together changes nothing, so
    sum(points_grad) + sum over rays of dL/do = 0; scaling a direction changes nothing, so d . dL/dd = 0 per ray.
    Both hold to rounding level (float64) relative to the sums' magnitudes."""
    case = common.config1(deg, q, fixed_quantiles=False)
    f = case.foam
    args = (f.points, f.attributes, f.adjacency, f.offsets, case.rays, case.start, case.quantiles)
    fwd = M.trace(*args, planes="exact", backward=False)
    m = MR.trace(*args, rgba=fwd["rgba"], grad_rgba=case.grad_rgba, grad_depth=case.grad_depth,
                 depth_indices=fwd.get("depth_indices"), planes="exact", quirks=False, ray_grad=True)
    rg = m["ray_grad"].reshape(-1, 6)
    pg = m["points_grad"]
    total = pg.value.sum(0) + rg[:, :3].sum(0)
    mag = pg.abs.sum(0) + np.abs(rg[:, :3]).sum(0)
    assert (mag > 0).all()
    assert (np.abs(total) <= 1e-11 * mag).all(), (total, mag)
    d = case.rays.reshape(-1, 6)[:, 3:].astype(np.float64)
    dot = (d * rg[:, 3:]).sum(1)
    assert (np.abs(dot) <= 1e-13 * np.linalg.norm(d, axis=1) * np.linalg.norm(rg[:, 3:], axis=1) + 1e-300).all()


@pytest.mark.parametrize("deg,q", [(3, 2), (2, 3), (0, 0)])
def test_ray_grad_modes_differ_by_stabilisers_only(deg, q):
    """quirks=True (the 1e-6 stabilisers in dL/dalpha, the rgb == 0 mask) and quirks=False (neither) use the
    same planes and gd_q, so their ray gradients differ by stabiliser-sized amounts only."""
    case = common.config1(deg, q, fixed_quantiles=False)
    f = case.foam
    args = (f.points, f.attributes, f.adjacency, f.offsets, case.rays, case.start, case.quantiles)
    fwd = M.trace(*args, backward=False)
    kw = dict(rgba=fwd["rgba"], grad_rgba=case.grad_rgba, grad_depth=case.grad_depth,
              depth_indices=fwd.get("depth_indices"), ray_grad=True)
    quirk = MR.trace(*args, quirks=True, **kw)["ray_grad"].reshape(-1, 6)
    true = MR.trace(*args, quirks=False, **kw)["ray_grad"].reshape(-1, 6)
    assert np.abs(true).max() > 0 and not np.array_equal(quirk, true)
    # the stabilisers perturb dL/dalpha by about 1e-6 / (1 - alpha) relative: 1e-6 for most cells, more on
    # the few rays that cross a nearly opaque cell.  Relative to each ray's largest origin / direction entry:
    for group in (slice(0, 3), slice(3, 6)):
        scale = np.maximum(np.abs(true[:, group]).max(1, keepdims=True), 1e-30)
        rel = (np.abs(quirk[:, group] - true[:, group]) / scale).max(1)
        assert np.median(rel) <= 2e-6 and np.quantile(rel, 0.99) <= 1e-3 and rel.max() <= 0.1, \
            (np.median(rel), np.quantile(rel, 0.99), rel.max())


# ------------------------------------------------------------------ the kernel sources on the emulator
def emu_ray_impl(sh_degree, attr_dtype, f, tape, **settings):
    import emu_rays

    pipe = emu_rays.EmuRayPipeline(sh_degree, attr_dtype)
    scene = (f.points, f.attributes.astype(attr_dtype), f.adjacency, f.offsets)

    def run(rays, start, dq, g, gd, err, backward):
        fwd = pipe.trace_forward(*scene, rays, start, dq, return_contribution=True, record_tape=tape,
                                 scene_version=7 if tape else 0, **settings)
        if not backward:
            return fwd
        args = (None,) * 6 if tape else scene + (rays, start)
        bwd = pipe.trace_backward(*args, fwd["rgba"], g.astype(attr_dtype), None if tape else dq,
                                  fwd.get("depth_indices"), gd, err, use_tape=tape,
                                  scene_version=7 if tape else 0, ray_grad=True, **settings)
        return {**fwd, **bwd}
    return run


def run_emu_ray_case(case, attr_dtype, mode, tape, monkeypatch, **settings):
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    f = case.foam
    err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(attr_dtype)
    return MR.check_implementation(
        emu_ray_impl(f.sh_degree, attr_dtype, f, tape, **settings), f.points, f.attributes.astype(attr_dtype),
        f.adjacency, f.offsets, case.rays, case.start, case.quantiles, case.grad_rgba.astype(attr_dtype),
        case.grad_depth, err, ray_grad=True, **settings)


@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
@pytest.mark.parametrize("mode", ["cached", "direct"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("deg,q", [(0, 0), (1, 2), (2, 3), (3, 2), (3, 0), (0, 3)])
def test_emulated_ray_grad_within_model_bounds(deg, q, dtype, mode, tape, monkeypatch):
    """Every output, ray_grad included, within the model's bounds."""
    case = common.config1(deg, q, fixed_quantiles=False)
    report = run_emu_ray_case(case, dtype, mode, tape, monkeypatch)
    assert report["rays_compared"] == report["rays"] - report["ambiguous"]


@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
def test_emulated_ray_grad_small_scene_within_model_bounds(tape, monkeypatch):
    case = common.scene_case(num_points=1500, width=48, height=32, q=2)
    run_emu_ray_case(case, np.float32, "cached", tape, monkeypatch)


@pytest.mark.parametrize("mode", ["cached", "direct"])
def test_default_backward_leaves_ray_grad_untouched(mode, monkeypatch):
    """Without the flag a sentinel-filled ray_grad comes back byte for byte; points_grad and attr_grad are the
    same with and without ray gradients, up to the order of their atomic sums (which already varies from run to
    run): both lie within the model's per-entry bounds."""
    import emu_rays

    monkeypatch.setenv("RFB_BWD_MODE", mode)
    case = common.config1(3, 2, fixed_quantiles=False)
    f = case.foam
    pipe = emu_rays.EmuRayPipeline(3, np.float32)
    scene = (f.points, f.attributes, f.adjacency, f.offsets)
    fwd = pipe.trace_forward(*scene, case.rays, case.start, case.quantiles)
    args = scene + (case.rays, case.start, fwd["rgba"], case.grad_rgba.astype(np.float32), case.quantiles,
                    fwd["depth_indices"], case.grad_depth)
    sentinel = np.full(case.rays.shape, np.nan, np.float32).view(np.uint32)
    sentinel[...] = 0x7fc0dead
    buf = sentinel.copy().view(np.float32)
    plain = pipe.trace_backward(*args, ray_grad_buffer=buf)
    assert np.array_equal(buf.view(np.uint32), sentinel)
    rays = pipe.trace_backward(*args, ray_grad=True)
    assert np.isfinite(rays["ray_grad"]).all() and np.abs(rays["ray_grad"]).max() > 0
    m = M.trace(*scene, case.rays, case.start, case.quantiles, rgba=fwd["rgba"], grad_rgba=case.grad_rgba,
                grad_depth=case.grad_depth, depth_indices=fwd["depth_indices"])
    assert not m["ambiguous"].any()
    for out in (plain, rays):
        M.compare({k: out[k] for k in ("points_grad", "attr_grad")}, m)


def test_ray_grad_flag_without_buffer_is_an_error():
    import emu_rays

    case = common.config1(0, 0)
    f = case.foam
    pipe = emu_rays.EmuRayPipeline(0, np.float32)
    scene = (f.points, f.attributes, f.adjacency, f.offsets)
    fwd = pipe.trace_forward(*scene, case.rays, case.start)
    lib = pipe.lib
    import ctypes
    from radfoam_b200 import _lib as abi

    opts = abi.LaunchOpts(0, 0, abi.FLAG_RAY_GRAD)
    settings = abi.TraceSettings(0.001, 1024)
    c = lambda a, dt: np.ascontiguousarray(a, dt)  # noqa: E731
    keep = [c(f.points, np.float32), c(f.attributes, np.float32), c(f.adjacency, np.uint32),
            c(f.offsets, np.uint32), c(case.rays, np.float32), c(case.start, np.uint32), fwd["rgba"],
            c(case.grad_rgba, np.float32), np.empty((f.num_points, 3), np.float32),
            np.empty((f.num_points, f.attributes.shape[1]), np.float32)]
    p = [a.ctypes.data_as(ctypes.c_void_p) for a in keep]
    rc = lib.rfb_trace_backward(pipe.handle, ctypes.byref(settings), f.num_points, p[0], p[1], keep[2].size, p[2],
                                p[3], case.rays.size // 6, p[4], p[5], 0, None, None, p[6], p[7], None, None, None,
                                p[8], p[9], None, ctypes.byref(opts), None)
    assert rc != 0 and b"ray_grad" in lib.rfb_last_error()


def test_accumulate_rays_matches_trace_backward(monkeypatch):
    """The split backward's rfb_trace_backward_accumulate_rays gives the same ray_grad as rfb_trace_backward."""
    import emu_rays

    monkeypatch.setenv("RFB_BWD_MODE", "cached")
    case = common.config1(2, 2, fixed_quantiles=False)
    f = case.foam
    pipe = emu_rays.EmuRayPipeline(2, np.float32)
    scene = (f.points, f.attributes, f.adjacency, f.offsets)
    fwd = pipe.trace_forward(*scene, case.rays, case.start, case.quantiles)
    args = scene + (case.rays, case.start, fwd["rgba"], case.grad_rgba.astype(np.float32), case.quantiles,
                    fwd["depth_indices"], case.grad_depth)
    full = pipe.trace_backward(*args, ray_grad=True)["ray_grad"]
    _, split = pipe.trace_backward_accumulate(*args, ray_grad=True)
    assert np.array_equal(full.view(np.uint32), split.view(np.uint32))
