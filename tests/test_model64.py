"""CPU tests of the float64 model with error bounds (tests/model64.py) and of its comparator.

They establish that the model is sound before it judges any kernel: its true-derivative mode matches
finite differences of its own forward; its reference mode differs from the true derivative exactly where
SURVEY.md A.5 says; the reference's kernels' stored outputs lie inside its per-entry bounds; the
comparator catches changes the max-normalised bar misses; and the product's kernel sources, run on the
CPU emulator, pass the same comparison."""
import glob
import os
import sys
import warnings

import numpy as np
import pytest

import common
import model64 as M
from radfoam_b200 import foam

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))

GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))
                if not os.path.basename(p).startswith(("benchmark", "farthest")))


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def load(path):
    z = dict(np.load(path))
    scene = (z["points"], z["attributes"], z["adjacency"], z["offsets"])
    settings = (float(z["weight_threshold"]), int(z["max_intersections"]))
    return z, scene, settings


def golden_model(z, scene, settings):
    q = z.get("quantiles")
    m = M.trace(*scene, z["rays"], z["start"], q, *settings, rgba=z["out_rgba"], grad_rgba=z["grad_rgba"],
                grad_depth=z.get("grad_depth"), depth_indices=z.get("out_depth_indices"))
    # the stored gradients include every ray's terms: leave out what an ambiguous ray could have touched
    skip = M.rows_reachable(m, z["offsets"], z["adjacency"], z["points"], z["attributes"], z["rays"],
                            z["start"], q, *settings)
    return m, skip


def golden_outputs(z):
    return {k[4:]: v for k, v in z.items() if k.startswith("out_")}


# ------------------------------------------------------------------ the reference inside the bounds
def test_all_golden_cases_present():
    assert len(GOLDEN) == 11


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_outputs_within_model_bounds(path):
    """Every output of the reference's kernels (integers exactly, floats per entry) on unambiguous rays and
    on every scatter row no ambiguous ray can reach.  The fp16 case's gradients are half atomics."""
    z, scene, settings = load(path)
    m, skip = golden_model(z, scene, settings)
    report = M.compare(golden_outputs(z), m, half_atomics=True, skip_rows=skip)
    print("\n" + M.format_report(os.path.basename(path)[:-4], report))
    assert report["rays_compared"] >= 0.99 * report["rays"]


# ------------------------------------------------------------------ the comparator's discriminating power
def single_ray_terms(z, scene, settings, ray):
    """The model's gradient terms of one ray alone (flat index), with the reference's saved outputs."""
    sl = np.unravel_index(ray, z["rays"].shape[:-1])
    q = z.get("quantiles")
    one = lambda a: None if a is None else a[sl][None]      # noqa: E731
    return M.trace(*scene, one(z["rays"]), one(z["start"]), one(q), *settings, rgba=one(z["out_rgba"]),
                   grad_rgba=one(z["grad_rgba"]), grad_depth=one(z.get("grad_depth")),
                   depth_indices=one(z.get("out_depth_indices")))


@pytest.mark.parametrize("key", ["points_grad", "attr_grad"])
def test_lost_ray_contribution_on_a_small_row_is_caught(key):
    """Drop one ray's terms from a row below 1e-4 of the largest: the per-entry bound fails, the old bar
    (1e-5 of max |ref|) passes."""
    z, scene, settings = load(os.path.join(os.path.dirname(__file__), "golden", "config1_deg3_q2.npz"))
    m, skip = golden_model(z, scene, settings)
    ref = z["out_" + key].astype(np.float64)
    scale = np.abs(ref).max()
    bound = m[key].bound()
    small = np.flatnonzero((np.abs(ref).max(1) < 1e-4 * scale) & (m[key].count > 1) & ~skip)
    assert small.size
    rays_ok = np.flatnonzero(~m["ambiguous"].reshape(-1))
    for ray in rays_ok:
        t = single_ray_terms(z, scene, settings, ray)[key]
        rows = small[t.count[small] > 0]
        for row in rows:
            col = int(np.argmax(np.abs(t.value[row])))
            c = t.value[row, col]
            if bound[row, col] < abs(c) < 1e-5 * scale:
                mutated = z["out_" + key].copy()
                mutated[row, col] -= np.float32(c)
                got = golden_outputs(z)
                got[key] = mutated
                assert common.grad_error(mutated, z["out_" + key]) <= 1e-5
                with pytest.raises(M.Mismatch, match=key):
                    M.compare(got, m, half_atomics=True, skip_rows=skip)
                return
    pytest.fail("no small row with a removable ray term")


def test_half_atomic_gradients_fail_the_rounded_once_bound():
    """The reference's fp16 gradients are half atomics; ours are accumulated in fp32 and rounded once.  The
    tighter of the two bounds rejects the former, which the old fp16 bar (2e-2 of max) accepts."""
    z, scene, settings = load(os.path.join(os.path.dirname(__file__), "golden", "config1_deg3_q2_half.npz"))
    m, skip = golden_model(z, scene, settings)
    got = golden_outputs(z)
    M.compare(got, m, half_atomics=True, skip_rows=skip)
    assert common.grad_error(got["attr_grad"].astype(np.float32), m["attr_grad"].value) <= 2e-2
    with pytest.raises(M.Mismatch, match="attr_grad"):
        M.compare(got, m, half_atomics=False, skip_rows=skip)


# ------------------------------------------------------------------ finite differences
def fd_case(kind, deg, q):
    if kind == "config1":
        case = common.config1(deg, q, fixed_quantiles=False)
        f, rays, start, dq = case.foam, case.rays[::4, ::4], case.start[::4, ::4], case.quantiles
        dq = None if dq is None else dq[::4, ::4]
    else:
        f = foam.small_foam(96, sh_degree=deg, seed=deg + 3)
        rays = foam.pinhole_rays(8, 8, (0.2, -2.5, 0.4), fov=0.8)
        start = np.full((8, 8), foam.nearest_point(f.points, (0.2, -2.5, 0.4)), dtype=np.uint32)
        dq = None if q == 0 else np.sort(np.random.default_rng(deg).uniform(0.1, 0.9, (8, 8, q)),
                                         axis=-1)[..., ::-1].astype(np.float32).copy()
    return f, rays, start, dq


@pytest.mark.parametrize("loss", ["rgb", "alpha", "depth"])
@pytest.mark.parametrize("kind,deg,q", [("config1", 0, 1), ("config1", 1, 3), ("config1", 2, 0),
                                        ("config1", 3, 2), ("small_foam", 0, 3), ("small_foam", 3, 1)])
def test_true_derivative_matches_finite_differences(kind, deg, q, loss):
    if loss == "depth" and q == 0:
        pytest.skip("no depth quantiles")
    f, rays, start, dq = fd_case(kind, deg, q)
    pts = f.points.astype(np.float64)
    attrs = f.attributes.astype(np.float64)
    batch = rays.shape[:-1]
    rng = np.random.default_rng(17)
    g = rng.normal(size=batch + (4,))
    g[..., :3] *= loss == "rgb"
    g[..., 3] *= loss == "alpha"
    gd = None if dq is None else rng.normal(size=batch + (q,)) * (loss == "depth")
    kw = dict(planes="exact", weight_threshold=0.0 if loss == "depth" else 0.001)

    def value(p, a):
        out = M.trace(p, a, f.adjacency, f.offsets, rays, start, dq, backward=False, **kw)
        v = (g * out["rgba"]).sum()
        if gd is not None:
            v += (gd * np.where(out["depth_indices"] == M.NONE, 0.0, out["depth"])).sum()
        return v, out

    _, base = value(pts, attrs)
    m = M.trace(pts, attrs, f.adjacency, f.offsets, rays, start, dq, rgba=base["rgba"], grad_rgba=g,
                grad_depth=gd, depth_indices=base.get("depth_indices"), quirks=False, **kw)
    pg, ag = m["points_grad"].value, m["attr_grad"].value
    h = 1e-6
    checked = 0
    for arr, grad, name in ((pts, pg, "points"), (attrs, ag, "attributes")):
        cols = [arr.shape[1] - 1, 0, arr.shape[1] // 2] if name == "attributes" else [0, 1, 2]
        for col in cols:
            rows = np.flatnonzero(np.abs(grad[:, col]) > 1e-4 * np.abs(grad).max())
            if name == "attributes" and col == arr.shape[1] - 1:
                # a step across the density gate sigma > 1e-6 switches the colour on: not differentiable there
                rows = rows[np.abs(arr[rows, col] - 1e-6) > 2 * h]
            for row in rng.permutation(rows)[:4]:
                plus, minus = arr.copy(), arr.copy()
                plus[row, col] += h
                minus[row, col] -= h
                vp, op = value(plus, attrs) if name == "points" else value(pts, plus)
                vm, om = value(minus, attrs) if name == "points" else value(pts, minus)
                if not (np.array_equal(op["num_intersections"], base["num_intersections"])
                        and np.array_equal(om["num_intersections"], base["num_intersections"])):
                    continue                                  # the walk changed: not differentiable here
                fd = (vp - vm) / (2 * h)
                assert abs(fd - grad[row, col]) <= 1e-5 * (abs(grad[row, col]) + 1e-3 * np.abs(grad).max()), \
                    (name, row, col, fd, grad[row, col])
                checked += 1
    assert checked >= 6


# ------------------------------------------------------------------ quirk structure
@pytest.mark.parametrize("deg,q", [(3, 2), (1, 3)])
def test_quirks_differ_from_true_derivative_only_where_a5_says(deg, q):
    """Exact planes: (reference backward) - (true derivative) is nonzero on points only at each ray's first
    composited cell (the origin term), last composited cell and its successor (the two accumulators never
    written); on SH coefficients nowhere; on density only by stabiliser-sized amounts."""
    case = common.config1(deg, q, fixed_quantiles=False)
    f = case.foam
    args = (f.points, f.attributes, f.adjacency, f.offsets, case.rays, case.start, case.quantiles)
    fwd = M.trace(*args, planes="exact", backward=False)
    assert not fwd["skipped"].any()
    # grad_depth is zero here: the depth term's dL/dt0 quirk (gd / sigma instead of gd, see model64) touches
    # every cell a quantile falls in, which the row pattern below does not single out
    kw = dict(rgba=fwd["rgba"], grad_rgba=case.grad_rgba, grad_depth=np.zeros_like(case.grad_depth),
              depth_indices=fwd.get("depth_indices"), planes="exact")
    quirk = M.trace(*args, quirks=True, **kw)
    true = M.trace(*args, quirks=False, **kw)
    comp = fwd["last_cell"] >= 0
    allowed = np.zeros(f.num_points, dtype=bool)
    for k in ("first_cell", "last_cell", "last_next"):
        allowed[fwd[k][comp]] = True
    dp = quirk["points_grad"].value - true["points_grad"].value
    scale = np.abs(true["points_grad"].value).max()
    tol = 1e-9 * scale + 1e-4 * true["points_grad"].abs      # the stabilisers, through dL/ddelta
    assert (np.abs(dp[~allowed]) <= tol[~allowed]).all()
    # the quirks are not vacuous: the allowed rows do differ
    assert (np.abs(dp[allowed]) > 1e-3 * scale).any()
    da = quirk["attr_grad"].value - true["attr_grad"].value
    assert np.array_equal(da[:, :-1], np.zeros_like(da[:, :-1]))
    dens = true["attr_grad"].abs[:, -1]
    # the 1e-6 stabilisers perturb dL/dalpha by about 1e-6 / (1 - alpha) relative
    assert (np.abs(da[:, -1]) <= 1e-4 * dens + 1e-12).all()


# ------------------------------------------------------------------ the kernel sources on the emulator
def emu_impl(sh_degree, attr_dtype, f, tape, **settings):
    import emu

    pipe = emu.EmuPipeline(sh_degree, attr_dtype)
    scene = (f.points, f.attributes.astype(attr_dtype), f.adjacency, f.offsets)

    def run(rays, start, dq, g, gd, err, backward):
        fwd = pipe.trace_forward(*scene, rays, start, dq, return_contribution=True, record_tape=tape,
                                 scene_version=7 if tape else 0, **settings)
        if not backward:
            return fwd
        args = (None,) * 6 if tape else scene + (rays, start)
        bwd = pipe.trace_backward(*args, fwd["rgba"], g.astype(attr_dtype), None if tape else dq,
                                  fwd.get("depth_indices"), gd, err, use_tape=tape,
                                  scene_version=7 if tape else 0, **settings)
        return {**fwd, **bwd}
    return run


def run_emu_case(case, attr_dtype, mode, tape, monkeypatch, **settings):
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    f = case.foam
    err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(attr_dtype)
    report = M.check_implementation(
        emu_impl(f.sh_degree, attr_dtype, f, tape, **settings), f.points, f.attributes.astype(attr_dtype),
        f.adjacency, f.offsets, case.rays, case.start, case.quantiles, case.grad_rgba.astype(attr_dtype),
        case.grad_depth, err, **settings)
    return report


@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
@pytest.mark.parametrize("mode", ["cached", "direct"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("deg,q", [(0, 0), (1, 2), (2, 3), (3, 2), (3, 0), (0, 3)])
def test_emulated_kernels_within_model_bounds(deg, q, dtype, mode, tape, monkeypatch):
    case = common.config1(deg, q, fixed_quantiles=False)
    report = run_emu_case(case, dtype, mode, tape, monkeypatch)
    print("\n" + M.format_report(f"emu deg{deg} q{q} {np.dtype(dtype).name} {mode} tape={tape}", report))


@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
def test_emulated_kernels_small_scene_within_model_bounds(tape, monkeypatch):
    case = common.scene_case(num_points=1500, width=48, height=32, q=2)
    report = run_emu_case(case, np.float32, "cached", tape, monkeypatch)
    print("\n" + M.format_report(f"emu scene1500 tape={tape}", report))


def test_compare_fp16_overflow_to_inf():
    """An fp16 scatter entry whose sum reaches 65520 rounds to inf of its sign; a wrong sign, or inf where the bound
    stays below the overflow, is still a mismatch."""
    s = M.Scatter(3, 1)
    s.add(np.array([0, 1, 2]), [0], M.EV(np.array([[7e4], [-7e4], [6e4]])))
    s.flush()
    m = {"ambiguous": np.zeros(0, dtype=bool), "attr_grad": s}
    ok = np.array([[np.inf], [-np.inf], [6e4]], dtype=np.float16)
    M.compare({"attr_grad": ok}, m, per_ray=False)
    for bad in ([[-np.inf], [-np.inf], [6e4]], [[np.inf], [-np.inf], [np.inf]]):
        with pytest.raises(M.Mismatch):
            M.compare({"attr_grad": np.array(bad, dtype=np.float16)}, m, per_ray=False)
