"""The CUDA kernels on stale scenes (tests/stale_cases.py), held to the float64 model and to the reference's kernels.

A training step traces points that have moved since the adjacency was built: the optimizer moves them every step,
the triangulation is rebuilt only every few dozen steps.  On such a foam most rays skip cells with t1 <= t0, the
backward recomputes a composited cell's entry plane after skipped cells instead of carrying the previous exit plane
over, and rays can stop inside the scene.  Every case here prints and asserts floors on that staleness, and holds
every output entry to the model as tests/test_gpu_model64.py does: integers exactly and floats within their bound
on the unambiguous rays, every scatter row within its per-entry bound, ray gradients within theirs."""
import time
import warnings

import numpy as np
import pytest

import common
import masked_frame as MF
import model64 as M
import model64_rays as MR
import refgold
import stale_cases as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def staleness(case, floors, rays=None):
    f = case.foam
    m = M.trace(f.points, f.attributes, f.adjacency, f.offsets, case.rays, case.start, case.quantiles,
                backward=False)
    st = S.stats(m, f.points, rays)
    S.assert_floors(st, *floors)
    return st


def device_impl(torch, f, attr_dtype, tape, contribution=True, ray_grad=False, pipe=None, paths=None):
    """check_implementation's ``impl`` on the product's Pipeline.  ``paths`` collects, per backward, the path that
    ran: "replay" when its forward recorded the whole walk into the tape, "re-walk" when the tape is off or the
    recording overflowed the tape pool (the backward then walks again)."""
    import radfoam_b200

    half = attr_dtype == np.float16
    pipe = pipe or radfoam_b200.create_pipeline(f.sh_degree, "float16" if half else "float32")
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    scene = [dev(x) for x in (f.points, f.attributes.astype(attr_dtype), f.adjacency, f.offsets)]
    if tape:  # scene tensors that require grad make the forward record the walk tape
        scene[0].requires_grad_(True)
        scene[1].requires_grad_(True)
    pipe.record_tape = tape

    def run(rays, start, dq, g, gd, err, backward):
        rays_d, start_d, dq_d = dev(rays), dev(start), dev(dq)
        fwd = pipe.trace_forward(*scene, rays_d, start_d, depth_quantiles=dq_d,
                                 return_contribution=contribution or not backward)
        out = {k: v.cpu().numpy() for k, v in fwd.items()}
        if backward:
            if paths is not None:
                status = pipe.tape_status() if tape else None
                replay = tape and status["used_chunks"] > 0 and not status["overflowed"]
                paths.append("replay" if replay else "re-walk")
            bwd = pipe.trace_backward(*scene, rays_d, start_d, fwd["rgba"], dev(g), dq_d, fwd.get("depth_indices"),
                                      dev(gd), dev(err), return_ray_grad=ray_grad)
            out.update({k: v.cpu().numpy() for k, v in bwd.items() if k != "ray_grad" or ray_grad})
        torch.cuda.synchronize()
        return out
    return run


def check_case(torch, name, case, attr_dtype=np.float32, tape=False, contribution=True, ray_grad=False):
    """Hold one case to the model on a new pipeline.  With the tape on, a first recording that overflows the tape pool
    (which then grows) re-walks; the case is traced again on the same pipeline, and that backward must replay.  Every
    run is held to the model.  Returns the last report and the backward path of every run."""
    import radfoam_b200

    f = case.foam
    pipe = radfoam_b200.create_pipeline(f.sh_degree, "float16" if attr_dtype == np.float16 else "float32")
    err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(attr_dtype)
    paths = []
    for step in range(2):
        t = time.perf_counter()
        impl = device_impl(torch, f, attr_dtype, tape, contribution, ray_grad, pipe, paths)
        report = MR.check_implementation(impl, f.points, f.attributes.astype(attr_dtype), f.adjacency, f.offsets,
                                         case.rays, case.start, case.quantiles, case.grad_rgba.astype(attr_dtype),
                                         case.grad_depth, err, contribution=contribution, ray_grad=ray_grad)
        assert report["rays_compared"] == report["rays"] - report["ambiguous"]
        assert report["ambiguous"] < 0.05 * report["rays"]
        print("\n" + M.format_report(f"{name} step {step}", report)
              + f" | ambiguous {report['ambiguous']} | backward {paths[-1]} ({time.perf_counter() - t:.1f} s)")
        if not tape or paths[-1] == "replay":
            break
    assert paths[-1] == ("replay" if tape else "re-walk"), paths
    return report, paths


# ------------------------------------------------------------------ config 1, every kernel instantiation
@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
@pytest.mark.parametrize("mode", ["cached", "direct"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("q", [0, 2])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_config1_stale_within_model_bounds(torch_cuda, deg, q, dtype, mode, tape, monkeypatch):
    """Config 1 with its points moved: noise of half the nearest-neighbour distance at odd degrees, a coherent field
    of the median spacing at even ones."""
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    kind, frac, floors = (("noise", 0.5, (0.6, 0.08, 1)) if deg % 2 else ("field", 1.0, (0.4, 0.05, 0)))
    case = S.stale_case(common.config1(deg, q, fixed_quantiles=False), frac, kind, seed=1)
    st = staleness(case, floors)
    check_case(torch_cuda, f"stale config1 {kind} f={frac} deg{deg} q{q} {np.dtype(dtype).name} {mode} tape={tape}",
               case, dtype, tape)
    print(f"  {st}")


# ------------------------------------------------------------------ the 20 k shell scene
SCENE_FLOORS = {0.2: (0.3, 0.015, 0), 0.5: (0.8, 0.07, 100)}


def scene20k_stale(frac, inside):
    return S.stale_case(common.scene_case(inside=inside), frac, "noise", seed=2)


@pytest.mark.parametrize("contribution", [True, False], ids=["contribution", "training"])
@pytest.mark.parametrize("inside", [False, True], ids=["outside", "inside"])
@pytest.mark.parametrize("frac", [0.2, 0.5])
def test_scene20k_stale_within_model_bounds(torch_cuda, frac, inside, contribution):
    """With ray gradients and the tape on.  Without ``return_contribution`` the forward runs the fast kernel and its
    exact twin that a training step runs (with it, only the per-ray scan mode); both are held to the model.  A first
    recording that overflows the tape pool re-walks; the second step then replays (check_case)."""
    case = scene20k_stale(frac, inside)
    st = staleness(case, SCENE_FLOORS[frac])
    check_case(torch_cuda, f"stale scene20k f={frac} inside={inside} contribution={contribution}", case, tape=True,
               contribution=contribution, ray_grad=True)
    print(f"  {st}")


def test_random_batch_stale_within_model_bounds(torch_cuda):
    """An unordered batch from 16 cameras on the moved points, start cells from ``starting_points`` on them."""
    import radfoam_b200

    torch = torch_cuda
    base = common.random_ray_case()
    f = S.stale(base.foam, 0.3, "noise", seed=3)
    start = radfoam_b200.starting_points(torch.from_numpy(base.rays).cuda(), torch.from_numpy(f.points).cuda())
    case = common.Case(f, base.rays, start.cpu().numpy(), base.quantiles)
    case.grad_rgba, case.grad_depth = base.grad_rgba, base.grad_depth
    assert np.array_equal(case.start, S.start_cells(f.points, base.rays))
    st = staleness(case, (0.4, 0.03, 1))
    check_case(torch, "stale random batch 20k", case, tape=True, ray_grad=True)
    print(f"  {st}")


# ------------------------------------------------------------------ a training sequence on one pipeline
def test_training_sequence_on_one_pipeline(torch_cuda):
    """Three steps of TraceRays autograd with the tape on, the points moved in place between steps as an optimizer
    step does (the scene mirrors are invalidated through the tensors' _version, the tape key changes with them),
    start cells from ``starting_points`` on each step's points.  Each step is held to the model of its points."""
    import radfoam_b200
    from radfoam_b200 import foam

    torch = torch_cuda
    base = common.scene_case()
    f = base.foam
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    pipe = radfoam_b200.create_pipeline(3)
    pts = dev(f.points).requires_grad_(True)
    attrs = dev(f.attributes).requires_grad_(True)
    adj, off = dev(f.adjacency), dev(f.offsets)
    rays, dq = dev(base.rays), dev(base.quantiles)
    moved = f.points.copy()
    for step in range(3):
        if step:
            delta = S.displacement(moved, 0.25, "noise", seed=40 + step).astype(np.float32)
            with torch.no_grad():
                pts.add_(dev(delta))
            moved = pts.detach().cpu().numpy()
        start = radfoam_b200.starting_points(rays, pts)
        case = common.Case(foam.Foam(moved, f.attributes, f.adjacency, f.offsets, 3), base.rays,
                           start.cpu().numpy(), base.quantiles)
        m0 = M.trace(moved, f.attributes, f.adjacency, f.offsets, base.rays, case.start, base.quantiles,
                     backward=False)
        st = S.stats(m0, moved)
        amb = m0["ambiguous"]
        g = np.where(amb[..., None], 0, base.grad_rgba).astype(np.float32)
        gd = np.where(amb[..., None], 0, base.grad_depth).astype(np.float32)
        pts.grad = attrs.grad = None
        rgba, depth, _, nint, _ = radfoam_b200.TraceRays.apply(pipe, pts, attrs, adj, off, rays, start, dq, False)
        status = pipe.tape_status()
        ((rgba * dev(g)).sum() + (depth * dev(gd)).sum()).backward()
        got = {"rgba": rgba.detach().cpu().numpy(), "depth": depth.detach().cpu().numpy(),
               "num_intersections": nint.cpu().numpy(), "points_grad": pts.grad.cpu().numpy(),
               "attr_grad": attrs.grad.cpu().numpy()}
        di = pipe.trace_forward(pts.detach(), attrs.detach(), adj, off, rays, start, depth_quantiles=dq)
        got["depth_indices"] = di["depth_indices"].cpu().numpy()
        m = M.trace(moved, f.attributes, f.adjacency, f.offsets, base.rays, case.start, base.quantiles,
                    rgba=got["rgba"], grad_rgba=g, grad_depth=gd, depth_indices=got["depth_indices"])
        report = M.compare(got, m)
        replay = status["used_chunks"] > 0 and not status["overflowed"]
        print("\n" + M.format_report(f"training step {step}", report) + f" | ambiguous {int(amb.sum())} | backward "
              f"{'replay' if replay else 're-walk (tape overflowed)'} | {st}")
        if step:
            # the first recording sized the tape pool; the stale steps after it replay
            assert replay, status
            S.assert_floors(st, 0.2 * step, 0.01 * step)


# ------------------------------------------------------------------ the parameter form
def test_params_stale_step_within_model_bounds(torch_cuda):
    """One stale step through the parameter form (bound parameters, re-layout and finalize kernels)."""
    from test_gpu_param_scene import check_params_case

    case = scene20k_stale(0.5, False)
    st = staleness(case, SCENE_FLOORS[0.5])
    check_params_case(torch_cuda, "params stale scene20k f=0.5", case, np.float32, tape=True)
    print(f"  {st}")


# ------------------------------------------------------------------ full size: config 4
def test_config4_stale_fullframe_within_model_bounds(torch_cuda, monkeypatch):
    """Config 4's 1 M-point foam with its points moved by f = 0.2, the 1920x1080 frame (more CTAs than the sorted
    replay takes, so the default replay is unsorted).  S = a dense block, one lane per warp and the longest walks,
    about 1 M model ray-steps; the unsorted and sorted replay, the re-walk, the direct backward and the replay with
    ray gradients."""
    import bench
    from test_gpu_fullframe_model64 import SORTED_REPLAY_MAX_CTAS, Frame

    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    moved = S.stale(f, 0.2, "noise", seed=4).points
    fr = Frame(torch_cuda, 1 << 20, 1920, 1080, points=moved)
    ctas = MF.cta_count(1080, 1920)
    assert ctas > SORTED_REPLAY_MAX_CTAS
    status = fr.pipe.tape_status()
    cx, cy = 1920 // 2 // 16 * 16, 1080 // 2 // 8 * 8
    nint = fr.num_intersections.reshape(-1).astype(np.int64)
    sel = np.unique(np.concatenate([MF.block(1080, 1920, cx - 32, cy - 16, 64, 32),
                                    MF.one_lane_per_warp(1080, 1920, 2048), MF.longest(nint, 256)]))
    steps = int(nint[sel].sum())
    assert steps < 1_500_000, steps
    runs = {"replay unsorted": fr.run(monkeypatch),
            "replay sorted": fr.run(monkeypatch, order="1"),
            "re-walk": fr.run(monkeypatch, tape=False),
            "direct": fr.run(monkeypatch, mode="direct"),
            "replay unsorted ray_grad": fr.run(monkeypatch, ray_grad=True)}
    m = {}
    fr.check("stale config4 1080p f=0.2", sel, runs, model=m)
    st = S.stats(m, moved)
    print(f"stale config4: {ctas} CTAs, tape {status}, {steps} model ray-steps; S: {st}")
    S.assert_floors(st, 0.2, 0.005)


# ------------------------------------------------------------------ negative control
def test_stale_outputs_fail_the_unmoved_model(torch_cuda):
    """The stale run's outputs held to the model of the unmoved foam must not pass: the check sees the move."""
    base = common.scene_case()
    case = scene20k_stale(0.2, False)
    f, f0 = case.foam, base.foam
    impl = device_impl(torch_cuda, f, np.float32, tape=True)
    with pytest.raises(M.Mismatch):
        M.check_implementation(impl, f0.points, f0.attributes, f0.adjacency, f0.offsets, case.rays, case.start,
                               case.quantiles, case.grad_rgba, case.grad_depth)


# ------------------------------------------------------------------ the reference's kernels on stale scenes
def stale_ref_cases():
    """name -> (case, attr dtype) of the stored reference outputs (tests/golden/make_golden_reference.py stale)."""
    import bench
    from radfoam_b200 import foam

    cases = {}
    for frac in (0.2, 0.5):
        for inside in (False, True):
            cases[f"scene20k_f{frac}_{'inside' if inside else 'outside'}"] = lambda frac=frac, inside=inside: \
                scene20k_stale(frac, inside)
    cases["random60k"] = lambda: S.stale_case(common.random_ray_case(num_points=60000, num_rays=100000), 0.2, "noise",
                                              seed=5)

    def config4():
        f = bench.load_or_build_foam(1 << 20, lambda m: None)
        moved = S.stale(f, 0.2, "noise", seed=4)
        cam = (2.5, 2.5, 2.5)
        rays = foam.pinhole_rays(1920, 1080, cam, fov=0.9)
        start = np.full((1080, 1920), foam.nearest_point(moved.points, cam), dtype=np.uint32)
        return common.Case(moved, rays, start, common._quantiles((1080, 1920), 2, 23), seed=7)
    cases["config4"] = config4
    return cases


REF_CASES = stale_ref_cases()


@pytest.mark.parametrize("name", list(REF_CASES))
def test_stale_matches_reference_kernels(torch_cuda, name):
    """Traversal integers equal, rgba / depth within 1e-5, gradients within 1e-5 of max|ref| (or 4x the reference's
    own run-to-run noise), on the default replay path."""
    from test_gpu_parity import assert_forward_equal, run_ours

    case = REF_CASES[name]()
    ref = refgold.load("stale", name)
    got = run_ours(torch_cuda, case, tape=True, repeat=2)
    assert_forward_equal(got, ref)
    noise = float(ref["grad_noise"])
    err = max(refgold.grad_error(got[k], ref, k) for k in ("points_grad", "attr_grad"))
    print(f"\n{name}: gradients {err:.2e} of max|ref| (reference vs itself {noise:.2e})")
    assert err <= max(1e-5, 4 * noise)
