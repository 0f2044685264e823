"""Ray gradients dL/d(origin, direction) of the CUDA kernels: every output held to the float64 model with
per-entry bounds (tests/model64_rays.py, ``ray_grad=True``), bit-identical ray gradients across the three backward
paths, ray layouts and runs, and the autograd ops' ``rays.grad``."""
import time
import warnings

import numpy as np
import pytest

import common
import fuzz_cases
import model64 as M
import model64_rays as MR

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


def device_impl(torch, f, attr_dtype, tape=False, pipe=None, statuses=None, **settings):
    """The product's Pipeline, ray gradients requested, as check_implementation's ``impl``."""
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
        fwd = pipe.trace_forward(*scene, rays_d, start_d, depth_quantiles=dq_d, return_contribution=True, **settings)
        if statuses is not None:
            statuses.append(pipe.tape_status()["overflowed"])
        out = {k: v.cpu().numpy() for k, v in fwd.items()}
        if backward:
            bwd = pipe.trace_backward(*scene, rays_d, start_d, fwd["rgba"], dev(g), dq_d, fwd.get("depth_indices"),
                                      dev(gd), dev(err), return_ray_grad=True, **settings)
            out.update({k: v.cpu().numpy() for k, v in bwd.items()})
        torch.cuda.synchronize()
        return out
    return run


def check_case(torch, name, case, attr_dtype=np.float32, tape=False, ray_error=True, impl=None, **settings):
    f = case.foam
    err = None
    if ray_error:
        err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(attr_dtype)
    t = time.perf_counter()
    report = MR.check_implementation(
        impl or device_impl(torch, f, attr_dtype, tape, **settings), f.points, f.attributes.astype(attr_dtype),
        f.adjacency, f.offsets, case.rays, case.start, case.quantiles, case.grad_rgba.astype(attr_dtype),
        case.grad_depth, err, ray_grad=True, **settings)
    print("\n" + M.format_report(name, report) + f" ({time.perf_counter() - t:.1f} s)")
    return report


# ------------------------------------------------------------------ against the model
@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
@pytest.mark.parametrize("mode", ["cached", "direct"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("q", [0, 2, 3])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_config1_ray_grad_within_model_bounds(torch_cuda, deg, q, dtype, mode, tape, monkeypatch):
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    check_case(torch_cuda, f"config1 deg{deg} q{q} {np.dtype(dtype).name} {mode} tape={tape}",
               common.config1(deg, q, fixed_quantiles=q != 3), dtype, tape)


@pytest.mark.parametrize("inside", [False, True], ids=["outside", "inside"])
def test_scene_ray_grad_within_model_bounds(torch_cuda, inside):
    """20 k-point shell scene.  From inside, the first recording overflows the tape pool (the backward
    re-walks), the second is replayed; both are held to the model."""
    import radfoam_b200

    case = common.scene_case(inside=inside)
    check_case(torch_cuda, f"scene20k inside={inside}", case)
    if inside:
        statuses = []
        impl = device_impl(torch_cuda, case.foam, np.float32, True, pipe=radfoam_b200.create_pipeline(3),
                           statuses=statuses)
        for step in range(2):
            check_case(torch_cuda, f"scene20k inside tape step {step}", case, ray_error=False, impl=impl)
        assert statuses[0] and not statuses[-1], statuses


@pytest.mark.parametrize("kwargs", [dict(max_intersections=1), dict(max_intersections=7),
                                    dict(weight_threshold=0.0), dict(weight_threshold=0.5)])
def test_trace_settings_ray_grad_within_model_bounds(torch_cuda, kwargs):
    check_case(torch_cuda, f"scene20k {kwargs}", common.scene_case(), **kwargs)


def test_random_ray_batch_ray_grad_within_model_bounds(torch_cuda):
    check_case(torch_cuda, "random rays 20k", common.random_ray_case())


@pytest.mark.parametrize("seed", list(range(9000, 9020)))
def test_fuzz_case_ray_grad_within_model_bounds(torch_cuda, seed):
    """Tie-heavy scenes; a case is only dropped when fewer than half of its rays can be compared."""
    scene_kind, ray_kind, f, rays, start, dq, kw = fuzz_cases.make_case(seed)
    m = M.trace(f.points, f.attributes, f.adjacency, f.offsets, rays, start, dq, backward=False,
                **{"weight_threshold": 0.001, "max_intersections": 1024, **kw})
    share = float(m["ambiguous"].mean())
    if share > 0.5:
        pytest.skip(f"{100 * share:.0f}% of the rays are ambiguous")
    check_case(torch_cuda, f"fuzz {seed}", common.Case(f, rays, start, dq, seed=seed), **kw)


CAMERA = (2.5, 2.5, 2.5)


def test_config4_crop_ray_grad_within_model_bounds(torch_cuda):
    """Config 4's 1 M-point foam: a 128x64 crop of the 1080p frame, traced as its own image with the tape on."""
    import bench
    from radfoam_b200 import foam

    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    rays = foam.pinhole_rays(1920, 1080, CAMERA, fov=0.9)[508:572, 896:1024].copy()
    start = np.full(rays.shape[:-1], foam.nearest_point(f.points, CAMERA), dtype=np.uint32)
    case = common.Case(f, rays, start, common._quantiles(rays.shape[:-1], 2, 22))
    check_case(torch_cuda, "config4 crop fp32", case, tape=True, ray_error=False)


# ------------------------------------------------------------------ determinism
def test_ray_grad_bit_identical_across_paths_layouts_and_runs(torch_cuda, monkeypatch):
    """ray_grad is a per-thread sum (no atomics): direct, cached re-walk and cached replay, an image layout and
    the same rays as a flat batch, and repeated runs all give the same bits."""
    import radfoam_b200

    torch = torch_cuda
    case = common.scene_case(q=2)
    f = case.foam
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    pts, attrs = dev(f.points).requires_grad_(True), dev(f.attributes).requires_grad_(True)
    adj, off = dev(f.adjacency), dev(f.offsets)
    results = {}
    for layout in ("image", "flat"):
        shape = case.rays.shape if layout == "image" else (-1, 6)
        rays = dev(case.rays.reshape(shape))
        start = dev(case.start.reshape(shape[:-1]))
        dq = dev(case.quantiles.reshape(tuple(shape[:-1]) + (2,)))
        g = dev(case.grad_rgba.reshape(tuple(shape[:-1]) + (4,)))
        gd = dev(case.grad_depth.reshape(tuple(shape[:-1]) + (2,)))
        for mode, tape in (("direct", False), ("cached", False), ("cached", True)):
            monkeypatch.setenv("RFB_BWD_MODE", mode)
            pipe = radfoam_b200.create_pipeline(f.sh_degree)
            pipe.record_tape = tape
            overflowed = []
            for run in range(3):  # the first recording may overflow the tape pool (re-walk); the pool then grows
                fwd = pipe.trace_forward(pts, attrs, adj, off, rays, start, depth_quantiles=dq)
                if tape:
                    overflowed.append(pipe.tape_status()["overflowed"])
                bwd = pipe.trace_backward(pts, attrs, adj, off, rays, start, fwd["rgba"], g, dq,
                                          fwd["depth_indices"], gd, return_ray_grad=True)
                results[(layout, mode, tape, run)] = bwd["ray_grad"].reshape(-1, 6).cpu().numpy().view(np.uint32)
            assert not tape or not overflowed[-1], overflowed  # the last run was a replay
    ref = results[("image", "direct", False, 0)]
    assert np.abs(ref.view(np.float32)).max() > 0
    for key, v in results.items():
        assert np.array_equal(v, ref), key


# ------------------------------------------------------------------ autograd
def _torch_case(torch, deg=3, q=2):
    case = common.config1(deg, q, fixed_quantiles=False)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    return case, dev


@pytest.mark.parametrize("op", ["TraceRays", "FoamScene_fused", "FoamScene_unfused"])
def test_autograd_rays_grad_equals_pipeline_ray_grad(torch_cuda, op):
    """rays.grad through the autograd ops equals the pipeline call's ray_grad for the same upstream gradients."""
    import radfoam_b200
    from radfoam_b200.scene_io import FoamScene

    torch = torch_cuda
    case, dev = _torch_case(torch)
    f = case.foam
    pipe = radfoam_b200.create_pipeline(3)
    rays = dev(case.rays).requires_grad_(True)
    start, dq = dev(case.start), dev(case.quantiles)
    g, gd = dev(case.grad_rgba), dev(case.grad_depth)
    adj, off = dev(f.adjacency), dev(f.offsets)
    if op == "TraceRays":
        pts, attrs = dev(f.points).requires_grad_(True), dev(f.attributes).requires_grad_(True)
        rgba, depth, _, _, _ = radfoam_b200.TraceRays.apply(pipe, pts, attrs, adj, off, rays, start, dq, False)
    else:
        a = dev(f.attributes)
        # density parameter whose activation softplus(x, beta=10) gives the foam's density back
        dens = a[:, -1:].clamp_min(1e-6)
        raw = torch.where(dens * 10 > 20, dens, torch.log(torch.expm1(dens * 10)) / 10)
        scene = FoamScene(dev(f.points).requires_grad_(True), raw.clone().requires_grad_(True),
                          a[:, :3].clone().requires_grad_(True), a[:, 3:-1].clone().requires_grad_(True),
                          adj, off, sh_degree=3)
        rgba, depth, _, _, _ = scene.forward(pipe, rays, start, dq, fused=op == "FoamScene_fused")
        pts, attrs = scene.get_trace_data()[:2]
        attrs = attrs.detach()
    ((rgba * g).sum() + (depth * gd).sum()).backward()
    assert rays.grad is not None and rays.grad.shape == rays.shape
    direct = radfoam_b200.create_pipeline(3)
    fwd = direct.trace_forward(pts.detach(), attrs.detach(), adj, off, rays.detach(), start, depth_quantiles=dq)
    bwd = direct.trace_backward(pts.detach(), attrs.detach(), adj, off, rays.detach(), start, fwd["rgba"], g, dq,
                                fwd["depth_indices"], gd, scrub_nonfinite=True, return_ray_grad=True)
    assert torch.equal(rgba.detach(), fwd["rgba"])
    assert np.array_equal(rays.grad.cpu().numpy().view(np.uint32), bwd["ray_grad"].cpu().numpy().view(np.uint32))


def test_autograd_rays_grad_only_when_requested(torch_cuda):
    import radfoam_b200

    torch = torch_cuda
    case, dev = _torch_case(torch)
    f = case.foam
    pipe = radfoam_b200.create_pipeline(3)
    pts = dev(f.points).requires_grad_(True)
    rays = dev(case.rays)
    rgba, *_ = radfoam_b200.TraceRays.apply(pipe, pts, dev(f.attributes), dev(f.adjacency), dev(f.offsets), rays,
                                            dev(case.start), None, False)
    rgba.sum().backward()
    assert rays.grad is None and pts.grad is not None


def _rotation(w, torch):
    """Rodrigues: rotation matrix of the axis-angle vector w (torch ops, differentiable)."""
    th = torch.linalg.norm(w)
    k = w / th
    zero = torch.zeros((), dtype=w.dtype, device=w.device)
    K = torch.stack([torch.stack([zero, -k[2], k[1]]), torch.stack([k[2], zero, -k[0]]),
                     torch.stack([-k[1], k[0], zero])])
    eye = torch.eye(3, dtype=w.dtype, device=w.device)
    return eye + torch.sin(th) * K + (1 - torch.cos(th)) * K @ K


def test_pose_gradient_matches_finite_differences(torch_cuda):
    """A camera pose (translation t, axis-angle rotation w) moves a fixed bundle of rays; autograd through
    TraceRays gives dL/d(t, w), checked against central differences of the device forward.  Step and tolerance
    were rehearsed on the CPU emulator with the same scene and loss: central differences with h = 3e-5 agree
    with the chained ray gradient to 0.3 % of the largest component (h = 3e-4 is still curvature-dominated at
    3 %, h = 1e-5 already fp32-noise-dominated at 0.4 %); the bar is 2 %."""
    import radfoam_b200
    from radfoam_b200 import foam

    torch = torch_cuda
    f = foam.small_foam(400, sh_degree=2, seed=11)
    cam = (0.2, -2.5, 0.4)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    base = dev(foam.pinhole_rays(24, 16, cam, fov=0.8)).double()
    start = dev(np.full((16, 24), foam.nearest_point(f.points, cam), dtype=np.uint32))
    g = dev(np.random.default_rng(3).normal(size=(16, 24, 4)).astype(np.float32))
    scene = [dev(a) for a in (f.points, f.attributes, f.adjacency, f.offsets)]
    pipe = radfoam_b200.create_pipeline(2)

    def loss(p):
        R = _rotation(p[3:], torch)
        rays = torch.cat([base[..., :3] + p[:3], base[..., 3:] @ R.T], -1).float()
        rgba, *_ = radfoam_b200.TraceRays.apply(pipe, *scene, rays, start, None, False)
        return (rgba.double() * g).sum()

    p0 = torch.tensor([0.01, -0.02, 0.03, 0.02, -0.01, 0.015], dtype=torch.float64, device="cuda")
    p = p0.clone().requires_grad_(True)
    loss(p).backward()
    ana = p.grad.cpu().numpy()
    h = 3e-5
    with torch.no_grad():
        fd = np.array([float(loss(p0 + h * e) - loss(p0 - h * e)) / (2 * h)
                       for e in torch.eye(6, dtype=torch.float64, device="cuda")])
    err = np.abs(fd - ana).max() / np.abs(ana).max()
    print(f"\npose: autograd {np.round(ana, 3)} fd {np.round(fd, 3)} max err {err:.2e} of max")
    assert err <= 2e-2
