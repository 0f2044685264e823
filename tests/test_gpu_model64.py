"""The CUDA kernels against the float64 model with per-entry error bounds (tests/model64.py).

Every output entry is compared: integers exactly and floats within their own bound on the rays whose walk
has no near-tie decision, every scatter row (gradients, contribution, point_error) within its per-entry
bound, rows without any term exactly zero.  Ambiguous rays get zero upstream gradients in both the model
and the kernel run.  The model reads nothing but the inputs and the kernels' saved forward outputs."""
import time
import warnings

import numpy as np
import pytest

import common
import fuzz_cases
import model64 as M

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
    """The product's Pipeline as check_implementation's ``impl``."""
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
                                      dev(gd), dev(err), **settings)
            out.update({k: v.cpu().numpy() for k, v in bwd.items() if k != "ray_grad"})
        torch.cuda.synchronize()
        return out
    return run


def check_case(torch, name, case, attr_dtype=np.float32, tape=False, ray_error=True, **settings):
    f = case.foam
    err = None
    if ray_error:
        err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(attr_dtype)
    t = time.perf_counter()
    report = M.check_implementation(
        device_impl(torch, f, attr_dtype, tape, **settings), f.points, f.attributes.astype(attr_dtype),
        f.adjacency, f.offsets, case.rays, case.start, case.quantiles, case.grad_rgba.astype(attr_dtype),
        case.grad_depth, err, **settings)
    print("\n" + M.format_report(name, report) + f" ({time.perf_counter() - t:.1f} s)")
    return report


@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
@pytest.mark.parametrize("mode", ["cached", "direct"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("q", [0, 2, 3])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_config1_within_model_bounds(torch_cuda, deg, q, dtype, mode, tape, monkeypatch):
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    check_case(torch_cuda, f"config1 deg{deg} q{q} {np.dtype(dtype).name} {mode} tape={tape}",
               common.config1(deg, q, fixed_quantiles=q != 3), dtype, tape)


@pytest.mark.parametrize("inside", [False, True], ids=["outside", "inside"])
def test_scene_within_model_bounds(torch_cuda, inside):
    """20 k-point shell scene.  From inside, the first recording overflows the tape pool (the backward
    re-walks); the second is replayed.  Both are held to the model."""
    import radfoam_b200

    case = common.scene_case(inside=inside)
    check_case(torch_cuda, f"scene20k inside={inside}", case)
    if inside:
        pipe = radfoam_b200.create_pipeline(3)
        statuses = []
        impl = device_impl(torch_cuda, case.foam, np.float32, True, pipe=pipe, statuses=statuses)
        f = case.foam
        for step in range(2):
            report = M.check_implementation(impl, f.points, f.attributes, f.adjacency, f.offsets, case.rays,
                                            case.start, case.quantiles, case.grad_rgba, case.grad_depth)
            print("\n" + M.format_report(f"scene20k inside tape step {step}", report))
        assert statuses[0] and not statuses[-1], statuses


@pytest.mark.parametrize("kwargs", [dict(max_intersections=1), dict(max_intersections=7),
                                    dict(weight_threshold=0.0), dict(weight_threshold=0.5)])
def test_trace_settings_within_model_bounds(torch_cuda, kwargs):
    check_case(torch_cuda, f"scene20k {kwargs}", common.scene_case(), **kwargs)


def test_random_ray_batch_within_model_bounds(torch_cuda):
    check_case(torch_cuda, "random rays 20k", common.random_ray_case())


FUZZ_SEEDS = list(range(9000, 9060))


@pytest.mark.parametrize("seed", FUZZ_SEEDS)
def test_fuzz_case_within_model_bounds(torch_cuda, seed):
    """Tie-heavy scenes: exact lattices and axis rays make many rays ambiguous.  A case is only dropped
    when fewer than half of its rays can be compared."""
    scene_kind, ray_kind, f, rays, start, dq, kw = fuzz_cases.make_case(seed)
    case = common.Case(f, rays, start, dq, seed=seed)
    m = M.trace(f.points, f.attributes, f.adjacency, f.offsets, rays, start, dq, backward=False,
                **{"weight_threshold": 0.001, "max_intersections": 1024, **kw})
    share = float(m["ambiguous"].mean())
    print(f"\nfuzz {seed} {scene_kind}/{ray_kind}: {100 * share:.0f}% of {m['ambiguous'].size} rays ambiguous")
    if share > 0.5:
        pytest.skip(f"{100 * share:.0f}% of the rays are ambiguous")
    check_case(torch_cuda, f"fuzz {seed}", case, **kw)


# ------------------------------------------------------------------ at size: config 4
CAMERA = (2.5, 2.5, 2.5)


@pytest.fixture(scope="module")
def config4():
    import bench

    return bench.load_or_build_foam(1 << 20, lambda m: None)


def test_config4_frame_rows_within_model_bounds(torch_cuda, config4):
    """The full 1920x1080 frame with the tape on; forward outputs on 16 rows spread over the frame."""
    from radfoam_b200 import foam

    f = config4
    rays = foam.pinhole_rays(1920, 1080, CAMERA, fov=0.9)
    start = np.full((1080, 1920), foam.nearest_point(f.points, CAMERA), dtype=np.uint32)
    case = common.Case(f, rays, start, common._quantiles((1080, 1920), 2, 21))
    got = device_impl(torch_cuda, f, np.float32, tape=True)(rays, start, case.quantiles, case.grad_rgba,
                                                             case.grad_depth, None, True)
    rows = np.linspace(0, 1079, 16).astype(int)
    t = time.perf_counter()
    m = M.trace(f.points, f.attributes, f.adjacency, f.offsets, rays[rows], start[rows], case.quantiles[rows],
                backward=False)
    steps = int(m["num_intersections"].sum())
    dt = time.perf_counter() - t
    sub = {k: got[k][rows] for k in ("rgba", "depth", "depth_indices", "num_intersections")}
    report = M.compare(sub, m)
    print(f"\nconfig4 16 rows: {report['rays_compared']}/{report['rays']} rays compared; model "
          f"{steps / dt / 1e6:.2f} M ray-steps/s")


@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
def test_config4_crop_gradients_within_model_bounds(torch_cuda, config4, dtype):
    """Every row of points_grad / attr_grad for a 128x64 crop of the frame traced as its own image.  (The
    model runs at about 0.04 M ray-steps/s at this foam size, which keeps the crop this small.)"""
    from radfoam_b200 import foam

    f = config4
    rays = foam.pinhole_rays(1920, 1080, CAMERA, fov=0.9)[508:572, 896:1024].copy()
    start = np.full(rays.shape[:-1], foam.nearest_point(f.points, CAMERA), dtype=np.uint32)
    case = common.Case(f, rays, start, common._quantiles(rays.shape[:-1], 2, 22))
    check_case(torch_cuda, f"config4 crop {np.dtype(dtype).name}", case, dtype, tape=True, ray_error=False)
