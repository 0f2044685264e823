"""Full-size backward launches held per entry to the float64 model (tests/model64_rays.py), by masking the upstream
gradients to a set S of rays (tests/masked_frame.py).

The launches are the frames bench.py and tests/test_gpu_configs.py trace: config 4 (1 M-point foam, 1920x1080) and
the 2 M-point foam at 3840x2160 with max_intersections = 96 (config 5's step-budget edge).  With more than 5,280
CTAs the forward does not sort the replay's tiles, so these are the launches that run the unsorted replay.  The
full frame is traced forward and backward; only S has nonzero upstream gradients.  Every row of points_grad,
attr_grad and point_error is compared (rows no ray of S touches must be exactly zero), S's per-ray outputs and
ray gradients are compared, and ray_grad must be exactly zero on every other ray of the frame.  The model traces
S once per case, and every device path of the case is held to that one result."""
import time
import warnings

import numpy as np
import pytest

import common
import masked_frame as MF
import model64 as M

pytestmark = pytest.mark.gpu

CAMERA = (2.5, 2.5, 2.5)
SORTED_REPLAY_MAX_CTAS = 132 * 5 * 8   # up to this many CTAs the forward orders the replay's tiles longest-first


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


class Frame:
    """A foam on the device and one camera's full frame, with a seeded upstream of the common.Case kind."""

    def __init__(self, torch, num_points, width, height, attr_dtype=np.float32, points=None, **settings):
        """``points``: trace the foam with these points instead of its own (a stale foam: moved points, the same
        adjacency); the camera's start cell is their nearest point."""
        import bench
        import radfoam_b200
        from radfoam_b200 import foam

        self.torch, self.settings, self.attr_dtype = torch, settings, attr_dtype
        f = self.foam = bench.load_or_build_foam(num_points, lambda m: None)
        if points is not None:
            f = self.foam = foam.Foam(points, f.attributes, f.adjacency, f.offsets, f.sh_degree)
        self.scene = (f.points, f.attributes.astype(attr_dtype), f.adjacency, f.offsets)
        rays = foam.pinhole_rays(width, height, CAMERA, fov=0.9)
        start = np.full((height, width), foam.nearest_point(f.points, CAMERA), dtype=np.uint32)
        self.case = common.Case(f, rays, start, common._quantiles((height, width), 2, 23), seed=num_points % 1000)
        self.ray_error = np.random.default_rng(4).uniform(0, 1, size=(height, width)).astype(attr_dtype)
        assert MF.cta_count(height, width) > SORTED_REPLAY_MAX_CTAS
        dev = self.dev
        self.scene_d = [dev(x) for x in self.scene]
        self.scene_d[0].requires_grad_(True)   # scene tensors that require grad make the forward record the tape
        self.scene_d[1].requires_grad_(True)
        self.rays_d, self.start_d, self.dq_d = dev(rays), dev(start), dev(self.case.quantiles)
        self.pipe = radfoam_b200.create_pipeline(f.sh_degree, "float16" if attr_dtype == np.float16 else "float32")
        for _ in range(3):   # the first recordings may overflow the tape pool, which then grows
            fwd = self.forward()
            if not self.pipe.tape_status()["overflowed"]:
                break
        self.num_intersections = fwd["num_intersections"].cpu().numpy()

    def dev(self, a):
        return None if a is None else self.torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def forward(self):
        return self.pipe.trace_forward(*self.scene_d, self.rays_d, self.start_d, depth_quantiles=self.dq_d,
                                       **self.settings)

    def run(self, monkeypatch, mode="cached", tape=True, order=None, ray_grad=False):
        """A full-frame forward and backward on one backward path, as masked_frame.check_paths's ``run``.
        ``order``: RFB_REPLAY_ORDER for the recording forward ("1": sorted replay), None for the default."""
        from radfoam_b200 import _lib

        def run(g, gd, err):
            monkeypatch.setenv("RFB_BWD_MODE", mode)
            if order is None:
                monkeypatch.delenv("RFB_REPLAY_ORDER", raising=False)
            else:
                monkeypatch.setenv("RFB_REPLAY_ORDER", order)
            self.pipe.record_tape = tape
            fwd = self.forward()
            replay = self.pipe._tape_flag(self.rays_d, self.start_d, self.pipe._scene_version) == _lib.FLAG_USE_TAPE
            assert replay == tape
            if tape:
                status = self.pipe.tape_status()
                assert status["used_chunks"] > 0 and not status["overflowed"], status
            bwd = self.pipe.trace_backward(*self.scene_d, self.rays_d, self.start_d, fwd["rgba"], self.dev(g),
                                           self.dq_d, fwd["depth_indices"], self.dev(gd), self.dev(err),
                                           return_ray_grad=ray_grad, **self.settings)
            out = {k: v.cpu().numpy() for k, v in fwd.items()}
            out.update({k: v.cpu().numpy() for k, v in bwd.items() if k != "ray_grad" or ray_grad})
            self.torch.cuda.synchronize()
            self.pipe.record_tape = True
            return out
        return run

    def check(self, name, sel, runs, model=None):
        frame = MF.MaskedFrame(self.case.rays, self.case.start, self.case.quantiles, sel)
        t = time.perf_counter()
        reports = MF.check_paths(self.scene, frame, frame.batch(self.case.grad_rgba.astype(self.attr_dtype)),
                                 frame.batch(self.case.grad_depth), frame.batch(self.ray_error), runs,
                                 model=model, **self.settings)
        dt = time.perf_counter() - t
        for path, report in reports.items():
            print("\n" + M.format_report(f"{name} {path}", report))
            # long walks have many decisions, so a larger share of them has a near-tie than in the crop tests
            assert report["rays_compared"] == frame.sel.size - report["ambiguous"] > 0.5 * frame.sel.size
        print(f"{name}: {frame.sel.size} rays in S, {len(runs)} paths ({dt:.1f} s)")
        return reports


def frame_sets(height, width, nint, lanes=4096, longest=2048):
    cx, cy = width // 2 // 16 * 16, height // 2 // 8 * 8
    return {"dense": MF.block(height, width, cx - 64, cy - 32, 64, 32),
            "dense offset": MF.block(height, width, cx + 3, cy + 1, 64, 32),
            "one lane per warp": MF.one_lane_per_warp(height, width, lanes),
            "longest": MF.longest(nint, longest)}


def test_config4_fullframe_every_path_within_model_bounds(torch_cuda, monkeypatch):
    """Config 4, fp32, 1920x1080; S = dense blocks, one lane per warp and the 2,048 longest rays.  The unsorted
    replay (what bench.py runs), the sorted replay, the cached re-walk and the direct backward, and the unsorted
    replay and the direct backward again with ray gradients."""
    fr = Frame(torch_cuda, 1 << 20, 1920, 1080)
    sets = frame_sets(1080, 1920, fr.num_intersections)
    sel = np.unique(np.concatenate(list(sets.values())))
    runs = {"replay unsorted": fr.run(monkeypatch),
            "replay sorted": fr.run(monkeypatch, order="1"),
            "re-walk": fr.run(monkeypatch, tape=False),
            "direct": fr.run(monkeypatch, mode="direct"),
            "replay unsorted ray_grad": fr.run(monkeypatch, ray_grad=True),
            "direct ray_grad": fr.run(monkeypatch, mode="direct", ray_grad=True)}
    fr.check("config4 1080p fp32", sel, runs)


def test_config4_fullframe_fp16_within_model_bounds(torch_cuda, monkeypatch):
    """Config 4 with fp16 attributes: dense blocks and one lane per warp on the unsorted replay; the gradients are
    accumulated in fp32 and rounded once."""
    fr = Frame(torch_cuda, 1 << 20, 1920, 1080, np.float16)
    sets = frame_sets(1080, 1920, fr.num_intersections)
    sel = np.unique(np.concatenate([sets["dense"], sets["dense offset"], sets["one lane per warp"]]))
    fr.check("config4 1080p fp16", sel, {"replay unsorted": fr.run(monkeypatch)})


def test_4k_step_budget_fullframe_within_model_bounds(torch_cuda, monkeypatch):
    """The 2 M-point foam at 3840x2160 with max_intersections = 96: 2,048 of the rays that run out of steps and one
    lane in each of 2,048 warps, on the unsorted replay with and without ray gradients."""
    fr = Frame(torch_cuda, 1 << 21, 3840, 2160, max_intersections=96)
    nint = fr.num_intersections
    assert float((nint == 97).mean()) > 0.2, "the case must exhaust the step budget"
    sel = np.unique(np.concatenate([MF.budget_exhausted(nint, 96, 2048), MF.one_lane_per_warp(2160, 3840, 2048)]))
    runs = {"replay unsorted": fr.run(monkeypatch), "replay unsorted ray_grad": fr.run(monkeypatch, ray_grad=True)}
    fr.check("2M 4K budget96", sel, runs)
