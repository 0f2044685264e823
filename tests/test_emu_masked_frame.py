"""The masked-frame harness (tests/masked_frame.py) on the CPU kernel-logic emulator (tests/emu/emu_rays.py).

The emulator compiles the product's host code, so RFB_REPLAY_ORDER reaches both replay schedules of the tape
backward at a size it can run: the 20 k-point scene at 160x96 with the tape on.  Each kind of ray set is held to the
float64 model with ``ray_grad``, and a harness that scatters S's upstream one pixel to the side must fail the
per-entry check."""
import os
import sys
import warnings

import numpy as np
import pytest

import common
import masked_frame as MF
import model64 as M

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))

VERSION = 7


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


@pytest.fixture(scope="module")
def frame_case():
    """The scene, an emulated pipeline whose tape pool has grown to the frame, and the frame's forward."""
    import emu_rays

    case = common.scene_case()
    f = case.foam
    pipe = emu_rays.EmuRayPipeline(f.sh_degree)
    scene = (f.points, f.attributes, f.adjacency, f.offsets)
    for _ in range(2):  # the first recording overflows the initial pool, which then grows
        fwd = pipe.trace_forward(*scene, case.rays, case.start, case.quantiles, record_tape=True,
                                 scene_version=VERSION)
    assert not pipe.tape_status()["overflowed"]
    return case, pipe, scene, fwd


def ray_sets(height, width, nint):
    return {"dense aligned": MF.block(height, width, 48, 32, 32, 16),
            "dense offset (3, 1)": MF.block(height, width, 83, 49, 32, 16),
            "one lane per warp": MF.one_lane_per_warp(height, width, 240),
            "longest": MF.longest(nint, 256)}


def emu_run(pipe, scene, case, order, ray_grad, monkeypatch):
    """One full-frame forward and tape-replay backward on the emulator with the given replay schedule."""
    import emu

    def run(g, gd, err):
        monkeypatch.setenv("RFB_REPLAY_ORDER", order)
        fwd = pipe.trace_forward(*scene, case.rays, case.start, case.quantiles, record_tape=True,
                                 scene_version=VERSION)
        status = pipe.tape_status()
        assert status["used_chunks"] > 0 and not status["overflowed"], status
        assert (emu.tape_schedule(pipe) is not None) == (order == "1")   # sorted replay iff asked for
        bwd = pipe.trace_backward(*(None,) * 6, fwd["rgba"], g, None, fwd["depth_indices"], gd, err, use_tape=True,
                                  scene_version=VERSION, ray_grad=ray_grad)
        return {**fwd, **bwd}
    return run


def upstream(case, frame):
    err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(np.float32)
    return frame.batch(case.grad_rgba), frame.batch(case.grad_depth), frame.batch(err)


@pytest.mark.parametrize("kind", ["dense aligned", "dense offset (3, 1)", "one lane per warp", "longest"])
def test_masked_frame_within_model_bounds(frame_case, kind, monkeypatch):
    """Unsorted and sorted replay, with and without ray gradients, held to one model result for S."""
    case, pipe, scene, fwd = frame_case
    h, w = case.rays.shape[:2]
    assert MF.cta_count(h, w) == 120
    frame = MF.MaskedFrame(case.rays, case.start, case.quantiles, ray_sets(h, w, fwd["num_intersections"])[kind])
    runs = {f"order={o} ray_grad={r}": emu_run(pipe, scene, case, o, r, monkeypatch)
            for o in ("0", "1") for r in (True, False)}
    reports = MF.check_paths(scene, frame, *upstream(case, frame), runs)
    for name, report in reports.items():
        print("\n" + M.format_report(f"scene20k masked {kind} {name}", report))
        assert report["rays_compared"] == frame.sel.size - report["ambiguous"] > 0.9 * frame.sel.size
        assert report["attr_grad"]["compared"] > 0


@pytest.mark.parametrize("order", ["0", "1"])
def test_masked_frame_shifted_upstream_is_caught(frame_case, order, monkeypatch):
    """Negative control: S's upstream scattered one pixel to the side of where the model puts it."""
    case, pipe, scene, fwd = frame_case
    h, w = case.rays.shape[:2]
    sets = ray_sets(h, w, fwd["num_intersections"])
    for kind in ("dense aligned", "one lane per warp"):
        shifted = MF.MaskedFrame(case.rays, case.start, case.quantiles, sets[kind], shift=1)
        runs = {"shifted": emu_run(pipe, scene, case, order, False, monkeypatch)}
        with pytest.raises(M.Mismatch, match="points_grad|attr_grad|point_error"):
            MF.check_paths(scene, shifted, *upstream(case, shifted), runs)
