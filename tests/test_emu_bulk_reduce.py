"""The warp-aggregated backward sends the gradient row of a lane that is alone in its cell as one bulk reduction
(cp.reduce.async.bulk: shared memory -> global, through the TMA unit) instead of 13 scattered 16-byte REDs.  Checked
on the CPU emulator (tests/emu), which counts the 16-byte REDs (the bulk reduction is emulated with plain atomics):
  * the replay backward's 16-byte RED count per ray-step falls to what the cache evictions and the
    position-gradient flushes need, while its gradients stay complete (below);
  * its gradients lie inside tests/model64.py's per-entry bounds;
  * it agrees with the direct backward (RFB_BWD_MODE=direct, which keeps per-lane 16-byte REDs) up to reduction
    order, in fp32 and fp16, with and without ray gradients; ray gradients are per-thread sums and agree bit for bit.
"""
import os
import sys

import numpy as np
import pytest

import common
import model64 as M

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
import emu_rays  # noqa: E402


@pytest.fixture(scope="module")
def case():
    return common.scene_case(num_points=1500, width=48, height=32, q=2)


def run(case, dtype, mode, ray, monkeypatch):
    """Recording forward + replay backward; returns (backward outputs, reduction counters of the backward,
    ray-steps on the tape)."""
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    f = case.foam
    pipe = emu_rays.EmuRayPipeline(3, dtype)
    scene = (f.points, f.attributes.astype(dtype), f.adjacency, f.offsets)
    fwd = pipe.trace_forward(*scene, case.rays, case.start, case.quantiles, scene_version=3, record_tape=True)
    emu.red_counters()
    bwd = pipe.trace_backward(*scene, case.rays, case.start, fwd["rgba"], case.grad_rgba.astype(dtype),
                              case.quantiles, fwd["depth_indices"], case.grad_depth, scene_version=3,
                              use_tape=mode == "cached", ray_grad=ray)
    counts = emu.red_counters()
    h, w = case.rays.shape[:2]
    steps = int(emu.tape_records(pipe, h, w)[2].sum())
    return bwd, counts, steps


def test_lone_rows_leave_without_16_byte_reds(case, monkeypatch):
    _, c, steps = run(case, np.float32, "cached", False, monkeypatch)
    # 16-byte REDs per ray-step on this scene: 5.35 when lone rows left as 13 REDs each; the cache evictions,
    # its drain and the position-gradient flushes alone come to 1.39
    assert c["red_v4"] / steps < 2.0, c["red_v4"] / steps


@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
def test_replay_backward_within_model_bounds(case, dtype, monkeypatch):
    monkeypatch.setenv("RFB_BWD_MODE", "cached")
    f = case.foam
    pipe = emu.EmuPipeline(3, dtype)
    scene = (f.points, f.attributes.astype(dtype), f.adjacency, f.offsets)

    def impl(rays, start, dq, g, gd, err, backward):
        fwd = pipe.trace_forward(*scene, rays, start, dq, return_contribution=True, record_tape=True,
                                 scene_version=5)
        if not backward:
            return fwd
        bwd = pipe.trace_backward(*(None,) * 6, fwd["rgba"], g.astype(dtype), None, fwd.get("depth_indices"), gd,
                                  err, use_tape=True, scene_version=5)
        return {**fwd, **bwd}

    err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(dtype)
    with np.errstate(all="ignore"):  # the model's bounds of rays that never reach a cell divide by zero
        report = M.check_implementation(impl, f.points, f.attributes.astype(dtype), f.adjacency, f.offsets,
                                        case.rays, case.start, case.quantiles, case.grad_rgba.astype(dtype),
                                        case.grad_depth, err)
    print("\n" + M.format_report(f"emu bulk rows scene1500 {np.dtype(dtype).name}", report))


@pytest.mark.parametrize("ray", [False, True], ids=["scene", "scene+rays"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
def test_replay_backward_matches_direct(case, dtype, ray, monkeypatch):
    got, _, _ = run(case, dtype, "cached", ray, monkeypatch)
    want, _, _ = run(case, dtype, "direct", ray, monkeypatch)
    for k in ("points_grad", "attr_grad"):
        g, w = got[k].astype(np.float32), want[k].astype(np.float32)
        # summation order only; fp16 outputs are rounded once from the fp32 sums, so one fp16 ulp more
        bar = 1e-5 * np.abs(w).max() + (np.spacing(np.abs(want[k])).astype(np.float32) if dtype == np.float16 else 0)
        assert np.all(np.abs(g - w) <= bar), (k, float(np.abs(g - w).max()))
    if ray:
        assert np.array_equal(got["ray_grad"].view(np.uint32), want["ray_grad"].view(np.uint32))
