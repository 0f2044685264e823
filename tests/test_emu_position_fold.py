"""The warp-aggregated backward holds each composited cell's gradient row until the lane's next composited step has
finished that cell's position gradient, and sends both together, so the position gradient needs no 16-byte RED of
its own.  Checked on the CPU emulator (tests/emu), which counts the 16-byte REDs; test_emu_bulk_reduce.py checks that
the gradients stay what the direct backward computes.
"""
import os
import sys

import numpy as np
import pytest

import common

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
import emu_rays  # noqa: E402


@pytest.fixture(scope="module")
def case():
    return common.scene_case(num_points=1500, width=48, height=32, q=2)


@pytest.mark.parametrize("ray", [False, True], ids=["scene", "scene+rays"])
def test_position_gradients_ride_in_their_rows(case, ray, monkeypatch):
    monkeypatch.setenv("RFB_BWD_MODE", "cached")
    f = case.foam
    pipe = emu_rays.EmuRayPipeline(3, np.float32)
    scene = (f.points, f.attributes, f.adjacency, f.offsets)
    fwd = pipe.trace_forward(*scene, case.rays, case.start, case.quantiles, scene_version=3, record_tape=True)
    emu.red_counters()
    pipe.trace_backward(*scene, case.rays, case.start, fwd["rgba"], case.grad_rgba, case.quantiles,
                        fwd["depth_indices"], case.grad_depth, scene_version=3, use_tape=True, ray_grad=ray)
    c = emu.red_counters()
    h, w = case.rays.shape[:2]
    steps = int(emu.tape_records(pipe, h, w)[2].sum())
    # 16-byte REDs per ray-step on this scene: 1.39 when every position gradient left as its own RED (0.93 of
    # them); the cache evictions and the drain alone come to 0.46
    assert c["red_v4"] / steps < 0.6, c["red_v4"] / steps
