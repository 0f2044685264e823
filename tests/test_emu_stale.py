"""The kernel sources, run on the CPU emulator, against the float64 model on stale scenes (tests/stale_cases.py): the
1,500-point shell scene with its points moved and its adjacency kept, which is what most training steps trace.

Every case compares all of its non-ambiguous rays, and asserts floors on its staleness: the share of rays that skip
a cell, the share of composited cells entered after skipped ones (the backward's entry plane is then recomputed
instead of carried over from the previous exit plane) and the rays stranded inside the hull."""
import warnings

import numpy as np
import pytest

import common
import model64 as M
import stale_cases as S
from test_model64 import run_emu_case
from test_model64_rays import run_emu_ray_case

FRACS = (0.05, 0.2, 0.5, 1.0)
PATHS = (("cached", True), ("cached", False), ("direct", True), ("direct", False))
# (kind, f) -> floors (share of rays skipping a cell, share of composited cells re-entered, rays stranded): about
# half of what the seeded cases have
FLOORS = {("noise", 0.05): (0.005, 2e-4, 0), ("noise", 0.2): (0.15, 0.015, 10), ("noise", 0.5): (0.45, 0.06, 200),
          ("noise", 1.0): (0.4, 0.1, 200), ("field", 0.05): (0.001, 5e-5, 0), ("field", 0.2): (0.006, 4e-4, 0),
          ("field", 0.5): (0.03, 0.0025, 0), ("field", 1.0): (0.12, 0.01, 1)}


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def stale_scene(kind, frac, sh_degree):
    base = common.scene_case(num_points=1500, width=48, height=32, q=2, sh_degree=sh_degree)
    case = S.stale_case(base, frac, kind, seed=FRACS.index(frac) + 10 * S.KINDS.index(kind))
    f = case.foam
    m = M.trace(f.points, f.attributes, f.adjacency, f.offsets, case.rays, case.start, case.quantiles,
                backward=False)
    st = S.stats(m, f.points)
    S.assert_floors(st, *FLOORS[kind, frac])
    assert m["ambiguous"].mean() < 0.05
    return case, st


def test_fresh_scene_is_not_stale():
    """The floors mean something: the unmoved scene is below them."""
    base = common.scene_case(num_points=1500, width=48, height=32, q=2)
    f = base.foam
    m = M.trace(f.points, f.attributes, f.adjacency, f.offsets, base.rays, base.start, base.quantiles, backward=False)
    st = S.stats(m, f.points)
    assert st.skipped < FLOORS["noise", 0.2][0] and st.reentered < FLOORS["noise", 0.2][1] and st.stranded == 0


@pytest.mark.parametrize("path", range(len(PATHS)), ids=[f"{m}-{'tape' if t else 'rewalk'}" for m, t in PATHS])
@pytest.mark.parametrize("frac", FRACS)
@pytest.mark.parametrize("kind", S.KINDS)
def test_emulated_kernels_stale_within_model_bounds(kind, frac, path, monkeypatch):
    """Forward and backward on every backward path; the degree and the attribute dtype rotate over the cases."""
    mode, tape = PATHS[path]
    i = FRACS.index(frac)
    deg = (i + path) % 4
    dtype = np.float16 if (S.KINDS.index(kind) + i + path) % 2 else np.float32
    case, st = stale_scene(kind, frac, deg)
    report = run_emu_case(case, dtype, mode, tape, monkeypatch)
    assert report["rays_compared"] == report["rays"] - report["ambiguous"]
    print(f"\n{kind} f={frac}: {st}\n" + M.format_report(
        f"emu stale deg{deg} {np.dtype(dtype).name} {mode} tape={tape} ambiguous {report['ambiguous']}", report))


@pytest.mark.parametrize("mode,tape", [("cached", True), ("direct", False)], ids=["cached-tape", "direct-rewalk"])
@pytest.mark.parametrize("frac", FRACS)
@pytest.mark.parametrize("kind", S.KINDS)
def test_emulated_ray_grad_stale_within_model_bounds(kind, frac, mode, tape, monkeypatch):
    """Every output, ray_grad included: the ray gradient's t0 plane is the previous composited cell's exit plane,
    which on a stale scene lies cells behind the current one."""
    deg = 3 - FRACS.index(frac)
    case, st = stale_scene(kind, frac, deg)
    report = run_emu_ray_case(case, np.float32, mode, tape, monkeypatch)
    assert report["rays_compared"] == report["rays"] - report["ambiguous"]
    print(f"\n{kind} f={frac}: {st}\n" + M.format_report(f"emu stale ray_grad deg{deg} {mode} tape={tape}", report))
