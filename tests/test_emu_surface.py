"""Surface extraction (rfb_surface_count / rfb_surface_write) on the CPU kernel-logic emulator (tests/emu) against
the float64 model (tests/surface_model.py): general-position, tie-heavy and stale foams, empty rows, duplicate
points, SH degrees 0-3 in fp32 and fp16, the count/write agreement, and rgb equal to the emulated sample_field."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import fuzz_cases
import stale_cases
import surface_model as sm
from radfoam_b200 import _lib as abi
from radfoam_b200 import foam

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
import emu  # noqa: E402


def extract(pipe, points, attrs, adjacency, offsets, inside, bounds=None):
    """(surface dict, totals) from the two emulated passes, sized from the count's totals as the Python layer does."""
    lib = pipe.lib
    pts, att = np.ascontiguousarray(points, np.float32), np.ascontiguousarray(attrs, pipe.dtype)
    adj, off = np.ascontiguousarray(adjacency, np.uint32), np.ascontiguousarray(offsets, np.uint32)
    ins = np.ascontiguousarray(inside, np.uint8)
    lo, hi = sm.bounding_box(pts) if bounds is None else bounds
    box = abi.Box((ctypes.c_float * 3)(*map(float, lo)), (ctypes.c_float * 3)(*map(float, hi)))
    e = adj.size
    scratch = np.zeros((int(lib.rfb_surface_scratch_bytes(e)) + 7) // 8, np.uint64)
    emu._check(lib.rfb_surface_count(emu._p(pts), pts.shape[0], e, emu._p(adj) if e else None, emu._p(off),
                                     emu._p(ins), ctypes.byref(box), emu._p(scratch), None))
    nv, npoly, over = (int(x) for x in scratch[:3])
    out = {"vertices": np.full((nv, 3), np.nan, np.float32), "offsets": np.full(npoly + 1, -1, np.int64),
           "cells": np.full((npoly, 2), 7, np.uint32), "rgb": np.full((npoly, 3), np.nan, pipe.dtype)}
    emu._check(lib.rfb_surface_write(pipe.handle, emu._p(pts), pts.shape[0], emu._p(att), e, emu._p(adj) if e else None,
                                     emu._p(off), emu._p(ins), ctypes.byref(box), emu._p(scratch),
                                     emu._p(out["vertices"]), emu._p(out["offsets"]), emu._p(out["cells"]),
                                     emu._p(out["rgb"]), None))
    return out, (nv, npoly, over), scratch


def check_against_model(out, points, adjacency, offsets, inside, bounds=None):
    """Every polygon the model emits (CSR order) is there with its cells; general-position polygons vertex for
    vertex within the bound, near-degenerate ones by area and Hausdorff distance; nothing else is emitted except
    polygons below the area tolerance."""
    lo, hi = sm.bounding_box(points) if bounds is None else bounds
    scale = float(np.linalg.norm(np.asarray(hi, np.float64) - np.asarray(lo, np.float64))) or 1.0
    want = sm.surface(points, adjacency, offsets, inside, bounds)
    off = out["offsets"]
    assert off[0] == 0 and off[-1] == out["vertices"].shape[0] and np.all(np.diff(off) >= 3)
    got = {(int(c[0]), int(c[1]), k): out["vertices"][off[k]:off[k + 1]].astype(np.float64)
           for k, c in enumerate(out["cells"])}
    rows = sm.rows_of(offsets)
    # CSR order: the emitted (i, j) sequence is a subsequence of the entries in order
    keys = [(int(rows[q.entry]), int(adjacency[q.entry])) for q in want]
    got_keys = [(k[0], k[1]) for k in got]
    area_tol = (1e-6 * scale) ** 2
    gi = 0
    for q, key in zip(want, keys):
        while gi < len(got_keys) and got_keys[gi] != key:
            extra = got[(*got_keys[gi], gi)]
            assert np.linalg.norm(sm.area_vector(extra)) <= area_tol, f"extra polygon {got_keys[gi]}"
            gi += 1
        if gi == len(got_keys):
            assert np.linalg.norm(sm.area_vector(q.vertices)) <= area_tol, f"missing polygon {key}"
            continue
        v = got[(*key, gi)]
        gi += 1
        if not q.degenerate and v.shape == q.vertices.shape:
            k = int(np.argmin(np.linalg.norm(v - q.vertices[0], axis=1)))
            err = np.abs(np.roll(v, -k, axis=0) - q.vertices)
            assert np.all(err <= sm.vertex_bound(q.vertices, scale)), (key, err.max())
        else:
            assert not (not q.degenerate and np.linalg.norm(sm.area_vector(q.vertices)) > area_tol), \
                f"general-position polygon {key}: {v.shape[0]} vertices, model {q.vertices.shape[0]}"
            aw, ag = sm.area_vector(q.vertices), sm.area_vector(v)
            assert np.linalg.norm(aw - ag) <= 1e-6 * scale ** 2, key
            assert sm.hausdorff(v, q.vertices) <= 1e-6 * scale, key
    for rest in range(gi, len(got_keys)):
        assert np.linalg.norm(sm.area_vector(got[(*got_keys[rest], rest)])) <= area_tol, "extra polygon"
    return want


def sample_rgb(pipe, points, attrs, adjacency, offsets, cells):
    """rfb_sample_field at p_i along p_i - p_j (renormalised by the kernel)."""
    p = np.ascontiguousarray(points, np.float32)
    i, j = cells[:, 0].astype(np.int64), cells[:, 1].astype(np.int64)
    q = np.ascontiguousarray(p[i])
    d = np.ascontiguousarray(p[i] - p[j])
    m = q.shape[0]
    att = np.ascontiguousarray(attrs, pipe.dtype)
    adj, off = np.ascontiguousarray(adjacency, np.uint32), np.ascontiguousarray(offsets, np.uint32)
    c, dens, rgb = np.empty(m, np.uint32), np.empty(m, pipe.dtype), np.empty((m, 3), pipe.dtype)
    emu._check(pipe.lib.rfb_sample_field(pipe.handle, emu._p(p), p.shape[0], emu._p(att), emu._p(adj), emu._p(off),
                                         emu._p(q), m, emu._p(np.ascontiguousarray(i.astype(np.uint32))), emu._p(d),
                                         emu._p(c), emu._p(dens), emu._p(rgb), None))
    assert np.array_equal(c.astype(np.int64), i)
    return rgb


def run_case(f, inside, deg=0, dtype=np.float32, bounds=None, attrs=None):
    pipe = emu.EmuPipeline(deg, dtype)
    attrs = f.attributes if attrs is None else attrs
    out, (nv, npoly, over), _ = extract(pipe, f.points, attrs, f.adjacency, f.offsets, inside, bounds)
    assert over == 0
    again, _, _ = extract(pipe, f.points, attrs, f.adjacency, f.offsets, inside, bounds)
    for k in out:  # deterministic, and every counted slot was written
        assert out[k].tobytes() == again[k].tobytes(), k
    assert not np.isnan(out["vertices"]).any() and (out["offsets"] >= 0).all()
    want = check_against_model(out, f.points, f.adjacency, f.offsets, inside, bounds)
    return pipe, out, want


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_small_foam_all_degrees(deg, dtype):
    f = foam.small_foam(160, sh_degree=deg, seed=deg)
    f.attributes = f.attributes.astype(dtype)
    inside = np.linalg.norm(f.points, axis=1) < 0.6
    pipe, out, want = run_case(f, inside, deg, dtype)
    assert len(want) > 20
    rgb = sample_rgb(pipe, f.points, f.attributes, f.adjacency, f.offsets, out["cells"])
    assert out["rgb"].tobytes() == rgb.tobytes(), "rgb is sample_field's colour, bit for bit"
    # the volume of an occupied set clear of the box, from the kernel's polygons
    lo, hi = sm.bounding_box(f.points)
    off = out["offsets"]
    got = sm.enclosed_volume([out["vertices"][off[k]:off[k + 1]] for k in range(off.size - 1)])
    assert abs(got - sm.enclosed_volume([q.vertices for q in want])) <= 1e-5 * abs(got)


@pytest.mark.parametrize("seed", range(6))
def test_tie_heavy_scenes(seed):
    rng = np.random.default_rng(500 + seed)
    kind = fuzz_cases.SCENE_KINDS[seed % len(fuzz_cases.SCENE_KINDS)]
    f = fuzz_cases.make_scene(rng, kind, int(rng.integers(40, 160)), 0)
    inside = rng.random(f.num_points) < 0.4
    run_case(f, inside)


@pytest.mark.parametrize("kind", stale_cases.KINDS)
def test_stale_adjacency(kind):
    f = stale_cases.stale(foam.small_foam(150, sh_degree=1, seed=3), 0.3, kind, seed=4)
    inside = np.linalg.norm(f.points, axis=1) < 0.7
    pipe, out, _ = run_case(f, inside, deg=1)
    rgb = sample_rgb(pipe, f.points, f.attributes, f.adjacency, f.offsets, out["cells"])
    assert out["rgb"].tobytes() == rgb.tobytes()


def test_empty_rows_duplicates_repeats_and_bounds():
    f = foam.small_foam(120, seed=6)
    rows = [list(f.adjacency[f.offsets[i]:f.offsets[i + 1]]) for i in range(f.num_points)]
    rows[5] = []                               # an empty row
    rows[9] = rows[9] + [rows[9][0]]           # a repeated entry: a repeated polygon
    pts = f.points.copy()
    pts[11] = pts[rows[11][0]]                 # a duplicate point: no plane, no polygon between them
    adj = np.array([a for r in rows for a in r], np.uint32)
    off = np.zeros(f.num_points + 1, np.uint32)
    off[1:] = np.cumsum([len(r) for r in rows])
    g = foam.Foam(pts, f.attributes, adj, off, f.sh_degree)
    inside = np.zeros(f.num_points, bool)
    inside[[5, 9, 11]] = True
    inside[np.linalg.norm(pts, axis=1) < 0.4] = True
    _, out, _ = run_case(g, inside)
    c = [tuple(x) for x in out["cells"].astype(np.int64)]
    assert c.count((9, int(rows[9][0]))) == 2 or inside[rows[9][0]]
    assert all(i != 5 for i, _ in c)
    # a smaller box clips the polygons to it
    run_case(g, inside, bounds=(np.full(3, -0.5), np.full(3, 0.45)))


def test_nothing_inside_everything_inside_and_nonfinite():
    f = foam.small_foam(60, seed=2)
    pipe = emu.EmuPipeline(0)
    for inside in (np.zeros(60, bool), np.ones(60, bool)):
        out, tot, _ = extract(pipe, f.points, f.attributes, f.adjacency, f.offsets, inside)
        assert tot == (0, 0, 0) and out["offsets"].tolist() == [0]
    pts = f.points.copy()
    pts[3] = np.nan
    pts[7, 1] = np.inf
    inside = np.ones(60, bool)
    inside[::2] = False
    out, (nv, npoly, over), _ = extract(pipe, pts, f.attributes, f.adjacency, f.offsets, inside,
                                        bounds=(np.full(3, -1.0), np.full(3, 1.0)))
    assert npoly > 0 and out["offsets"][-1] == nv and np.isfinite(out["vertices"]).all()
    assert all(3 not in c and 7 not in c for c in out["cells"].tolist())


def test_argument_checks():
    pipe = emu.EmuPipeline(0)
    f = foam.small_foam(30, seed=1)
    with pytest.raises(RuntimeError, match="bounds"):
        extract(pipe, f.points, f.attributes, f.adjacency, f.offsets, np.ones(30, bool),
                bounds=(np.ones(3), np.zeros(3)))
    box = abi.Box()
    with pytest.raises(RuntimeError, match="NULL"):
        emu._check(pipe.lib.rfb_surface_count(None, 30, 0, None, None, None, ctypes.byref(box), None, None))
    with pytest.raises(RuntimeError, match="pipeline is NULL"):
        emu._check(pipe.lib.rfb_surface_write(None, None, 0, None, 0, None, None, None, ctypes.byref(box), None, None,
                                              None, None, None, None))


def test_shuffled_lane_schedule():
    """The scan's warp shuffles and shared-memory handoffs under the emulator's shuffled resume order."""
    code = f"""
import sys
sys.path[:0] = [{HERE!r}, {os.path.dirname(HERE)!r}]
import test_emu_surface as t
t._shuffled_body()
print("ok")
"""
    env = dict(os.environ, RFB_EMU_SHUFFLE="11")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stderr[-2000:]


def _shuffled_body():
    f = foam.small_foam(200, sh_degree=2, seed=9)
    inside = np.linalg.norm(f.points, axis=1) < 0.6
    pipe, out, want = run_case(f, inside, deg=2)
    assert len(want) > 20
    rgb = sample_rgb(pipe, f.points, f.attributes, f.adjacency, f.offsets, out["cells"])
    assert out["rgb"].tobytes() == rgb.tobytes()
