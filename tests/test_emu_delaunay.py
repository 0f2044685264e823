"""The Delaunay adjacency kernels (rfb_delaunay_count / rfb_delaunay_write) on the CPU kernel-logic emulator
(tests/emu), judged against Qhull and the float64 model (tests/delaunay_model.py): every entry that differs from
Qhull's graph must have a face of area <= TAU |p_i - p_j|^2 (outside the box, or a zero-area tie)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import delaunay_emu as de
import delaunay_model as dm
import fuzz_cases
from radfoam_b200 import foam
from radfoam_b200.delaunay import TriangulationFailedError

HERE = os.path.dirname(os.path.abspath(__file__))


def check_structure(adj, off, n):
    assert off.shape == (n + 1,) and off[0] == 0 and off[-1] == adj.size
    assert np.all(np.diff(off.astype(np.int64)) >= 0)
    rows = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
    assert np.all(adj < n) and not np.any(adj == rows)
    same = rows[1:] == rows[:-1]
    assert np.all(adj[1:][same] > adj[:-1][same]), "rows not strictly ascending"
    fwd = np.sort((rows.astype(np.int64) << 32) | adj.astype(np.int64))
    bwd = np.sort((adj.astype(np.int64) << 32) | rows.astype(np.int64))
    assert np.array_equal(fwd, bwd), "not symmetric"


def check(points, bounds=None, all_points=False, ref=None):
    """Build, check the structure and every difference from the reference graph (Qhull's, or the brute-force one);
    returns (adjacency, offsets, totals, differences)."""
    adj, off, totals = de.build(points, bounds)
    check_structure(adj, off, points.shape[0])
    qa, qo = foam.delaunay_adjacency(points) if ref is None else ref
    lo, hi = de.box_of(points, bounds)
    diffs = dm.judge(points, adj, off, qa, qo, lo.astype(np.float64), hi.astype(np.float64), all_points)
    bad = [d for d in diffs if d[2] > dm.TAU]
    assert not bad, f"{len(bad)} differences with a face above the tolerance, e.g. {bad[:5]}"
    return adj, off, totals, diffs


def uniform(n, seed=0):
    return np.random.default_rng(seed).uniform(-1, 1, (n, 3)).astype(np.float32)


def test_small_foam():
    check(foam.small_foam(256).points)


def test_uniform_4k_and_a_large_box_recovers_far_hull_edges():
    p = uniform(4096, 1)
    adj, off, totals, diffs = check(p)
    dropped = [d for d in diffs if d[3]]
    assert dropped and not [d for d in diffs if not d[3]], "the default box drops far hull edges and adds none"
    _, _, _, diffs_big = check(p, bounds=(-1e4 * np.ones(3), 1e4 * np.ones(3)))
    assert len(diffs_big) < len(diffs)
    print(f"uniform 4k: {len(dropped)} Qhull entries dropped by the default box, {len(diffs_big)} by a 1e4 box; "
          f"{int(totals[3])} cells on the overflow path")


def test_scene_foam_20k_far_field():
    p = foam.scene_foam(20000).points
    _, _, totals, diffs = check(p)
    assert totals[3] > 0, "hull cells take the overflow path"
    print(f"scene_foam(20000): {len(diffs)} entries differ from Qhull (all justified), {int(totals[3])} overflow cells")


@pytest.mark.parametrize("kind,noise", [("lattice", 0.0), ("lattice", 1e-7), ("bcc", None), ("cluster", None),
                                        ("scaled", 1e-3), ("scaled", 1e3)])
def test_fuzz_kinds(kind, noise):
    rng = np.random.default_rng(3)
    if kind == "lattice":
        g = np.stack(np.meshgrid(*[np.linspace(-1, 1, 10)] * 3, indexing="ij"), -1).reshape(-1, 3)
        p = (g + rng.normal(0, noise, size=g.shape) if noise else g).astype(np.float32)
    elif kind == "scaled":
        p = (rng.uniform(-1, 1, size=(1500, 3)) * noise).astype(np.float32)
    else:
        p = fuzz_cases.make_scene(rng, kind, 1500, 0).points
    p = np.unique(p, axis=0)
    check(p)


def test_hub_takes_the_overflow_path():
    rng = np.random.default_rng(5)
    u = rng.normal(size=(500, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    p = np.concatenate([np.zeros((1, 3)), u * (1 + rng.normal(0, 1e-3, (500, 1)))]).astype(np.float32)
    adj, off, totals, _ = check(p)
    assert totals[3] > 0
    assert off[1] - off[0] > 400, "the centre is a hub"


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4])
def test_tiny_sets_against_brute_force(n):
    p = uniform(n, 9 + n)
    lo, hi = de.box_of(p) if n else (np.zeros(3), np.zeros(3))
    if n < 2:
        adj, off, _ = de.build(p)
        assert adj.size == 0 and np.array_equal(off, np.zeros(n + 1, np.uint32))
        return
    check(p, ref=dm.brute_graph(p, lo.astype(np.float64), hi.astype(np.float64)), all_points=True)


@pytest.mark.parametrize("kind", ["coplanar", "collinear"])
def test_degenerate_sets_against_brute_force(kind):
    rng = np.random.default_rng(13)
    p = rng.uniform(-1, 1, (30, 3))
    if kind == "coplanar":
        p[:, 2] = 0.0
    else:
        p = np.outer(rng.uniform(-1, 1, 30), [1.0, 2.0, -0.5])
    p = np.unique(p.astype(np.float32), axis=0)
    lo, hi = de.box_of(p)
    ref = dm.brute_graph(p, lo.astype(np.float64), hi.astype(np.float64))
    adj, off, _, _ = check(p, ref=ref, all_points=True)
    if kind == "collinear":  # a chain: every inner point has its two neighbours along the line
        assert adj.size == 2 * (p.shape[0] - 1)


def test_duplicates_and_nan_raise():
    p = uniform(300, 2)
    p[200] = p[10]
    with pytest.raises(TriangulationFailedError):
        de.build(p)
    q = uniform(300, 2)
    q[5, 2] = np.nan
    with pytest.raises(TriangulationFailedError):
        de.build(q)


def test_order_changes_nothing_and_a_small_pool_is_grown():
    p = uniform(2000, 4)
    a, o, _ = de.build(p)
    b, ob, _ = de.build(p, order=np.random.default_rng(0).permutation(p.shape[0]), pool=16)
    assert np.array_equal(o, ob) and np.array_equal(a, b)


def test_shuffled_lane_schedule_is_byte_identical():
    """RFB_EMU_SHUFFLE resumes the emulated lanes in a pseudo-random order: the build must not change by one byte."""
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r); import delaunay_emu as de; "
            "from radfoam_b200 import foam; p = foam.scene_foam(3000).points; a, o, _ = de.build(p); "
            "sys.stdout.buffer.write(a.tobytes() + o.tobytes())") % (HERE, os.path.dirname(HERE))
    runs = [subprocess.run([sys.executable, "-c", code], capture_output=True, check=True,
                           env=dict(os.environ, **({"RFB_EMU_SHUFFLE": s} if s else {}))).stdout
            for s in ("", "1", "7")]
    assert runs[0] == runs[1] == runs[2] and len(runs[0]) > 0
