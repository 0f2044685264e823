"""The float64 judge of the Delaunay adjacency (tests/delaunay_model.py) against Qhull and against brute force, so that
a model that under-reported face areas -- and would excuse any kernel error as 'justified' -- fails here."""
import numpy as np
import pytest

import delaunay_model as dm
from radfoam_b200 import foam
from radfoam_b200.delaunay import default_bounds


def generic(n, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (n, 3)).astype(np.float32)


def box(points, scale=None):
    lo, hi = default_bounds(points.min(0), points.max(0))
    lo, hi = lo.astype(np.float64), hi.astype(np.float64)
    if scale:
        lo, hi = lo - scale * (hi - lo), hi + scale * (hi - lo)
    return lo, hi


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_brute_force_equals_qhull_in_a_large_box(seed):
    p = generic(30, seed)
    lo, hi = box(p, 1e3)
    adj, off = dm.brute_graph(p, lo, hi)
    qa, qo = foam.delaunay_adjacency(p)
    assert np.array_equal(dm.codes(adj, off), dm.codes(qa, qo))


@pytest.mark.parametrize("seed", [3, 4])
def test_qhull_rows_and_all_points_give_the_same_areas(seed):
    """Qhull's row of i is a superset of i's Voronoi neighbours: clipping against it gives the area clipping against
    every point gives, on every Qhull edge, inside the default box."""
    p = generic(40, seed)
    lo, hi = box(p)
    qa, qo = foam.delaunay_adjacency(p)
    inside = 0
    for i in range(p.shape[0]):
        row = qa[qo[i]:qo[i + 1]]
        for j in row:
            a_row = dm.face_area(p, i, int(j), row, lo, hi)
            a_all = dm.face_area(p, i, int(j), range(p.shape[0]), lo, hi)
            d2 = float(((p[i].astype(np.float64) - p[j]) ** 2).sum())
            assert abs(a_row - a_all) <= 1e-9 * d2
            inside += a_all > dm.TAU * d2
    assert inside > 0.8 * qa.size, "most Qhull faces lie inside the default box"


@pytest.mark.parametrize("seed", [5, 6])
def test_every_face_inside_the_box_is_a_qhull_edge_and_above_tau(seed):
    p = generic(35, seed)
    lo, hi = box(p)
    adj, off = dm.brute_graph(p, lo, hi)
    qa, qo = foam.delaunay_adjacency(p)
    got, ref = dm.codes(adj, off), dm.codes(qa, qo)
    assert np.isin(got, ref).all(), "a face inside the box that Qhull does not have"
    for code in got.tolist():
        i, j = code >> 32, code & 0xFFFFFFFF
        d2 = float(((p[i].astype(np.float64) - p[j]) ** 2).sum())
        assert dm.face_area(p, i, j, qa[qo[i]:qo[i + 1]], lo, hi) > dm.TAU * d2


def test_a_removed_edge_is_flagged():
    p = generic(200, 7)
    lo, hi = box(p)
    qa, qo = foam.delaunay_adjacency(p)
    # drop the entry (i, j) with the largest face from both rows
    i = 0
    row = qa[qo[i]:qo[i + 1]]
    areas = [dm.face_area(p, i, int(j), row, lo, hi) for j in row]
    j = int(row[int(np.argmax(areas))])
    keep = np.ones(qa.size, bool)
    keep[qo[i] + int(np.argmax(areas))] = False
    rj = qa[qo[j]:qo[j + 1]]
    keep[qo[j] + int(np.nonzero(rj == i)[0][0])] = False
    rows = np.repeat(np.arange(p.shape[0]), np.diff(qo.astype(np.int64)))[keep]
    adj = qa[keep]
    off = np.zeros(p.shape[0] + 1, np.uint32)
    off[1:] = np.cumsum(np.bincount(rows, minlength=p.shape[0]))
    diffs = dm.judge(p, adj, off, qa, qo, lo, hi)
    assert sorted((d[0], d[1]) for d in diffs) == sorted([(i, j), (j, i)])
    assert all(d[2] > 1e-3 and d[3] for d in diffs)
