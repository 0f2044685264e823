"""The float64 surface model (tests/surface_model.py) against scipy.spatial.Voronoi on points in general position:
every finite Voronoi ridge inside the box is the model's polygon (same vertex cycle), the polygons of an occupied set
clear of the box enclose exactly the occupied cells' volume, and lattice ties are flagged as near-degenerate."""
import numpy as np
import pytest
from scipy.spatial import ConvexHull, Voronoi

import fuzz_cases
import surface_model as sm
from radfoam_b200 import foam


def test_faces_are_the_voronoi_ridges():
    f = foam.small_foam(300, seed=11)
    lo, hi = sm.bounding_box(f.points)
    scale = float(np.linalg.norm(hi - lo))
    vor = Voronoi(f.points.astype(np.float64))
    rows = sm.rows_of(f.offsets)
    entry = {(int(rows[e]), int(f.adjacency[e])): e for e in range(f.adjacency.size)}
    checked = 0
    for (a, b), rv in zip(vor.ridge_points, vor.ridge_vertices):
        if -1 in rv:
            continue
        rverts = vor.vertices[rv]
        if (rverts < lo).any() or (rverts > hi).any():
            continue
        for i, j in ((a, b), (b, a)):
            got, deg = sm.face(f.points, f.adjacency, f.offsets, lo, hi, int(i), entry[(int(i), int(j))])
            assert not deg
            want = rverts if np.dot(sm.area_vector(rverts), f.points[j] - f.points[i]) > 0 else rverts[::-1]
            assert sm.same_cycle(want, got, 1e-9 * scale), (i, j)
            # counter-clockwise seen from j: the right-hand normal points from i to j
            assert np.dot(sm.area_vector(got), f.points[j].astype(np.float64) - f.points[i]) > 0
            checked += 1
    assert checked > 500


def test_volume_of_an_occupied_set_clear_of_the_box():
    f = foam.small_foam(400, seed=12)
    p = f.points.astype(np.float64)
    inside = np.linalg.norm(p, axis=1) < 0.5  # well inside [-1, 1]^3: the occupied cells are bounded
    vor = Voronoi(p)
    want = 0.0
    for i in np.flatnonzero(inside):
        region = vor.regions[vor.point_region[i]]
        assert -1 not in region
        want += ConvexHull(vor.vertices[region]).volume
    polys = sm.surface(f.points, f.adjacency, f.offsets, inside)
    assert len(polys) > 50
    assert not any(q.degenerate for q in polys)
    got = sm.enclosed_volume([q.vertices for q in polys])
    assert abs(got - want) <= 1e-9 * want, (got, want)


def test_lattice_ties_are_flagged():
    rng = np.random.default_rng(0)
    while True:
        f = fuzz_cases.make_scene(rng, "lattice", 64, 0)
        if np.allclose(f.points * 3, np.round(f.points * 3), atol=0):  # the exact lattice, no jitter
            break
    inside = np.zeros(f.num_points, bool)
    inside[np.argmin(np.linalg.norm(f.points, axis=1))] = True
    polys = sm.surface(f.points, f.adjacency, f.offsets, inside)
    assert polys and any(q.degenerate for q in polys)


@pytest.mark.parametrize("seed", [0, 1])
def test_empty_and_full_masks(seed):
    f = foam.small_foam(80, seed=seed)
    assert sm.surface(f.points, f.adjacency, f.offsets, np.zeros(80, bool)) == []
    assert sm.surface(f.points, f.adjacency, f.offsets, np.ones(80, bool)) == []
