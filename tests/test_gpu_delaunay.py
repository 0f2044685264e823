"""radfoam_b200.delaunay_adjacency and Triangulation on the GPU: against Qhull, with every difference justified by the
float64 model (tests/delaunay_model.py), structure, determinism, and Triangulation driven as radfoam_model/scene.py
drives it."""
import numpy as np
import pytest
import torch

import delaunay_model as dm
import fuzz_cases
import radfoam_b200
from radfoam_b200 import foam
from radfoam_b200.delaunay import default_bounds

pytestmark = pytest.mark.gpu


def build(points, bounds=None):
    adj, off = radfoam_b200.delaunay_adjacency(torch.from_numpy(np.ascontiguousarray(points)).cuda(), bounds)
    return adj.cpu().numpy(), off.cpu().numpy()


def check_structure(adj, off, n):
    assert off.shape == (n + 1,) and off[0] == 0 and off[-1] == adj.size and np.all(np.diff(off.astype(np.int64)) >= 0)
    rows = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
    assert np.all(adj < n) and not np.any(adj == rows)
    for i in range(n) if n <= 5000 else []:
        assert np.all(np.diff(adj[off[i]:off[i + 1]].astype(np.int64)) > 0)
    if n > 5000:  # ascending rows, vectorised: within a row each entry exceeds the one before
        same = rows[1:] == rows[:-1]
        assert np.all(adj[1:][same] > adj[:-1][same])
    fwd = (rows.astype(np.int64) << 32) | adj.astype(np.int64)
    bwd = (adj.astype(np.int64) << 32) | rows.astype(np.int64)
    assert np.array_equal(np.sort(fwd), np.sort(bwd)), "not symmetric"


def check_against_qhull(points, adj, off, bounds=None):
    """Differences from Qhull's graph, every one justified by the model; returns how many there are."""
    qa, qo = foam.delaunay_adjacency(points)
    p = points.astype(np.float32)
    lo, hi = default_bounds(p.min(0), p.max(0))
    if bounds is not None:
        lo, hi = np.minimum(lo, np.float32(bounds[0])), np.maximum(hi, np.float32(bounds[1]))
    diffs = dm.judge(points, adj, off, qa, qo, lo.astype(np.float64), hi.astype(np.float64))
    bad = [d for d in diffs if d[2] > dm.TAU]
    assert not bad, f"{len(bad)} differences from Qhull with a face above the tolerance, e.g. {bad[:5]}"
    return len(diffs)


@pytest.mark.parametrize("kind", ["scene", "uniform"])
def test_200k_against_qhull_and_model(kind):
    n = 200_000
    points = (foam.scene_foam(n, seed=5).points if kind == "scene"
              else np.random.default_rng(5).uniform(-1, 1, (n, 3)).astype(np.float32))
    adj, off = build(points)
    check_structure(adj, off, points.shape[0])
    diffs = check_against_qhull(points, adj, off)
    print(f"{kind} 200k: {adj.size} entries, {diffs} entries differ from Qhull, all justified by the model")


@pytest.mark.parametrize("kind,seed", [(k, s) for k in ("lattice", "bcc", "cluster", "scaled", "uniform")
                                       for s in (0, 1)])
def test_fuzz_kinds(kind, seed):
    f = fuzz_cases.make_scene(np.random.default_rng(100 * seed + len(kind)), kind, 3000, 0)
    adj, off = build(f.points)
    check_structure(adj, off, f.points.shape[0])
    check_against_qhull(f.points, adj, off)


def test_builds_are_byte_identical():
    points = torch.from_numpy(foam.scene_foam(50_000, seed=3).points).cuda()
    a = radfoam_b200.delaunay_adjacency(points)
    for _ in range(2):
        b = radfoam_b200.delaunay_adjacency(points)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_triangulation_as_scene_drives_it():
    rng = np.random.default_rng(7)
    points = torch.from_numpy((rng.normal(size=(20_000, 3)) * 25).astype(np.float32)).cuda()
    tri = radfoam_b200.Triangulation(points)
    perm = tri.permutation().to(torch.long)
    assert torch.equal(torch.sort(perm).values, torch.arange(points.size(0), device="cuda"))
    primal = points[perm]
    adj, off = tri.point_adjacency().cpu().numpy(), tri.point_adjacency_offsets().cpu().numpy()
    check_structure(adj, off, primal.size(0))
    check_against_qhull(primal.cpu().numpy(), adj, off)
    # a training step moves the points; the incremental rebuild keeps their order
    moved = primal + 0.05 * torch.randn_like(primal)
    assert tri.rebuild(moved, incremental=True) is False
    assert torch.equal(tri.permutation(), perm.to(torch.int32).view(torch.uint32))
    adj, off = tri.point_adjacency().cpu().numpy(), tri.point_adjacency_offsets().cpu().numpy()
    check_against_qhull(moved.cpu().numpy(), adj, off)
    # densification changes N: the rebuild sorts again
    grown = torch.cat([moved, moved[:100] + 0.01])
    assert tri.rebuild(grown, incremental=True) is True
    perm2 = tri.permutation().to(torch.long)
    adj, off = tri.point_adjacency().cpu().numpy(), tri.point_adjacency_offsets().cpu().numpy()
    check_against_qhull(grown[perm2].cpu().numpy(), adj, off)
    with pytest.raises(RuntimeError, match="not provided"):
        tri.tets()


def test_duplicate_raises_and_the_perturb_retry_succeeds():
    rng = np.random.default_rng(11)
    p = rng.uniform(-1, 1, (5000, 3)).astype(np.float32)
    p[4000] = p[17]
    points = torch.from_numpy(p).cuda()
    tri = radfoam_b200.Triangulation(torch.from_numpy(rng.uniform(-1, 1, (5000, 3)).astype(np.float32)).cuda())
    with pytest.raises(radfoam_b200.TriangulationFailedError):
        tri.rebuild(points, incremental=True)
    # scene.py's loop: perturb, retry non-incrementally
    perturbation, del_points = 1e-6, points
    for _ in range(25):
        try:
            assert tri.rebuild(del_points, incremental=False) is True
            break
        except radfoam_b200.TriangulationFailedError:
            perturbation *= 2
            del_points = points + perturbation * torch.randn_like(points)
    else:
        pytest.fail("the perturb-retry loop did not succeed")
    assert tri.point_adjacency_offsets().numel() == 5001
    bad = points.clone()
    bad[3, 1] = float("nan")
    with pytest.raises(radfoam_b200.TriangulationFailedError):
        radfoam_b200.delaunay_adjacency(bad)


@pytest.mark.parametrize("kind,param", [("lattice", 0.0), ("lattice", 1e-7), ("scaled", 1e-3), ("scaled", 1e3)])
def test_pinned_tie_and_scale_cases(kind, param):
    """The exact and barely jittered lattices and the 1e-3 / 1e3 scalings, which make_scene only draws at random."""
    rng = np.random.default_rng(17)
    if kind == "lattice":
        g = np.stack(np.meshgrid(*[np.linspace(-1, 1, 16)] * 3, indexing="ij"), -1).reshape(-1, 3)
        p = (g + rng.normal(0, param, size=g.shape) if param else g).astype(np.float32)
    else:
        p = (rng.uniform(-1, 1, size=(4000, 3)) * param).astype(np.float32)
    p = np.unique(p, axis=0)
    adj, off = build(p)
    check_structure(adj, off, p.shape[0])
    check_against_qhull(p, adj, off)
