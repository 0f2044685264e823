"""Surface extraction on the GPU through Pipeline.extract_surface: against the float64 model (tests/surface_model.py)
at 2k and 50k points and on a random sample of the config-4 foam (1,048,576 points), the enclosed volume, watertightness,
rgb bit for bit against sample_field, determinism, a trace step with extraction in between, and argument checks."""
import os
import sys

import numpy as np
import pytest

import surface_model as sm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run(torch, f, deg=None, dtype="float32", **kw):
    import radfoam_b200

    deg = f.sh_degree if deg is None else deg
    tdt = torch.float16 if dtype == "float16" else torch.float32
    pipe = radfoam_b200.create_pipeline(deg, dtype)
    args = (dev(torch, f.points), dev(torch, f.attributes).to(tdt), dev(torch, f.adjacency), dev(torch, f.offsets))
    return pipe, args, pipe.extract_surface(*args, **kw)


def host(out):
    return {k: v.cpu().numpy() for k, v in out.items()}


def compare(out, f, inside, entries=None):
    """The kernel's polygons against the model's, on every entry or on a sample of emitted ones."""
    lo, hi = sm.bounding_box(f.points)
    scale = float(np.linalg.norm(hi - lo))
    o = host(out)
    off = o["offsets"]
    rows = sm.rows_of(f.offsets)
    emitted_entries = []
    # the entry of each emitted polygon: the emitted (i, j) pairs follow CSR order
    cand = np.flatnonzero(inside[rows] & ~inside[f.adjacency])
    pairs = {}
    for e in cand:
        pairs.setdefault((int(rows[e]), int(f.adjacency[e])), []).append(int(e))
    for c in o["cells"].astype(np.int64):
        emitted_entries.append(pairs[(int(c[0]), int(c[1]))].pop(0))
    emitted_entries = np.array(emitted_entries, np.int64)
    sel = np.arange(len(emitted_entries)) if entries is None else entries
    want = {q.entry: q for q in sm.surface(f.points, f.adjacency, f.offsets, inside,
                                           entries=emitted_entries[sel] if entries is not None else None)}
    area_tol = (1e-6 * scale) ** 2
    if entries is None:  # the polygon sets are equal, except polygons below the area tolerance
        emitted = set(emitted_entries.tolist())
        for e, q in want.items():
            assert e in emitted or np.linalg.norm(sm.area_vector(q.vertices)) <= area_tol, e
    checked = 0
    for k in sel:
        e = int(emitted_entries[k])
        v = o["vertices"][off[k]:off[k + 1]].astype(np.float64)
        q = want.get(e)
        if q is None:
            assert np.linalg.norm(sm.area_vector(v)) <= area_tol, e
            continue
        if not q.degenerate and v.shape == q.vertices.shape:
            r = int(np.argmin(np.linalg.norm(v - q.vertices[0], axis=1)))
            assert np.all(np.abs(np.roll(v, -r, axis=0) - q.vertices) <= sm.vertex_bound(q.vertices, scale)), e
        else:
            assert np.linalg.norm(sm.area_vector(v) - sm.area_vector(q.vertices)) <= 1e-6 * scale ** 2, e
            assert sm.hausdorff(v, q.vertices) <= 1e-6 * scale, e
        checked += 1
    return checked


def polygons(o):
    off = o["offsets"]
    return [o["vertices"][off[k]:off[k + 1]].astype(np.float64) for k in range(off.size - 1)]


def occupied_volume(points, inside):
    from scipy.spatial import ConvexHull, Voronoi

    vor = Voronoi(points.astype(np.float64))
    total = 0.0
    for i in np.flatnonzero(inside):
        region = vor.regions[vor.point_region[i]]
        assert -1 not in region
        total += ConvexHull(vor.vertices[region]).volume
    return total


def watertight(o, tol):
    """After welding vertices within ``tol``, every undirected polygon edge occurs an even number of times."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    from scipy.spatial import cKDTree

    v = o["vertices"].astype(np.float64)
    pairs = cKDTree(v).query_pairs(tol, output_type="ndarray")
    graph = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(v.shape[0], v.shape[0]))
    _, vid = connected_components(graph, directed=False)
    off = o["offsets"]
    a = vid
    nxt = np.arange(a.size) + 1
    nxt[off[1:] - 1] = off[:-1]
    b = vid[nxt]
    edges = np.sort(np.stack([a, b], 1), axis=1)
    edges = edges[edges[:, 0] != edges[:, 1]]
    _, counts = np.unique(edges, axis=0, return_counts=True)
    return bool(np.all(counts % 2 == 0)), int((counts % 2).sum())


@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_2k_against_model_volume_watertight(torch_cuda, dtype):
    from radfoam_b200 import foam

    torch = torch_cuda
    f = foam.small_foam(2000, sh_degree=3, seed=21)
    inside = np.linalg.norm(f.points, axis=1) < 0.6
    pipe, args, out = run(torch, f, dtype=dtype, inside=dev(torch, inside))
    assert compare(out, f, inside) > 500
    o = host(out)
    vol = sm.enclosed_volume(polygons(o))
    want = occupied_volume(f.points, inside)
    assert abs(vol - want) <= 1e-5 * want, (vol, want)
    ok, odd = watertight(o, 1e-6)
    assert ok, f"{odd} unpaired edges"
    # triangles: a fan per polygon, V - 2P of them, each inside its polygon's vertex run
    tri = o["triangles"]
    assert tri.shape == (o["vertices"].shape[0] - 2 * (o["offsets"].size - 1), 3)
    tri_area = 0.5 * np.linalg.norm(np.cross(o["vertices"][tri[:, 1]] - o["vertices"][tri[:, 0]],
                                             o["vertices"][tri[:, 2]] - o["vertices"][tri[:, 0]]), axis=1).sum()
    assert abs(tri_area - sum(np.linalg.norm(sm.area_vector(v)) for v in polygons(o))) <= 1e-4 * tri_area


def test_50k_shell_threshold(torch_cuda):
    from radfoam_b200 import foam

    torch = torch_cuda
    f = foam.scene_foam(50000, sh_degree=1, seed=7)
    # the shell's occupied cells (a threshold also selects a few cells of the far field, unbounded ones among them)
    inside = (f.attributes[:, -1] > 0.5) & (np.linalg.norm(f.points, axis=1) < 2.0)
    pipe, args, out = run(torch, f, inside=dev(torch, inside))
    o = host(out)
    npoly = o["offsets"].size - 1
    assert npoly > 10000
    rng = np.random.default_rng(0)
    assert compare(out, f, inside, entries=np.sort(rng.choice(npoly, 3000, replace=False))) > 2500
    vol = sm.enclosed_volume(polygons(o))
    want = occupied_volume(f.points, inside)
    assert abs(vol - want) <= 1e-5 * want, (vol, want)
    ok, odd = watertight(o, 1e-6)
    assert ok, f"{odd} unpaired edges"
    # rgb: sample_field at p_i along p_i - p_j (the kernel renormalises the direction), bit for bit
    for dtype in ("float32", "float16"):
        pipe, args, out = run(torch, f, dtype=dtype, threshold=0.5)
        c = out["cells"].to(torch.int64)
        assert bool((args[1][c[:, 0], -1] > 0.5).all()) and not bool((args[1][c[:, 1], -1] > 0.5).any())
        pts = args[0]
        s = pipe.sample_field(*args, pts[c[:, 0]], pts[c[:, 0]] - pts[c[:, 1]], hint=c[:, 0])
        assert torch.equal(s["cell"].to(torch.int64), c[:, 0])
        assert torch.equal(s["rgb"], out["rgb"]), dtype
    # two calls give identical bytes
    again = pipe.extract_surface(*args, threshold=0.5)
    for k in out:
        assert torch.equal(out[k], again[k]), k


def test_config4_sample(torch_cuda):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench

    torch = torch_cuda
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    inside = f.attributes[:, -1] > 0.5
    pipe, args, out = run(torch, f, threshold=0.5)
    npoly = out["offsets"].numel() - 1
    assert npoly > 100000
    rng = np.random.default_rng(4)
    assert compare(out, f, inside, entries=np.sort(rng.choice(npoly, 2000, replace=False))) > 1900


def test_tape_replay_unchanged_with_extraction_between(torch_cuda):
    """A recorded walk tape is still replayed, and the gradients are unchanged, when extract_surface runs between a
    step's forward and backward on the same pipeline."""
    import common
    import radfoam_b200

    torch = torch_cuda
    case = common.scene_case(20000, 160, 96, 2)
    f = case.foam
    pts, attrs = dev(torch, f.points).requires_grad_(True), dev(torch, f.attributes).requires_grad_(True)
    adj, off = dev(torch, f.adjacency), dev(torch, f.offsets)
    rays, start, dq = dev(torch, case.rays), dev(torch, case.start), dev(torch, case.quantiles)
    g, gd = dev(torch, case.grad_rgba), dev(torch, case.grad_depth)

    def step(pipe, middle):
        out = pipe.trace_forward(pts, attrs, adj, off, rays, start, depth_quantiles=dq)
        if middle:
            s = pipe.extract_surface(pts, attrs, adj, off, threshold=0.5)
            assert s["offsets"].numel() > 1
        before = radfoam_b200.pipeline.launch_count()
        grads = pipe.trace_backward(pts, attrs, adj, off, rays, start, out["rgba"], g, dq, out["depth_indices"], gd)
        torch.cuda.synchronize()
        return grads, radfoam_b200.pipeline.launch_count() - before

    ref, ref_launches = step(radfoam_b200.create_pipeline(3), False)
    got, launches = step(radfoam_b200.create_pipeline(3), True)
    assert launches == ref_launches
    for k in ("points_grad", "attr_grad"):
        assert common.grad_error(got[k].cpu().numpy(), ref[k].cpu().numpy()) <= 1e-6, k


def test_validation_and_empty(torch_cuda):
    from radfoam_b200 import foam

    torch = torch_cuda
    f = foam.small_foam(200, sh_degree=0, seed=3)
    pipe, args, out = run(torch, f, inside=torch.zeros(200, dtype=torch.bool, device="cuda"))
    assert out["offsets"].tolist() == [0] and out["vertices"].shape == (0, 3) and out["cells"].shape == (0, 2)
    assert out["triangles"].shape == (0, 3) and out["rgb"].shape == (0, 3)
    pts, attrs, adj, off = args
    inside = torch.ones(200, dtype=torch.bool, device="cuda")
    for kw, match in ((dict(), "exactly one"), (dict(threshold=0.1, inside=inside), "exactly one"),
                      (dict(inside=inside.to(torch.uint8)), "bool"), (dict(inside=inside[:10]), "bool"),
                      (dict(inside=inside.cpu()), "bool"),
                      (dict(threshold=0.1, bounds=([1, 1, 1], [0, 0, 0])), "bounds"),
                      (dict(threshold=0.1, bounds=([0, 0], [1, 1])), "bounds")):
        with pytest.raises(RuntimeError, match=match):
            pipe.extract_surface(pts, attrs, adj, off, **kw)
    with pytest.raises(RuntimeError, match="float32"):
        pipe.extract_surface(pts.double(), attrs, adj, off, threshold=0.1)
    with pytest.raises(RuntimeError, match="uint32"):
        pipe.extract_surface(pts, attrs, adj.to(torch.int64), off, threshold=0.1)
    with pytest.raises(RuntimeError, match="dimension"):
        pipe.extract_surface(pts, attrs[:, :2], adj, off, threshold=0.1)
    with pytest.raises(RuntimeError, match="CUDA"):
        pipe.extract_surface(pts.cpu(), attrs, adj, off, threshold=0.1)
