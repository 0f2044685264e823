"""Point location and field sampling on the GPU through the public wrappers (locate_points, Pipeline.sample_field,
SampleField): 2 M secondary-ray origins on the config-4 foam, the tracer's own colour, autograd against the float64
model, a trace step with sampling in between, and CUDA-graph capture."""
import os
import sys

import numpy as np
import pytest

import locate_model as lm

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF
GAP = 8 * lm.U32  # as tests/test_emu_locate.py: fp32 d2 keeps the order of distances further apart than this


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def config4(torch_cuda):
    """The 1080p bench frame on the 1,048,576-point foam: each pixel's median-depth point (a secondary ray's origin)
    and the cell the forward reported there (depth_indices)."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    import radfoam_b200

    torch = torch_cuda
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    fr = bench.make_frame(f, 1920, 1080)
    pts, attrs, adj, off = dev(torch, f.points), dev(torch, f.attributes), dev(torch, f.adjacency), dev(torch, f.offsets)
    rays, start = dev(torch, fr["rays"]), dev(torch, fr["start"])
    pipe = radfoam_b200.create_pipeline(3)
    dq = torch.full((1080, 1920, 1), 0.5, device="cuda")
    out = pipe.trace_forward(pts, attrs, adj, off, rays, start, depth_quantiles=dq)
    depth, idx = out["depth"][..., 0], lm.as_long(out["depth_indices"][..., 0])  # uint32 tensors cannot be indexed
    hit = torch.isfinite(depth) & (idx != NONE)
    o = (rays[..., :3] + depth[..., None] * rays[..., 3:])[hit]
    hint = idx[hit]
    # 2 M distinct origins: the frame's surface points and, to fill up, the same points nudged off them
    m = 2 * 1024 * 1024
    g = torch.Generator(device="cuda").manual_seed(0)
    extra = m - o.shape[0]
    pick = torch.randint(0, o.shape[0], (extra,), device="cuda", generator=g)
    o = torch.cat([o, o[pick] + 1e-3 * torch.randn((extra, 3), device="cuda", generator=g)])
    hint = torch.cat([hint, hint[pick]]).to(torch.uint32)
    return dict(foam=f, pts=pts, attrs=attrs, adj=adj, off=off, pipe=pipe, queries=o.contiguous(), hint=hint)


def check_all(torch, c, q, got):
    """cKDTree rule on every query, brute-force nearest_point on a 4,096 subsample, local minimum everywhere."""
    import radfoam_b200
    from scipy.spatial import cKDTree

    adj64, off64 = lm.as_long(c["adj"]), lm.as_long(c["off"])
    assert lm.local_min(c["pts"], adj64, off64, q, got).all()
    sub = torch.randperm(q.shape[0], device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))[:4096]
    brute = radfoam_b200.nearest_point(c["pts"], q[sub])
    assert torch.equal(lm.as_long(brute), lm.as_long(got)[sub])
    p64, q64, g = c["foam"].points.astype(np.float64), q.cpu().numpy().astype(np.float64), got.cpu().numpy()
    d, i = cKDTree(p64).query(q64, k=2, workers=-1)
    d1, d2 = d[:, 0] ** 2, d[:, 1] ** 2
    clear = d2 - d1 > GAP * (d1 + d2)
    assert np.array_equal(g[clear], i[clear, 0].astype(np.uint32))
    dg = ((p64[g.astype(np.int64)] - q64) ** 2).sum(1)
    assert np.all(dg - d1 <= GAP * (dg + d1))


@pytest.mark.parametrize("with_hint", [True, False])
def test_secondary_origins_2m(torch_cuda, config4, with_hint):
    import radfoam_b200

    torch, c = torch_cuda, config4
    q = c["queries"]
    got = radfoam_b200.locate_points(c["pts"], c["adj"], c["off"], q, hint=c["hint"] if with_hint else None)
    assert got.dtype == torch.uint32 and got.shape == q.shape[:-1]
    check_all(torch, c, q, got)


def test_sample_field_rgb_is_the_tracers_cell_colour(torch_cuda):
    """A 1-cell-deep probe: with every density huge the first cell absorbs the whole ray (alpha rounds to 1), so the
    ray's colour is that cell's colour bit for bit; rays from the sampled points along the sampled directions.  Rays
    that leave their first cell within a few 1e-4 (alpha below 1) reach a second cell and are not compared."""
    import radfoam_b200
    from radfoam_b200 import foam

    torch = torch_cuda
    for dtype in ("float32", "float16"):
        for deg in (0, 1, 2, 3):
            f = foam.scene_foam(20000, sh_degree=deg, seed=3)
            attrs = f.attributes.copy()
            attrs[:, -1] = 1e4
            rng = np.random.default_rng(deg)
            q = rng.uniform(-1.2, 1.2, size=(4096, 3)).astype(np.float32)
            d = rng.normal(size=(4096, 3)).astype(np.float32)
            pipe = radfoam_b200.create_pipeline(deg, dtype)
            tdt = torch.float16 if dtype == "float16" else torch.float32
            pts, at, adj, off = dev(torch, f.points), dev(torch, attrs).to(tdt), dev(torch, f.adjacency), dev(torch, f.offsets)
            s = pipe.sample_field(pts, at, adj, off, dev(torch, q), dev(torch, d))
            rays = torch.cat([dev(torch, q), dev(torch, d)], -1)
            # traced in fp32 on the same (fp16-representable) values, so that "fully opaque" is exact: an fp16
            # rgba would round an alpha of 1 - 2^-13 to 1
            out = radfoam_b200.create_pipeline(deg).trace_forward(pts, at.float(), adj, off, rays, s["cell"])
            # one cell entered and fully opaque: the ray's colour is w * rgb with w = alpha = 1
            full = (out["rgba"][:, 3] == 1) & (lm.as_long(out["num_intersections"][:, 0]) == 1)
            assert full.float().mean() > 0.8
            assert torch.equal(out["rgba"][full, :3].to(tdt), s["rgb"][full]), (dtype, deg)
            assert torch.equal(s["density"], at[lm.as_long(s["cell"]), -1])


@pytest.mark.parametrize("dtype", ["float32", "float16"])
@pytest.mark.parametrize("deg", [0, 3])
def test_autograd_matches_float64_model(torch_cuda, deg, dtype):
    import radfoam_b200
    from radfoam_b200 import foam

    torch = torch_cuda
    f = foam.small_foam(300, sh_degree=deg, seed=deg)
    rng = np.random.default_rng(7)
    g = np.linspace(-0.95, 0.95, 40)
    q = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)  # ~200 per cell
    d = rng.normal(size=q.shape).astype(np.float32)
    tdt = torch.float16 if dtype == "float16" else torch.float32
    npdt = np.float16 if dtype == "float16" else np.float32
    attrs = dev(torch, f.attributes.astype(npdt)).requires_grad_(True)
    pipe = radfoam_b200.create_pipeline(deg, dtype)
    pts = dev(torch, f.points).requires_grad_(True)
    density, rgb, cell = radfoam_b200.SampleField.apply(pipe, pts, attrs, dev(torch, f.adjacency),
                                                        dev(torch, f.offsets), dev(torch, q), dev(torch, d), None)
    wd, wr = (rng.normal(size=s).astype(npdt) for s in (density.shape, rgb.shape))
    ((density * dev(torch, wd)).sum() + (rgb * dev(torch, wr)).sum()).backward()
    assert pts.grad is None
    want, bound = lm.field_grad64(f.num_points, deg, cell.cpu().numpy(), d, rgb.detach().cpu().numpy(), wr, wd, npdt)
    err = np.abs(attrs.grad.cpu().numpy().astype(np.float64) - want)
    assert np.all(err <= bound)
    c_ = cell.cpu().numpy()
    _, want_rgb, rb = lm.field64(f.attributes.astype(npdt), c_, d, deg, npdt)
    assert np.all(np.abs(rgb.detach().cpu().numpy().astype(np.float64) - want_rgb) <= rb)
    with pytest.raises(RuntimeError, match="queries"):
        radfoam_b200.SampleField.apply(pipe, pts, attrs, dev(torch, f.adjacency), dev(torch, f.offsets),
                                       dev(torch, q).requires_grad_(True), dev(torch, d), None)
    with pytest.raises(RuntimeError, match="directions"):
        radfoam_b200.SampleField.apply(pipe, pts, attrs, dev(torch, f.adjacency), dev(torch, f.offsets),
                                       dev(torch, q), dev(torch, d).requires_grad_(True), None)


def test_sampling_between_trace_forward_and_backward(torch_cuda):
    """A recorded walk tape is still replayed, and the gradients are unchanged, when sample_field and its backward
    run between a step's forward and backward on the same pipeline."""
    import common
    import radfoam_b200

    torch = torch_cuda
    case = common.scene_case(20000, 160, 96, 2)
    f = case.foam
    pts, attrs = dev(torch, f.points).requires_grad_(True), dev(torch, f.attributes).requires_grad_(True)
    adj, off = dev(torch, f.adjacency), dev(torch, f.offsets)
    rays, start, dq = dev(torch, case.rays), dev(torch, case.start), dev(torch, case.quantiles)
    g, gd = dev(torch, case.grad_rgba), dev(torch, case.grad_depth)
    q = torch.rand((50000, 3), device="cuda") * 2 - 1
    dirs = torch.randn((50000, 3), device="cuda")

    def step(pipe, middle):
        out = pipe.trace_forward(pts, attrs, adj, off, rays, start, depth_quantiles=dq)
        if middle:
            s = pipe.sample_field(pts, attrs, adj, off, q, dirs)
            pipe.sample_field_backward(f.num_points, s["cell"], dirs, s["rgb"], torch.ones_like(s["rgb"]),
                                       torch.ones_like(s["density"]))
        before = radfoam_b200.pipeline.launch_count()
        grads = pipe.trace_backward(pts, attrs, adj, off, rays, start, out["rgba"], g, dq, out["depth_indices"], gd)
        torch.cuda.synchronize()
        return grads, radfoam_b200.pipeline.launch_count() - before

    ref, ref_launches = step(radfoam_b200.create_pipeline(3), False)
    pipe = radfoam_b200.create_pipeline(3)
    got, launches = step(pipe, True)
    assert launches == ref_launches  # the same kernels: the tape replay and nothing rebuilt
    for k in ("points_grad", "attr_grad"):
        assert common.grad_error(got[k].cpu().numpy(), ref[k].cpu().numpy()) <= 1e-6, k


def test_cuda_graph_capture(torch_cuda):
    import radfoam_b200
    from radfoam_b200 import foam

    torch = torch_cuda
    for dtype in ("float32", "float16"):
        f = foam.scene_foam(20000, sh_degree=2, seed=4)
        tdt = torch.float16 if dtype == "float16" else torch.float32
        pts, attrs = dev(torch, f.points), dev(torch, f.attributes).to(tdt)
        adj, off = dev(torch, f.adjacency), dev(torch, f.offsets)
        pipe = radfoam_b200.create_pipeline(2, dtype)
        q = torch.rand((100000, 3), device="cuda") * 3 - 1.5
        d = torch.randn((100000, 3), device="cuda")
        gr = torch.randn((100000, 3), device="cuda").to(tdt)
        eager = (radfoam_b200.locate_points(pts, adj, off, q), pipe.sample_field(pts, attrs, adj, off, q, d))
        eager_grad = pipe.sample_field_backward(f.num_points, eager[1]["cell"], d, eager[1]["rgb"], gr,
                                                eager[1]["density"])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                cells = radfoam_b200.locate_points(pts, adj, off, q)
                out = pipe.sample_field(pts, attrs, adj, off, q, d)
                grad = pipe.sample_field_backward(f.num_points, out["cell"], d, out["rgb"], gr, out["density"])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(lm.as_long(cells), lm.as_long(eager[0]))
        assert torch.equal(lm.as_long(out["cell"]), lm.as_long(eager[1]["cell"]))
        assert torch.equal(out["rgb"], eager[1]["rgb"]) and torch.equal(out["density"], eager[1]["density"])
        torch.testing.assert_close(grad.float(), eager_grad.float(), rtol=1e-3, atol=1e-3)


def test_validation(torch_cuda):
    import radfoam_b200
    from radfoam_b200 import foam

    torch = torch_cuda
    f = foam.small_foam(64, seed=1)
    p, a, o = dev(torch, f.points), dev(torch, f.adjacency), dev(torch, f.offsets)
    q = torch.zeros((5, 2, 3), device="cuda")
    assert radfoam_b200.locate_points(p, a, o, q).shape == (5, 2)
    assert torch.all(lm.as_long(radfoam_b200.locate_points(p, a, o, q, hint=7)) ==
                     lm.as_long(radfoam_b200.locate_points(p, a, o, q)))
    with pytest.raises(RuntimeError, match="uint32"):
        radfoam_b200.locate_points(p, a.to(torch.int64), o, q)
    with pytest.raises(RuntimeError, match="num_points \\+ 1"):
        radfoam_b200.locate_points(p, a, o[:-1], q)
    with pytest.raises(RuntimeError, match="float32"):
        radfoam_b200.locate_points(p, a, o, q.double())
    with pytest.raises(RuntimeError, match="batch shape"):
        radfoam_b200.locate_points(p, a, o, q, hint=torch.zeros(10, dtype=torch.int64, device="cuda"))
    assert radfoam_b200.locate_points(p, a, o, q[:0]).numel() == 0
