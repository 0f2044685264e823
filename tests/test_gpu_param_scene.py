"""The parameter-form scene -- the default training path (FoamScene.forward(fused=True) -> TraceRaysParams) --
against the float64 model (tests/model64.py) and the softplus references (tests/param_model.py).

build_cells_params_kernel evaluates cat(att_dc, att_sh, scale * softplus(density, beta=10)).to(dtype) per value;
finalize_params_kernel rounds the attribute gradient to the attribute dtype, scrubs it and chains it through
softplus.  The model takes its attributes from the torch glue evaluated on CUDA (FoamScene.get_trace_data), whose
softplus is itself held to the float64 softplus bounds first, so the check is not circular.  A seeded tenth of the
raw densities sits at softplus' edges: around the x*10 > 20 switch, on the linear branch, at 0 and in the tail
where expf goes subnormal and then to 0.

The density gradient's bound: the kernel forms (fl(g * scale) * z) / (z + 1) with z = expf(fl(raw * 10)); the
fp32 product raw * 10 is the model's exact input (param_model takes it from numpy fp32), so beyond the attribute
gradient's own bound B (Scatter.bound) the EV rules add 4u|z| for expf and one rounding for each of g * scale,
* z, z + 1 and the division: |chain| * B + 8u |value| to first order, plus the subnormal terms of expf."""
import time
import warnings

import numpy as np
import pytest

import common
import model64 as M
import param_model as P

pytestmark = pytest.mark.gpu

SCALE = 1.7


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(autouse=True)
def _quiet():
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        yield


def edge_params(f, seed=31):
    """(att_dc, att_sh, raw [N,1], edge rows): the foam's colours, the raw densities that give its densities
    through scale * softplus(., beta=10), a seeded tenth of them overwritten with the edge set."""
    a = f.attributes.shape[1]
    sigma = np.maximum(f.attributes[:, -1:].astype(np.float64) / SCALE, 1e-30)
    with np.errstate(all="ignore"):
        raw = np.where(10.0 * sigma > 20.0, sigma, np.log(np.expm1(10.0 * sigma)) / 10.0).astype(np.float32)
    rows = np.random.default_rng(seed).choice(f.num_points, f.num_points // 10, replace=False)
    raw[rows, 0] = np.resize(P.EDGE_RAW, rows.size)
    return f.attributes[:, :3].copy(), f.attributes[:, 3:a - 1].copy(), raw, rows


def glue_scene(torch, f, att_dc, att_sh, raw, dtype):
    """FoamScene (the torch glue) on CUDA with the attribute dtype of the pipeline."""
    from radfoam_b200 import scene_io

    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    scene = scene_io.FoamScene(dev(f.points), dev(raw), dev(att_dc), dev(att_sh), dev(f.adjacency), dev(f.offsets),
                               sh_degree=f.sh_degree, activation_scale=SCALE)
    scene.attr_dtype = torch.float16 if dtype == np.float16 else torch.float32
    return scene


def check_torch_softplus(torch, raw):
    """The glue's softplus (torch on CUDA) within the float64 softplus bounds."""
    got = torch.nn.functional.softplus(torch.from_numpy(raw).cuda(), beta=10).cpu().numpy().astype(np.float64)
    want = P.softplus_beta10(raw)
    bad = np.abs(got - want.v) > want.e
    assert not bad.any(), f"torch softplus outside its float64 bound at raw {raw[bad][:4]}"


def hold(name, got, value, bound, count):
    """Scatter-style comparison of one gradient block: rows without a term exactly zero, the rest within bound.
    Returns model64.compare's tightness entry."""
    got = np.asarray(got, np.float64).reshape(value.shape)
    zero = count == 0
    if (got[zero] != 0).any():
        raise M.Mismatch(f"{name}: {int((got[zero] != 0).any(1).sum())} rows without any term are nonzero")
    sel = count > 0
    M._within(name, got[sel], value[sel], bound[sel])
    scale = np.abs(value[sel]).max() if sel.any() else 0.0
    return dict(entries=int(value.size), compared=int(sel.sum() * value.shape[1]),
                median_bound_over_abs=float(np.median(bound[sel] / np.maximum(np.abs(value[sel]), 1e-300)))
                if sel.any() else 0.0,
                tighter_than_1e5_max=float((bound[sel] < 1e-5 * scale).mean()) if sel.any() else 1.0)


def hold_param_grads(m, grads, raw, half, tag=""):
    """att_dc ‖ att_sh against the model's attr_grad[:, :A-1]; density against chain(raw) * attr_grad[:, A-1]."""
    s = m["attr_grad"]
    a = s.c
    b = s.bound("fp32_half" if half else "fp32")
    att = np.concatenate([grads["att_dc_grad"].reshape(-1, 3), grads["att_sh_grad"].reshape(s.n, a - 4)], axis=1)
    rep = hold(f"{tag}att_dc|att_sh", att, s.value[:, :a - 1], b[:, :a - 1], s.count)
    up = M.EV(s.value[:, a - 1:], b[:, a - 1:]) * float(np.float32(SCALE))
    want = P.softplus_beta10_backward(up, raw)
    hold(f"{tag}density_grad", grads["density_grad"], want.v, np.broadcast_to(want.e, want.v.shape), s.count)
    return rep


def params_impl(torch, f, att_dc, att_sh, raw, dtype, tape, last, statuses):
    """check_implementation's ``impl``: the product's Pipeline with the parameters bound, attributes=None."""
    import radfoam_b200

    half = dtype == np.float16
    pipe = radfoam_b200.create_pipeline(f.sh_degree, "float16" if half else "float32")
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    pts, adj, off = dev(f.points), dev(f.adjacency), dev(f.offsets)
    params = [dev(att_dc), dev(att_sh), dev(raw)]
    if tape:  # trainable tensors make the forward record the walk tape
        for t in [pts] + params:
            t.requires_grad_(True)
    pipe.bind_scene_params(*params, SCALE)
    pipe.record_tape = tape

    def run(rays, start, dq, g, gd, err, backward):
        rays_d, start_d, dq_d = dev(rays), dev(start), dev(dq)
        fwd = pipe.trace_forward(pts, None, adj, off, rays_d, start_d, depth_quantiles=dq_d, return_contribution=True)
        if backward and tape:
            if pipe.tape_status()["overflowed"]:  # the first recording sized the pool; record again to replay
                fwd = pipe.trace_forward(pts, None, adj, off, rays_d, start_d, depth_quantiles=dq_d,
                                         return_contribution=True)
            statuses.append(pipe.tape_status())
        out = {k: v.cpu().numpy() for k, v in fwd.items()}
        if backward:
            bwd = pipe.trace_backward_params(pts, adj, off, rays_d, start_d, fwd["rgba"], dev(g), dq_d,
                                             fwd.get("depth_indices"), dev(gd), dev(err))
            last.update({k: v.cpu().numpy() for k, v in bwd.items()})
            out["points_grad"] = last["points_grad"]
            if "point_error" in last:
                out["point_error"] = last["point_error"]
        torch.cuda.synchronize()
        return out
    return run


def check_params_case(torch, name, case, dtype, tape, edge_rows=None, ray_error=True):
    f = case.foam
    att_dc, att_sh, raw, rows = edge_params(f)
    check_torch_softplus(torch, raw)
    attrs = glue_scene(torch, f, att_dc, att_sh, raw, dtype).get_trace_data()[1].detach().cpu().numpy()
    err = None
    if ray_error:
        err = np.random.default_rng(4).uniform(0, 1, size=case.rays.shape[:-1]).astype(dtype)
    last, statuses = {}, []
    t = time.perf_counter()
    report, m = M.check_implementation(
        params_impl(torch, f, att_dc, att_sh, raw, dtype, tape, last, statuses), f.points, attrs, f.adjacency,
        f.offsets, case.rays, case.start, case.quantiles, case.grad_rgba.astype(dtype), case.grad_depth, err,
        return_model=True)
    report["attr_grad"] = hold_param_grads(m, last, raw, dtype == np.float16)
    composited = int((m["contribution"].count[rows] > 0).sum())
    if tape:
        assert statuses and all(s["used_chunks"] > 0 and not s["overflowed"] for s in statuses), statuses
    print("\n" + M.format_report(name, report).replace("attr_grad", "att_dc|att_sh+density")
          + f" | edge cells composited {composited}/{rows.size} ({time.perf_counter() - t:.1f} s)")
    return composited


@pytest.mark.parametrize("tape", [False, True], ids=["rewalk", "tape"])
@pytest.mark.parametrize("mode", ["cached", "direct"])
@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("q", [0, 2])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_config1_params_within_model_bounds(torch_cuda, deg, q, dtype, mode, tape, monkeypatch):
    monkeypatch.setenv("RFB_BWD_MODE", mode)
    check_params_case(torch_cuda, f"params config1 deg{deg} q{q} {np.dtype(dtype).name} {mode} tape={tape}",
                      common.config1(deg, q), dtype, tape)


@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
def test_edge_density_scene_within_model_bounds(torch_cuda, dtype):
    """20 k-point shell scene, degree 3, tape on: at least 50 edge-density cells must be composited."""
    composited = check_params_case(torch_cuda, f"params edge scene20k {np.dtype(dtype).name}",
                                   common.scene_case(20000, 160, 96, q=2), dtype, tape=True)
    assert composited >= 50, f"only {composited} edge-density cells composited"


@pytest.mark.parametrize("dtype", [np.float32, np.float16], ids=["fp32", "fp16"])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_fused_forward_and_gradients_equal_torch_glue(torch_cuda, deg, dtype):
    """The fused path against the torch glue on the edge-density scene: per-ray forward outputs bit for bit
    (rgba, depth, depth_indices, num_intersections); contribution (atomic order) within the model's bound; the
    four parameter gradients of both paths -- TraceRaysParams and torch autograd through get_trace_data +
    TraceRays -- within the model's bounds on a 80x48 crop (the model's cost keeps it that size)."""
    import radfoam_b200
    from radfoam_b200 import render

    torch = torch_cuda
    half = dtype == np.float16
    case = common.scene_case(20000, 160, 96, q=2, sh_degree=deg)
    f = case.foam
    att_dc, att_sh, raw, rows = edge_params(f)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    name = "float16" if half else "float32"
    glue = glue_scene(torch, f, att_dc, att_sh, raw, dtype)
    points, attributes, adj, off = glue.get_trace_data()
    rays, start, dq = dev(case.rays), dev(case.start), dev(case.quantiles)
    want = radfoam_b200.create_pipeline(deg, name).trace_forward(points, attributes, adj, off, rays, start,
                                                                  depth_quantiles=dq)
    fused = radfoam_b200.create_pipeline(deg, name)
    fused.bind_scene_params(glue.att_dc, glue.att_sh, glue.density, SCALE)
    got = fused.trace_forward(points, None, adj, off, rays, start, depth_quantiles=dq)
    fused.bind_scene_params(None, None, None)
    for k in ("rgba", "depth", "depth_indices", "num_intersections"):
        assert torch.equal(got[k], want[k]), f"{k}: fused forward differs from the torch glue"

    # gradients and contribution on a crop, both paths through their autograd ops
    crop = (slice(24, 72), slice(40, 120))
    rays_c, start_c, dq_c = case.rays[crop].copy(), case.start[crop].copy(), case.quantiles[crop].copy()
    m0 = M.trace(f.points, attributes.detach().cpu().numpy(), f.adjacency, f.offsets, rays_c, start_c, dq_c,
                 backward=False)
    amb = m0["ambiguous"]
    g = np.where(amb[..., None], 0, case.grad_rgba[crop]).astype(dtype)
    gd = np.where(amb[..., None], 0, case.grad_depth[crop]).astype(np.float32)
    results = {}
    for path in ("glue", "fused"):
        scene = glue_scene(torch, f, att_dc, att_sh, raw, dtype)
        params = [scene.primal_points, scene.att_dc, scene.att_sh, scene.density]
        for t in params:
            t.requires_grad_(True)
        pipe = radfoam_b200.create_pipeline(deg, name)
        if path == "fused":
            out = render.TraceRaysParams.apply(pipe, *params, SCALE, scene.point_adjacency,
                                               scene.point_adjacency_offsets, dev(rays_c), dev(start_c), dev(dq_c),
                                               True)
        else:
            pts_, attrs_, adj_, off_ = scene.get_trace_data()
            out = render.TraceRays.apply(pipe, pts_, attrs_, adj_, off_, dev(rays_c), dev(start_c), dev(dq_c), True)
        rgba, depth, contribution = out[0], out[1], out[2]
        ((rgba * dev(g)).sum().float() + (depth * dev(gd)).sum()).backward()
        results[path] = dict(rgba=rgba.detach().cpu().numpy(), contribution=contribution.detach().cpu().numpy(),
                             grads=[t.grad.cpu().numpy() for t in params])
    assert np.array_equal(results["glue"]["rgba"].view(np.uint8), results["fused"]["rgba"].view(np.uint8))
    m = M.trace(f.points, attributes.detach().cpu().numpy(), f.adjacency, f.offsets, rays_c, start_c, dq_c,
                rgba=results["glue"]["rgba"], grad_rgba=g, grad_depth=gd)
    for path, r in results.items():
        pg, dcg, shg, dg = r["grads"]
        report = M.compare({"points_grad": pg}, m, per_ray=False)
        if not amb.any():
            report.update(M.compare({"contribution": r["contribution"]}, m, per_ray=False))
        report["attr_grad"] = hold_param_grads(m, dict(att_dc_grad=dcg, att_sh_grad=shg, density_grad=dg), raw, half,
                                               tag=f"{path} ")
        report.update(rays=int(amb.size), rays_compared=int((~amb).sum()))
        print("\n" + M.format_report(f"{path} deg{deg} {np.dtype(dtype).name} crop", report)
              .replace("attr_grad", "att_dc|att_sh+density"))
