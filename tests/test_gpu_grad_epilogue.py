"""The gradient epilogues on the device: what the optimizer reads, held bit for bit to tests/param_model.py.

* finalize_grads_kernel and finalize_params_kernel on crafted accumulators (fp16 overflow, subnormals and ties,
  NaN / +-inf / -0 / FLT_MAX, scrub on and off; up to 300 001 points, where the grid-stride loop wraps at degree
  0), the density gradient against torch's own softplus_backward on CUDA and within its float64 bound;
* reduce_finalize_peers_kernel with W "ranks" that are W buffers of this one device (peer pointers to the same
  device are legal arguments): every instantiation (WORLD 2, 4, 8 and the generic loop), ragged blocks, ranks
  without a block, and a rank that loops over more blocks than its grid covers;
* a ray-sharded training step emulated on one GPU (image bands, one pipeline per rank, the peer reduction),
  held to the float64 model -- the only check of the sharded gradient path that runs on a one-GPU machine.

Every output is a view into a larger allocation whose other bytes hold a sentinel that must survive."""
import time
import warnings

import numpy as np
import pytest

import common
import epilogue_harness as H
import model64 as M
import param_model as P

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float16]
IDS = ["fp32", "fp16"]
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


def _pipe(deg, dtype):
    import radfoam_b200

    return radfoam_b200.create_pipeline(deg, "float16" if dtype == np.float16 else "float32")


@pytest.mark.parametrize("scrub", [False, True], ids=["raw", "scrub"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 3, 16, 17, 1000, 300001])
def test_finalize_crafted_accumulator(torch_cuda, n, deg, dtype, scrub):
    mem = H.TorchMemory(torch_cuda)
    pipe = _pipe(deg, dtype)
    contents = H._crafted(n, deg, n * 10 + deg, 0.25)
    H.prime_accumulator(mem, pipe._lib, pipe._handle, deg, n, contents)
    pts, attr = H.finalize_outputs(mem, pipe._lib, pipe._handle, deg, dtype, n, scrub)
    want_pts, want_attr = P.finalize(contents, deg, dtype, scrub)
    pts.check("points_grad", want_pts)
    attr.check("attr_grad", want_attr)


@pytest.mark.parametrize("scrub", [False, True], ids=["raw", "scrub"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 17, 1000, 300001])
def test_finalize_params_crafted_accumulator(torch_cuda, n, deg, dtype, scrub):
    """The parameter-form epilogue with the softplus edge densities bound: att_dc / att_sh / points bit for bit,
    density_grad bit for bit with torch.ops.aten.softplus_backward(g * scale, raw, 10, 20) on CUDA (what the
    unfused glue's autograd computes) and within the float64 bound."""
    torch = torch_cuda
    mem = H.TorchMemory(torch)
    pipe = _pipe(deg, dtype)
    a = P.attr_dim(deg)
    raw = H.edge_raw_density(n, seed=n + deg)
    raw_d = torch.from_numpy(raw).cuda()
    pipe.bind_scene_params(torch.zeros((n, 3), device="cuda"), torch.zeros((n, a - 4), device="cuda"), raw_d, SCALE)
    contents = H._crafted(n, deg, n * 10 + deg + 5, 0.25)
    H.prime_accumulator(mem, pipe._lib, pipe._handle, deg, n, contents)
    out = H.finalize_params_outputs(mem, pipe._lib, pipe._handle, deg, n, scrub)
    want = P.finalize_params(contents, raw, SCALE, deg, dtype, scrub)
    for k in ("points_grad", "att_dc_grad", "att_sh_grad"):
        if out[k] is not None:
            out[k].check(k, want[k])
    g = torch.from_numpy(want["density_column"]).cuda()  # the rounded, scrubbed attribute gradient's last column
    torch_grad = torch.ops.aten.softplus_backward(g * SCALE, raw_d, 10, 20)
    out["density_grad"].check("density_grad vs torch softplus_backward", torch_grad.cpu().numpy())
    got = out["density_grad"].out.cpu().numpy().astype(np.float64)
    v, e = want["density_grad"].v, np.broadcast_to(want["density_grad"].e, want["density_grad"].v.shape)
    ok = np.isfinite(v) & np.isfinite(e)
    bad = np.abs(got[ok] - v[ok]) > e[ok]
    assert not bad.any(), f"density_grad: {int(bad.sum())} entries outside the float64 bound"
    pipe.bind_scene_params(None, None, None)


@pytest.mark.parametrize("scrub", [False, True], ids=["raw", "scrub"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8, 16])
def test_peer_reduce_finalize_one_device(torch_cuda, world, deg, dtype, scrub):
    """N in {1, 15, 16, 17, 16W - 1 (the last rank has no block), 200 003 (a rank loops over more blocks than its
    grid of 132 * 16 CTAs covers)}.  After all ranks, every rank's outputs equal finalize(peer_sum(accs)) and
    rfb_trace_backward_finalize on an external accumulator holding that sum."""
    mem = H.TorchMemory(torch_cuda)
    pipe = _pipe(deg, dtype)
    for n in sorted({1, 15, 16, 17, 16 * world - 1, 200003}):
        accs = H.rank_accumulators(n, deg, world)
        want_pts, want_attr = H.run_peers(mem, pipe._lib, pipe._handle, deg, dtype, accs, scrub)
        H.prime_accumulator(mem, pipe._lib, pipe._handle, deg, n, P.peer_sum(accs))
        pts, attr = H.finalize_outputs(mem, pipe._lib, pipe._handle, deg, dtype, n, scrub)
        pts.check("points_grad", want_pts)
        attr.check("attr_grad", want_attr)
        pipe.set_grad_accumulator(None)


# ---------------------------------------------------------------- a ray-sharded step on one device
def sharded_impl(torch, f, world, keep):
    """check_implementation's ``impl``: the image dealt to ``world`` ranks as 8-row bands (radfoam_b200.sharded),
    one pipeline per rank accumulating into its rank buffer, then every rank's peer reduction."""
    import radfoam_b200
    from radfoam_b200 import sharded

    deg, n = f.sh_degree, f.num_points
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    scene = [dev(x) for x in (f.points, f.attributes, f.adjacency, f.offsets)]
    pipes = [radfoam_b200.create_pipeline(deg) for _ in range(world)]
    single = radfoam_b200.create_pipeline(deg)
    o_attr, o_pts, _, total = H.peer_layout(n, deg, np.float32)
    bufs = [torch.zeros(total, dtype=torch.uint8, device="cuda") for _ in range(world)]
    for p, b in zip(pipes, bufs):
        p.set_grad_accumulator(b[:o_attr].view(torch.float32).view(n, P.grad_row(deg)))
    import ctypes

    table = lambda off: (ctypes.c_void_p * world)(*[b.data_ptr() + off for b in bufs])  # noqa: E731
    a = P.attr_dim(deg)

    def run(rays, start, dq, g, gd, err, backward):
        image = rays.ndim == 3
        part = ((lambda t, r: sharded.shard_image(t, r, world)) if image
                else (lambda t, r: sharded.shard_flat(t, r, world)))
        rays_d, start_d, dq_d, g_d, gd_d = dev(rays), dev(start), dev(dq), dev(g), dev(gd)
        shard = lambda t, r: None if t is None else part(t, r).contiguous()  # noqa: E731
        fwd = []
        for r, p in enumerate(pipes):
            fwd.append(p.trace_forward(*scene, shard(rays_d, r), shard(start_d, r), depth_quantiles=shard(dq_d, r),
                                       return_contribution=True))
        join = ((lambda k: sharded.unshard_image([o[k] for o in fwd], rays.shape[0])) if image
                else (lambda k: torch.cat([o[k] for o in fwd])))
        out = {k: join(k) for k in fwd[0] if k != "contribution"}
        out["contribution"] = sum(o["contribution"] for o in fwd)
        ref = single.trace_forward(*scene, rays_d, start_d, depth_quantiles=dq_d)
        for k in ("rgba", "depth", "depth_indices", "num_intersections"):
            if k in ref:
                assert torch.equal(out[k], ref[k]), f"{k}: the reassembled shards differ from one pipeline's trace"
        out = {k: v.cpu().numpy() for k, v in out.items()}
        if backward:
            for r, p in enumerate(pipes):
                p.trace_backward_accumulate(*scene, shard(rays_d, r), shard(start_d, r), fwd[r]["rgba"],
                                            shard(g_d, r), shard(dq_d, r), fwd[r].get("depth_indices"),
                                            shard(gd_d, r))
            torch.cuda.synchronize()
            for r, p in enumerate(pipes):
                p.reduce_finalize_peers(world, r, n, table(0), table(o_attr), table(o_pts), torch.device("cuda"),
                                        scrub_nonfinite=True)
            torch.cuda.synchronize()
            tails = [b[o_attr:].clone() for b in bufs]
            for r in range(1, world):
                assert torch.equal(tails[r], tails[0]), f"rank {r}'s gradients differ from rank 0's"
            out["attr_grad"] = bufs[0][o_attr:o_attr + 4 * n * a].view(torch.float32).view(n, a).cpu().numpy()
            out["points_grad"] = bufs[0][o_pts:o_pts + 12 * n].view(torch.float32).view(n, 3).cpu().numpy()
            keep["rank_accumulators"] = world
        torch.cuda.synchronize()
        return out
    return run


@pytest.mark.parametrize("world", [2, 3])
def test_ray_sharded_step_on_one_device_within_model_bounds(torch_cuda, world):
    case = common.scene_case()
    f = case.foam
    keep = {}
    t = time.perf_counter()
    report = M.check_implementation(sharded_impl(torch_cuda, f, world, keep), f.points, f.attributes, f.adjacency,
                                    f.offsets, case.rays, case.start, case.quantiles, case.grad_rgba, case.grad_depth)
    print("\n" + M.format_report(f"sharded W={world} scene20k", report) + f" ({time.perf_counter() - t:.1f} s)")
    assert keep.get("rank_accumulators") == world
