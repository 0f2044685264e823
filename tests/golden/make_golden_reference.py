"""Store what the reference's own kernels compute for every GPU test that compares with them (read through
tests/refgold.py).  Needs a GPU and oracle/_ref (`make -C oracle ref ref_py REF=<upstream radfoam checkout>`):

    python tests/golden/make_golden_reference.py OUTDIR [GROUP ...]   # then copy OUTDIR/*.npz to tests/golden/reference/

Each test module provides the function that runs the reference on exactly its inputs.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import common  # noqa: E402
import fuzz_cases  # noqa: E402
import refgold  # noqa: E402
import test_gpu_configs as configs  # noqa: E402
import test_gpu_farthest as farthest  # noqa: E402
import test_gpu_fullsize as fullsize  # noqa: E402
import test_gpu_fuzz as fuzz  # noqa: E402
import test_gpu_parity as parity  # noqa: E402
import test_gpu_reference_op as reference_op  # noqa: E402
import test_gpu_stale_model64 as stale  # noqa: E402
from oracle import ref_gpu  # noqa: E402


def make_parity(tmp):
    recs = {}
    for name, make in parity.REF_CASES.items():
        case = make()
        ref = parity.run_ref_gpu(torch, case, return_contribution=name.startswith("config1"))
        recs[name] = refgold.record(ref, exact=parity.REF_EXACT, sampled=[k for k in parity.REF_SAMPLED if k in ref])
        if name.startswith("scene60k"):
            ref2 = parity.run_ref_gpu(torch, case)
            recs[name]["grad_noise"] = np.float64(max(common.grad_error(ref2[k], ref[k])
                                                      for k in ("points_grad", "attr_grad")))
    half = parity.run_ref_gpu(torch, common.scene_case(), attr_dtype="float16", backward=False)
    recs["scene20k_half"] = refgold.record(half, exact=("num_intersections", "depth_indices"), sampled=("rgba",),
                                           rows=1024)
    for model in ("pinhole", "fisheye"):
        for dt in ("float16", "float32"):
            recs[f"benchmark_{model}_{dt}"] = refgold.record(parity.benchmark_frame(torch, model, dt, reference=True),
                                                             exact=("adjacent_diff", "frame"))
    frames = parity.checkpoint_frames(torch, tmp, reference=True)
    recs["pt_checkpoint"] = refgold.record({f"frame{k}": f for k, f in enumerate(frames)},
                                           exact=[f"frame{k}" for k in range(len(frames))])
    return recs


def make_fuzz():
    recs = {}
    for seed in fuzz.SEEDS:
        _, _, f, rays, start, dq, kw = fuzz_cases.make_case(seed)
        full = dict(weight_threshold=0.001, max_intersections=1024)
        full.update(kw)
        ref = parity.run_ref_gpu(torch, common.Case(f, rays, start, dq, seed=seed), **full)
        recs.setdefault(fuzz.group(seed), {})[f"seed{seed}"] = fuzz.reference_record(ref)
    for i, case, kw in fuzz.single_rays_3736():
        ref = parity.run_ref_gpu(torch, case, weight_threshold=0.0, max_intersections=1024)
        recs.setdefault(fuzz.group_3736(i), {})[f"seed3736_ray{i}"] = fuzz.reference_record(ref, entries=1 << 14)
    return recs


def make_farthest():
    recs = {}
    for make in ("edge", "scene200k"):
        f = farthest.reference_case(make)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
        idx, radius = ref_gpu.farthest_neighbor(d(f.points), d(f.adjacency), d(f.offsets))
        recs[make] = refgold.record({"indices": idx.cpu().numpy(), "radius": radius.cpu().numpy()},
                                    exact=("indices", "radius"))
    return recs


def make_reference_op():
    mod = reference_op.load_reference_op()
    recs = {}
    for with_error in (False, True):
        case = reference_op.op_case()
        for contribution, name in ((False, "op_error%d"), (True, "op_contribution_error%d")):
            res = reference_op.drive(torch, mod.TraceRays, reference_op.ReferencePipeline(), case, with_error,
                                     contribution=contribution)
            recs[name % int(with_error)] = reference_op.reference_record(res)
    recs["error_map"] = reference_op.reference_error_map(torch)
    return recs


def make_configs():
    recs = {name: configs.reference_record(torch, *args) for name, args in configs.CASES.items()}
    ref_gpu.load().rfref_release_pool()
    return recs


def make_fullsize():
    world = fullsize.make_world()
    return {"config2": fullsize.reference_record(world)}


def make_stale():
    """Stale scenes (moved points, the adjacency kept): integers whole, floats and gradients on sampled rows, and the
    reference's run-to-run gradient noise."""
    recs = {}
    for name, make in stale.REF_CASES.items():
        case = make()
        ref = parity.run_ref_gpu(torch, case)
        recs[name] = refgold.record(ref, exact=parity.REF_EXACT, sampled=[k for k in parity.REF_SAMPLED if k in ref])
        ref2 = parity.run_ref_gpu(torch, case)
        recs[name]["grad_noise"] = np.float64(max(common.grad_error(ref2[k], ref[k])
                                                  for k in ("points_grad", "attr_grad")))
        print(name, "reference noise", float(recs[name]["grad_noise"]), flush=True)
    return recs


def main(outdir):
    import pathlib
    import tempfile

    assert ref_gpu.available(), "oracle/_ref is not built"
    os.makedirs(outdir, exist_ok=True)
    groups = {"parity": lambda: make_parity(pathlib.Path(tempfile.mkdtemp())), "fuzz": make_fuzz, "farthest": make_farthest,
              "reference_op": make_reference_op, "fullsize": make_fullsize, "configs": make_configs, "stale": make_stale}
    only = sys.argv[2:] or list(groups)
    for name in only:
        recs = groups[name]()
        torch.cuda.synchronize()
        files = recs if name == "fuzz" else {name: recs}  # fuzz: {file: records}
        for fname, frecs in files.items():
            path = os.path.join(outdir, fname + ".npz")
            refgold.save(path, frecs)
            print(fname, len(frecs), "cases", os.path.getsize(path), "bytes", flush=True)


if __name__ == "__main__":
    main(sys.argv[1])
