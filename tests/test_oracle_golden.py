"""CPU tests: the restatement oracle/radfoam_oracle.c against golden vectors produced by the
reference's OWN kernels (oracle/_ref = /root/reference/src/tracing/pipeline.cu compiled
unmodified against oracle/eigen_shim) on a B200 -- tests/golden/make_golden.py made them.
This is what pins the oracle: the reference ships no tests or fixtures for this path."""
import glob
import os

import numpy as np
import pytest

import common
import model64
from oracle import oracle

GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))
                if not os.path.basename(p).startswith(("benchmark", "farthest")))


def test_golden_vectors_present():
    assert len(GOLDEN) >= 10


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_reproduces_reference_kernel_outputs(path):
    z = dict(np.load(path))
    half = z["attributes"].dtype == np.float16
    q = z.get("quantiles")
    settings = (float(z["weight_threshold"]), int(z["max_intersections"]))
    scene = (z["points"], z["attributes"], z["adjacency"], z["offsets"])
    fwd = oracle.trace_forward(*scene, z["rays"], z["start"], q, *settings, return_contribution=True)
    # integer traversal outputs: bit-exact against the reference's kernels
    assert np.array_equal(fwd["num_intersections"], z["out_num_intersections"])
    if q is not None:
        assert np.array_equal(fwd["depth_indices"], z["out_depth_indices"])
    if half:
        # fp16 mode rounds rgba to half and accumulates with order-dependent half adds
        np.testing.assert_allclose(fwd["rgba"].astype(np.float32), z["out_rgba"].astype(np.float32),
                                   rtol=2e-3, atol=1e-3)
        # its gradients are half atomics like the reference's: each entry within the float64 model's
        # half-atomic bound, on the oracle's own saved outputs
        bwd = oracle.trace_backward(*scene, z["rays"], z["start"], fwd["rgba"], z["grad_rgba"], q,
                                    fwd.get("depth_indices"), z.get("grad_depth"), None, *settings)
        m = model64.trace(*scene, z["rays"], z["start"], q, *settings, rgba=fwd["rgba"], grad_rgba=z["grad_rgba"],
                          grad_depth=z.get("grad_depth"), depth_indices=fwd.get("depth_indices"))
        skip = model64.rows_reachable(m, z["offsets"], z["adjacency"], z["points"], z["attributes"], z["rays"],
                                      z["start"], q, *settings)
        model64.compare({k: np.asarray(bwd[k]) for k in ("points_grad", "attr_grad")}, m, half_atomics=True,
                        skip_rows=skip, per_ray=False)
        return
    ref = {k[4:]: v for k, v in z.items() if k.startswith("out_")}
    common.assert_forward_close_cpu(fwd, ref, z["attributes"])
    bwd = oracle.trace_backward(*scene, z["rays"], z["start"], z["out_rgba"], z["grad_rgba"], q,
                                z.get("out_depth_indices"), z.get("grad_depth"), None, *settings)
    for k in ("points_grad", "attr_grad"):
        assert common.nonfinite_mismatch(bwd[k], ref[k]) == 0
        assert common.grad_error(bwd[k], ref[k]) <= common.CPU_GRAD_TOL, k


def test_golden_inputs_are_the_seeded_cases():
    """The fixtures hold the inputs they were made from; they must equal what the seeded
    generators produce today, or generator drift would silently detach the GPU tests (which
    regenerate inputs) from the CPU tests (which read them)."""
    z = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "config1_deg3_q2.npz")))
    case = common.config1(3, 2)
    assert np.array_equal(z["points"], case.foam.points)
    assert np.array_equal(z["attributes"], case.foam.attributes)
    assert np.array_equal(z["adjacency"], case.foam.adjacency)
    assert np.array_equal(z["rays"], case.rays)
    assert np.array_equal(z["grad_rgba"], case.grad_rgba)


BENCH = os.path.join(os.path.dirname(__file__), "golden", "benchmark2k.npz")


@pytest.mark.parametrize("tag", ["f16", "f32"])
@pytest.mark.parametrize("model", ["pinhole", "fisheye"])
def test_oracle_trace_benchmark_reproduces_reference_frames(tag, model):
    """trace_benchmark (in-kernel cast_ray + RGBA8 packing, benchmark.py's FPS path): the CPU
    restatement vs frames the reference's own benchmark<> kernel rendered on a B200
    (tests/golden/make_golden_benchmark.py).  RGBA8 truncates v*255, so an expf-level difference
    may move a channel by one LSB on a few pixels; nothing larger is allowed."""
    z = dict(np.load(BENCH))
    cam = {k: z[f"cam_{model}_{k}"] for k in ("position", "forward", "right", "up")}
    cam.update(fov=float(z[f"cam_{model}_fov"]), width=64, height=48, model=model)
    # the offsets the reference was given (its own prefetch) equal the restatement's
    diff = oracle.prefetch_adjacent_diff(z["points"], z["adjacency"], z["offsets"])
    assert np.array_equal(diff.view(np.uint16), z["adjacent_diff"].view(np.uint16))
    img = oracle.trace_benchmark(z["points"], z["attributes_" + tag], z["adjacency"], z["offsets"], diff, cam,
                                 int(z[f"start_{model}"][0]), weight_threshold=0.05)
    a = img.view(np.uint8).reshape(48, 64, 4).astype(np.int32)
    b = z[f"image_{tag}_{model}"].view(np.uint8).reshape(48, 64, 4).astype(np.int32)
    assert (b[..., :3].sum(axis=-1) > 0).mean() > 0.2      # the golden frame is not empty
    assert np.abs(a - b).max() <= 1
    assert (a != b).any(axis=-1).mean() < 5e-3
