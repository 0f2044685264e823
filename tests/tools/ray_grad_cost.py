"""What requesting ray gradients costs: the backward ray kernel's time on the bench frame (BASELINE config 4:
1,048,576-point foam, 1920x1080, Q = 2, sh degree 3, walk tape on), without and with ``return_ray_grad``.
The two are alternated step by step in one process: 5 warm-up steps each, then 20 timed steps each.  Each step
is a recording forward and a backward; the backward kernel is timed with the pipeline's CUDA events around it
(``last_kernel_ms("backward")``) and the whole ``trace_backward`` call with events on the stream.
Prints one JSON record (GPU name and power limit included) and writes it to --out when given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001 - the record says what could not be read
        return {"gpu_info_error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    import radfoam_b200

    assert torch.cuda.is_available(), "needs a GPU"
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    fr = bench.make_frame(f, 1920, 1080)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    pts, attrs = dev(f.points).requires_grad_(True), dev(f.attributes).requires_grad_(True)
    adj, off = dev(f.adjacency), dev(f.offsets)
    rays, start, dq = dev(fr["rays"]), dev(fr["start"]), dev(fr["dq"])
    g, gd = dev(fr["grad_rgba"]), dev(fr["grad_depth"])
    pipe = radfoam_b200.create_pipeline(3)
    pipe.set_profiling(True)
    times = {False: {"kernel_ms": [], "call_ms": []}, True: {"kernel_ms": [], "call_ms": []}}

    def step(with_rays, record):
        fwd = pipe.trace_forward(pts, attrs, adj, off, rays, start, depth_quantiles=dq)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        pipe.trace_backward(pts, attrs, adj, off, rays, start, fwd["rgba"], g, dq, fwd["depth_indices"], gd,
                            scrub_nonfinite=True, return_ray_grad=with_rays)
        e1.record()
        torch.cuda.synchronize()
        if record:
            times[with_rays]["kernel_ms"].append(pipe.last_kernel_ms("backward"))
            times[with_rays]["call_ms"].append(e0.elapsed_time(e1))

    for _ in range(args.warmup):
        for with_rays in (False, True):
            step(with_rays, False)
    overflowed = pipe.tape_status()["overflowed"]
    for _ in range(args.steps):
        for with_rays in (False, True):
            step(with_rays, True)

    def stats(v):
        return {"median": round(float(np.median(v)), 4), "min": round(float(np.min(v)), 4),
                "max": round(float(np.max(v)), 4)}

    rec = {"what": "backward kernel time at config 4 (1,048,576 points, 1920x1080, Q=2, sh 3, tape on), "
                   "without / with return_ray_grad, alternated step by step",
           "warmup": args.warmup, "steps": args.steps, "tape_overflowed_after_warmup": overflowed,
           **gpu_info(), "torch": torch.__version__,
           "without_ray_grad": {k: stats(v) for k, v in times[False].items()},
           "with_ray_grad": {k: stats(v) for k, v in times[True].items()}}
    k0, k1 = rec["without_ray_grad"]["kernel_ms"]["median"], rec["with_ray_grad"]["kernel_ms"]["median"]
    rec["kernel_ratio_median"] = round(k1 / k0, 4)
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(rec, indent=2) + "\n")


if __name__ == "__main__":
    main()
