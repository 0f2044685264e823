"""Kernel time of trace_visualization at config 4 (1,048,576 points, 1920x1080 pinhole from (2.5, 2.5, 2.5)), fp32 and
fp16 attributes: this library's kernel in every mode, the reference's visualization kernel (oracle/ref_vis.py) in
every mode, and trace_benchmark (ours and the reference's) on the same camera.  Calls are alternated round-robin within
one process after a warm-up; each call's kernel time comes from torch.profiler's device timestamps (our calls are a
fast kernel + its exact-scan twin, which returns at once unless a ray needs the exact scan: both are summed).
Medians over --reps calls.

    python tests/tools/vis_bench.py [--reps 25] [--warmup 3] [--out profiles/h100_visualization.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import vis_cases as V  # noqa: E402

import radfoam_b200  # noqa: E402


# kernel names, mangled or demangled
def OURS_VIS(n): return "visualization_kernel" in n  # noqa: E302,E704
def OURS_BENCH(n): return "benchmark_kernel" in n  # noqa: E302,E704
def REF_VIS(n): return "visualization" in n and "visualization_kernel" not in n  # noqa: E302,E704
def REF_BENCH(n): return "benchmark" in n and "benchmark_kernel" not in n  # noqa: E302,E704


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle import ref_gpu, ref_vis

    have_ref = ref_gpu.available() and ref_vis.available()
    f = bench.load_or_build_foam(1 << 20, print)
    cam = V.config4_camera()
    start = V.foam.nearest_point(f.points, cam["position"])
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    tabs = [d(t) for t in V.tables("ramp")]
    ptrs = d(np.array([t.data_ptr() for t in tabs], dtype=np.int64))
    sizes = d(np.array([t.shape[0] for t in tabs], dtype=np.int32))
    result = {"workload": "config 4: 1,048,576 points, 1920x1080 pinhole, weight_threshold 0.001, "
                          "max_intersections 1024, ramp colour tables (256 entries)",
              "reps": args.reps, "warmup": args.warmup, "unit": "ms (median kernel time per call)", **gpu_info()}
    for dtype in ("float32", "float16"):
        attrs = f.attributes.astype(np.float16 if dtype == "float16" else np.float32)
        scene = [d(f.points), d(attrs), d(f.adjacency), d(f.offsets)]
        pipe = radfoam_b200.create_pipeline(3, dtype)
        diff = pipe.prefetch_adjacent_diff(scene[0], scene[2], scene[3])
        start_t = d(np.array([start], np.uint32))
        frame = torch.zeros((cam["height"], cam["width"]), dtype=torch.uint32, device="cuda")
        calls = []  # (label, kernel-name predicate, number of matching kernels the call launches, fn)
        for mode in V.MODES:
            calls.append((f"ours_{mode}", OURS_VIS, 2,
                          lambda m=mode: pipe.trace_visualization(*scene, diff, cam, start, frame, mode=m,
                                                                  cmap_table=tabs)))
        calls.append(("ours_trace_benchmark", OURS_BENCH, 2,
                      lambda: pipe.trace_benchmark(*scene, diff, cam, start_t, frame)))
        if have_ref:
            for mode in V.MODES:
                calls.append((f"reference_{mode}", REF_VIS, 1,
                              lambda m=mode: ref_vis.trace_visualization(*scene, diff, cam, start, ptrs, sizes, frame,
                                                                         mode=m)))
            calls.append(("reference_trace_benchmark", REF_BENCH, 1,
                          lambda: ref_gpu.trace_benchmark(*scene, diff, cam, start_t, frame)))
        for _ in range(args.warmup):
            for _, _, _, fn in calls:
                fn()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                for _, _, _, fn in calls:
                    fn()
            torch.cuda.synchronize()
        kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                          and ("visualization" in e.name or "benchmark" in e.name)),
                         key=lambda e: e.time_range.start)
        times = {label: [] for label, *_ in calls}
        it = iter(kernels)
        for _ in range(args.reps):
            for label, key, count, _ in calls:
                total = 0.0
                for _ in range(count):
                    e = next(it)
                    assert key(e.name), (label, e.name)
                    total += (e.time_range.end - e.time_range.start) / 1000.0
                times[label].append(total)
        res = {label: round(float(np.median(v)), 4) for label, v in times.items()}
        res.update({label + "_spread": round(float(np.max(v) - np.min(v)), 4) for label, v in times.items()})
        if have_ref:
            for mode in V.MODES:
                res[f"speedup_{mode}"] = round(res[f"reference_{mode}"] / res[f"ours_{mode}"], 3)
            res["speedup_trace_benchmark"] = round(res["reference_trace_benchmark"] / res["ours_trace_benchmark"], 3)
        result[dtype] = res
        print(dtype, json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
