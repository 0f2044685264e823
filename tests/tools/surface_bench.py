"""Time surface extraction (rfb_surface_count: count + scan, then rfb_surface_write) on the config-4 foam (1,048,576
points, SH degree 3, fp32), with the threshold selecting the synthetic foam's shell cells (density > 0.5).

CUDA events around the two library calls, warm-up first, median of --reps; also the whole Pipeline.extract_surface
call (its one device-to-host read of the totals included).  Prints one JSON line with polygons, vertices, the card's
name and power limit, and writes it to --out when given.

    python tests/tools/surface_bench.py --reps 15 --out profiles/h100_surface.json
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--threshold", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    import radfoam_b200
    from radfoam_b200 import _lib

    assert torch.cuda.is_available(), "surface_bench needs a GPU"
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    pts, attrs, adj, off = t(f.points), t(f.attributes), t(f.adjacency), t(f.offsets)
    pipe = radfoam_b200.create_pipeline(3)
    inside = (attrs[:, -1] > args.threshold).contiguous()
    surf = pipe.extract_surface(pts, attrs, adj, off, inside=inside)  # output sizes, and a warm-up
    lib = _lib.load()
    box = _lib.Box()
    lo, hi = torch.stack([pts.amin(0), pts.amax(0)]).cpu().tolist()
    box.lo[:], box.hi[:] = lo, hi
    n, e = pts.size(0), adj.numel()
    scratch = torch.empty((int(lib.rfb_surface_scratch_bytes(e)) + 7) // 8, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def count():
        _lib.check(lib.rfb_surface_count(pts.data_ptr(), n, e, adj.data_ptr(), off.data_ptr(), inside.data_ptr(),
                                         ctypes.byref(box), scratch.data_ptr(), stream))

    def write():
        _lib.check(lib.rfb_surface_write(pipe._handle, pts.data_ptr(), n, attrs.data_ptr(), e, adj.data_ptr(),
                                         off.data_ptr(), inside.data_ptr(), ctypes.byref(box), scratch.data_ptr(),
                                         surf["vertices"].data_ptr(), surf["offsets"].data_ptr(),
                                         surf["cells"].data_ptr(), surf["rgb"].data_ptr(), stream))

    def timed(fn, reps):
        ms = []
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))

    c = timed(count, args.reps)
    w = timed(write, args.reps)
    both = timed(lambda: (count(), write()), args.reps)
    whole = timed(lambda: pipe.extract_surface(pts, attrs, adj, off, inside=inside), args.reps)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rec = {"workload": "config 4 (1,048,576 points, SH degree 3, fp32), shell cells: density > %g" % args.threshold,
           "points": n, "csr_entries": e, "occupied_cells": int(inside.sum()),
           "polygons": int(surf["offsets"].numel() - 1), "vertices": int(surf["vertices"].shape[0]),
           "count_and_scan_ms": {"median": c[0], "min": c[1], "max": c[2]},
           "write_ms": {"median": w[0], "min": w[1], "max": w[2]},
           "count_scan_write_ms": {"median": both[0], "min": both[1], "max": both[2]},
           "extract_surface_call_ms": {"median": whole[0], "min": whole[1], "max": whole[2]},
           "reps": args.reps, "device": torch.cuda.get_device_name(0),
           "nvidia_smi_name_power_limit_max_sm_clock": smi[0] if smi else None}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
