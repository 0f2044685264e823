"""Time radfoam_b200.delaunay_adjacency on the H100 and compare its graph with Qhull's at 1 M points.

Foams: scene_foam(1048576) (config 4's foam), 1 M uniform points in [-1, 1]^3 and scene_foam(4194304).  Per foam:
the whole call with CUDA events (warm-up, then the median of --reps), the per-phase kernel times from one
torch.profiler run (order = the Morton sort in torch, tree, clip, overflow, assembly), the cells the overflow
kernel finished, the degree histogram, and the entries a box 1000x larger than the default adds (edges the default
box drops).  For config 4's foam also Qhull's single-core time in the same run and every entry that differs from
Qhull's graph with its model area (the Qhull entries the default box drops).  Prints and writes one JSON document
(--out, rewritten after every foam) with the card's name and power limit.

    python tests/tools/delaunay_bench.py --reps 10 --out profiles/h100_delaunay.json
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PHASES = {"order": ("radix", "sort", "elementwise", "reduce", "index", "arange", "Morton"),
          "tree": ("delaunay_gather", "delaunay_leaf", "delaunay_level"),
          "clip": ("delaunay_clip",), "overflow": ("delaunay_overflow",),
          "assembly": ("delaunay_extra", "delaunay_count", "scan_", "delaunay_fill", "delaunay_sort")}


def scene_points(n):
    """scene_foam(n)'s points without its Qhull adjacency (the generator triangulates unconditionally)."""
    import numpy as np

    from radfoam_b200 import foam
    real = foam.delaunay_adjacency
    foam.delaunay_adjacency = lambda p: (np.zeros(0, np.uint32), np.zeros(p.shape[0] + 1, np.uint32))
    try:
        return foam.scene_foam(n).points
    finally:
        foam.delaunay_adjacency = real


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="1048576,4194304")
    ap.add_argument("--no-qhull", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch

    import radfoam_b200
    from radfoam_b200 import _lib, delaunay, foam

    assert torch.cuda.is_available(), "delaunay_bench needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else None, "reps": args.reps,
              "foams": {}}
    sizes = [int(s) for s in args.sizes.split(",")]
    cases = [(f"scene_{n}", lambda n=n: scene_points(n)) for n in sizes]
    cases.insert(1, ("uniform_1048576", lambda: np.random.default_rng(0).uniform(-1, 1, (1 << 20, 3)).astype(np.float32)))
    lib = _lib.load()
    for name, make in cases:
        pts_np = make()
        pts = torch.from_numpy(pts_np).cuda()
        t0 = time.time()
        adj, off = radfoam_b200.delaunay_adjacency(pts)  # warm-up
        torch.cuda.synchronize()
        print(name, f"warm-up call {time.time() - t0:.3f} s", flush=True)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            radfoam_b200.delaunay_adjacency(pts)
            torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            radfoam_b200.delaunay_adjacency(pts)
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        phases = {k: 0.0 for k in PHASES}
        for ev in prof.key_averages():
            t = ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
            if t > 0:
                print(f"  {ev.key[:70]:70s} {t:10.3f} ms", flush=True)
            for k, keys in PHASES.items():
                if any(s in ev.key for s in keys):
                    phases[k] += t
                    break
        # totals of one build: overflow cells, one-sided entries
        n = pts.size(0)
        order = delaunay.morton_order(pts).to(torch.int32).view(torch.uint32)
        p = pts_np.astype(np.float32)
        lo, hi = delaunay.default_bounds(p.min(0), p.max(0))
        box = _lib.Box()
        box.lo[:], box.hi[:] = lo.tolist(), hi.tolist()
        pool = max(32 * n + 4096, int(adj.numel()) + 4096)
        scratch = torch.empty((int(lib.rfb_delaunay_scratch_bytes(n, pool)) + 7) // 8, dtype=torch.int64,
                              device="cuda")
        _lib.check(lib.rfb_delaunay_count(pts.data_ptr(), n, order.data_ptr(), ctypes.byref(box), pool,
                                          scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
        totals = scratch[:8].cpu().tolist()
        deg = np.diff(off.cpu().numpy().astype(np.int64))
        hist = np.bincount(deg)
        entry = {"num_points": n, "edges_directed": int(adj.numel()), "ms_median": float(np.median(ms)),
                 "ms_all": [round(x, 3) for x in ms], "phase_ms_profiler": {k: round(v, 3) for k, v in phases.items()},
                 "overflow_cells": int(totals[3]), "one_sided_entries": int(totals[0]),
                 "degree_min": int(deg.min()), "degree_max": int(deg.max()), "degree_mean": float(deg.mean()),
                 "degree_histogram": {int(d): int(c) for d, c in enumerate(hist) if c}}
        # the edges the default box drops, against a box 1000x larger on every side
        big = (lo - 1000.0 * (hi - lo), hi + 1000.0 * (hi - lo))
        t0 = time.time()
        badj, boff = radfoam_b200.delaunay_adjacency(pts, big)
        torch.cuda.synchronize()
        entry["large_box_call_s"] = time.time() - t0
        import delaunay_model as dm
        dcode, bcode = dm.codes(adj.cpu().numpy(), off.cpu().numpy()), dm.codes(badj.cpu().numpy(), boff.cpu().numpy())
        entry["large_box_adds_entries"] = int(np.setdiff1d(bcode, dcode, assume_unique=True).size)
        entry["large_box_drops_entries"] = int(np.setdiff1d(dcode, bcode, assume_unique=True).size)
        del badj, boff
        if name == "scene_1048576" and not args.no_qhull:
            t0 = time.time()
            qa, qo = foam.delaunay_adjacency(pts_np)
            entry["qhull_s"] = time.time() - t0
            diffs = dm.judge(pts_np, adj.cpu().numpy(), off.cpu().numpy(), qa, qo, lo.astype(np.float64),
                             hi.astype(np.float64))
            entry["qhull_entries"] = int(qa.size)
            entry["differ_from_qhull"] = len(diffs)
            entry["differ_in_qhull_only"] = sum(1 for d in diffs if d[3])
            entry["differ_max_area_rel"] = max([d[2] for d in diffs] or [0.0])
            entry["differ_over_tau"] = sum(1 for d in diffs if d[2] > dm.TAU)
            entry["differences"] = [[int(d[0]), int(d[1]), float(d[2]), bool(d[3])] for d in diffs[:200]]
        result["foams"][name] = entry
        if args.out:  # after every foam, so that a run cut short keeps what it measured
            with open(args.out, "w") as fh:
                json.dump(result, fh, indent=1)
        print(name, json.dumps({k: v for k, v in entry.items() if k not in ("differences", "degree_histogram")}),
              flush=True)
        del pts, adj, off, scratch
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
