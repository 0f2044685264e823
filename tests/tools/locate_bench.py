"""Point location and field sampling on the config-4 foam (1,048,576 points, bench.py's synthetic scene):

* locate_points for 2 M distinct queries of two kinds -- the 1080p bench frame's median-depth points (secondary-ray
  origins; with and without their depth_indices as hints, padded to 2,097,152 with copies nudged by 1e-3) and
  uniform points of the foam's bounding box --, with the mean / max number of walk moves per query (counted by
  the torch restatement in tests/locate_model.py from the same seeds);
* the seed sample size swept (RFB_LOCATE_SAMPLE), to show the trade-off between the sample scan and the walk;
* nearest_point (the tiled brute force) at M = 1,024 and 4,096, for its slope;
* Pipeline.sample_field forward (with directions) and sample_field_backward at 2 M queries, sh degree 3, fp32.

Times are CUDA-event medians over --reps calls after --warmup calls.  Prints one JSON record (GPU name and power
limit included) and writes it to --out when given."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

SWEEP = (256, 1024, 2048, 4096, 8192, 16384)
DEFAULT_SAMPLE = 2048  # kLocateSample in radfoam_b200/csrc/radfoam_b200.cu
STATS_SUBSAMPLE = 1 << 18


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import bench
    import locate_model as lm
    import radfoam_b200
    from ray_grad_cost import gpu_info

    assert torch.cuda.is_available(), "needs a GPU"
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    fr = bench.make_frame(f, 1920, 1080)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    pts, attrs, adj, off = dev(f.points), dev(f.attributes), dev(f.adjacency), dev(f.offsets)
    adj64, off64 = lm.as_long(adj), lm.as_long(off)
    rays, start = dev(fr["rays"]), dev(fr["start"])
    pipe = radfoam_b200.create_pipeline(3)
    out = pipe.trace_forward(pts, attrs, adj, off, rays, start,
                             depth_quantiles=torch.full((1080, 1920, 1), 0.5, device="cuda"))
    depth, idx = out["depth"][..., 0], lm.as_long(out["depth_indices"][..., 0])
    hit = torch.isfinite(depth) & (idx != lm.NONE)
    sec = (rays[..., :3] + depth[..., None] * rays[..., 3:])[hit]
    sec_hint = idx[hit]
    m = 1 << 21
    g = torch.Generator(device="cuda").manual_seed(0)
    pick = torch.randint(0, sec.shape[0], (m - sec.shape[0],), device="cuda", generator=g)
    sec = torch.cat([sec, sec[pick] + 1e-3 * torch.randn((pick.numel(), 3), device="cuda", generator=g)]).contiguous()
    sec_hint = torch.cat([sec_hint, sec_hint[pick]]).to(torch.uint32)
    lo, hi = pts.min(0).values, pts.max(0).values
    box = (lo + (hi - lo) * torch.rand((m, 3), device="cuda", generator=g)).contiguous()
    dirs = torch.randn((m, 3), device="cuda", generator=g)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return {"median_ms": round(float(np.median(ts)), 4), "min_ms": round(float(np.min(ts)), 4),
                "max_ms": round(float(np.max(ts)), 4)}

    def moves(q, seeds, cells):
        cells_model, mv = lm.walk(pts, adj64, off64, q, seeds)
        assert torch.equal(cells_model, lm.as_long(cells)), "the model's walk ends where the kernel's does"
        mv = mv.double()
        return {"mean_moves": round(float(mv.mean()), 3), "max_moves": int(mv.max()), "over_queries": q.shape[0]}

    rec = {"what": "locate_points / sample_field on the config-4 foam (1,048,576 points), 2,097,152 queries",
           "warmup": args.warmup, "reps": args.reps, **gpu_info(), "torch": torch.__version__,
           "default_sample": DEFAULT_SAMPLE, "locate": {}, "sample_sweep": {}, "nearest_point": {}}

    def locate(q, h, sample):
        if sample is None:
            os.environ.pop("RFB_LOCATE_SAMPLE", None)
        else:
            os.environ["RFB_LOCATE_SAMPLE"] = str(sample)
        cells = radfoam_b200.locate_points(pts, adj, off, q, hint=h)
        r = timed(lambda: radfoam_b200.locate_points(pts, adj, off, q, hint=h))
        r["Mqueries_per_s"] = round(q.shape[0] / r["median_ms"] / 1e3, 1)
        return cells, r

    # the shipped configuration (no override), walk statistics over all queries
    for name, q, h in (("secondary_origins_hinted", sec, sec_hint), ("secondary_origins", sec, None),
                       ("uniform_box", box, None)):
        cells, r = locate(q, h, None)
        seeds = lm.as_long(h) if h is not None else lm.sample_seeds(pts, q, DEFAULT_SAMPLE)
        r.update(moves(q, seeds, cells))
        rec["locate"][name] = r
    # seed sample sweep, walk statistics over a subsample
    sub = torch.randperm(m, device="cuda", generator=g)[:STATS_SUBSAMPLE]
    for sample in SWEEP:
        for name, q in (("secondary_origins", sec), ("uniform_box", box)):
            cells, r = locate(q, None, sample)
            r.update(moves(q[sub], lm.sample_seeds(pts, q[sub], sample), lm.as_long(cells)[sub]))
            rec["sample_sweep"][f"{name}_S{sample}"] = r
    os.environ.pop("RFB_LOCATE_SAMPLE", None)
    # the brute force's slope
    for mq in (1024, 4096):
        q = sec[:mq].contiguous()
        r = timed(lambda: radfoam_b200.nearest_point(pts, q))
        r["us_per_query"] = round(1e3 * r["median_ms"] / mq, 3)
        rec["nearest_point"][f"M{mq}"] = r
    # field sampling, degree 3 fp32, secondary origins with hints and random directions
    s = pipe.sample_field(pts, attrs, adj, off, sec, dirs, hint=sec_hint)
    rec["sample_field_forward"] = timed(lambda: pipe.sample_field(pts, attrs, adj, off, sec, dirs, hint=sec_hint))
    gr, gd = torch.randn_like(s["rgb"]), torch.randn_like(s["density"])
    rec["sample_field_backward"] = timed(
        lambda: pipe.sample_field_backward(f.num_points, s["cell"], dirs, s["rgb"], gr, gd))
    cells = lm.as_long(s["cell"])
    rec["sample_field_backward"]["distinct_cells"] = int(torch.unique(cells).numel())
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(json.dumps(rec, indent=2) + "\n")


if __name__ == "__main__":
    main()
