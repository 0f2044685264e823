"""Frames of the reference's OWN visualization kernel (oracle/ref_vis.py: Pipeline::trace_visualization on a surface,
copied out) for every case of tests/vis_cases.py, plus SHA-256 digests and sampled rows of config 4's 1920x1080
frames in every mode.  Needs a GPU and oracle/_ref:
    python tests/golden/make_golden_visualization.py [out_dir]      (then copy visualization.npz to
                                                                    tests/golden/reference/)"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import vis_cases as V  # noqa: E402
from oracle import ref_gpu, ref_vis  # noqa: E402


def d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def cmap_arrays(tables):
    keep = [d(t) for t in tables]
    ptrs = d(np.array([t.data_ptr() for t in keep], dtype=np.int64))
    sizes = d(np.array([t.shape[0] for t in keep], dtype=np.int32))
    return keep, ptrs, sizes


def reference_frame(f, attrs, cam, start, c):
    scene = [d(f.points), d(attrs), d(f.adjacency), d(f.offsets)]
    diff = ref_gpu.prefetch_adjacent_diff(scene[0], scene[2], scene[3])
    keep, ptrs, sizes = cmap_arrays(V.tables(c["tables"]))
    out = torch.zeros((cam["height"], cam["width"]), dtype=torch.uint32, device="cuda")
    kw = V.vis_kwargs(c)
    ref_vis.trace_visualization(*scene, diff, cam, start, ptrs, sizes, out, **kw)
    torch.cuda.synchronize()
    del keep
    return out.cpu().numpy()


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "reference")
    os.makedirs(out_dir, exist_ok=True)
    rec = {}
    for c in V.cases():
        f, cam = V.scene(c["scene"]), V.case_camera(c)
        img = reference_frame(f, V.case_attributes(c), cam, V.start_index(c["scene"], cam), c)
        rec[c["name"]] = img
        print(c["name"], "nonzero pixels:", float((img & 0xFFFFFF != 0).mean()), flush=True)
    import bench

    f4 = bench.load_or_build_foam(1 << 20, print)
    cam = V.config4_camera()
    start = V.foam.nearest_point(f4.points, cam["position"])
    for c in V.FULL_CASES:
        img = reference_frame(f4, f4.attributes, cam, start, c)
        rec[c["name"] + "#sha256"] = np.frombuffer(hashlib.sha256(img.tobytes()).digest(), dtype=np.uint8).copy()
        rec[c["name"] + "#rows"] = img[V.FULL_ROWS]
        print(c["name"], "nonzero pixels:", float((img & 0xFFFFFF != 0).mean()), flush=True)
    np.savez_compressed(os.path.join(out_dir, "visualization.npz"), **rec)
    print("written", len(rec), "arrays to", out_dir)


if __name__ == "__main__":
    main()
