"""Inputs of the trace_visualization checks: scenes, cameras, test-made colour tables and the case list the
reference's frames were stored for (tests/golden/make_golden_visualization.py -> tests/golden/reference/
visualization.npz).  Everything is regenerated from seeds; the colour tables are made here, not taken from any
viewer (the library ships no colour-map data)."""
from __future__ import annotations

import functools

import numpy as np

from radfoam_b200 import foam

W, H = 64, 48
MODES = ("rgb", "depth", "alpha", "intersections")
MAPS = ("gray", "viridis", "inferno", "turbo")


def _ramp(n: int, phase: float) -> np.ndarray:
    x = np.linspace(0.0, 1.0, n, dtype=np.float64)[:, None]
    return np.clip(np.concatenate([x, (1 - x) * 0.5 + 0.25 * np.sin(6 * x + phase) + 0.25, x[::-1]], axis=1),
                   0, 1).astype(np.float32)


def _random(n: int, seed: int) -> np.ndarray:
    # values a little outside [0, 1] so the saturating pack is exercised
    return np.random.default_rng(seed).uniform(-0.25, 1.25, size=(n, 3)).astype(np.float32)


def tables(kind: str) -> list:
    """Four float32 [L_k, 3] tables, indexed by colour map (gray, viridis, inferno, turbo)."""
    if kind == "ramp":
        return [_ramp(256, k) for k in range(4)]
    if kind == "random":
        return [_random(256, 10 + k) for k in range(4)]
    if kind == "mixed":  # lengths 1, 2, 7 and 256, random and ramp values
        return [_random(1, 20), _ramp(2, 1.0), _random(7, 21), _ramp(256, 2.0)]
    raise KeyError(kind)


@functools.lru_cache(maxsize=None)
def scene(name: str) -> foam.Foam:
    if name == "c1":  # BASELINE config 1's foam
        return foam.small_foam(256, sh_degree=3, seed=0)
    if name == "s20k":  # the 20k shell scene of test_gpu_parity.test_trace_benchmark
        return foam.scene_foam(20000)
    if name == "s20k_zero":  # the same with every third cell's density set to zero
        f = scene("s20k")
        attrs = f.attributes.copy()
        attrs[::3, -1] = 0.0
        return foam.Foam(f.points, attrs, f.adjacency, f.offsets, f.sh_degree)
    raise KeyError(name)


def camera(scene_name: str, model: str, width: int = W, height: int = H) -> dict:
    if model == "exact":
        # forward has an x component of 1e-25: the pixel column with u = 0 gets a direction component far below
        # 2^-60, which the ranked face scan is not proven for, so the exact-scan twin re-renders the frame
        return {"position": np.array([0.0, 0.0, 3.0], np.float32),
                "forward": np.array([1e-25, 0.0, -1.0], np.float32),
                "right": np.array([1.0, 0.0, 0.0], np.float32), "up": np.array([0.0, 1.0, 0.0], np.float32),
                "fov": 0.9, "width": width, "height": height, "model": "pinhole"}
    fov = 0.9 if model == "pinhole" else 1.2
    if scene_name == "c1":
        return foam.camera_dict((0.0, 0.0, -3.0), up=(0.0, 1.0, 0.0), fov=fov, width=width, height=height,
                                model=model)
    return foam.camera_dict((2.5, 2.5, 2.5), fov=fov, width=width, height=height, model=model)


def start_index(scene_name: str, cam: dict) -> int:
    return foam.nearest_point(scene(scene_name).points, cam["position"])


DEFAULTS = dict(color_map="turbo", tables="ramp", bg_color=(1.0, 1.0, 1.0), checker_bg=False, max_depth=6.0,
                depth_quantile=0.5, weight_threshold=0.001, max_intersections=1024)


def _case(name, scene_name, dtype, model, mode, **kw):
    c = dict(DEFAULTS)
    c.update(kw)
    c.update(name=name, scene=scene_name, dtype=dtype, model=model, mode=mode)
    return c


def cases() -> list:
    out = []
    # every mode x camera model x attribute dtype, on both scenes
    for sc in ("c1", "s20k"):
        for dt in ("float32", "float16"):
            for model in ("pinhole", "fisheye"):
                for mode in MODES:
                    kw = {}
                    if mode == "intersections":
                        kw = dict(color_map="inferno", tables="random", max_intersections=200)
                    if mode == "rgb" and model == "fisheye":
                        kw = dict(checker_bg=True)
                    out.append(_case(f"{sc}_{dt}_{model}_{mode}", sc, dt, model, mode, **kw))
    # colour tables of 1, 2, 7 and 256 entries (one per colour map), random and ramp values
    for k, cmap in enumerate(MAPS):
        for mode in ("depth", "intersections"):
            out.append(_case(f"mixed_{cmap}_{mode}", "s20k", "float32", "pinhole", mode, color_map=cmap,
                             tables="mixed", max_intersections=150))
        out.append(_case(f"random_{cmap}_depth", "c1", "float32", "fisheye", "depth", color_map=cmap,
                         tables="random", max_depth=4.5))
    # backgrounds
    out.append(_case("bg_colour", "s20k", "float32", "pinhole", "rgb", bg_color=(0.2, 0.6, 0.9)))
    out.append(_case("bg_checker_black", "c1", "float16", "pinhole", "rgb", checker_bg=True, bg_color=(0, 0, 0)))
    out.append(_case("bg_black", "s20k", "float16", "fisheye", "rgb", bg_color=(0.0, 0.0, 0.0)))
    # edge cases
    out.append(_case("quantile_never_reached", "s20k", "float32", "pinhole", "depth", depth_quantile=1e-30))
    out.append(_case("max_depth_tiny", "s20k", "float32", "pinhole", "depth", max_depth=1e-3))
    out.append(_case("max_depth_saturates_int", "s20k", "float32", "fisheye", "depth", max_depth=1e-9,
                     tables="mixed", color_map="turbo"))
    out.append(_case("max_depth_saturates_int_short", "s20k", "float32", "pinhole", "depth", max_depth=1e-9,
                     tables="mixed", color_map="inferno"))
    out.append(_case("zero_density_depth", "s20k_zero", "float32", "pinhole", "depth"))
    out.append(_case("zero_density_quantile_above_one", "s20k_zero", "float32", "fisheye", "depth",
                     depth_quantile=1.5, tables="random"))
    out.append(_case("zero_density_quantile_one", "s20k_zero", "float16", "pinhole", "depth", depth_quantile=1.0,
                     tables="mixed", color_map="inferno"))
    out.append(_case("zero_density_rgb", "s20k_zero", "float32", "fisheye", "rgb"))
    out.append(_case("steps_exhausted", "s20k", "float32", "pinhole", "intersections", max_intersections=3))
    out.append(_case("steps_exhausted_alpha", "s20k", "float32", "pinhole", "alpha", max_intersections=3))
    out.append(_case("no_threshold_rgb", "s20k", "float32", "pinhole", "rgb", weight_threshold=0.0))
    out.append(_case("no_threshold_intersections", "c1", "float32", "fisheye", "intersections",
                     weight_threshold=0.0, max_intersections=64))
    for mode in MODES:
        out.append(_case(f"exact_scan_{mode}", "s20k", "float32", "exact", mode, max_intersections=300))
    return out


def case_camera(c: dict) -> dict:
    return camera(c["scene"], c["model"])


def case_attributes(c: dict) -> np.ndarray:
    return scene(c["scene"]).attributes.astype(np.float16 if c["dtype"] == "float16" else np.float32)


def vis_kwargs(c: dict) -> dict:
    """Keyword arguments of Pipeline.trace_visualization (minus cmap_table)."""
    return dict(mode=c["mode"], color_map=c["color_map"], bg_color=tuple(float(v) for v in c["bg_color"]),
                checker_bg=bool(c["checker_bg"]), max_depth=float(c["max_depth"]),
                depth_quantile=float(c["depth_quantile"]), weight_threshold=float(c["weight_threshold"]),
                max_intersections=int(c["max_intersections"]))


# config 4 at full size: 1,048,576 points, 1920x1080 pinhole from (2.5, 2.5, 2.5), every mode
FULL_W, FULL_H = 1920, 1080
FULL_ROWS = np.linspace(0, FULL_H - 1, 12).astype(np.int64)
FULL_CASES = [dict(DEFAULTS, name=f"config4_{mode}", mode=mode, dtype="float32",
                   **({"max_intersections": 400, "color_map": "inferno"} if mode == "intersections" else {}))
              for mode in MODES]


def config4_camera() -> dict:
    return foam.camera_dict((2.5, 2.5, 2.5), fov=0.9, width=FULL_W, height=FULL_H, model="pinhole")
