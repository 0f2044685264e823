"""Scene container and the ``.pt`` checkpoint format of the reference (SURVEY.md §8f.3) -- the data formats on
either side of the tracing path, so that a trained radfoam checkpoint can be fed to this library unchanged.

Mirrors, with the same tensor names, shapes and dtypes:
  * ``RadFoamScene.save_pt / load_pt``          radfoam_model/scene.py:614-656
        {"xyz" f32[N,3], "density" f32[N,1] (pre-activation), "color_dc" f32[N,3], "color_sh" f32[N,3((1+deg)^2-1)],
         "adjacency" int64[E], "adjacency_offsets" int64[N+1]}
  * ``get_primal_density / get_primal_attributes / get_trace_data``   scene.py:202-217
        density = activation_scale * softplus(raw, beta=10);  attributes = cat(color_dc, color_sh, density).to(attr_dtype)
  * the camera dictionaries and the FPS loop of benchmark.py:57-139.
Pure torch plumbing (runs on CPU tensors too); the kernels are reached through ``radfoam_b200.Pipeline``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

PT_KEYS = ("xyz", "density", "color_dc", "color_sh", "adjacency", "adjacency_offsets")


def sh_coefficient_count(sh_degree: int) -> int:
    """Columns of ``color_sh`` (scene.py:636): everything but the DC term, three channels."""
    return 3 * ((1 + sh_degree) * (1 + sh_degree) - 1)


class FoamScene:
    """The tensors of a radiance foam and the views the tracer consumes (no optimiser, no triangulation)."""

    def __init__(self, xyz, density, color_dc, color_sh, adjacency, adjacency_offsets, sh_degree=3,
                 attr_dtype=torch.float32, activation_scale=1.0):
        got = color_sh.shape[-1]
        exp = sh_coefficient_count(sh_degree)
        assert exp == got, f"Expected {exp} SH coeffs per-point, got {got}"  # scene.py:637-640
        n = xyz.shape[0]
        if density.shape != (n, 1) or color_dc.shape != (n, 3) or color_sh.shape[0] != n:
            raise RuntimeError("density [N,1], color_dc [N,3] and color_sh [N,*] must match xyz [N,3]")
        if adjacency_offsets.numel() != n + 1:
            raise RuntimeError("adjacency_offsets must have num_points + 1 elements")
        self.sh_degree = sh_degree
        self.attr_dtype = attr_dtype
        self.activation_scale = activation_scale
        self.primal_points = xyz
        self.density = density
        self.att_dc = color_dc.to(attr_dtype)
        self.att_sh = color_sh.to(attr_dtype)
        self.point_adjacency = adjacency if adjacency.dtype == torch.uint32 else _to_uint32(adjacency)
        self.point_adjacency_offsets = (adjacency_offsets if adjacency_offsets.dtype == torch.uint32
                                        else _to_uint32(adjacency_offsets))

    # ------------------------------------------------------------------ scene.py:202-217
    def get_primal_density(self):
        return self.activation_scale * F.softplus(self.density, beta=10)

    def get_primal_attributes(self):
        return torch.cat([self.att_dc, self.att_sh], dim=-1)

    def get_trace_data(self):
        attributes = torch.cat([self.get_primal_attributes(), self.get_primal_density()], dim=-1).to(self.attr_dtype)
        return self.primal_points, attributes, self.point_adjacency, self.point_adjacency_offsets

    # ------------------------------------------------------------------ scene.py:236-261
    def forward(self, pipeline, rays, start_point=None, depth_quantiles=None, return_contribution=False, fused=True):
        """``RadFoamScene.forward``: ``(rgba, depth, contribution, num_intersections, errbox)``.  ``fused`` (fp32
        parameters only) hands the parameters to the kernels instead of building the attribute matrix with torch
        ops -- same values, same gradients, 3-5 fewer passes over ``[N, 49]`` per step."""
        from . import pipeline as _p
        from .render import TraceRays, TraceRaysParams

        points = self.primal_points
        if start_point is None:
            start_point = _p.starting_points(rays, points)
        else:
            start_point = torch.broadcast_to(start_point, rays.shape[:-1])
        if fused and self.att_dc.dtype == torch.float32 and self.density.dtype == torch.float32:
            return TraceRaysParams.apply(pipeline, points, self.att_dc, self.att_sh, self.density,
                                         self.activation_scale, self.point_adjacency, self.point_adjacency_offsets,
                                         rays, start_point, depth_quantiles, return_contribution)
        points, attributes, adjacency, offsets = self.get_trace_data()
        return TraceRays.apply(pipeline, points, attributes, adjacency, offsets, rays, start_point, depth_quantiles,
                               return_contribution)

    # ------------------------------------------------------------------ scene.py:497-548
    def collect_error_map(self, pipeline, rays, rgbs, white_bkg=True, downsample=2, generator=None, fused=True):
        """The densification pass's error map (``RadFoamScene.collect_error_map``): for every view ``rays[v]``
        (``[V, H, W, 6]``, targets ``rgbs[V, H, W, 3]``) a randomly offset ``downsample``-strided sub-image is rendered
        with the contribution output, the L1 colour loss is back-propagated, and per point the gradient norm of its
        position is accumulated and the contribution maximised.  Returns ``(point_error [N,1], point_contribution [N,1])``.
        The scene's tensors must require grad; their ``.grad`` is cleared per view like ``zero_grad(set_to_none=True)``."""
        from . import pipeline as _p

        points = self.primal_points
        start_points = _p.starting_points(rays[:, 0, 0].to(points.device), points)
        point_error = torch.zeros_like(points[..., 0:1]).detach()
        point_contribution = torch.zeros_like(points[..., 0:1]).detach()
        params = [points, self.att_dc, self.att_sh, self.density]
        for v in range(rays.shape[0]):
            d = torch.randint(0, downsample, (2,), generator=generator)
            ray_batch = rays[v:v + 1, int(d[0])::downsample, int(d[1])::downsample, :].to(points.device)
            rgb_batch = rgbs[v:v + 1, int(d[0])::downsample, int(d[1])::downsample, :].to(points.device)
            rgba, _, contribution, _, _ = self.forward(pipeline, ray_batch, start_points[v], return_contribution=True,
                                                       fused=fused)
            opacity = rgba[..., -1:]
            rgb = rgba[..., :3] + (1 - opacity) if white_bkg else rgba[..., :3]
            (rgb_batch - rgb).abs().mean(dim=-1).sum().backward()
            point_error += points.grad.norm(dim=-1, keepdim=True).detach()
            point_contribution = torch.maximum(point_contribution, contribution.detach().to(point_contribution.dtype))
            for t in params:
                t.grad = None
        return point_error, point_contribution

    @property
    def num_points(self) -> int:
        return int(self.primal_points.shape[0])

    # ------------------------------------------------------------------ scene.py:614-656
    def save_pt(self, pt_path) -> None:
        torch.save({
            "xyz": self.primal_points.detach().float().cpu(),
            "density": self.density.detach().float().cpu(),
            "color_dc": self.att_dc.detach().float().cpu(),
            "color_sh": self.att_sh.detach().float().cpu(),
            "adjacency": self.point_adjacency.cpu().long(),
            "adjacency_offsets": self.point_adjacency_offsets.cpu().long(),
        }, pt_path)

    @classmethod
    def load_pt(cls, pt_path, sh_degree=3, attr_dtype=torch.float32, device="cuda", activation_scale=1.0):
        scene_data = torch.load(pt_path, map_location="cpu")
        missing = [k for k in PT_KEYS if k not in scene_data]
        if missing:
            raise KeyError(f"{pt_path}: not a radfoam scene checkpoint, missing {missing}")
        return cls(scene_data["xyz"].to(device), scene_data["density"].to(device),
                   scene_data["color_dc"].to(device), scene_data["color_sh"].to(device),
                   scene_data["adjacency"].to(device), scene_data["adjacency_offsets"].to(device),
                   sh_degree=sh_degree, attr_dtype=attr_dtype, activation_scale=activation_scale)

    @classmethod
    def from_foam(cls, foam, raw_density=None, attr_dtype=torch.float32, device="cuda", activation_scale=1.0):
        """From a synthetic ``radfoam_b200.foam.Foam`` (its last attribute column is the ACTIVATED density; the
        checkpoint stores the pre-activation value, so invert softplus_beta10 unless ``raw_density`` is given)."""
        a = torch.from_numpy(foam.attributes).to(torch.float32)
        if raw_density is None:
            sigma = (a[:, -1:] / activation_scale).clamp_min(1e-30).double()
            raw_density = torch.where(10.0 * sigma > 20.0, sigma, torch.log(torch.expm1(10.0 * sigma)) / 10.0).float()
        return cls(torch.from_numpy(foam.points).to(device), raw_density.to(device), a[:, :3].to(device),
                   a[:, 3:-1].to(device), torch.from_numpy(foam.adjacency).to(device),
                   torch.from_numpy(foam.offsets).to(device), sh_degree=foam.sh_degree, attr_dtype=attr_dtype,
                   activation_scale=activation_scale)


def save_surface_ply(path, surface) -> None:
    """Write a ``Pipeline.extract_surface`` result as a binary little-endian PLY mesh: one vertex element (``x y z``
    float, ``red green blue`` uchar: each vertex takes its polygon's colour, clamped to [0, 1] and truncated from
    ``x 255`` in float32 as the tracer's RGBA8 packing does) and one face element (``vertex_indices``: a uchar count
    and int indices).  Polygons are written as they are -- shared vertices are not welded.  The mesh counterpart of
    the reference's point-cloud ``save_ply`` (radfoam_model/scene.py:550-612)."""
    import numpy as np

    def host(t):
        return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)

    vertices = np.ascontiguousarray(host(surface["vertices"]), dtype=np.float32).reshape(-1, 3)
    offsets = host(surface["offsets"]).astype(np.int64).reshape(-1)
    rgb = host(surface["rgb"]).astype(np.float32).reshape(-1, 3)
    nv, npoly = vertices.shape[0], offsets.shape[0] - 1
    counts = np.diff(offsets)
    if npoly < 0 or rgb.shape[0] != npoly or offsets[0] != 0 or offsets[-1] != nv or (counts < 3).any() \
            or (counts > 255).any() or nv >= 2 ** 31:
        raise ValueError("not a surface: offsets[P+1] must partition the vertices into polygons of 3..255 vertices, "
                         "with one rgb row per polygon")
    # fmax(0, fmin(1, c)) maps NaN to 1, like fmaxf(0, fminf(1, c)) in the kernels
    colour = (np.fmax(np.float32(0), np.fmin(np.float32(1), rgb)) * np.float32(255)).astype(np.uint8)
    vrec = np.empty(nv, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"),
                               ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    vrec["x"], vrec["y"], vrec["z"] = vertices[:, 0], vertices[:, 1], vertices[:, 2]
    per_vertex = np.repeat(colour, counts, axis=0)
    vrec["red"], vrec["green"], vrec["blue"] = per_vertex[:, 0], per_vertex[:, 1], per_vertex[:, 2]
    # face k = [count_k][int32 indices offsets[k] .. offsets[k+1]-1]; it starts at byte k + 4 offsets[k]
    faces = np.empty(npoly + 4 * nv, dtype=np.uint8)
    faces[np.arange(npoly) + 4 * offsets[:-1]] = counts.astype(np.uint8)
    at = np.repeat(np.arange(npoly, dtype=np.int64), counts) + 1 + 4 * np.arange(nv, dtype=np.int64)
    faces[at[:, None] + np.arange(4)] = np.arange(nv, dtype="<i4").view(np.uint8).reshape(nv, 4)
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {nv}\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {npoly}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vrec.tobytes())
        f.write(faces.tobytes())


def _to_uint32(t):
    if t.numel() and (int(t.min()) < 0 or int(t.max()) > 0xFFFFFFFF):
        raise RuntimeError("adjacency values do not fit uint32")
    return t.to(torch.int64).to(torch.uint32)


# ---------------------------------------------------------------------- benchmark.py:57-84
def benchmark_cameras(c2w, fy, width, height, every=8):
    """Camera dictionaries for ``Pipeline.trace_benchmark`` from camera-to-world matrices ``[M,4,4]`` (or
    ``[M,3,4]``), one per ``every`` poses: right = +x column, up = -y column, forward = +z column,
    fov = 2 atan(height / (2 fy)).  Returns (cameras, positions[M',3])."""
    cameras, positions = [], []
    fov = float(2 * math.atan(height / (2 * fy)))
    for i in range(c2w.shape[0]):
        if i % every:
            continue
        position = c2w[i, :3, 3].contiguous()
        positions.append(position)
        cameras.append({"position": position, "forward": c2w[i, :3, 2].contiguous(),
                        "right": c2w[i, :3, 0].contiguous(), "up": (-c2w[i, :3, 1]).contiguous(), "fov": fov,
                        "width": width, "height": height, "model": "pinhole"})
    return cameras, torch.stack(positions, dim=0)


def benchmark_fps(pipeline, scene: FoamScene, cameras, positions, n_reps=5, weight_threshold=0.05):
    """The reference's FPS measurement (benchmark.py:86-139): fp16 or fp32 attributes as the scene holds them,
    precomputed half4 neighbour offsets, RGBA8 output, CUDA events around ``n_reps`` passes over the cameras."""
    from . import pipeline as _p

    points, attributes, adjacency, offsets = scene.get_trace_data()
    adjacent_offsets = pipeline.prefetch_adjacent_diff(points, adjacency, offsets)
    start_points = _p.nearest_point(points, positions.to(points.device))
    height, width = cameras[0]["height"], cameras[0]["width"]
    output = torch.zeros((len(cameras), height, width), dtype=torch.uint32, device=points.device)

    def one_pass():
        for i, camera in enumerate(cameras):
            pipeline.trace_benchmark(points, attributes, adjacency, offsets, adjacent_offsets, camera,
                                     start_points[i:i + 1], output[i], weight_threshold=weight_threshold)

    one_pass()  # warm-up, as upstream
    torch.cuda.synchronize()
    start_event, end_event = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start_event.record()
    for _ in range(n_reps):
        one_pass()
    end_event.record()
    torch.cuda.synchronize()
    total_ms = start_event.elapsed_time(end_event)
    return {"fps": n_reps * len(cameras) / (total_ms / 1000.0), "total_ms": total_ms, "frames": len(cameras),
            "output": output}
