"""Pipeline.trace_visualization / rfb_trace_visualization{,_rgba8} on the GPU: every frame byte-identical to the one the
reference's own visualization kernel rendered for the same inputs (tests/golden/reference/visualization.npz, made by
tests/golden/make_golden_visualization.py), through the linear-buffer entry point and through a real CUDA surface,
plus cross-checks that need no reference: the RGB frame over black equals trace_benchmark's frame with its rows
reversed, and a redraw of an unchanged scene equals a fresh pipeline's frame."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

import vis_cases as V

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "visualization.npz")


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def to_dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def scene_tensors(torch, f, attrs):
    return [to_dev(torch, x) for x in (f.points, attrs, f.adjacency, f.offsets)]


def cmap_tensors(torch, kind):
    return [to_dev(torch, t) for t in V.tables(kind)]


def render(torch, pipe, f, attrs, cam, start, c, scene=None):
    import radfoam_b200  # noqa: F401

    scene = scene or scene_tensors(torch, f, attrs)
    diff = pipe.prefetch_adjacent_diff(scene[0], scene[2], scene[3])
    frame = pipe.trace_visualization(*scene, diff, cam, start, cmap_table=cmap_tensors(torch, c["tables"]),
                                     **V.vis_kwargs(c))
    torch.cuda.synchronize()
    return frame.cpu().numpy()


# ---------------------------------------------------------------- the CUDA runtime's surface API, through ctypes
class _Cudart:
    def __init__(self):
        import torch  # noqa: F401  (its CUDA runtime is the one loaded below)

        path = None
        try:
            import nvidia.cuda_runtime as m

            cand = os.path.join(list(m.__path__)[0], "lib", "libcudart.so.12")
            path = cand if os.path.exists(cand) else None
        except ImportError:
            pass
        self.lib = ctypes.CDLL(path or "libcudart.so.12")
        P = ctypes.c_void_p
        self.lib.cudaMallocArray.argtypes = [ctypes.POINTER(P), P, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint]
        self.lib.cudaCreateSurfaceObject.argtypes = [ctypes.POINTER(ctypes.c_uint64), P]
        self.lib.cudaDestroySurfaceObject.argtypes = [ctypes.c_uint64]
        self.lib.cudaFreeArray.argtypes = [P]
        self.lib.cudaMemcpy2DFromArray.argtypes = [P, ctypes.c_size_t, P, ctypes.c_size_t, ctypes.c_size_t,
                                                   ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int]

    def check(self, rc):
        assert rc == 0, f"CUDA runtime error {rc}"

    def surface(self, width, height):
        """(array, surface object) of width x height RGBA8 texels (cudaArraySurfaceLoadStore)."""
        fmt = (ctypes.c_int * 5)(8, 8, 8, 8, 1)  # cudaChannelFormatDesc, cudaChannelFormatKindUnsigned
        arr = ctypes.c_void_p()
        self.check(self.lib.cudaMallocArray(ctypes.byref(arr), ctypes.cast(fmt, ctypes.c_void_p), width, height, 2))
        res = (ctypes.c_uint64 * 32)()  # cudaResourceDesc: resType = cudaResourceTypeArray (0), res.array.array
        res[1] = arr.value
        surf = ctypes.c_uint64()
        self.check(self.lib.cudaCreateSurfaceObject(ctypes.byref(surf), ctypes.cast(res, ctypes.c_void_p)))
        return arr, surf.value

    def read_and_free(self, torch, arr, surf, width, height):
        out = torch.empty((height, width), dtype=torch.uint32, device="cuda")
        torch.cuda.synchronize()
        self.check(self.lib.cudaMemcpy2DFromArray(ctypes.c_void_p(out.data_ptr()), 4 * width, arr, 0, 0, 4 * width,
                                                  height, 3))  # cudaMemcpyDeviceToDevice
        self.check(self.lib.cudaDestroySurfaceObject(surf))
        self.check(self.lib.cudaFreeArray(arr))
        return out.cpu().numpy()


@pytest.fixture(scope="module")
def cudart(torch_cuda):
    return _Cudart()


def render_surface(torch, cudart, f, attrs, cam, start, c):
    """The same frame through rfb_trace_visualization into a CUDA surface, then copied out."""
    from radfoam_b200 import _lib

    lib = _lib.load()
    handle = ctypes.c_void_p()
    _lib.check(lib.rfb_create_pipeline(f.sh_degree, 1 if attrs.dtype == np.float16 else 0, ctypes.byref(handle)))
    try:
        scene = scene_tensors(torch, f, attrs)
        diff = torch.zeros((f.adjacency.size, 4), dtype=torch.float16, device="cuda")
        _lib.check(lib.rfb_prefetch_adjacent_diff(scene[0].data_ptr(), f.points.shape[0], f.adjacency.size,
                                                  scene[2].data_ptr(), scene[3].data_ptr(), diff.data_ptr(), None))
        tabs = cmap_tensors(torch, c["tables"])
        ptrs = to_dev(torch, np.array([t.data_ptr() for t in tabs], dtype=np.int64))
        sizes = to_dev(torch, np.array([t.shape[0] for t in tabs], dtype=np.int32))
        cm = _lib.CMapTable(ptrs.data_ptr(), sizes.data_ptr())
        camera = _lib.Camera()
        for k in ("position", "forward", "right", "up"):
            getattr(camera, k)[:] = [float(v) for v in cam[k]]
        camera.fov, camera.width, camera.height = float(cam["fov"]), cam["width"], cam["height"]
        camera.model = 0 if cam["model"] == "pinhole" else 1
        vis = _lib.VisualizationSettings(_lib.VIS_MODES[c["mode"]], _lib.COLOR_MAPS[c["color_map"]],
                                         (ctypes.c_float * 3)(*c["bg_color"]), int(c["checker_bg"]),
                                         c["max_depth"], c["depth_quantile"])
        settings = _lib.TraceSettings(c["weight_threshold"], c["max_intersections"])
        arr, surf = cudart.surface(cam["width"], cam["height"])
        torch.cuda.synchronize()
        _lib.check(lib.rfb_trace_visualization(
            handle, ctypes.byref(settings), ctypes.byref(vis), ctypes.byref(camera), ctypes.byref(cm),
            f.points.shape[0], 0, scene[0].data_ptr(), scene[1].data_ptr(), scene[2].data_ptr(), scene[3].data_ptr(),
            diff.data_ptr(), start, surf, None, None))
        return cudart.read_and_free(torch, arr, surf, cam["width"], cam["height"])
    finally:
        lib.rfb_destroy_pipeline(handle)


CASES = V.cases()


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_frame_equals_reference_kernel_frame(torch_cuda, cudart, golden, c):
    import radfoam_b200

    torch = torch_cuda
    f, attrs, cam = V.scene(c["scene"]), V.case_attributes(c), V.case_camera(c)
    start = V.start_index(c["scene"], cam)
    pipe = radfoam_b200.create_pipeline(f.sh_degree, c["dtype"])
    ours = render(torch, pipe, f, attrs, cam, start, c)
    ref = golden[c["name"]]
    assert ours.shape == ref.shape == (cam["height"], cam["width"])
    bad = ours != ref
    assert not bad.any(), f"{int(bad.sum())} pixels differ from the reference kernel's, first at {np.argwhere(bad)[0]}"
    surf = render_surface(torch, cudart, f, attrs, cam, start, c)
    assert np.array_equal(surf, ours), "the surface frame differs from the linear-buffer frame"


def test_exact_scan_camera_needs_the_exact_twin():
    """The exact-scan cases really route rays through the exact twin: one pixel column has a direction component
    below 2^-60 (the same cast_ray arithmetic in float32 numpy: u = 0 there, so d_x = s * 1e-25)."""
    cam = V.camera("s20k", "exact")
    s = np.float32(1.0) / np.tan(np.float32(cam["fov"]) * np.float32(0.5), dtype=np.float32)
    dx = np.float32(s * cam["forward"][0])
    assert 0 < abs(dx) < 2.0 ** -60
    assert (V.W // 2) / V.W == 0.5


@pytest.mark.parametrize("model", ["pinhole", "fisheye"])
@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_rgb_over_black_equals_benchmark_frame(torch_cuda, model, dtype):
    """RGB mode with a black background and no checker is trace_benchmark's frame with its rows reversed, byte for
    byte (the 20k scene and 200x120 camera of test_gpu_parity.test_trace_benchmark)."""
    import radfoam_b200

    torch = torch_cuda
    f = V.scene("s20k")
    attrs = f.attributes.astype(np.float16 if dtype == "float16" else np.float32)
    cam = V.camera("s20k", model, 200, 120)
    start = V.start_index("s20k", cam)
    pipe = radfoam_b200.create_pipeline(3, dtype)
    scene = scene_tensors(torch, f, attrs)
    diff = pipe.prefetch_adjacent_diff(scene[0], scene[2], scene[3])
    bench = torch.zeros((120, 200), dtype=torch.uint32, device="cuda")
    pipe.trace_benchmark(*scene, diff, cam, to_dev(torch, np.array([start], np.uint32)), bench, weight_threshold=0.05)
    vis = pipe.trace_visualization(*scene, diff, cam, start, mode="rgb", bg_color=(0.0, 0.0, 0.0),
                                   weight_threshold=0.05)
    torch.cuda.synchronize()
    b = bench.cpu().numpy()
    assert (b & 0xFFFFFF != 0).mean() > 0.2  # the frame is not empty
    assert np.array_equal(vis.cpu().numpy(), b[::-1])


def test_redraw_of_unchanged_scene_equals_fresh_pipeline(torch_cuda):
    """A viewer redraws one scene many times: the second call reuses the mirrors (same scene version) and must give
    the bytes of a fresh pipeline, in every mode."""
    import radfoam_b200

    torch = torch_cuda
    f = V.scene("s20k")
    cam = V.camera("s20k", "fisheye")
    start = V.start_index("s20k", cam)
    pipe = radfoam_b200.create_pipeline(3)
    scene = scene_tensors(torch, f, f.attributes)
    diff = pipe.prefetch_adjacent_diff(scene[0], scene[2], scene[3])
    tabs = cmap_tensors(torch, "mixed")
    for mode in V.MODES:
        frames = [pipe.trace_visualization(*scene, diff, cam, start, mode=mode, cmap_table=tabs).cpu().numpy()
                  for _ in range(2)]
        fresh = radfoam_b200.create_pipeline(3).trace_visualization(*scene, diff, cam, start, mode=mode,
                                                                    cmap_table=tabs).cpu().numpy()
        assert np.array_equal(frames[0], frames[1]) and np.array_equal(frames[1], fresh), mode


def test_config4_frames_match_reference_hashes(torch_cuda, golden):
    """Config 4 (1,048,576 points) at 1920x1080 in every mode: SHA-256 of the whole frame and 12 sampled rows equal
    the reference kernel's."""
    import bench
    import radfoam_b200

    torch = torch_cuda
    f = bench.load_or_build_foam(1 << 20, lambda m: None)
    cam = V.config4_camera()
    start = V.foam.nearest_point(f.points, cam["position"])
    pipe = radfoam_b200.create_pipeline(3)
    scene = scene_tensors(torch, f, f.attributes)
    for c in V.FULL_CASES:
        img = render(torch, pipe, f, f.attributes, cam, start, c, scene=scene)
        assert np.array_equal(img[V.FULL_ROWS], golden[c["name"] + "#rows"]), c["name"]
        assert hashlib.sha256(img.tobytes()).digest() == golden[c["name"] + "#sha256"].tobytes(), c["name"]


def test_exact_twin_against_live_reference(torch_cuda):
    """Where oracle/_ref was built: the exact-twin camera's frames against the reference kernel run now."""
    from oracle import ref_gpu, ref_vis

    if not (ref_gpu.available() and ref_vis.available()):
        pytest.skip("oracle/_ref not built")
    import radfoam_b200

    torch = torch_cuda
    for c in (c for c in CASES if c["name"].startswith("exact_scan_")):
        f, attrs, cam = V.scene(c["scene"]), V.case_attributes(c), V.case_camera(c)
        start = V.start_index(c["scene"], cam)
        ours = render(torch, radfoam_b200.create_pipeline(3, c["dtype"]), f, attrs, cam, start, c)
        scene = scene_tensors(torch, f, attrs)
        diff = ref_gpu.prefetch_adjacent_diff(scene[0], scene[2], scene[3])
        tabs = cmap_tensors(torch, c["tables"])
        ptrs = to_dev(torch, np.array([t.data_ptr() for t in tabs], dtype=np.int64))
        sizes = to_dev(torch, np.array([t.shape[0] for t in tabs], dtype=np.int32))
        ref = torch.zeros((cam["height"], cam["width"]), dtype=torch.uint32, device="cuda")
        ref_vis.trace_visualization(*scene, diff, cam, start, ptrs, sizes, ref, **V.vis_kwargs(c))
        torch.cuda.synchronize()
        assert np.array_equal(ours, ref.cpu().numpy()), c["name"]
