"""trace_visualization without a GPU: the CPU restatement (tests/vis_oracle.c: rfo_trace_visualization) and the
product's kernel source on the CPU emulator (tests/emu), through both the linear entry point and the surface stand-in,
against the frames the reference's own visualization kernel rendered (tests/golden/reference/visualization.npz,
made by tests/golden/make_golden_visualization.py on an H100); and the C ABI's argument checks.

The reference's frames are byte-identical to the device kernel's (tests/test_gpu_visualization.py).  On the CPU,
expf / logf come from libm instead of libdevice; a last-bit difference moves an RGBA8 channel by one level at most
where the frame is a continuous function of it, and can flip a threshold decision (T > weight_threshold,
T' < depth_quantile) on a rare pixel.  The bars: at most 1 % of pixels differ at all, and at most 0.3 % by more than
one level.  The edge cases (non-finite and saturated colour-map inputs, exhausted step budgets) are held to the
same bars, so a wrong conversion rule, which changes whole regions, fails them."""
import ctypes
import os
import sys

import numpy as np
import pytest

import vis_cases as V

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "visualization.npz")
CASES = V.cases()


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def assert_frame_close(got, ref, name):
    assert got.shape == ref.shape
    a = got.view(np.uint8).reshape(*got.shape, 4).astype(np.int32)
    b = ref.view(np.uint8).reshape(*ref.shape, 4).astype(np.int32)
    diff = np.abs(a - b).max(axis=-1)
    assert (diff > 0).mean() <= 0.01, f"{name}: {(diff > 0).mean():.4f} of the pixels differ"
    assert (diff > 1).mean() <= 0.003, f"{name}: {(diff > 1).mean():.4f} of the pixels differ by more than 1"


def case_inputs(c):
    f, cam = V.scene(c["scene"]), V.case_camera(c)
    return f, V.case_attributes(c), cam, V.start_index(c["scene"], cam)


def test_golden_frames_cover_the_cases(golden):
    """Every case has a stored frame, and the stored frames show something (not one flat colour)."""
    for c in CASES:
        img = golden[c["name"]]
        assert img.shape == (V.H, V.W) and img.dtype == np.uint32, c["name"]
    flat = {c["name"] for c in CASES if len(np.unique(golden[c["name"]])) == 1}
    # flat by construction: a one-entry table, every ray out of steps (v = 1), every depth -inf / NaN
    assert flat == {"mixed_gray_depth", "mixed_gray_intersections", "steps_exhausted",
                    "zero_density_quantile_above_one"}, flat
    for c in V.FULL_CASES:
        assert golden[c["name"] + "#sha256"].shape == (32,)
        assert golden[c["name"] + "#rows"].shape == (V.FULL_ROWS.size, V.FULL_W)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_oracle_reproduces_reference_frames(golden, c):
    import vis_oracle
    from oracle import oracle

    f, attrs, cam, start = case_inputs(c)
    diff = oracle.prefetch_adjacent_diff(f.points, f.adjacency, f.offsets)
    img = vis_oracle.trace_visualization(f.points, attrs, f.adjacency, f.offsets, diff, cam, start,
                                     V.tables(c["tables"]), num_threads=0, **V.vis_kwargs(c))
    assert_frame_close(img, golden[c["name"]], c["name"])


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_emulated_kernel_reproduces_reference_frames(golden, c):
    import emu
    import emu_vis

    f, attrs, cam, start = case_inputs(c)
    diff = emu.prefetch_adjacent_diff(f.points, f.adjacency, f.offsets)
    pipe = emu.EmuPipeline(f.sh_degree, attrs.dtype)
    args = (pipe, f.points, attrs, f.adjacency, f.offsets, diff, cam, start, V.tables(c["tables"]))
    linear = emu_vis.trace_visualization(*args, **V.vis_kwargs(c))
    assert_frame_close(linear, golden[c["name"]], c["name"])
    surface = emu_vis.trace_visualization(*args, surface=True, **V.vis_kwargs(c))
    assert np.array_equal(surface, linear), "the surface frame differs from the linear-buffer frame"


def test_emulated_colour_map_edge_values():
    """The colour-map conversions of the kernel source on the emulator, against the C restatement, on a tiny foam
    where whole frames hit them: depth 0 (quantile never reached), ±inf / NaN depth (zero density), v far above 1
    and beyond the int range (tiny max_depth), v = 1 exactly (steps exhausted)."""
    import emu
    import emu_vis
    import vis_oracle

    f = V.scene("c1")
    attrs = f.attributes.copy()
    attrs[::2, -1] = 0.0
    cam = V.camera("c1", "pinhole", 24, 16)
    start = V.start_index("c1", cam)
    diff = emu.prefetch_adjacent_diff(f.points, f.adjacency, f.offsets)
    pipe = emu.EmuPipeline(3, np.float32)
    for kw in (dict(mode="depth", depth_quantile=1e-30), dict(mode="depth", depth_quantile=1.5),
               dict(mode="depth", depth_quantile=1.0), dict(mode="depth", max_depth=1e-9),
               dict(mode="depth", max_depth=-1e-9), dict(mode="intersections", max_intersections=2),
               dict(mode="intersections", max_intersections=0)):
        for tabs in ("mixed", "random"):
            for cmap in V.MAPS:
                args = (f.points, attrs, f.adjacency, f.offsets, diff, cam, start, V.tables(tabs))
                a = emu_vis.trace_visualization(pipe, *args, color_map=cmap, **kw)
                b = vis_oracle.trace_visualization(*args, color_map=cmap, **kw)
                assert np.array_equal(a, b), (kw, tabs, cmap)


def _emu_call(fn, pipe, vis=None, cam=None, table=None, pts=True, output=True):
    import emu
    from radfoam_b200 import _lib as abi

    f = V.scene("c1")
    buf = np.zeros((8, 8), dtype=np.uint32)
    diff = np.zeros((f.adjacency.size, 4), np.float16)
    arrays = [f.points, f.attributes, f.adjacency, f.offsets, diff]
    cam = cam or abi.Camera((ctypes.c_float * 3)(0, 0, -3), (ctypes.c_float * 3)(0, 0, 1),
                            (ctypes.c_float * 3)(1, 0, 0), (ctypes.c_float * 3)(0, 1, 0), 0.7, 8, 8, 0)
    vis = vis if vis is not None else abi.VisualizationSettings(0, 3, (ctypes.c_float * 3)(1, 1, 1), 0, 10.0, 0.5)
    from emu_vis import EmuSurface

    lib = pipe.lib
    surf = EmuSurface(buf.ctypes.data, buf.strides[0], 4 * buf.shape[1], buf.shape[0])
    out_arg = (emu._p(buf) if output else None) if fn == "rfb_trace_visualization_rgba8" else (
        ctypes.addressof(surf) if output else 0)
    rc = getattr(lib, fn)(pipe.handle, None, ctypes.byref(vis), ctypes.byref(cam), table, f.points.shape[0], 0,
                          *[emu._p(a) if pts or k else None for k, a in enumerate(arrays)], 0, out_arg, None, None)
    return rc, lib.rfb_last_error().decode()


@pytest.mark.parametrize("fn", ["rfb_trace_visualization", "rfb_trace_visualization_rgba8"])
def test_cabi_argument_checks(fn):
    import emu
    from radfoam_b200 import _lib as abi

    pipe = emu.EmuPipeline(3, np.float32)
    f = V.scene("c1")
    rc, msg = _emu_call(fn, pipe, pts=False)
    assert rc != 0 and "NULL argument" in msg and fn in msg
    rc, msg = _emu_call(fn, pipe, output=False)
    assert rc != 0 and "NULL argument" in msg
    for bad_mode in (-1, 4):
        rc, msg = _emu_call(fn, pipe, vis=abi.VisualizationSettings(bad_mode, 3, (ctypes.c_float * 3)(1, 1, 1), 0,
                                                                    10.0, 0.5))
        assert rc != 0 and "unknown visualization mode" in msg
    rc, msg = _emu_call(fn, pipe, vis=abi.VisualizationSettings(0, 7, (ctypes.c_float * 3)(1, 1, 1), 0, 10.0, 0.5))
    assert rc != 0 and "unknown color map" in msg
    for mode in (1, 3):  # depth and intersections read the table
        rc, msg = _emu_call(fn, pipe, vis=abi.VisualizationSettings(mode, 3, (ctypes.c_float * 3)(1, 1, 1), 0,
                                                                    10.0, 0.5))
        assert rc != 0 and "color map table" in msg
    for mode in (0, 2):  # RGB and alpha do not
        rc, msg = _emu_call(fn, pipe, vis=abi.VisualizationSettings(mode, 3, (ctypes.c_float * 3)(1, 1, 1), 0,
                                                                    10.0, 0.5))
        assert rc == 0, msg
    bad_cam = abi.Camera((ctypes.c_float * 3)(0, 0, -3), (ctypes.c_float * 3)(0, 0, 1), (ctypes.c_float * 3)(1, 0, 0),
                         (ctypes.c_float * 3)(0, 1, 0), 0.7, 8, 8, 5)
    rc, msg = _emu_call(fn, pipe, cam=bad_cam)
    assert rc != 0 and "camera model" in msg
    assert f.points.shape[0] > 0


def test_product_library_checks_need_no_gpu():
    """The product library's own entry points reject a NULL pipeline and NULL arguments before touching the GPU."""
    from radfoam_b200 import _lib

    lib = _lib.load()
    vis = _lib.VisualizationSettings(0, 3, (ctypes.c_float * 3)(1, 1, 1), 0, 10.0, 0.5)
    for fn, out in ((lib.rfb_trace_visualization, 0), (lib.rfb_trace_visualization_rgba8, None)):
        assert fn(None, None, ctypes.byref(vis), None, None, 0, 0, None, None, None, None, None, 0, out, None,
                  None) != 0
        assert b"pipeline is NULL" in lib.rfb_last_error()
