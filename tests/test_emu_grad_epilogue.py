"""The gradient epilogues on the CPU kernel emulator (tests/emu), on crafted accumulators: fp16 overflow and
subnormals, round-half-even ties, NaN / +-inf / -0 / FLT_MAX, scrub on and off, ragged row blocks and ranks without
a block.  finalize, finalize_params and the peer reduction are held bit for bit to tests/param_model.py (the
density gradient, whose expf is the host's here, within its float64 bound), with sentinel guards behind every
output.  tests/test_gpu_grad_epilogue.py runs the same harness on the device."""
import os
import sys

import numpy as np
import pytest

import epilogue_harness as H
import param_model as P

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402

DTYPES = [np.float32, np.float16]
IDS = ["fp32", "fp16"]


@pytest.fixture(autouse=True)
def _quiet():
    with np.errstate(all="ignore"):
        yield


def assert_density(got: np.ndarray, want, name="density_grad"):
    """Within the float64 bound where the reference is finite; the same inf / NaN where it is not."""
    v, e = want.v.reshape(got.shape), np.broadcast_to(want.e, want.v.shape).reshape(got.shape)
    g = got.astype(np.float64)
    fin = np.isfinite(v)
    assert np.array_equal(np.isnan(g[~fin]), np.isnan(v[~fin])), f"{name}: NaN where the reference has none"
    inf = np.isinf(v)
    assert np.array_equal(g[inf], v[inf]), f"{name}: infinities differ"
    ok = fin & np.isfinite(e)
    bad = np.abs(g[ok] - v[ok]) > e[ok]
    assert not bad.any(), f"{name}: {int(bad.sum())} entries outside the float64 bound"


def test_reference_rounding_and_crafted_inputs():
    """The references' own promises: fp16 rounding is round-half-even with overflow at 65520, the crafted
    accumulator carries every special, and the torch threshold branch is taken from the fp32 product."""
    h = np.array([65504, 65519.996, 65520, 1 + 2 ** -11, 1 + 3 * 2 ** -11, 2049, 2 ** -25, 1.5 * 2 ** -24,
                  2.5 * 2 ** -24, 1e-8], np.float32).astype(np.float16)
    assert h[0] == 65504 and h[1] == 65504 and np.isinf(h[2])
    assert h[3] == 1 and h[4] == 1 + 2 ** -9 and h[5] == 2048
    assert h[6] == 0 and h[7] == 2 * 2 ** -24 and h[8] == 2 * 2 ** -24 and h[9] == 0
    acc = P.crafted_accumulator(64, 3, 1)
    for s in P.SPECIALS:
        assert (np.isnan(acc).any() if np.isnan(s) else (acc.view(np.uint32) == np.float32(s).view(np.uint32)).any())
    xb = P.EDGE_RAW * np.float32(10)
    assert not (xb[0] > 20) and xb[1] > 20 and not (xb[2] > 20)     # 2.0f*10 == 20 exactly: log1p branch
    sp = P.softplus_beta10(P.EDGE_RAW)
    assert sp.v[5] == 2.5 and sp.v[7] == pytest.approx(np.log(2) / 10, rel=1e-15)
    assert sp.v[11] < 1e-44 and np.all(sp.e >= 0)


def test_unshard_image_of_uint32_outputs():
    """num_intersections and depth_indices are uint32: the ray-sharded reassembly must carry them bit for bit."""
    import torch

    from radfoam_b200 import sharded

    t = torch.arange(40 * 3, dtype=torch.int64).view(40, 3).mul_(0x01010101).to(torch.uint32)
    parts = [sharded.shard_image(t, r, 3) for r in range(3)]
    back = sharded.unshard_image(parts, 40)
    assert back.dtype == torch.uint32 and torch.equal(back.view(torch.int32), t.view(torch.int32))


@pytest.mark.parametrize("scrub", [False, True], ids=["raw", "scrub"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 3, 16, 17, 1000])
def test_finalize_crafted_accumulator(n, deg, dtype, scrub):
    mem = H.NumpyMemory()
    pipe = emu.EmuPipeline(deg, dtype)
    contents = P.crafted_accumulator(n, deg, seed=n * 10 + deg)
    H.prime_accumulator(mem, pipe.lib, pipe.handle, deg, n, contents)
    pts, attr = H.finalize_outputs(mem, pipe.lib, pipe.handle, deg, dtype, n, scrub)
    want_pts, want_attr = P.finalize(contents, deg, dtype, scrub)
    pts.check("points_grad", want_pts)
    attr.check("attr_grad", want_attr)


@pytest.mark.parametrize("scrub", [False, True], ids=["raw", "scrub"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 17, 1000])
def test_finalize_params_crafted_accumulator(n, deg, dtype, scrub):
    mem = H.NumpyMemory()
    pipe = emu.EmuPipeline(deg, dtype)
    raw = H.edge_raw_density(n, seed=n + deg)
    a = P.attr_dim(deg)
    pipe.bind_scene_params(np.zeros((n, 3), np.float32), np.zeros((n, a - 4), np.float32), raw, 1.7)
    contents = P.crafted_accumulator(n, deg, seed=n * 10 + deg + 5)
    H.prime_accumulator(mem, pipe.lib, pipe.handle, deg, n, contents)
    out = H.finalize_params_outputs(mem, pipe.lib, pipe.handle, deg, n, scrub)
    want = P.finalize_params(contents, pipe._params[2], 1.7, deg, dtype, scrub)
    for k in ("points_grad", "att_dc_grad", "att_sh_grad"):
        if out[k] is not None:
            out[k].check(k, want[k])
    assert mem.untouched(out["density_grad"].tail)
    assert_density(out["density_grad"].out, want["density_grad"])


@pytest.mark.parametrize("scrub", [False, True], ids=["raw", "scrub"])
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("deg", [0, 3])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8, 16])
def test_peer_reduce_finalize(world, deg, dtype, scrub):
    """Every instantiation of the peer kernel (WORLD 2, 4, 8 and the generic loop) at the row counts where its
    blocks go wrong: one row, a ragged single block, exactly one block, one row into the second, and 16W - 1
    (the last rank has no block: the host returns before launching)."""
    pipe = emu.EmuPipeline(deg, dtype)
    for n in sorted({1, 15, 16, 17, 16 * world - 1}):
        mem = H.NumpyMemory()
        accs = H.rank_accumulators(n, deg, world)
        want_pts, want_attr = H.run_peers(mem, pipe.lib, pipe.handle, deg, dtype, accs, scrub)
        H.prime_accumulator(mem, pipe.lib, pipe.handle, deg, n, P.peer_sum(accs))
        pts, attr = H.finalize_outputs(mem, pipe.lib, pipe.handle, deg, dtype, n, scrub)
        pts.check("points_grad", want_pts)
        attr.check("attr_grad", want_attr)
        pipe.lib.rfb_set_grad_accumulator(pipe.handle, None, 0)
