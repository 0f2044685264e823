"""Drives the gradient epilogues -- rfb_trace_backward_finalize, rfb_trace_backward_finalize_params and
rfb_reduce_finalize_peers -- on crafted accumulators, with every output a view into a larger allocation whose
tail (and every byte the kernel must not write) holds a sentinel pattern, and holds the results to
``param_model`` bit for bit.

One harness for two memories: ``NumpyMemory`` (the CPU kernel emulator, tests/emu) and ``TorchMemory`` (a CUDA
device; the comparisons run on the device so that large cases do not cross PCIe once per rank).  The peer kernel
takes W rank buffers laid out ``[accumulator | attr_grad | points_grad]`` with the 16-byte granules of
``radfoam_b200.sharded.ShardedTracer._peer_setup``; on one device they are W allocations of that device.
"""
from __future__ import annotations

import ctypes
import functools

import numpy as np

import param_model as P
from radfoam_b200 import _lib as abi

SENTINEL = 0xA5            # every byte of an output allocation before the kernel runs
# sentinel bytes after the last output element: more than the longest run of stores a ragged row block could make
# past its last row (15 rows of 49 fp32 attributes, then 15 position rows), so that an over-long store lands in
# the guard and is observed rather than leaving the allocation
GUARD = 4096
PEER_ROWS = 16             # rows per block of the peer reduction, dealt round-robin to the ranks


def _ceil16(n: int) -> int:
    return (n + 15) // 16 * 16


def _uint(dtype):
    return {2: np.uint16, 4: np.uint32}[np.dtype(dtype).itemsize]


class NumpyMemory:
    """Host arrays standing in for device memory (the emulated library dereferences them directly)."""

    def __init__(self):
        self._keep = []
        self.stream = None

    def alloc(self, nbytes: int):
        raw = np.empty(nbytes + 64, np.uint8)
        off = (-raw.ctypes.data) % 64
        a = raw[off:off + nbytes]
        a[...] = SENTINEL
        self._keep.append(raw)
        return a

    @staticmethod
    def ptr(buf, offset: int = 0) -> int:
        return buf.ctypes.data + offset

    @staticmethod
    def view(buf, offset: int, shape, dtype):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return buf[offset:offset + n].view(dtype).reshape(shape)

    @staticmethod
    def upload(a):
        return np.ascontiguousarray(a)

    @staticmethod
    def write(dst, src):
        dst[...] = src

    @staticmethod
    def same(got, want, rows=None) -> bool:
        """Bit-identical on the selected rows, any NaN matching any NaN."""
        if rows is not None:
            got, want = got[rows], want[rows]
        u = _uint(got.dtype)
        nan = np.isnan(want)
        return bool(np.array_equal(np.isnan(got), nan) and np.array_equal(got.view(u)[~nan], want.view(u)[~nan]))

    @staticmethod
    def untouched(got, rows=None) -> bool:
        if rows is not None:
            got = got[rows]
        return bool((np.ascontiguousarray(got).view(np.uint8) == SENTINEL).all())

    @staticmethod
    def host(a):
        return np.asarray(a)

    def sync(self):
        pass


class TorchMemory:
    """CUDA allocations of the current device; comparisons run there."""

    def __init__(self, torch):
        self.torch = torch
        self.stream = torch.cuda.current_stream().cuda_stream
        self._keep = []   # the library holds raw pointers (the accumulator): no allocation may be recycled

    def alloc(self, nbytes: int):
        buf = self.torch.full((nbytes,), SENTINEL, dtype=self.torch.uint8, device="cuda")
        self._keep.append(buf)
        return buf

    @staticmethod
    def ptr(buf, offset: int = 0) -> int:
        return buf.data_ptr() + offset

    def view(self, buf, offset: int, shape, dtype):
        td = {np.float32: self.torch.float32, np.float16: self.torch.float16}[np.dtype(dtype).type]
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return buf[offset:offset + n].view(td).view(tuple(shape))

    def upload(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def write(self, dst, src):
        dst.copy_(self.upload(src))

    def same(self, got, want, rows=None) -> bool:
        t = self.torch
        if rows is not None:
            got, want = got[rows], want[rows]
        it = {2: t.int16, 4: t.int32}[got.element_size()]
        nan = t.isnan(want)
        eq = (got.view(it) == want.view(it)) | (nan & t.isnan(got))
        return bool(eq.all()) and not bool((t.isnan(got) & ~nan).any())

    def untouched(self, got, rows=None) -> bool:
        if rows is not None:
            got = got[rows]
        return bool((got.contiguous().view(self.torch.uint8) == SENTINEL).all())

    @staticmethod
    def host(a):
        return a.cpu().numpy()

    def sync(self):
        self.torch.cuda.synchronize()


def _check(lib, rc):
    if rc:
        raise RuntimeError(lib.rfb_last_error().decode())


class Guarded:
    """One output array at the head of its own allocation, GUARD sentinel bytes behind it."""

    def __init__(self, mem, shape, dtype):
        self.mem, self.shape, self.dtype = mem, tuple(shape), np.dtype(dtype)
        nbytes = int(np.prod(shape)) * self.dtype.itemsize
        self.buf = mem.alloc(nbytes + GUARD)
        self.out = mem.view(self.buf, 0, shape, dtype)
        self.tail = self.buf[nbytes:]

    @property
    def ptr(self):
        return self.mem.ptr(self.buf)

    def check(self, name, want):
        assert self.mem.untouched(self.tail), f"{name}: a store ran past the end of the output"
        assert self.mem.same(self.out, self.mem.upload(np.asarray(want, self.dtype).reshape(self.shape))), \
            f"{name}: not bit-identical to the reference"


def prime_accumulator(mem, lib, handle, deg: int, n: int, contents: np.ndarray):
    """Point the pipeline's accumulator at a caller allocation, let a zero-ray backward zero-fill it and set the
    point count, then write ``contents`` into it.  Returns the accumulator view."""
    gr = P.grad_row(deg)
    buf = mem.alloc(n * gr * 4)
    acc = mem.view(buf, 0, (n, gr), np.float32)
    _check(lib, lib.rfb_set_grad_accumulator(handle, mem.ptr(buf), n * gr))
    _check(lib, lib.rfb_trace_backward_accumulate(handle, None, n, None, None, 0, None, None, 0, None, None, 0, None,
                                                  None, None, None, None, None, None, None, mem.stream))
    mem.sync()
    assert mem.same(acc, mem.upload(np.zeros((n, gr), np.float32))), "the zero-ray backward must zero-fill"
    mem.write(acc, contents)
    mem.sync()
    return acc


def finalize_outputs(mem, lib, handle, deg: int, dtype, n: int, scrub: bool):
    """rfb_trace_backward_finalize into guarded outputs: (points_grad, attr_grad) Guarded."""
    pts, attr = Guarded(mem, (n, 3), np.float32), Guarded(mem, (n, P.attr_dim(deg)), dtype)
    _check(lib, lib.rfb_trace_backward_finalize(handle, n, pts.ptr, attr.ptr,
                                                abi.FLAG_SCRUB_NONFINITE if scrub else 0, mem.stream))
    mem.sync()
    return pts, attr


def finalize_params_outputs(mem, lib, handle, deg: int, n: int, scrub: bool):
    """rfb_trace_backward_finalize_params into guarded outputs (a parameter-form scene must be bound)."""
    a = P.attr_dim(deg)
    out = {"points_grad": Guarded(mem, (n, 3), np.float32), "att_dc_grad": Guarded(mem, (n, 3), np.float32),
           "att_sh_grad": Guarded(mem, (n, a - 4), np.float32) if a > 4 else None,
           "density_grad": Guarded(mem, (n, 1), np.float32)}
    _check(lib, lib.rfb_trace_backward_finalize_params(
        handle, n, out["points_grad"].ptr, out["att_dc_grad"].ptr,
        out["att_sh_grad"].ptr if out["att_sh_grad"] else None, out["density_grad"].ptr,
        abi.FLAG_SCRUB_NONFINITE if scrub else 0, mem.stream))
    mem.sync()
    return out


def edge_raw_density(n: int, seed: int) -> np.ndarray:
    """[n, 1] raw densities: the softplus edge set (and NaN / +-inf) repeated, then seeded ordinary values."""
    rng = np.random.default_rng(seed)
    edges = np.concatenate([P.EDGE_RAW, P.EDGE_RAW_NONFINITE])
    raw = rng.normal(0.0, 1.0, size=n).astype(np.float32)
    k = min(n, 4 * edges.size)
    raw[:k] = np.resize(edges, k)
    return raw.reshape(n, 1)


# ---- the peer reduction ------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=16)
def _crafted(n: int, deg: int, seed: int, share: float) -> np.ndarray:
    return P.crafted_accumulator(n, deg, seed, share)


def rank_accumulators(n: int, deg: int, world: int) -> list:
    """W different crafted accumulators (three generated, rolled by rank: cheap at 200 k rows), specials thinned
    with W so that the rank sums are not mostly non-finite."""
    share = 0.3 / world
    return [np.roll(_crafted(n, deg, 100 + w % 3, share), 17 * w, axis=0) for w in range(world)]


def peer_layout(n: int, deg: int, dtype):
    """Byte offsets of one rank buffer [acc | attr (16-byte granules) | pts (16-byte granules) | guard]."""
    acc_b = n * P.grad_row(deg) * 4
    attr_b = _ceil16(n * P.attr_dim(deg) * np.dtype(dtype).itemsize)
    pts_b = _ceil16(n * 3 * 4)
    return acc_b, acc_b + attr_b, acc_b + attr_b + pts_b, acc_b + attr_b + pts_b + GUARD


def run_peers(mem, lib, handle, deg: int, dtype, accs: list, scrub: bool):
    """Every rank in turn on W same-device buffers.  After rank r, exactly the row blocks of ranks 0..r are
    written in every rank's outputs, bit-identical to finalize(peer_sum(accs)); all other output bytes, the
    granule padding, the guard and the accumulators keep their contents.  Returns the expected
    (points_grad, attr_grad) for further checks."""
    world, n = len(accs), accs[0].shape[0]
    a, gr = P.attr_dim(deg), P.grad_row(deg)
    o_attr, o_pts, o_end, total = peer_layout(n, deg, dtype)
    bufs = [mem.alloc(total) for _ in range(world)]
    acc_v = [mem.view(b, 0, (n, gr), np.float32) for b in bufs]
    for v, host in zip(acc_v, accs):
        mem.write(v, host)
    attr_v = [mem.view(b, o_attr, (n, a), dtype) for b in bufs]
    pts_v = [mem.view(b, o_pts, (n, 3), np.float32) for b in bufs]
    pad_attr = [b[o_attr + n * a * np.dtype(dtype).itemsize:o_pts] for b in bufs]
    pad_pts = [b[o_pts + n * 12:] for b in bufs]    # granule padding + guard
    want_pts, want_attr = P.finalize(P.peer_sum(accs), deg, dtype, scrub)
    want_pts_d, want_attr_d = mem.upload(want_pts), mem.upload(want_attr)
    accs_d = [mem.upload(x) for x in accs]
    owner = (np.arange(n) // PEER_ROWS) % world
    table = lambda off: (ctypes.c_void_p * world)(*[mem.ptr(b, off) for b in bufs])  # noqa: E731
    mem.sync()
    for rank in range(world):
        _check(lib, lib.rfb_reduce_finalize_peers(handle, world, rank, n, table(0), table(o_attr), table(o_pts), None,
                                                  abi.FLAG_SCRUB_NONFINITE if scrub else 0, mem.stream))
        mem.sync()
        done = mem.upload(owner <= rank)
        rest = mem.upload(owner > rank)
        for w in range(world):
            where = f"world {world} rank {rank} -> buffer {w}"
            assert mem.same(attr_v[w], want_attr_d, done), f"{where}: attr_grad of the finished blocks"
            assert mem.same(pts_v[w], want_pts_d, done), f"{where}: points_grad of the finished blocks"
            assert mem.untouched(attr_v[w], rest), f"{where}: attr_grad written outside the finished blocks"
            assert mem.untouched(pts_v[w], rest), f"{where}: points_grad written outside the finished blocks"
            assert mem.untouched(pad_attr[w]) and mem.untouched(pad_pts[w]), f"{where}: padding or guard written"
            assert mem.same(acc_v[w], accs_d[w]), f"{where}: an accumulator was modified"
    return want_pts, want_attr
