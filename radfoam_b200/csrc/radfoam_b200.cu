// C-ABI implementation (include/radfoam_b200.h) of the H100 foam tracer.
// Host side: argument checks, cached scene re-layout, kernel dispatch.
#include "../../include/radfoam_b200.h"

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <atomic>
#include <cstring>
#include <new>
#include <string>
#include <type_traits>

#include "foam_kernels.cuh"

// Kernel launch.  In the product this is the <<< >>> launch; the CPU kernel-logic emulator under tests/emu
// (test infrastructure, never loaded by the product) defines RFB_LAUNCH itself before this file is compiled.
#ifndef RFB_LAUNCH
#define RFB_UNPAREN(...) __VA_ARGS__
#define RFB_LAUNCH(kernel, grid, block, smem, stream, ...) \
    (RFB_UNPAREN kernel)<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif


namespace {

thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0}; // process-wide: autograd runs backward on its own thread
std::atomic<uint64_t> g_device_allocs{0}, g_device_frees{0}; // cudaMalloc / cudaFree calls made by this library

int fail(const std::string &msg) {
    g_last_error = msg;
    return 1;
}

#define RFB_CUDA(call)                                                                    \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess)                                                            \
            return fail(std::string("CUDA call failed at " __FILE__ ":") +                \
                        std::to_string(__LINE__) + ": " + cudaGetErrorString(e_));        \
    } while (0)

#define RFB_LAUNCHED()                                                                    \
    do {                                                                                  \
        ++g_launches;                                                                     \
        RFB_CUDA(cudaGetLastError());                                                     \
    } while (0)

struct DeviceBuffer {
    void *ptr = nullptr;
    size_t bytes = 0;
    // grow-only; reallocation synchronises, steady state does not
    cudaError_t ensure(size_t need) {
        if (need <= bytes)
            return cudaSuccess;
        if (ptr) {
            ++g_device_frees;
            cudaError_t e = cudaFree(ptr);
            ptr = nullptr;
            bytes = 0;
            if (e != cudaSuccess)
                return e;
        }
        size_t want = need + need / 16 + 256;
        ++g_device_allocs;
        cudaError_t e = cudaMalloc(&ptr, want);
        if (e == cudaSuccess)
            bytes = want;
        return e;
    }
    void release() {
        if (ptr)
            cudaFree(ptr);
        ptr = nullptr;
        bytes = 0;
    }
};

struct SceneKey {
    const void *points = nullptr, *attrs = nullptr, *adj = nullptr, *off = nullptr;
    const void *diff = nullptr; // non-null: faces were copied from this caller-built array
    uint32_t n = 0, e = 0;
    uint64_t version = 0;
    bool faces = false;
    bool operator==(const SceneKey &o) const {
        return points == o.points && attrs == o.attrs && adj == o.adj && off == o.off && diff == o.diff &&
               n == o.n && e == o.e && version == o.version;
    }
};

// Streaming multiprocessors of an H100 SXM; grid caps below are multiples of it.
constexpr int kNumSMs = 132;

int grid_for(uint64_t work_items, int block, int max_blocks = kNumSMs * 16) {
    uint64_t b = (work_items + block - 1) / block;
    if (b > (uint64_t)max_blocks)
        b = max_blocks;
    if (b < 1)
        b = 1;
    return (int)b;
}

// f(std::integral_constant<int, D>{}) for SH degree D: one kernel instantiation per degree
template <typename F>
auto with_degree(int deg, F &&f) {
    switch (deg) {
    case 0: return f(std::integral_constant<int, 0>{});
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    default: return f(std::integral_constant<int, 3>{});
    }
}

template <typename T>
struct TypeTag {
    using type = T;
};

// f(TypeTag<AttrT>{}) for the attribute dtype: __half for RFB_FLOAT16, else float
template <typename F>
auto with_attr_type(int attr_dtype, F &&f) {
    if (attr_dtype == RFB_FLOAT16)
        return f(TypeTag<__half>{});
    return f(TypeTag<float>{});
}

// The fast kernel and, right behind it, its exact twin (a no-op unless the fast one raised the flag);
// launch(std::integral_constant<int, MODE>{}) launches one of them.
template <typename F>
int launch_twins(F &&launch) {
    if (int rc = launch(std::integral_constant<int, rfb::kScanFast>{}))
        return rc;
    return launch(std::integral_constant<int, rfb::kScanExactTwin>{});
}

} // namespace

struct rfb_pipeline {
    int sh_degree;
    int attr_dtype;
    int device = -1;
    DeviceBuffer cells, sh_rows, faces, nbr, acc;
    SceneKey key;
    bool key_valid = false;
    // producer stream + completion event of the mirrors / of the tape: a consumer on another stream waits on it
    cudaStream_t scene_stream = nullptr, tape_stream = nullptr;
    cudaEvent_t scene_ready = nullptr, tape_ready = nullptr;
    // RFB_DEBUG=1: checksum of (points, attributes) taken when the mirrors were built, re-checked on every cache hit
    DeviceBuffer debug_sum;
    uint64_t scene_checksum = 0;
    uint32_t acc_points = 0;
    // caller-provided accumulator memory (rfb_set_grad_accumulator: a peer-mapped allocation for the fused
    // multi-GPU reduction); nullptr = the pipeline's own `acc`
    float *acc_external = nullptr;
    uint64_t acc_external_floats = 0;
    // parameter-form scene (rfb_bind_scene_params): attributes are derived from these inside the re-layout kernel
    rfb_scene_params params = {nullptr, nullptr, nullptr, 1.0f};
    bool params_bound = false;
    // walk tape (forward records, backward replays; see foam_kernels.cuh)
    DeviceBuffer scan_flag; // one word: a fast forward met a ray outside the ranked scan's domain (ScanMode)
    DeviceBuffer tape_pool, tape_table, tape_per_ray, tape_ctrl, tape_sched; // sched: [tile_steps | order]
    uint32_t tape_blocks = 0;
    bool tape_scheduled = false; // the last recording forward also built a tile order for the replay
    uint32_t tape_capacity = 0;      // chunks
    uint32_t tape_table_stride = 0;
    bool tape_valid = false;
    struct TapeKey {
        const void *rays = nullptr, *start = nullptr;
        uint32_t num_rays = 0, image_width = 0, max_steps = 0;
        float weight_threshold = 0.0f;
        uint64_t scene_version = 0;
    } tape_key;
    uint32_t *tape_readback = nullptr; // pinned host copy of ctrl, refreshed after every recording
    cudaEvent_t tape_readback_done = nullptr;
    bool tape_readback_pending = false;
    // optional live kernel timing (rfb_set_profiling): events around the ray kernels
    bool profiling = false;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr}; // fwd start/stop, bwd start/stop
    bool ev_valid[2] = {false, false};
};

namespace {

using namespace rfb;

int check_device(rfb_pipeline *p) {
    int dev = 0;
    RFB_CUDA(cudaGetDevice(&dev));
    if (p->device < 0)
        p->device = dev;
    else if (p->device != dev)
        return fail("pipeline was first used on CUDA device " + std::to_string(p->device) +
                    " but the current device is " + std::to_string(dev) +
                    " (create one pipeline per device)");
    return 0;
}

bool debug_checks() {
    static const bool on = [] {
        const char *e = getenv("RFB_DEBUG");
        return e && *e && *e != '0';
    }();
    return on;
}

// RFB_DEBUG only (synchronises): order-independent checksum of the caller's points and attributes
int scene_checksum(rfb_pipeline *p, uint32_t n, const float *points, const void *attrs, cudaStream_t stream,
                   uint64_t &out) {
    RFB_CUDA(p->debug_sum.ensure(sizeof(unsigned long long)));
    RFB_CUDA(cudaMemsetAsync(p->debug_sum.ptr, 0, sizeof(unsigned long long), stream));
    const int A = attr_dim(p->sh_degree);
    const uint64_t attr_words = (uint64_t)n * A * (p->attr_dtype == RFB_FLOAT16 ? 2 : 4) / 4;
    auto *sum = reinterpret_cast<unsigned long long *>(p->debug_sum.ptr);
    if (n) {
        RFB_LAUNCH((checksum_kernel), grid_for((uint64_t)n * 3, 256), 256, 0, stream,
                   reinterpret_cast<const uint32_t *>(points), (uint64_t)n * 3, sum);
        RFB_LAUNCH((checksum_kernel), grid_for(attr_words, 256), 256, 0, stream,
                   reinterpret_cast<const uint32_t *>(attrs), attr_words, sum);
    }
    unsigned long long host = 0;
    RFB_CUDA(cudaMemcpyAsync(&host, sum, sizeof(host), cudaMemcpyDeviceToHost, stream));
    RFB_CUDA(cudaStreamSynchronize(stream));
    out = host;
    return 0;
}

// Is `stream` being captured into a CUDA graph?  Then nothing host-visible may be attached to it: no events
// that the host (or another stream) later queries, no read-back.  A captured step replays with the buffers it
// was captured with; the library's bookkeeping (tape growth, cross-stream ordering) resumes outside the graph.
bool capturing(cudaStream_t stream) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &st) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return st != cudaStreamCaptureStatusNone;
}

// make `stream` wait for work recorded in `ev` on `producer` (no-op on the same stream)
int wait_for(cudaEvent_t ev, cudaStream_t producer, cudaStream_t stream) {
    if (ev && producer != stream && !capturing(stream))
        RFB_CUDA(cudaStreamWaitEvent(stream, ev, 0));
    return 0;
}

int mark(cudaEvent_t &ev, cudaStream_t &producer, cudaStream_t stream) {
    if (capturing(stream))
        return 0;
    if (!ev)
        RFB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    RFB_CUDA(cudaEventRecord(ev, stream));
    producer = stream;
    return 0;
}

// (Re)build the internal mirrors of the scene unless the caller vouches they are current.
int ensure_scene(rfb_pipeline *p, uint32_t n, const float *points, const void *attrs, uint32_t e,
                 const uint32_t *adj, const uint32_t *off, bool need_faces,
                 const rfb_launch_opts *opts, cudaStream_t stream, const void *caller_diff = nullptr) {
    if (int rc = check_device(p))
        return rc;
    SceneKey k;
    k.points = points;
    k.attrs = attrs;
    k.adj = adj;
    k.off = off;
    k.diff = caller_diff;
    k.n = n;
    k.e = e;
    k.version = opts ? opts->scene_version : 0;
    if (p->key_valid && k.version != 0 && k == p->key && (p->key.faces || !need_faces)) {
        if (debug_checks()) {
            uint64_t now = 0;
            if (int rc = scene_checksum(p, n, points, attrs, stream, now))
                return rc;
            if (now != p->scene_checksum)
                return fail("RFB_DEBUG: points/attributes changed but scene_version did not (stale scene mirrors; "
                            "bump rfb_launch_opts.scene_version whenever the scene tensors are written)");
        }
        return wait_for(p->scene_ready, p->scene_stream, stream);
    }
    p->key_valid = false;
    if (debug_checks())
        if (int rc = scene_checksum(p, n, points, attrs, stream, p->scene_checksum))
            return rc;

    const int A = attr_dim(p->sh_degree), SR = sh_row(p->sh_degree);
    RFB_CUDA(p->cells.ensure((size_t)n * sizeof(float4)));
    RFB_CUDA(p->sh_rows.ensure((size_t)n * SR * sizeof(float)));
    if (n && p->params_bound) {
        const int grid = grid_for((uint64_t)n * (SR / 4), 256 * 4, kNumSMs * 8);
        float4 *cells = reinterpret_cast<float4 *>(p->cells.ptr), *rows = reinterpret_cast<float4 *>(p->sh_rows.ptr);
        with_degree(p->sh_degree, [&](auto d) {
            with_attr_type(p->attr_dtype, [&](auto t) {
                RFB_LAUNCH((build_cells_params_kernel<typename decltype(t)::type, decltype(d)::value>), grid, 256, 0,
                           stream, points, p->params.att_dc, p->params.att_sh, p->params.density,
                           p->params.activation_scale, n, cells, rows);
            });
        });
        RFB_LAUNCHED();
    } else if (n) {
        const int grid = grid_for((uint64_t)n * (SR / 4), 256 * 4, kNumSMs * 8);
        float4 *cells = reinterpret_cast<float4 *>(p->cells.ptr), *rows = reinterpret_cast<float4 *>(p->sh_rows.ptr);
        with_degree(p->sh_degree, [&](auto d) {
            with_attr_type(p->attr_dtype, [&](auto t) {
                using AttrT = typename decltype(t)::type;
                RFB_LAUNCH((build_cells_kernel<AttrT, decltype(d)::value>), grid, 256, 0, stream, points,
                           reinterpret_cast<const AttrT *>(attrs), n, cells, rows);
            });
        });
        RFB_LAUNCHED();
    }
    if (need_faces) {
        size_t slots = (size_t)padded_slots(n, e); // rows padded to 4 faces, <= 3 slack per row
        RFB_CUDA(p->faces.ensure(slots * sizeof(uint2)));
        RFB_CUDA(p->nbr.ensure(slots * sizeof(uint32_t)));
        if (n && caller_diff) {
            RFB_LAUNCH((build_faces_from_diff_kernel), grid_for((uint64_t)n * 16, 256), 256, 0, stream,
                       reinterpret_cast<const uint2 *>(caller_diff), n, adj, off,
                       reinterpret_cast<uint2 *>(p->faces.ptr), reinterpret_cast<uint32_t *>(p->nbr.ptr));
            RFB_LAUNCHED();
        } else if (n) {
            RFB_LAUNCH((build_faces_kernel), grid_for((uint64_t)n * 16, 256), 256, 0, stream, points, n, adj,
                       off, reinterpret_cast<uint2 *>(p->faces.ptr),
                       reinterpret_cast<uint32_t *>(p->nbr.ptr));
            RFB_LAUNCHED();
        }
    }
    k.faces = need_faces;
    p->key = k;
    p->key_valid = true;
    return mark(p->scene_ready, p->scene_stream, stream);
}

void ray_grid(uint32_t num_rays, uint32_t image_width, uint32_t &blocks, uint32_t &blocks_x,
              uint32_t &width_used) {
    width_used = (image_width && num_rays % image_width == 0) ? image_width : 0;
    if (width_used) {
        uint32_t h = num_rays / width_used;
        blocks_x = (width_used + kTileW - 1) / kTileW;
        blocks = blocks_x * ((h + kTileH - 1) / kTileH);
    } else {
        blocks_x = 0;
        blocks = (num_rays + kBlock - 1) / kBlock;
    }
}

int profile_mark(rfb_pipeline *p, int which, cudaStream_t stream) {
    if (!p->profiling || capturing(stream))
        return 0;
    if (!p->ev[which])
        RFB_CUDA(cudaEventCreate(&p->ev[which]));
    RFB_CUDA(cudaEventRecord(p->ev[which], stream));
    if (which & 1)
        p->ev_valid[which >> 1] = true;
    return 0;
}

template <typename Faces>
int launch_forward(int deg, const ForwardParams &fp, const Faces &fa, uint32_t blocks, cudaStream_t stream) {
    auto launch = [&](auto mode) {
        return with_degree(deg, [&](auto d) {
            RFB_LAUNCH((forward_kernel<decltype(d)::value, Faces, decltype(mode)::value>), blocks, kBlock, 0, stream,
                       fp, fa);
            RFB_LAUNCHED();
            return 0;
        });
    };
    // with a contribution output (accumulated by atomics: a second pass would double it) one launch that chooses
    // per ray
    return fp.contrib ? launch(std::integral_constant<int, kScanPerRay>{}) : launch_twins(launch);
}

template <typename Faces>
int launch_forward_record(int deg, const ForwardParams &fp, const Faces &fa, const Tape &tape,
                          uint32_t blocks, cudaStream_t stream) {
    auto launch = [&](auto mode) {
        return with_degree(deg, [&](auto d) {
            RFB_LAUNCH((forward_record_kernel<decltype(d)::value, Faces, decltype(mode)::value>), blocks, kBlock, 0,
                       stream, fp, fa, tape);
            RFB_LAUNCHED();
            return 0;
        });
    };
    return fp.contrib ? launch(std::integral_constant<int, kScanPerRay>{}) : launch_twins(launch);
}

// The device view of the pipeline's tape buffers; `order` (the replay schedule) is left to the caller.
Tape pipeline_tape(const rfb_pipeline *p) {
    Tape tape = {};
    tape.pool = reinterpret_cast<uint2 *>(p->tape_pool.ptr);
    tape.table = reinterpret_cast<uint32_t *>(p->tape_table.ptr);
    tape.per_ray = reinterpret_cast<uint2 *>(p->tape_per_ray.ptr);
    tape.ctrl = reinterpret_cast<uint32_t *>(p->tape_ctrl.ptr);
    tape.capacity = p->tape_capacity;
    tape.table_stride = p->tape_table_stride;
    tape.tile_steps = reinterpret_cast<uint32_t *>(p->tape_sched.ptr);
    return tape;
}

// The walk's view of the pipeline's face mirror, with the caller's CSR offsets.
PaddedFaces padded_faces(const rfb_pipeline *p, const uint32_t *offsets) {
    PaddedFaces fa;
    fa.faces = reinterpret_cast<const uint2 *>(p->faces.ptr);
    fa.nbr = reinterpret_cast<const uint32_t *>(p->nbr.ptr);
    fa.off = offsets;
    return fa;
}

// Clears the exact-scan flag (ScanMode) a fast kernel raises for its twin and points `flag` at it.
int reset_exact_flag(rfb_pipeline *p, cudaStream_t stream, uint32_t *&flag) {
    RFB_CUDA(p->scan_flag.ensure(4 * sizeof(uint32_t)));
    RFB_CUDA(cudaMemsetAsync(p->scan_flag.ptr, 0, 4 * sizeof(uint32_t), stream));
    flag = reinterpret_cast<uint32_t *>(p->scan_flag.ptr);
    return 0;
}

// Size / reset the tape for a recording forward of `blocks` CTAs; fills `tape`.  The tape is an optimisation:
// when its memory cannot be had (the pool is a raw cudaMalloc next to the caller's own allocator), `ok` comes
// back false, the forward runs without recording and the backward re-walks.
int prepare_tape(rfb_pipeline *p, uint32_t blocks, uint32_t num_rays, uint32_t max_steps, Tape &tape,
                 cudaStream_t stream, bool &ok) {
    ok = false;
    const uint32_t num_warps = blocks * (kBlock / 32);
    const uint32_t stride = max_steps / kTapeChunk + 2;
    // grow the pool if the previous recording needed more chunks than it had
    // (no event query while a graph is being captured: "unsafe" runtime calls invalidate a global-mode capture)
    if (p->tape_readback_pending && !capturing(stream) && cudaEventQuery(p->tape_readback_done) == cudaSuccess) {
        p->tape_readback_pending = false;
        uint32_t wanted = p->tape_readback[0] > p->tape_readback[2] ? p->tape_readback[0] : p->tape_readback[2];
        if (wanted > p->tape_capacity)
            p->tape_capacity = wanted + wanted / 4;
    }
    uint64_t want = (uint64_t)num_warps; // first guess: one chunk (32 steps) per warp; grows on demand
    if (p->tape_capacity < want)
        p->tape_capacity = (uint32_t)(want < 0xFFFFFFF0ull ? want : 0xFFFFFFF0ull);
    const size_t chunk_bytes = (size_t)kTapeChunk * 32 * sizeof(uint2);
    size_t pool_bytes = (size_t)p->tape_capacity * chunk_bytes;
    if (pool_bytes > p->tape_pool.bytes) {
        // growing: never take more than half of what is free now (plus what the pool already holds)
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) {
            const size_t cap = (free_b + p->tape_pool.bytes) / 2;
            if (pool_bytes + pool_bytes / 16 + 256 > cap) {
                const uint64_t fit = cap / (chunk_bytes + chunk_bytes / 16 + 1);
                p->tape_capacity = (uint32_t)(fit < p->tape_capacity ? fit : p->tape_capacity);
                pool_bytes = (size_t)p->tape_capacity * chunk_bytes;
            }
        }
        cudaGetLastError();
    }
    if (p->tape_capacity < want || p->tape_pool.ensure(pool_bytes) != cudaSuccess ||
        p->tape_table.ensure((size_t)num_warps * stride * sizeof(uint32_t)) != cudaSuccess ||
        p->tape_per_ray.ensure((size_t)num_rays * sizeof(uint2)) != cudaSuccess ||
        p->tape_sched.ensure((size_t)blocks * 2 * sizeof(uint32_t)) != cudaSuccess ||
        p->tape_ctrl.ensure(4 * sizeof(uint32_t)) != cudaSuccess) {
        cudaGetLastError(); // out of memory is not sticky; forget it
        p->tape_capacity = 0; // start from the first guess next time
        return 0;
    }
    RFB_CUDA(cudaMemsetAsync(p->tape_ctrl.ptr, 0, 4 * sizeof(uint32_t), stream));
    p->tape_blocks = blocks;
    if (!p->tape_readback) {
        RFB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&p->tape_readback), 4 * sizeof(uint32_t)));
        RFB_CUDA(cudaEventCreateWithFlags(&p->tape_readback_done, cudaEventDisableTiming));
    }
    p->tape_table_stride = stride;
    tape = pipeline_tape(p);
    tape.order = tape.tile_steps + blocks;
    ok = true;
    return 0;
}

template <typename Faces>
int launch_backward(int deg, const BackwardParams &bp, const Faces &fa, const RayGradOut &rg, uint32_t blocks,
                    cudaStream_t stream) {
    auto launch = [&](auto ray) {
        return with_degree(deg, [&](auto d) {
            RFB_LAUNCH((backward_kernel<decltype(d)::value, Faces, decltype(ray)::value>), blocks, kBlock, 0, stream,
                       bp, fa, rg);
            RFB_LAUNCHED();
            return 0;
        });
    };
    return rg.ray_grad ? launch(std::true_type{}) : launch(std::false_type{});
}

template <int DEG, typename Faces, int SLOTS, int MIN_GROUP, int MIN_BLOCKS, bool REPLAY, bool RAY>
int launch_backward_cached_one(const BackwardParams &bp, const Faces &fa, const Tape &tape, const RayGradOut &rg,
                               uint32_t blocks, cudaStream_t stream) {
    constexpr int GR = grad_row(DEG);
    constexpr size_t smem = (size_t)(kBlock / 32) * ((32 * GR + SLOTS * GR + SLOTS + 3) & ~3) * sizeof(float);
    auto kernel = backward_cached_kernel<DEG, Faces, SLOTS, MIN_GROUP, MIN_BLOCKS, REPLAY, RAY>;
    // the attribute is per device and idempotent: set it once per (instantiation, device)
    static std::atomic<uint64_t> configured{0};
    int dev = 0;
    RFB_CUDA(cudaGetDevice(&dev));
    const uint64_t bit = 1ull << (dev & 63);
    if (!(configured.load(std::memory_order_relaxed) & bit)) {
        RFB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured.fetch_or(bit, std::memory_order_relaxed);
    }
    RFB_LAUNCH((kernel), blocks, kBlock, smem, stream, bp, fa, tape, rg);
    RFB_LAUNCHED();
    return 0;
}

// With a tape: the replay kernel and the re-walk kernel are both launched; the tape's overflow
// flag (device side) decides which one works.  Without: the re-walk kernel alone.
template <int DEG, typename Faces, int SLOTS, int MIN_GROUP, int MIN_BLOCKS, bool RAY>
int launch_backward_cached_cfg(const BackwardParams &bp, const Faces &fa, const Tape &tape, const RayGradOut &rg,
                               uint32_t blocks, cudaStream_t stream) {
    if (tape.pool)
        if (int rc = launch_backward_cached_one<DEG, Faces, SLOTS, MIN_GROUP, MIN_BLOCKS, true, RAY>(
                bp, fa, tape, rg, blocks, stream))
            return rc;
    return launch_backward_cached_one<DEG, Faces, SLOTS, MIN_GROUP, MIN_BLOCKS, false, RAY>(bp, fa, tape, rg,
                                                                                          blocks, stream);
}

// Shipped configuration: 4 cache slots per warp, groups of >= 6 lanes go through the cache, 5 CTAs/SM
// (<= 102 registers; the H100's 64 K registers per SM hold 5 CTAs of 128 threads at 96).  Fewer slots keep the
// per-warp staging small; 6 CTAs/SM would spill.  With 4 slots a CTA needs under 32 KB of shared memory, so 5 CTAs
// take about 150 KB of the H100's 228 KB per SM and the rest stays L1.
// Degree 3 gets 4 CTAs/SM (<= 128 registers): the row each lane holds until its next composited step (five values
// live across the step) made the 96-register build spill 108 bytes, and at 4 CTAs/SM the replay backward is 5 %
// faster on the bench frame (profiles/h100_backward_position_fold.json).
// With ray gradients (RAY) each thread also keeps its ray's sums (the G_k alone are (deg+1)^2 registers): those
// instantiations get fewer CTAs/SM, so that they do not spill -- 4 (<= 128 registers) for degrees 0-2 and 3
// (<= 168) for degree 3, which spills at 128.
template <int DEG, bool RAY>
constexpr int backward_min_blocks() { return !RAY ? (DEG == 3 ? 4 : 5) : DEG == 3 ? 3 : 4; }
template <typename Faces>
int launch_backward_cached(int deg, const BackwardParams &bp, const Faces &fa, const Tape &tape,
                           const RayGradOut &rg, uint32_t blocks, cudaStream_t stream) {
    auto launch = [&](auto ray) {
        return with_degree(deg, [&](auto d) {
            constexpr int DEG = decltype(d)::value;
            constexpr bool RAY = decltype(ray)::value;
            return launch_backward_cached_cfg<DEG, Faces, 4, 6, backward_min_blocks<DEG, RAY>(), RAY>(bp, fa, tape, rg,
                                                                                                  blocks, stream);
        });
    };
    return rg.ray_grad ? launch(std::true_type{}) : launch(std::false_type{});
}

template <typename Faces>
int launch_benchmark(int deg, const BenchmarkParams &bp, const Faces &fa, uint32_t blocks, cudaStream_t stream) {
    return launch_twins([&](auto mode) {
        return with_degree(deg, [&](auto d) {
            RFB_LAUNCH((benchmark_kernel<decltype(d)::value, Faces, decltype(mode)::value>), blocks, kBlock, 0, stream,
                       bp, fa);
            RFB_LAUNCHED();
            return 0;
        });
    });
}

template <typename Faces, typename Out>
int launch_visualization(int deg, const VisualizationParams &vp, const Faces &fa, const Out &out, uint32_t blocks,
                         cudaStream_t stream) {
    return launch_twins([&](auto mode) {
        return with_degree(deg, [&](auto d) {
            RFB_LAUNCH((visualization_kernel<decltype(d)::value, Faces, decltype(mode)::value, Out>), blocks, kBlock,
                       0, stream, vp, fa, out);
            RFB_LAUNCHED();
            return 0;
        });
    });
}

rfb_trace_settings settings_or_default(const rfb_trace_settings *s) {
    rfb_trace_settings d;
    d.weight_threshold = 0.001f; // default_trace_settings(), pipeline.h:15-20
    d.max_intersections = 1024;
    return s ? *s : d;
}

CameraParams camera_params(const rfb_camera *camera) {
    CameraParams c;
    memcpy(c.position, camera->position, sizeof(float) * 3);
    memcpy(c.forward, camera->forward, sizeof(float) * 3);
    memcpy(c.right, camera->right, sizeof(float) * 3);
    memcpy(c.up, camera->up, sizeof(float) * 3);
    c.fov = camera->fov;
    c.width = camera->width;
    c.height = camera->height;
    c.model = camera->model;
    return c;
}

// Scene mirrors for the entry points that take the caller's half4 adjacent_diff (trace_benchmark,
// trace_visualization).  The reference interface does not pass the adjacency size (pipeline.h:102-126); it is
// offsets[N].  Reading it costs a stream sync, paid only when the mirrors are (re)built.
int ensure_diff_scene(rfb_pipeline *p, uint32_t num_points, const float *points, const void *attributes,
                      const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets,
                      const void *adjacent_diff, const rfb_launch_opts *opts, cudaStream_t stream) {
    uint32_t num_edges = p->key_valid ? p->key.e : 0;
    {
        SceneKey probe;
        probe.points = points;
        probe.attrs = attributes;
        probe.adj = point_adjacency;
        probe.off = point_adjacency_offsets;
        probe.diff = adjacent_diff;
        probe.n = num_points;
        probe.e = num_edges;
        probe.version = opts ? opts->scene_version : 0;
        bool hit = p->key_valid && probe.version != 0 && probe == p->key && p->key.faces;
        if (!hit) {
            RFB_CUDA(cudaMemcpyAsync(&num_edges, point_adjacency_offsets + num_points, sizeof(uint32_t),
                                     cudaMemcpyDeviceToHost, stream));
            RFB_CUDA(cudaStreamSynchronize(stream));
        }
    }
    return ensure_scene(p, num_points, points, attributes, num_edges, point_adjacency, point_adjacency_offsets,
                        true, opts, stream, adjacent_diff);
}

// Shared body of rfb_trace_visualization{,_rgba8}: checks, mirrors, parameters, launch into `out`.
template <typename Out>
int trace_visualization(const char *fn, rfb_pipeline *p, const rfb_trace_settings *settings,
                        const rfb_visualization_settings *vis, const rfb_camera *camera,
                        const rfb_cmap_table *cmap_table, uint32_t num_points, const float *points,
                        const void *attributes, const uint32_t *point_adjacency,
                        const uint32_t *point_adjacency_offsets, const void *adjacent_diff, uint32_t start_index,
                        bool have_output, Out out, const rfb_launch_opts *opts, void *stream_) {
    const std::string name(fn);
    if (!p)
        return fail(name + ": pipeline is NULL");
    if (!vis || !camera || !points || !attributes || !point_adjacency || !point_adjacency_offsets ||
        !adjacent_diff || !have_output)
        return fail(name + ": NULL argument");
    if (vis->mode < RFB_VIS_RGB || vis->mode > RFB_VIS_INTERSECTIONS)
        return fail(name + ": unknown visualization mode " + std::to_string(vis->mode));
    if (vis->color_map < RFB_CMAP_GRAY || vis->color_map > RFB_CMAP_TURBO)
        return fail(name + ": unknown color map " + std::to_string(vis->color_map));
    const bool uses_cmap = vis->mode == RFB_VIS_DEPTH || vis->mode == RFB_VIS_INTERSECTIONS;
    if (uses_cmap && (!cmap_table || !cmap_table->data || !cmap_table->sizes))
        return fail(name + ": the depth and intersections modes need a color map table");
    if (camera->model != RFB_PINHOLE && camera->model != RFB_FISHEYE)
        return fail("Invalid camera model");
    if (start_index >= num_points)
        return fail(name + ": start_index is not a point of the scene");
    if (camera->width == 0 || camera->height == 0)
        return 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (int rc = ensure_diff_scene(p, num_points, points, attributes, point_adjacency, point_adjacency_offsets,
                                   adjacent_diff, opts, stream))
        return rc;
    rfb_trace_settings s = settings_or_default(settings);
    VisualizationParams vp;
    vp.cells = reinterpret_cast<const float4 *>(p->cells.ptr);
    vp.sh_rows = reinterpret_cast<const float *>(p->sh_rows.ptr);
    vp.cam = camera_params(camera);
    vp.start = start_index;
    vp.weight_threshold = s.weight_threshold;
    vp.max_steps = s.max_intersections;
    vp.mode = vis->mode;
    vp.color_map = vis->color_map;
    memcpy(vp.bg, vis->bg_color, sizeof(float) * 3);
    vp.checker_bg = vis->checker_bg;
    vp.max_depth = vis->max_depth;
    vp.depth_quantile = vis->depth_quantile;
    vp.cmap.data = uses_cmap ? cmap_table->data : nullptr;
    vp.cmap.sizes = uses_cmap ? cmap_table->sizes : nullptr;
    if (int rc = reset_exact_flag(p, stream, vp.exact_flag))
        return rc;
    vp.blocks_x = (camera->width + kTileW - 1) / kTileW;
    uint32_t blocks = vp.blocks_x * ((camera->height + kTileH - 1) / kTileH);
    return launch_visualization(p->sh_degree, vp, padded_faces(p, point_adjacency_offsets), out, blocks, stream);
}

} // namespace

extern "C" {

const char *rfb_last_error(void) { return g_last_error.c_str(); }
int rfb_abi_version(void) { return RFB_ABI_VERSION; }
uint64_t rfb_launch_count(void) { return g_launches.load(); }
void rfb_reset_launch_count(void) { g_launches.store(0); }
void rfb_device_alloc_counts(uint64_t *allocs, uint64_t *frees) {
    if (allocs)
        *allocs = g_device_allocs.load();
    if (frees)
        *frees = g_device_frees.load();
}

int rfb_create_pipeline(int sh_degree, int attr_dtype, rfb_pipeline **out) {
    if (!out)
        return fail("rfb_create_pipeline: out is NULL");
    *out = nullptr;
    if (attr_dtype != RFB_FLOAT32 && attr_dtype != RFB_FLOAT16)
        return fail("Unsupported attribute type");
    if (sh_degree < 0 || sh_degree > 3)
        return fail("Unsupported SH degree");
    rfb_pipeline *p = new (std::nothrow) rfb_pipeline();
    if (!p)
        return fail("out of host memory");
    p->sh_degree = sh_degree;
    p->attr_dtype = attr_dtype;
    *out = p;
    return 0;
}

void rfb_destroy_pipeline(rfb_pipeline *p) {
    if (!p)
        return;
    p->cells.release();
    p->sh_rows.release();
    p->faces.release();
    p->nbr.release();
    p->acc.release();
    p->scan_flag.release();
    p->tape_pool.release();
    p->tape_sched.release();
    p->tape_table.release();
    p->tape_per_ray.release();
    p->tape_ctrl.release();
    if (p->tape_readback)
        cudaFreeHost(p->tape_readback);
    if (p->tape_readback_done)
        cudaEventDestroy(p->tape_readback_done);
    for (auto &e : p->ev)
        if (e)
            cudaEventDestroy(e);
    if (p->scene_ready)
        cudaEventDestroy(p->scene_ready);
    if (p->tape_ready)
        cudaEventDestroy(p->tape_ready);
    p->debug_sum.release();
    delete p;
}

uint32_t rfb_attribute_dim(const rfb_pipeline *p) { return p ? (uint32_t)rfb::attr_dim(p->sh_degree) : 0; }
int rfb_attribute_type(const rfb_pipeline *p) { return p ? p->attr_dtype : -1; }
uint32_t rfb_grad_row_floats(const rfb_pipeline *p) { return p ? (uint32_t)rfb::grad_row(p->sh_degree) : 0; }
void rfb_invalidate_cache(rfb_pipeline *p) {
    if (p)
        p->key_valid = false;
}

int rfb_tape_status(rfb_pipeline *p, uint32_t *capacity_chunks, uint32_t *used_chunks,
                    uint32_t *overflowed) {
    if (!p || !capacity_chunks || !used_chunks || !overflowed)
        return fail("rfb_tape_status: NULL argument");
    if (!p->tape_valid || !p->tape_readback)
        return fail("rfb_tape_status: no recorded tape");
    RFB_CUDA(cudaEventSynchronize(p->tape_readback_done));
    *capacity_chunks = p->tape_capacity;
    *used_chunks = p->tape_readback[0] > p->tape_readback[2] ? p->tape_readback[0] : p->tape_readback[2];
    *overflowed = p->tape_readback[1];
    return 0;
}

void rfb_set_profiling(rfb_pipeline *p, int enabled) {
    if (p) {
        p->profiling = enabled != 0;
        p->ev_valid[0] = p->ev_valid[1] = false;
    }
}

int rfb_last_kernel_ms(rfb_pipeline *p, int which, float *ms) {
    if (!p || !ms || which < 0 || which > 1)
        return fail("rfb_last_kernel_ms: bad argument");
    if (!p->ev_valid[which])
        return fail("rfb_last_kernel_ms: no timed launch recorded (enable rfb_set_profiling first)");
    RFB_CUDA(cudaEventSynchronize(p->ev[2 * which + 1]));
    RFB_CUDA(cudaEventElapsedTime(ms, p->ev[2 * which], p->ev[2 * which + 1]));
    return 0;
}

int rfb_prefetch_adjacent_diff(const float *points, uint32_t num_points, uint32_t point_adjacency_size,
                               const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets,
                               void *adjacent_diff, void *stream) {
    (void)point_adjacency_size;
    if (num_points == 0)
        return 0;
    if (!points || !point_adjacency || !point_adjacency_offsets || !adjacent_diff)
        return fail("rfb_prefetch_adjacent_diff: NULL argument");
    RFB_LAUNCH((rfb::adjacent_diff_kernel), grid_for((uint64_t)num_points * 16, 256), 256, 0,
               (cudaStream_t)stream, points, num_points, point_adjacency, point_adjacency_offsets,
               reinterpret_cast<uint2 *>(adjacent_diff));
    RFB_LAUNCHED();
    return 0;
}

namespace {
// Stream-ordered scratch from the device's default memory pool; freed blocks stay in the pool (the default
// release threshold of 0 hands them back to the driver at the next synchronisation: ~2 ms per call measured).
int stream_scratch(void **ptr, size_t bytes, cudaStream_t stream) {
    static std::once_flag pool_once;
    std::call_once(pool_once, [] {
        int dev = 0;
        cudaMemPool_t pool = nullptr;
        uint64_t keep = ~0ull;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess)
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        cudaGetLastError();
    });
    if (cudaMallocAsync(ptr, bytes, stream) != cudaSuccess) {
        cudaGetLastError();
        return fail("out of device memory for " + std::to_string(bytes) + " bytes of scratch");
    }
    return 0;
}
} // namespace

int rfb_nearest_point(const float *points, uint32_t num_points, const float *queries,
                      uint32_t num_queries, uint32_t *indices, void *stream_) {
    if (num_queries == 0)
        return 0;
    if (!points || !queries || !indices)
        return fail("rfb_nearest_point: NULL argument");
    if (num_points == 0)
        return fail("rfb_nearest_point: empty point set");
    cudaStream_t stream = (cudaStream_t)stream_;
    unsigned long long *best = nullptr;
    if (int rc = stream_scratch(reinterpret_cast<void **>(&best), sizeof(unsigned long long) * num_queries, stream))
        return rc;
    cudaMemsetAsync(best, 0xFF, sizeof(unsigned long long) * num_queries, stream);
    const int grid = grid_for((uint64_t)num_points, rfb::kNNTile, kNumSMs * 4);
    RFB_LAUNCH((rfb::nearest_points_kernel), grid, 256, 0, stream, points, num_points, queries, num_queries,
               (const uint32_t *)nullptr, best);
    RFB_LAUNCH((rfb::nearest_points_finish_kernel), (num_queries + 255) / 256, 256, 0, stream, best, num_queries,
               indices);
    g_launches += 2;
    const cudaError_t launched = cudaGetLastError();
    cudaFreeAsync(best, stream); // stream-ordered: after the kernels above, also on the error path
    RFB_CUDA(launched);
    return 0;
}

int rfb_start_points(const float *points, uint32_t num_points, const float *rays, uint32_t num_rays,
                     uint32_t *start_point_index, void *stream_) {
    if (num_rays == 0)
        return 0;
    if (!points || !rays || !start_point_index)
        return fail("rfb_start_points: NULL argument");
    if (num_points == 0)
        return fail("rfb_start_points: empty point set");
    if (num_rays > 0x7FFFFFF0u)
        return fail("rfb_start_points: too many rays");
    cudaStream_t stream = (cudaStream_t)stream_;
    uint32_t table_size = 1024;
    while (table_size < 2u * num_rays)
        table_size <<= 1;
    // one scratch block: [best: R x u64][queries: R x 3 f32][table: T u32][query_of_slot: T u32]
    //                    [slot_of_ray: R u32][count: 4 u32]
    const size_t best_b = sizeof(unsigned long long) * (size_t)num_rays, query_b = 12 * (size_t)num_rays,
                 table_b = 4 * (size_t)table_size, slot_b = 4 * (size_t)num_rays;
    char *base = nullptr;
    if (int rc = stream_scratch(reinterpret_cast<void **>(&base), best_b + query_b + 2 * table_b + slot_b + 16, stream))
        return rc;
    auto *best = reinterpret_cast<unsigned long long *>(base);
    auto *queries = reinterpret_cast<float *>(base + best_b);
    auto *table = reinterpret_cast<uint32_t *>(base + best_b + query_b);
    auto *query_of_slot = table + table_size;
    auto *slot_of_ray = query_of_slot + table_size;
    auto *count = slot_of_ray + num_rays;
    cudaMemsetAsync(best, 0xFF, best_b, stream);
    cudaMemsetAsync(table, 0, table_b, stream);
    cudaMemsetAsync(count, 0, 16, stream);
    const uint32_t ray_grid = (num_rays + 255) / 256;
    RFB_LAUNCH((rfb::origin_slots_kernel), ray_grid, 256, 0, stream, rays, num_rays, table, table_size - 1,
               slot_of_ray, query_of_slot, queries, count);
    RFB_LAUNCH((rfb::nearest_points_kernel), grid_for((uint64_t)num_points, rfb::kNNTile, kNumSMs * 4), 256, 0, stream,
               points, num_points, (const float *)queries, 0u, (const uint32_t *)count, best);
    RFB_LAUNCH((rfb::start_points_scatter_kernel), ray_grid, 256, 0, stream, (const uint32_t *)slot_of_ray, num_rays,
               (const uint32_t *)query_of_slot, (const unsigned long long *)best, start_point_index);
    g_launches += 3;
    const cudaError_t launched = cudaGetLastError();
    cudaFreeAsync(base, stream);
    RFB_CUDA(launched);
    return 0;
}

int rfb_farthest_neighbor(const float *points, uint32_t num_points, const uint32_t *point_adjacency,
                          const uint32_t *point_adjacency_offsets, uint32_t *indices, float *cell_radius,
                          void *stream_) {
    if (num_points == 0)
        return 0;
    if (!points || !point_adjacency_offsets || !indices || !cell_radius)
        return fail("rfb_farthest_neighbor: NULL argument");
    // point_adjacency may be NULL only when every row is empty; the kernels never read it then
    cudaStream_t stream = (cudaStream_t)stream_;
    const uint32_t grid = (uint32_t)(((uint64_t)num_points + 255) / 256);
    RFB_LAUNCH((rfb::farthest_neighbor_kernel), grid, 256, 0, stream, points, point_adjacency,
               point_adjacency_offsets, num_points, indices, cell_radius);
    RFB_LAUNCHED();
    return 0;
}

} // extern "C"

namespace {
// Points in the seed sample of rfb_locate_points (DESIGN.md §4: the measured trade-off between the sample scan every
// query pays and the walk it shortens).  RFB_LOCATE_SAMPLE overrides it per call, for measuring that trade-off and
// for tests that want long walks on small foams; on a Delaunay adjacency the results do not depend on it (up to
// fp32 near-ties).
constexpr uint32_t kLocateSample = 2048;

LocateParams locate_params(const float *points, uint32_t num_points, const uint32_t *adj, const uint32_t *off,
                           const float *queries, uint32_t num_queries, const uint32_t *hints) {
    const char *e = getenv("RFB_LOCATE_SAMPLE");
    const long v = e ? atol(e) : 0;
    const uint32_t sample = v > 0 && v < (1l << 30) ? (uint32_t)v : kLocateSample;
    LocateParams lp;
    lp.points = points;
    lp.adj = adj;
    lp.off = off;
    lp.queries = queries;
    lp.hints = hints;
    lp.num_points = num_points;
    lp.num_queries = num_queries;
    lp.sample = sample < num_points ? sample : num_points;
    lp.stride = num_points / lp.sample;
    return lp;
}
} // namespace

extern "C" {

int rfb_locate_points(const float *points, uint32_t num_points, const uint32_t *point_adjacency,
                      const uint32_t *point_adjacency_offsets, const float *queries, uint32_t num_queries,
                      const uint32_t *hints, uint32_t *indices, void *stream) {
    if (num_queries == 0)
        return 0;
    // point_adjacency may be NULL only when every row is empty; the kernel never reads it then
    if (!points || !point_adjacency_offsets || !queries || !indices)
        return fail("rfb_locate_points: NULL argument");
    if (num_points == 0)
        return fail("rfb_locate_points: empty point set");
    const LocateParams lp = locate_params(points, num_points, point_adjacency, point_adjacency_offsets, queries,
                                          num_queries, hints);
    RFB_LAUNCH((rfb::locate_points_kernel), (num_queries + 255) / 256, 256, 0, (cudaStream_t)stream, lp, indices);
    RFB_LAUNCHED();
    return 0;
}

int rfb_sample_field(rfb_pipeline *p, const float *points, uint32_t num_points, const void *attributes,
                     const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets, const float *queries,
                     uint32_t num_queries, const uint32_t *hints, const float *directions, uint32_t *cells,
                     void *density, void *rgb, void *stream) {
    if (!p)
        return fail("rfb_sample_field: pipeline is NULL");
    if ((directions == nullptr) != (rgb == nullptr))
        return fail("rfb_sample_field: directions and rgb must both be given or both be NULL");
    if (num_queries == 0)
        return 0;
    if (!points || !attributes || !point_adjacency_offsets || !queries || !cells || !density)
        return fail("rfb_sample_field: NULL argument");
    if (num_points == 0)
        return fail("rfb_sample_field: empty point set");
    const LocateParams lp = locate_params(points, num_points, point_adjacency, point_adjacency_offsets, queries,
                                          num_queries, hints);
    with_degree(p->sh_degree, [&](auto d) {
        with_attr_type(p->attr_dtype, [&](auto t) {
            using AttrT = typename decltype(t)::type;
            RFB_LAUNCH((sample_field_kernel<decltype(d)::value, AttrT>), (num_queries + 255) / 256, 256, 0,
                       (cudaStream_t)stream, lp, reinterpret_cast<const AttrT *>(attributes), directions, cells,
                       reinterpret_cast<AttrT *>(density), reinterpret_cast<AttrT *>(rgb));
        });
    });
    RFB_LAUNCHED();
    return 0;
}

int rfb_sample_field_backward(rfb_pipeline *p, uint32_t num_points, uint32_t num_queries, const uint32_t *cells,
                              const float *directions, const void *rgb, const void *rgb_grad,
                              const void *density_grad, void *attribute_grad, void *stream_) {
    if (!p)
        return fail("rfb_sample_field_backward: pipeline is NULL");
    if (rgb_grad && (!directions || !rgb))
        return fail("rfb_sample_field_backward: rgb_grad needs the directions and the forward's rgb");
    if (num_points == 0)
        return 0;
    if (!attribute_grad || (num_queries && !cells))
        return fail("rfb_sample_field_backward: NULL argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    const uint64_t entries = (uint64_t)num_points * attr_dim(p->sh_degree);
    const bool half = p->attr_dtype == RFB_FLOAT16;
    // fp32 attributes: accumulate in place; fp16: in stream-ordered fp32 scratch, rounded once at the end
    float *acc = reinterpret_cast<float *>(attribute_grad);
    if (half)
        if (int rc = stream_scratch(reinterpret_cast<void **>(&acc), entries * sizeof(float), stream))
            return rc;
    cudaMemsetAsync(acc, 0, entries * sizeof(float), stream);
    if (num_queries) {
        with_degree(p->sh_degree, [&](auto d) {
            with_attr_type(p->attr_dtype, [&](auto t) {
                using AttrT = typename decltype(t)::type;
                RFB_LAUNCH((sample_field_backward_kernel<decltype(d)::value, AttrT>),
                           (num_queries + kSampleBwdBlock - 1) / kSampleBwdBlock, kSampleBwdBlock, 0, stream, cells,
                           num_queries, num_points, directions, reinterpret_cast<const AttrT *>(rgb),
                           reinterpret_cast<const AttrT *>(rgb_grad), reinterpret_cast<const AttrT *>(density_grad),
                           acc);
            });
        });
        ++g_launches;
    }
    if (half) {
        RFB_LAUNCH((round_to_half_kernel), grid_for(entries, 256), 256, 0, stream, (const float *)acc, entries,
                   reinterpret_cast<__half *>(attribute_grad));
        ++g_launches;
    }
    const cudaError_t launched = cudaGetLastError();
    if (half)
        cudaFreeAsync(acc, stream); // stream-ordered: after the kernels above, also on the error path
    RFB_CUDA(launched);
    return 0;
}

int rfb_trace_forward(rfb_pipeline *p, const rfb_trace_settings *settings, uint32_t num_points,
                      const float *points, const void *attributes, uint32_t point_adjacency_size,
                      const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets,
                      uint32_t num_rays, const float *rays, const uint32_t *start_point_index,
                      uint32_t num_depth_quantiles, const float *depth_quantiles, void *ray_rgba,
                      float *quantile_depths, uint32_t *quantile_point_indices,
                      uint32_t *num_intersections, void *point_contribution,
                      const rfb_launch_opts *opts, void *stream_) {
    if (!p)
        return fail("rfb_trace_forward: pipeline is NULL");
    if (num_rays == 0)
        return 0;
    if (p->params_bound)
        attributes = p->params.density; // identity for the mirror cache; the values come from the bound parameters
    if (!points || !attributes || !point_adjacency || !point_adjacency_offsets || !rays ||
        !start_point_index || !ray_rgba)
        return fail("rfb_trace_forward: NULL argument");
    if (depth_quantiles && num_depth_quantiles && (!quantile_depths || !quantile_point_indices))
        return fail("rfb_trace_forward: depth_quantiles given without output buffers");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (int rc = ensure_scene(p, num_points, points, attributes, point_adjacency_size, point_adjacency,
                              point_adjacency_offsets, true, opts, stream))
        return rc;
    rfb_trace_settings s = settings_or_default(settings);
    ForwardParams fp;
    fp.cells = reinterpret_cast<const float4 *>(p->cells.ptr);
    fp.sh_rows = reinterpret_cast<const float *>(p->sh_rows.ptr);
    fp.rays = rays;
    fp.start = start_point_index;
    fp.quantiles = num_depth_quantiles ? depth_quantiles : nullptr;
    fp.rgba = ray_rgba;
    fp.qdepth = quantile_depths;
    fp.qidx = quantile_point_indices;
    fp.nint = num_intersections;
    fp.contrib = point_contribution;
    fp.num_rays = num_rays;
    fp.num_q = num_depth_quantiles;
    fp.weight_threshold = s.weight_threshold;
    fp.max_steps = s.max_intersections;
    fp.out_half = p->attr_dtype == RFB_FLOAT16;
    uint32_t blocks;
    ray_grid(num_rays, opts ? opts->image_width : 0, blocks, fp.blocks_x, fp.image_width);
    const PaddedFaces fa = padded_faces(p, point_adjacency_offsets);
    if (int rc = reset_exact_flag(p, stream, fp.exact_flag))
        return rc;
    bool record = opts && (opts->flags & RFB_FLAG_RECORD_TAPE) && opts->scene_version != 0;
    p->tape_valid = false;
    Tape tape = {};
    if (record)
        if (int rc = prepare_tape(p, blocks, num_rays, s.max_intersections, tape, stream, record))
            return rc;
    if (int rc = profile_mark(p, 0, stream))
        return rc;
    if (int rc = record ? launch_forward_record(p->sh_degree, fp, fa, tape, blocks, stream)
                        : launch_forward(p->sh_degree, fp, fa, blocks, stream))
        return rc;
    if (int rc = profile_mark(p, 1, stream))
        return rc;
    if (record) {
        // the replay's longest-first schedule (small launches only: see tape_order_kernel)
        const char *sched = getenv("RFB_REPLAY_ORDER"); // "0" never, "1" always (for measuring)
        p->tape_scheduled = sched ? sched[0] == '1' : blocks <= kNumSMs * 5u * 8u;
        if (p->tape_scheduled) {
            RFB_LAUNCH((tile_steps_kernel), (blocks + 7) / 8, 256, 0, stream, (const uint2 *)tape.per_ray, num_rays,
                       fp.image_width, fp.blocks_x, blocks, tape.tile_steps);
            RFB_LAUNCH((tape_order_kernel), 1, 1024, 0, stream, (const uint32_t *)tape.tile_steps, blocks, blocks,
                       tape.order);
            g_launches += 1;
            RFB_LAUNCHED();
        }
        if (!capturing(stream)) {
            RFB_CUDA(cudaMemcpyAsync(p->tape_readback, p->tape_ctrl.ptr, 4 * sizeof(uint32_t),
                                     cudaMemcpyDeviceToHost, stream));
            RFB_CUDA(cudaEventRecord(p->tape_readback_done, stream));
            p->tape_readback_pending = true;
        }
        p->tape_key.rays = rays;
        p->tape_key.start = start_point_index;
        p->tape_key.num_rays = num_rays;
        p->tape_key.image_width = fp.image_width;
        p->tape_key.max_steps = s.max_intersections;
        p->tape_key.weight_threshold = s.weight_threshold;
        p->tape_key.scene_version = opts->scene_version;
        p->tape_valid = true;
        if (int rc = mark(p->tape_ready, p->tape_stream, stream))
            return rc;
    }
    return 0;
}

int rfb_trace_backward_accumulate(rfb_pipeline *p, const rfb_trace_settings *settings,
                                  uint32_t num_points, const float *points, const void *attributes,
                                  uint32_t point_adjacency_size, const uint32_t *point_adjacency,
                                  const uint32_t *point_adjacency_offsets, uint32_t num_rays,
                                  const float *rays, const uint32_t *start_point_index,
                                  uint32_t num_depth_quantiles, const float *depth_quantiles,
                                  const uint32_t *quantile_point_indices, const void *ray_rgba,
                                  const void *ray_rgba_grad, const float *depth_grad,
                                  const void *ray_error, void *point_error,
                                  const rfb_launch_opts *opts, void *stream) {
    return rfb_trace_backward_accumulate_rays(p, settings, num_points, points, attributes, point_adjacency_size,
                                              point_adjacency, point_adjacency_offsets, num_rays, rays,
                                              start_point_index, num_depth_quantiles, depth_quantiles,
                                              quantile_point_indices, ray_rgba, ray_rgba_grad, depth_grad, ray_error,
                                              point_error, nullptr, opts, stream);
}

int rfb_trace_backward_accumulate_rays(rfb_pipeline *p, const rfb_trace_settings *settings,
                                       uint32_t num_points, const float *points, const void *attributes,
                                       uint32_t point_adjacency_size, const uint32_t *point_adjacency,
                                       const uint32_t *point_adjacency_offsets, uint32_t num_rays,
                                       const float *rays, const uint32_t *start_point_index,
                                       uint32_t num_depth_quantiles, const float *depth_quantiles,
                                       const uint32_t *quantile_point_indices, const void *ray_rgba,
                                       const void *ray_rgba_grad, const float *depth_grad,
                                       const void *ray_error, void *point_error, float *ray_grad,
                                       const rfb_launch_opts *opts, void *stream_) {
    if (!p)
        return fail("rfb_trace_backward: pipeline is NULL");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (int rc = check_device(p))
        return rc;
    const int GR = grad_row(p->sh_degree);
    size_t acc_bytes = (size_t)num_points * GR * sizeof(float);
    float *acc_ptr = p->acc_external;
    if (acc_ptr) {
        if ((uint64_t)num_points * GR > p->acc_external_floats)
            return fail("rfb_trace_backward: the accumulator given to rfb_set_grad_accumulator is too small");
    } else {
        RFB_CUDA(p->acc.ensure(acc_bytes));
        acc_ptr = reinterpret_cast<float *>(p->acc.ptr);
    }
    RFB_CUDA(cudaMemsetAsync(acc_ptr, 0, acc_bytes, stream));
    p->acc_points = num_points;
    if (num_rays == 0)
        return 0;
    if (p->params_bound)
        attributes = p->params.density;
    if (!points || !attributes || !point_adjacency || !point_adjacency_offsets || !rays ||
        !start_point_index || !ray_rgba || !ray_rgba_grad)
        return fail("rfb_trace_backward: NULL argument");
    if (depth_quantiles && num_depth_quantiles && (!quantile_point_indices || !depth_grad))
        return fail("depth_grad must be provided if depth_quantiles is provided");
    if (int rc = ensure_scene(p, num_points, points, attributes, point_adjacency_size, point_adjacency,
                              point_adjacency_offsets, true, opts, stream))
        return rc;
    rfb_trace_settings s = settings_or_default(settings);
    BackwardParams bp;
    bp.cells = reinterpret_cast<const float4 *>(p->cells.ptr);
    bp.sh_rows = reinterpret_cast<const float *>(p->sh_rows.ptr);
    bp.rays = rays;
    bp.start = start_point_index;
    bp.quantiles = num_depth_quantiles ? depth_quantiles : nullptr;
    bp.qidx = quantile_point_indices;
    bp.rgba = ray_rgba;
    bp.rgba_grad = ray_rgba_grad;
    bp.depth_grad = depth_grad;
    bp.ray_error = ray_error;
    bp.point_error = ray_error ? point_error : nullptr;
    bp.acc = acc_ptr;
    bp.num_rays = num_rays;
    bp.num_q = num_depth_quantiles;
    bp.weight_threshold = s.weight_threshold;
    bp.max_steps = s.max_intersections;
    bp.io_half = p->attr_dtype == RFB_FLOAT16;
    uint32_t blocks;
    ray_grid(num_rays, opts ? opts->image_width : 0, blocks, bp.blocks_x, bp.image_width);
    const PaddedFaces fa = padded_faces(p, point_adjacency_offsets);
    if (int rc = profile_mark(p, 2, stream))
        return rc;
    const char *mode = getenv("RFB_BWD_MODE"); // "direct" | "cached" (experiment switch)
    bool cached = mode ? strcmp(mode, "direct") != 0 : true;
    // replay the forward's walk tape when the caller vouches the inputs are those of the last
    // recording forward (and everything the walk depends on matches)
    Tape tape = {};
    const rfb_pipeline::TapeKey &tk = p->tape_key;
    if (cached && opts && (opts->flags & RFB_FLAG_USE_TAPE) && p->tape_valid && opts->scene_version != 0 &&
        tk.scene_version == opts->scene_version && tk.rays == rays && tk.start == start_point_index &&
        tk.num_rays == num_rays && tk.image_width == bp.image_width && tk.max_steps == s.max_intersections &&
        tk.weight_threshold == s.weight_threshold) {
        tape = pipeline_tape(p);
        tape.order = (blocks == p->tape_blocks && p->tape_scheduled) ? tape.tile_steps + blocks : nullptr;
        if (int rc = wait_for(p->tape_ready, p->tape_stream, stream))
            return rc;
    }
    RayGradOut rg;
    rg.ray_grad = ray_grad;
    rg.scrub = (opts && (opts->flags & RFB_FLAG_SCRUB_NONFINITE)) ? 1 : 0;
    if (int rc = cached ? launch_backward_cached(p->sh_degree, bp, fa, tape, rg, blocks, stream)
                        : launch_backward(p->sh_degree, bp, fa, rg, blocks, stream))
        return rc;
    return profile_mark(p, 3, stream);
}

int rfb_grad_accumulator(rfb_pipeline *p, float **ptr, uint64_t *num_floats) {
    if (!p || !ptr || !num_floats)
        return fail("rfb_grad_accumulator: NULL argument");
    *ptr = p->acc_external ? p->acc_external : reinterpret_cast<float *>(p->acc.ptr);
    *num_floats = (uint64_t)p->acc_points * grad_row(p->sh_degree);
    return 0;
}

int rfb_set_grad_accumulator(rfb_pipeline *p, float *ptr, uint64_t num_floats) {
    if (!p)
        return fail("rfb_set_grad_accumulator: pipeline is NULL");
    if (ptr && (reinterpret_cast<uintptr_t>(ptr) & 15u))
        return fail("rfb_set_grad_accumulator: the accumulator must be 16-byte aligned");
    p->acc_external = ptr;
    p->acc_external_floats = ptr ? num_floats : 0;
    p->acc_points = 0;
    return 0;
}

int rfb_reduce_finalize_peers(rfb_pipeline *p, uint32_t world, uint32_t rank, uint32_t num_points,
                              const float *const *peer_acc, void *const *peer_attribute_grad,
                              float *const *peer_points_grad, const rfb_multicast *multicast, uint32_t flags,
                              void *stream_) {
    if (!p || !peer_acc || !peer_attribute_grad || !peer_points_grad)
        return fail("rfb_reduce_finalize_peers: NULL argument");
    if (multicast && (!multicast->acc || !multicast->attribute_grad || !multicast->points_grad))
        return fail("rfb_reduce_finalize_peers: incomplete multicast addresses");
    if (multicast && ((reinterpret_cast<uintptr_t>(multicast->acc) | reinterpret_cast<uintptr_t>(multicast->attribute_grad) |
                       reinterpret_cast<uintptr_t>(multicast->points_grad)) & 15u))
        return fail("rfb_reduce_finalize_peers: multicast addresses must be 16-byte aligned");
    if (world == 0 || world > (uint32_t)kMaxPeers || rank >= world)
        return fail("rfb_reduce_finalize_peers: world must be 1.." + std::to_string(kMaxPeers) + " and rank < world");
    if (num_points == 0)
        return 0;
    PeerReduceParams pr;
    for (uint32_t w = 0; w < world; ++w) {
        if (!peer_acc[w] || !peer_attribute_grad[w] || !peer_points_grad[w])
            return fail("rfb_reduce_finalize_peers: NULL peer pointer");
        if ((reinterpret_cast<uintptr_t>(peer_acc[w]) | reinterpret_cast<uintptr_t>(peer_attribute_grad[w]) |
             reinterpret_cast<uintptr_t>(peer_points_grad[w])) & 15u)
            return fail("rfb_reduce_finalize_peers: peer arrays must be 16-byte aligned");
        pr.acc[w] = peer_acc[w];
        pr.attr_grad[w] = peer_attribute_grad[w];
        pr.points_grad[w] = peer_points_grad[w];
    }
    pr.world = world;
    pr.num_points = num_points;
    // this rank's share: whole blocks of kPeerRows rows, dealt round-robin so that every rank streams from
    // the whole array (no rank's HBM serves one reader only)
    const uint32_t num_blocks = (num_points + kPeerRows - 1) / kPeerRows;
    pr.first_block = rank;
    pr.block_stride = world;
    pr.scrub = (flags & RFB_FLAG_SCRUB_NONFINITE) ? 1 : 0;
    pr.rank = rank;
    const char *dbg = getenv("RFB_PEER_DEBUG");
    pr.debug_mode = dbg ? atoi(dbg) : 0;
    pr.mc_acc = multicast ? multicast->acc : nullptr;
    pr.mc_attr_grad = multicast ? multicast->attribute_grad : nullptr;
    pr.mc_points_grad = multicast ? multicast->points_grad : nullptr;
    const uint32_t mine = (num_blocks + world - 1 - rank) / world;
    if (mine == 0)
        return 0;
    int grid = (int)(mine < kNumSMs * 16u ? mine : kNumSMs * 16u);
    cudaStream_t stream = (cudaStream_t)stream_;
    with_degree(p->sh_degree, [&](auto d) {
        with_attr_type(p->attr_dtype, [&](auto t) {
            constexpr int DEG = decltype(d)::value;
            using AttrT = typename decltype(t)::type;
            switch (world) {
            case 2: RFB_LAUNCH((reduce_finalize_peers_kernel<DEG, AttrT, 2>), grid, 256, 0, stream, pr); break;
            case 4: RFB_LAUNCH((reduce_finalize_peers_kernel<DEG, AttrT, 4>), grid, 256, 0, stream, pr); break;
            case 8: RFB_LAUNCH((reduce_finalize_peers_kernel<DEG, AttrT, 8>), grid, 256, 0, stream, pr); break;
            default: RFB_LAUNCH((reduce_finalize_peers_kernel<DEG, AttrT, 0>), grid, 256, 0, stream, pr); break;
            }
        });
    });
    RFB_LAUNCHED();
    return 0;
}

int rfb_trace_backward_finalize(rfb_pipeline *p, uint32_t num_points, float *points_grad,
                                void *attribute_grad, uint32_t flags, void *stream_) {
    if (!p)
        return fail("rfb_trace_backward_finalize: pipeline is NULL");
    if (num_points == 0)
        return 0;
    if (!points_grad || !attribute_grad)
        return fail("rfb_trace_backward_finalize: NULL argument");
    if (num_points != p->acc_points)
        return fail("rfb_trace_backward_finalize: no accumulated gradients for this point count");
    cudaStream_t stream = (cudaStream_t)stream_;
    const int A = attr_dim(p->sh_degree);
    const int grid = grid_for((uint64_t)num_points * A, 256 * 4, kNumSMs * 8);
    int scrub = (flags & RFB_FLAG_SCRUB_NONFINITE) ? 1 : 0;
    const float *acc_ptr = p->acc_external ? p->acc_external : reinterpret_cast<const float *>(p->acc.ptr);
    with_degree(p->sh_degree, [&](auto d) {
        with_attr_type(p->attr_dtype, [&](auto t) {
            using AttrT = typename decltype(t)::type;
            RFB_LAUNCH((finalize_grads_kernel<AttrT, decltype(d)::value>), grid, 256, 0, stream, acc_ptr, num_points,
                       points_grad, reinterpret_cast<AttrT *>(attribute_grad), scrub);
        });
    });
    RFB_LAUNCHED();
    return 0;
}

int rfb_bind_scene_params(rfb_pipeline *p, const rfb_scene_params *params) {
    if (!p)
        return fail("rfb_bind_scene_params: pipeline is NULL");
    p->key_valid = false;
    if (!params) {
        p->params_bound = false;
        return 0;
    }
    if (!params->att_dc || !params->density || (p->sh_degree > 0 && !params->att_sh))
        return fail("rfb_bind_scene_params: NULL parameter array");
    p->params = *params;
    p->params_bound = true;
    return 0;
}

int rfb_trace_backward_finalize_params(rfb_pipeline *p, uint32_t num_points, float *points_grad,
                                       float *att_dc_grad, float *att_sh_grad, float *density_grad,
                                       uint32_t flags, void *stream_) {
    if (!p)
        return fail("rfb_trace_backward_finalize_params: pipeline is NULL");
    if (!p->params_bound)
        return fail("rfb_trace_backward_finalize_params: no parameter-form scene is bound");
    if (num_points == 0)
        return 0;
    if (!points_grad || !att_dc_grad || !density_grad || (p->sh_degree > 0 && !att_sh_grad))
        return fail("rfb_trace_backward_finalize_params: NULL argument");
    if (num_points != p->acc_points)
        return fail("rfb_trace_backward_finalize_params: no accumulated gradients for this point count");
    cudaStream_t stream = (cudaStream_t)stream_;
    const int A = attr_dim(p->sh_degree);
    const int grid = grid_for((uint64_t)num_points * A, 256 * 4, kNumSMs * 8);
    int scrub = (flags & RFB_FLAG_SCRUB_NONFINITE) ? 1 : 0;
    const float *acc_ptr = p->acc_external ? p->acc_external : reinterpret_cast<const float *>(p->acc.ptr);
    with_degree(p->sh_degree, [&](auto d) {
        with_attr_type(p->attr_dtype, [&](auto t) {
            RFB_LAUNCH((finalize_params_kernel<typename decltype(t)::type, decltype(d)::value>), grid, 256, 0, stream,
                       acc_ptr, p->params.density, p->params.activation_scale, num_points, points_grad, att_dc_grad,
                       att_sh_grad, density_grad, scrub);
        });
    });
    RFB_LAUNCHED();
    return 0;
}

int rfb_trace_backward(rfb_pipeline *p, const rfb_trace_settings *settings, uint32_t num_points,
                       const float *points, const void *attributes, uint32_t point_adjacency_size,
                       const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets,
                       uint32_t num_rays, const float *rays, const uint32_t *start_point_index,
                       uint32_t num_depth_quantiles, const float *depth_quantiles,
                       const uint32_t *quantile_point_indices, const void *ray_rgba,
                       const void *ray_rgba_grad, const float *depth_grad, const void *ray_error,
                       float *ray_grad, float *points_grad, void *attribute_grad, void *point_error,
                       const rfb_launch_opts *opts, void *stream) {
    if (p && p->params_bound)
        return fail("rfb_trace_backward: a parameter-form scene is bound; use rfb_trace_backward_accumulate + "
                    "rfb_trace_backward_finalize_params");
    // without RFB_FLAG_RAY_GRAD ray_grad is not written, like the reference kernel (SURVEY.md A.5 quirk 4)
    const bool want_rays = opts && (opts->flags & RFB_FLAG_RAY_GRAD);
    if (want_rays && !ray_grad)
        return fail("rfb_trace_backward: RFB_FLAG_RAY_GRAD is set but ray_grad is NULL");
    if (int rc = rfb_trace_backward_accumulate_rays(
            p, settings, num_points, points, attributes, point_adjacency_size, point_adjacency,
            point_adjacency_offsets, num_rays, rays, start_point_index, num_depth_quantiles,
            depth_quantiles, quantile_point_indices, ray_rgba, ray_rgba_grad, depth_grad, ray_error,
            point_error, want_rays ? ray_grad : nullptr, opts, stream))
        return rc;
    return rfb_trace_backward_finalize(p, num_points, points_grad, attribute_grad,
                                       opts ? opts->flags : 0, stream);
}

int rfb_trace_benchmark(rfb_pipeline *p, const rfb_trace_settings *settings, uint32_t num_points,
                        const float *points, const void *attributes, const uint32_t *point_adjacency,
                        const uint32_t *point_adjacency_offsets, const void *adjacent_diff,
                        const rfb_camera *camera, const uint32_t *start_point_index,
                        uint32_t *output_rgba, const rfb_launch_opts *opts, void *stream_) {
    if (!p)
        return fail("rfb_trace_benchmark: pipeline is NULL");
    if (!points || !attributes || !point_adjacency || !point_adjacency_offsets || !adjacent_diff ||
        !camera || !start_point_index || !output_rgba)
        return fail("rfb_trace_benchmark: NULL argument");
    if (camera->model != RFB_PINHOLE && camera->model != RFB_FISHEYE)
        return fail("Invalid camera model");
    if (camera->width == 0 || camera->height == 0)
        return 0;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (int rc = ensure_diff_scene(p, num_points, points, attributes, point_adjacency, point_adjacency_offsets,
                                   adjacent_diff, opts, stream))
        return rc;
    rfb_trace_settings s = settings_or_default(settings);
    BenchmarkParams bp;
    bp.cells = reinterpret_cast<const float4 *>(p->cells.ptr);
    bp.sh_rows = reinterpret_cast<const float *>(p->sh_rows.ptr);
    bp.start = start_point_index;
    bp.out = output_rgba;
    bp.cam = camera_params(camera);
    bp.weight_threshold = s.weight_threshold;
    bp.max_steps = s.max_intersections;
    if (int rc = reset_exact_flag(p, stream, bp.exact_flag))
        return rc;
    bp.blocks_x = (camera->width + kTileW - 1) / kTileW;
    uint32_t blocks = bp.blocks_x * ((camera->height + kTileH - 1) / kTileH);
    // the caller's offsets, re-laid-out (copied, not recomputed) into the padded face rows
    return launch_benchmark(p->sh_degree, bp, padded_faces(p, point_adjacency_offsets), blocks, stream);
}

int rfb_trace_visualization(rfb_pipeline *p, const rfb_trace_settings *settings,
                            const rfb_visualization_settings *vis_settings, const rfb_camera *camera,
                            const rfb_cmap_table *cmap_table, uint32_t num_points, uint32_t num_tets,
                            const float *points, const void *attributes, const uint32_t *point_adjacency,
                            const uint32_t *point_adjacency_offsets, const void *adjacent_diff,
                            uint32_t start_index, uint64_t output_surface, const rfb_launch_opts *opts,
                            void *stream) {
    (void)num_tets; // accepted and unused, as in the reference
    SurfaceOut out;
    out.surf = (cudaSurfaceObject_t)output_surface;
    return trace_visualization("rfb_trace_visualization", p, settings, vis_settings, camera, cmap_table, num_points,
                               points, attributes, point_adjacency, point_adjacency_offsets, adjacent_diff,
                               start_index, output_surface != 0, out, opts, stream);
}

int rfb_trace_visualization_rgba8(rfb_pipeline *p, const rfb_trace_settings *settings,
                                  const rfb_visualization_settings *vis_settings, const rfb_camera *camera,
                                  const rfb_cmap_table *cmap_table, uint32_t num_points, uint32_t num_tets,
                                  const float *points, const void *attributes, const uint32_t *point_adjacency,
                                  const uint32_t *point_adjacency_offsets, const void *adjacent_diff,
                                  uint32_t start_index, uint32_t *output_rgba, const rfb_launch_opts *opts,
                                  void *stream) {
    (void)num_tets;
    LinearOut out;
    out.out = output_rgba;
    out.width = camera ? camera->width : 0u;
    return trace_visualization("rfb_trace_visualization_rgba8", p, settings, vis_settings, camera, cmap_table,
                               num_points, points, attributes, point_adjacency, point_adjacency_offsets,
                               adjacent_diff, start_index, output_rgba != nullptr, out, opts, stream);
}

} // extern "C"
