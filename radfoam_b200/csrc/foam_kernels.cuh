// Kernels of the H100 foam tracer: scene re-layout, forward, backward, benchmark.
// See foam_device.cuh for the spec references.
#pragma once

#include "foam_device.cuh"

namespace rfb {

// ------------------------------------------------------------------ re-layout
// cells[i] = (point, density); sh_rows[i] = SH coefficients padded to 16 bytes.
// Replaces per-step gathers of 3 + 49 scalars by aligned 128-bit loads.  A streaming pass over 416 MB at 1 M points
// that runs in every training step: flat over the output's 16-byte vectors (consecutive threads, consecutive
// vectors; the row length is a compile-time constant so the index split is a multiply-shift), four vectors per thread
// in flight.
template <typename AttrT, int DEG>
__global__ void __launch_bounds__(256) build_cells_kernel(const float *__restrict__ points,
                                                          const AttrT *__restrict__ attrs, uint32_t num_points,
                                                          float4 *__restrict__ cells, float4 *__restrict__ sh_rows) {
    constexpr uint32_t A = attr_dim(DEG), VPR = sh_row(DEG) / 4; // vectors per row
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)num_points * VPR;
#pragma unroll 4
    for (uint64_t v = gid; v < total; v += stride) {
        const uint64_t i = v / VPR;
        const uint32_t s0 = 4u * (uint32_t)(v % VPR);
        const AttrT *row = attrs + i * A;
        float4 o;
        o.x = s0 + 0 < A - 1 ? (float)row[s0 + 0] : 0.0f;
        o.y = s0 + 1 < A - 1 ? (float)row[s0 + 1] : 0.0f;
        o.z = s0 + 2 < A - 1 ? (float)row[s0 + 2] : 0.0f;
        o.w = s0 + 3 < A - 1 ? (float)row[s0 + 3] : 0.0f;
        sh_rows[v] = o;
    }
    for (uint64_t i = gid; i < num_points; i += stride)
        cells[i] = make_float4(points[3 * i], points[3 * i + 1], points[3 * i + 2], (float)attrs[i * A + (A - 1)]);
}

// F.softplus(x, beta=10) and its derivative exactly as torch evaluates them on CUDA (softplus_kernel /
// softplus_backward_kernel: threshold 20 on x*beta; log1p(exp(.)) / beta;  z / (z + 1) with z = exp(x*beta)).
__device__ __forceinline__ float softplus_beta10(float x) {
    const float xb = x * 10.0f;
    return xb > 20.0f ? x : log1pf(expf(xb)) / 10.0f;
}
__device__ __forceinline__ float softplus_beta10_backward(float grad_out, float x) {
    const float xb = x * 10.0f;
    if (xb > 20.0f)
        return grad_out;
    const float z = expf(xb);
    return (grad_out * z) / (z + 1.0f);
}

// The re-layout straight from the model's parameters -- RadFoamScene.get_trace_data (scene.py:202-217) fused in:
//   attributes = cat(att_dc, att_sh, activation_scale * softplus(density, beta=10)).to(attr_dtype)
// is never materialised; the cast is applied per value (AttrT = __half: round to fp16, then widen).  Same flat
// streaming form as build_cells_kernel.
template <typename AttrT, int DEG>
__global__ void __launch_bounds__(256) build_cells_params_kernel(const float *__restrict__ points,
                                                                 const float *__restrict__ att_dc,
                                                                 const float *__restrict__ att_sh,
                                                                 const float *__restrict__ density,
                                                                 float activation_scale, uint32_t num_points,
                                                                 float4 *__restrict__ cells,
                                                                 float4 *__restrict__ sh_rows) {
    constexpr uint32_t A = attr_dim(DEG), VPR = sh_row(DEG) / 4, REST = A - 4; // REST: columns of att_sh
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)num_points * VPR;
    auto value = [&](uint64_t i, uint32_t s) -> float {
        float v = 0.0f;
        if (s < 3)
            v = att_dc[3 * i + s];
        else if (s < A - 1)
            v = att_sh[i * REST + (s - 3)];
        return (float)(AttrT)v;
    };
#pragma unroll 4
    for (uint64_t v = gid; v < total; v += stride) {
        const uint64_t i = v / VPR;
        const uint32_t s0 = 4u * (uint32_t)(v % VPR);
        sh_rows[v] = make_float4(value(i, s0), value(i, s0 + 1), value(i, s0 + 2), value(i, s0 + 3));
    }
    for (uint64_t i = gid; i < num_points; i += stride) {
        const float sigma = activation_scale * softplus_beta10(density[i]);
        cells[i] = make_float4(points[3 * i], points[3 * i + 1], points[3 * i + 2], (float)(AttrT)sigma);
    }
}

// faces[padded_begin(i) + f] = half4(RN(points[adj[e]] - points[i]), 0),
// nbr[...] = adj[e]  (the reference's prefetch_adjacent_diff_kernel,
// pipeline.cu:546-568, writes the same values in CSR order).  16 lanes per row.  Bound by the 16 M neighbour
// gathers (L2); gathering from the float4 cell mirror instead of the packed points (one
// 128-bit load instead of three scalar ones) moves a third more bytes per gather.
__global__ void build_faces_kernel(const float *__restrict__ points, uint32_t num_points,
                                   const uint32_t *__restrict__ adj,
                                   const uint32_t *__restrict__ off, uint2 *__restrict__ faces,
                                   uint32_t *__restrict__ nbr) {
    const uint32_t group = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    const uint32_t lane = threadIdx.x & 15;
    const uint32_t stride = (gridDim.x * blockDim.x) >> 4;
    // The pass is a chain of dependent loads per row (offsets -> adjacency -> neighbour point), so it is bound by
    // how many rows are in flight: every 16-lane group works on kRows rows at once, level by level.
    constexpr int kRows = 2;
    for (uint32_t base = group; base < num_points; base += kRows * stride) {
        uint32_t row[kRows], a[kRows], nf[kRows];
        float px[kRows], py[kRows], pz[kRows];
#pragma unroll
        for (int k = 0; k < kRows; ++k) { // level 1: offsets and own point
            row[k] = base + k * stride;
            const bool live = row[k] < num_points;
            const uint32_t i = live ? row[k] : base;
            a[k] = __ldg(off + i);
            nf[k] = live ? __ldg(off + i + 1) - a[k] : 0u;
            px[k] = __ldg(points + 3 * (uint64_t)i);
            py[k] = __ldg(points + 3 * (uint64_t)i + 1);
            pz[k] = __ldg(points + 3 * (uint64_t)i + 2);
        }
        uint32_t passes = 0;
#pragma unroll
        for (int k = 0; k < kRows; ++k)
            passes = max(passes, (nf[k] + 15u) >> 4);
        for (uint32_t pass = 0; pass < passes; ++pass) {
            const uint32_t f = 16u * pass + lane;
            uint32_t j[kRows];
#pragma unroll
            for (int k = 0; k < kRows; ++k) // level 2: neighbour ids
                j[k] = f < nf[k] ? __ldg(adj + a[k] + f) : 0u;
            float qx[kRows], qy[kRows], qz[kRows];
#pragma unroll
            for (int k = 0; k < kRows; ++k) { // level 3: neighbour points
                qx[k] = __ldg(points + 3 * (uint64_t)j[k]);
                qy[k] = __ldg(points + 3 * (uint64_t)j[k] + 1);
                qz[k] = __ldg(points + 3 * (uint64_t)j[k] + 2);
            }
#pragma unroll
            for (int k = 0; k < kRows; ++k) {
                const uint32_t nf4 = (nf[k] + 3u) & ~3u;
                if (f < nf4) {
                    uint2 rec = make_uint2(0u, 0u); // pad: zero face, dp == 0 never wins
                    if (f < nf[k]) {
                        __half2 hxy = __floats2half2_rn(__fsub_rn(qx[k], px[k]), __fsub_rn(qy[k], py[k]));
                        __half2 hzw = __floats2half2_rn(__fsub_rn(qz[k], pz[k]), 0.0f);
                        rec.x = *reinterpret_cast<uint32_t *>(&hxy);
                        rec.y = *reinterpret_cast<uint32_t *>(&hzw);
                    }
                    const uint32_t dst = padded_begin(a[k], row[k]) + f;
                    faces[dst] = rec;
                    nbr[dst] = f < nf[k] ? j[k] : 0u;
                }
            }
        }
    }
}

// Same padded layout, but the offsets are COPIED from a caller-built half4[E] array (what
// trace_benchmark is given, pipeline.h:117-126) instead of derived from the points.
__global__ void build_faces_from_diff_kernel(const uint2 *__restrict__ diff, uint32_t num_points,
                                             const uint32_t *__restrict__ adj,
                                             const uint32_t *__restrict__ off, uint2 *__restrict__ faces,
                                             uint32_t *__restrict__ nbr) {
    uint32_t group = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    uint32_t lane = threadIdx.x & 15;
    uint32_t stride = (gridDim.x * blockDim.x) >> 4;
    for (uint32_t i = group; i < num_points; i += stride) {
        uint32_t a = __ldg(off + i), b = __ldg(off + i + 1);
        uint32_t dst = padded_begin(a, i);
        uint32_t nf = b - a, nf4 = (nf + 3u) & ~3u;
        for (uint32_t f = lane; f < nf4; f += 16) {
            uint2 rec = make_uint2(0u, 0u);
            uint32_t j = 0;
            if (f < nf) {
                rec = ldg2(diff + a + f);
                rec.y &= 0x0000FFFFu; // the 4th half is never read by the reference; keep it zero
                j = __ldg(adj + a + f);
            }
            faces[dst + f] = rec;
            nbr[dst + f] = j;
        }
    }
}

// reference-layout adjacent_diff (CSR order), for rfb_prefetch_adjacent_diff
__global__ void adjacent_diff_kernel(const float *__restrict__ points, uint32_t num_points,
                                     const uint32_t *__restrict__ adj,
                                     const uint32_t *__restrict__ off, uint2 *__restrict__ out) {
    uint32_t group = (blockIdx.x * blockDim.x + threadIdx.x) >> 4;
    uint32_t lane = threadIdx.x & 15;
    uint32_t stride = (gridDim.x * blockDim.x) >> 4;
    for (uint32_t i = group; i < num_points; i += stride) {
        uint32_t a = __ldg(off + i), b = __ldg(off + i + 1);
        float px = __ldg(points + 3 * (uint64_t)i), py = __ldg(points + 3 * (uint64_t)i + 1),
              pz = __ldg(points + 3 * (uint64_t)i + 2);
        for (uint32_t e = a + lane; e < b; e += 16) {
            uint32_t j = __ldg(adj + e);
            float qx = __ldg(points + 3 * (uint64_t)j), qy = __ldg(points + 3 * (uint64_t)j + 1),
                  qz = __ldg(points + 3 * (uint64_t)j + 2);
            __half2 hxy = __floats2half2_rn(__fsub_rn(qx, px), __fsub_rn(qy, py));
            __half2 hzw = __floats2half2_rn(__fsub_rn(qz, pz), 0.0f);
            uint2 rec;
            rec.x = *reinterpret_cast<uint32_t *>(&hxy);
            rec.y = *reinterpret_cast<uint32_t *>(&hzw);
            out[e] = rec;
        }
    }
}

// RFB_DEBUG: order-independent checksum of a word array (sum of word * odd multiplier of its index)
__global__ void checksum_kernel(const uint32_t *__restrict__ words, uint64_t count, unsigned long long *sum) {
    unsigned long long local = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x)
        local += (unsigned long long)words[i] * (2ull * i + 1ull);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        local += __shfl_down_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0)
        atomicAdd(sum, local);
}

// ------------------------------------------------------------------ forward
struct ForwardParams {
    const float4 *cells;
    const float *sh_rows;
    const float *rays;
    const uint32_t *start;
    const float *quantiles; // [R][Q] or null
    void *rgba;             // [R][4] f32 or f16
    float *qdepth;          // [R][Q]
    uint32_t *qidx;         // [R][Q]
    uint32_t *nint;         // [R] or null
    void *contrib;          // [N] f32 or f16, or null
    uint32_t num_rays;
    uint32_t num_q;
    uint32_t image_width;
    uint32_t blocks_x;
    float weight_threshold;
    uint32_t max_steps;
    int out_half;
    uint32_t *exact_flag; // device word: raised by a fast kernel that met a ray outside the ranked scan's domain
};

// MODE (ScanMode): kScanFast = ranked scan, raises *exact_flag for a ray it is not proven for; kScanExactTwin = the
// same kernel with the exact scan, launched right behind the fast one, a no-op unless the flag is up (it then
// overwrites every output); kScanPerRay = one launch that chooses per ray (used when `contrib` is accumulated
// with atomics, which a second pass would double).
template <int DEG, typename Faces, int MODE>
__global__ void __launch_bounds__(kBlock) forward_kernel(const ForwardParams p, const Faces fa) {
    if (MODE == kScanExactTwin && *p.exact_flag == 0u)
        return;
    uint32_t r;
    if (!thread_ray(p.num_rays, p.image_width, p.blocks_x, r))
        return;

    RayGeom ray;
    load_ray(p.rays, r, ray);
    if (MODE == kScanFast && needs_exact_scan(ray.dx, ray.dy, ray.dz))
        *p.exact_flag = 1u;
    float sh[sh_dim(DEG)];
    sh_basis<DEG>(ray.dx, ray.dy, ray.dz, sh);

    const uint32_t Q = p.quantiles ? p.num_q : 0u;
    const float *qv = p.quantiles + (uint64_t)r * p.num_q;
    uint32_t qi = 0;
    float cq = Q ? __ldg(qv) : 0.0f;

    float T = 1.0f;
    float cr = 0.0f, cg = 0.0f, cb = 0.0f;

    auto cell_fn = [&](uint32_t cell, const float4 &pc, float t0, float t1, const float4 &, uint32_t) -> bool {
        const float s = pc.w;
        const float Tn = composite_cell<DEG>(p.sh_rows, sh, cell, s, t0, t1, T, cr, cg, cb, [&](float w) {
            if (p.contrib) {
                if (p.out_half)
                    atomicAdd(reinterpret_cast<__half *>(p.contrib) + cell, __float2half_rn(w));
                else
                    atomicAdd(reinterpret_cast<float *>(p.contrib) + cell, w);
            }
        });
        while (qi < Q && Tn < cq) {
            p.qdepth[(uint64_t)r * Q + qi] = __fadd_rn(t0, __fdiv_rn(logf(__fdiv_rn(T, cq)), s));
            p.qidx[(uint64_t)r * Q + qi] = cell;
            qi++;
            if (qi < Q)
                cq = __ldg(qv + qi);
        }
        T = Tn;
        return T > p.weight_threshold;
    };

    uint32_t n = MODE == kScanPerRay
                     ? walk(fa, p.cells, ray, __ldg(p.start + r), p.max_steps, cell_fn)
                     : walk<MODE == kScanExactTwin>(fa, p.cells, ray, __ldg(p.start + r), p.max_steps, cell_fn);

    while (qi < Q) {
        p.qdepth[(uint64_t)r * Q + qi] = -1.0f;
        p.qidx[(uint64_t)r * Q + qi] = kNone;
        qi++;
    }
    float a = __fsub_rn(1.0f, T);
    if (p.out_half) {
        __half2 lo = __floats2half2_rn(cr, cg), hi = __floats2half2_rn(cb, a);
        uint2 v;
        v.x = *reinterpret_cast<uint32_t *>(&lo);
        v.y = *reinterpret_cast<uint32_t *>(&hi);
        reinterpret_cast<uint2 *>(p.rgba)[r] = v;
    } else {
        reinterpret_cast<float4 *>(p.rgba)[r] = make_float4(cr, cg, cb, a);
    }
    if (p.nint)
        p.nint[r] = n;
}

// ------------------------------------------------------------------ the walk tape
// A training step traces every ray twice: forward, then the backward re-walk
// (pipeline.cu:132-343 repeats trace<>()).  The face scan is ~2/3 of the walk's instructions,
// so when a backward pass is expected the forward records, per ray and visited cell,
// (cell, t1) -- 8 bytes -- and the backward replays that instead of re-scanning faces.  The
// record stream is identical to what the re-walk would compute (same kernel arithmetic), so
// results do not change.  Layout: all lanes of a warp are at the same step index k in the same
// loop iteration, so warp w writes rows of 32 records; rows are grouped in chunks of kTapeChunk
// steps (8 KB) handed out by a bump allocator, chunk ids in table[w][k / kTapeChunk].  If the
// pool runs out the overflow flag is raised and the backward re-walks (still correct); the host
// grows the pool for the next step.
constexpr int kTapeChunk = 32;     // steps per chunk
constexpr uint32_t kTapeNoChunk = 0xFFFFFFFFu;

struct Tape {
    uint2 *pool;        // [capacity][kTapeChunk][32] records (cell, float_as_uint(t1))
    uint32_t *table;    // [num_warps][table_stride] chunk ids
    uint2 *per_ray;     // [R] (number of records, cell entered after the last record)
    uint32_t *ctrl;     // [0] bump cursor, [1] overflow flag
    uint32_t capacity;  // chunks in the pool
    uint32_t table_stride;
    // Longest-first schedule of the replay: a ray is a serial chain of dependent loads (microseconds per step when
    // the SM is nearly empty), so a 250-step ray that happens to sit in one of the LAST tiles the hardware
    // dispatches keeps the kernel alive long after everything else has drained, a larger share of the backward
    // the smaller the launch.  After the recording forward,
    // tile_steps_kernel takes each tile's longest record count from per_ray (a pass of its own: touching the
    // forward kernel's epilogue for it cost 7 registers and an occupancy step), tape_order_kernel sorts the
    // tiles by that, descending, and the replay's CTA b works on tile order[b]: the long chains start first
    // and the short ones fill the tail.
    uint32_t *tile_steps; // [blocks]
    uint32_t *order;      // [blocks] tiles, longest first
};

// tile_steps[b] = max over the rays of tile b of the recorded step count (one warp per tile)
__global__ void __launch_bounds__(256) tile_steps_kernel(const uint2 *__restrict__ per_ray, uint32_t num_rays,
                                                         uint32_t image_width, uint32_t blocks_x, uint32_t blocks,
                                                         uint32_t *__restrict__ tile_steps) {
    const uint32_t tile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (tile >= blocks)
        return;
    uint32_t longest = 0;
    for (uint32_t t = lane; t < (uint32_t)kBlock; t += 32) { // thread t of the ray kernels' CTA `tile`
        uint32_t r;
        bool has;
        if (image_width == 0) {
            r = tile * kBlock + t;
            has = r < num_rays;
        } else {
            const uint32_t bx = tile % blocks_x, by = tile / blocks_x, warp = t >> 5, l = t & 31;
            const uint32_t x = bx * kTileW + (warp % kWarpsX) * 8 + (l & 7), y = by * kTileH + (warp / kWarpsX) * 4 + (l >> 3);
            r = y * image_width + x;
            has = x < image_width && y < num_rays / image_width;
        }
        if (has)
            longest = max(longest, per_ray[r].x);
    }
    longest = __reduce_max_sync(0xffffffffu, longest);

    if (lane == 0)
        tile_steps[tile] = longest;
}

// The replay's tile order (one CTA): the `budget` longest tiles first, by descending length (counting sort, bins
// of one step, the last bin open-ended; whole bins only), then all the others in their original, spatially
// coherent order.  Sorting ALL tiles removes most of the tail but
// scatters neighbouring tiles in time, and the lost L2 sharing of cells and gradient rows costs more than the tail
// on a full frame while it pays on a 1/8 shard, where the launch is fewer
// than three waves of CTAs whose durations differ widely.  So the host sorts everything for launches of up to 8 waves
// and keeps the dispatch order (no schedule at all) above that.
constexpr int kOrderBins = 2048;
__global__ void __launch_bounds__(1024) tape_order_kernel(const uint32_t *__restrict__ tile_steps, uint32_t blocks,
                                                          uint32_t budget, uint32_t *__restrict__ order) {
    __shared__ uint32_t bin_start[kOrderBins];
    __shared__ uint32_t warp_total[32];
    __shared__ uint32_t s_cut, s_running;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kOrderBins; i += blockDim.x)
        bin_start[i] = 0;
    __syncthreads();
    auto bin_of = [&](uint32_t b) { return (uint32_t)kOrderBins - 1u - min(tile_steps[b], (uint32_t)kOrderBins - 1u); };
    for (uint32_t b = threadIdx.x; b < blocks; b += blockDim.x)
        atomicAdd(&bin_start[bin_of(b)], 1u); // longest -> bin 0
    __syncthreads();
    if (warp == 0) { // exclusive scan of the counts by one warp (64 bins per lane) + the cut between long and rest
        constexpr int PER = kOrderBins / 32;
        uint32_t local = 0;
        for (int i = 0; i < PER; ++i)
            local += bin_start[lane * PER + i];
        uint32_t incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
            if ((int)lane >= o)
                incl += v;
        }
        uint32_t run = incl - local;
        uint32_t my_cut = 0, my_long = 0; // bins [0, my_cut) are long; their tile count
        for (int i = 0; i < PER; ++i) {
            const uint32_t c = bin_start[lane * PER + i];
            bin_start[lane * PER + i] = run;
            run += c;
            if (run <= budget) {
                my_cut = lane * PER + i + 1;
                my_long = run;
            }
        }
        // prefixes are nested, so the largest prefix within the budget is the max over the lanes
        const uint32_t cut = __reduce_max_sync(0xffffffffu, my_cut);
        const uint32_t nlong = __reduce_max_sync(0xffffffffu, my_long);
        if (lane == 0) {
            s_cut = cut;
            s_running = nlong;
        }
    }
    __syncthreads();
    const uint32_t cut = s_cut;
    for (uint32_t b = threadIdx.x; b < blocks; b += blockDim.x) { // the long tiles, longest first
        const uint32_t bin = bin_of(b);
        if (bin < cut)
            order[atomicAdd(&bin_start[bin], 1u)] = b;
    }
    for (uint32_t base = 0; base < blocks; base += blockDim.x) { // the rest, in index order (stable compaction)
        const uint32_t b = base + threadIdx.x;
        const bool keep = b < blocks && bin_of(b) >= cut;
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0)
            warp_total[warp] = __popc(ballot);
        __syncthreads();
        uint32_t before = 0;
        for (uint32_t w = 0; w < warp; ++w)
            before += warp_total[w];
        if (keep)
            order[s_running + before + __popc(ballot & ((1u << lane) - 1u))] = b;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t total = 0;
            for (uint32_t w = 0; w < blockDim.x / 32; ++w)
                total += warp_total[w];
            s_running += total;
        }
        __syncthreads();
    }
}

// Forward with an explicit warp-synchronous loop (all lanes stay in the loop until the warp is
// done, so lane 0 can allocate tape chunks for the warp) that records the tape.
// MODE: kScanFast / kScanExactTwin / kScanPerRay as for forward_kernel.  The twin allocates its tape chunks from a
// cursor of its own (ctrl[2]), i.e. it re-uses the pool from the start and overwrites the fast kernel's table.
template <int DEG, typename Faces, int MODE>
__global__ void __launch_bounds__(kBlock) forward_record_kernel(const ForwardParams p, const Faces fa,
                                                                const Tape tape) {
    if (MODE == kScanExactTwin && *p.exact_flag == 0u)
        return;
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int CURSOR = MODE == kScanExactTwin ? 2 : 0;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gwarp = blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
    uint32_t r;
    bool done = !thread_ray(p.num_rays, p.image_width, p.blocks_x, r);
    const bool has_ray = !done;

    RayGeom ray = {0.f, 0.f, 0.f, 0.f, 0.f, 1.f};
    float sh[sh_dim(DEG)];
    uint32_t Q = 0, qi = 0;
    const float *qv = nullptr;
    float cq = 0.0f;
    uint32_t cur = 0;
    float4 pc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (has_ray) {
        load_ray(p.rays, r, ray);
        Q = p.quantiles ? p.num_q : 0u;
        qv = p.quantiles + (uint64_t)r * p.num_q;
        cq = Q ? __ldg(qv) : 0.0f;
        cur = __ldg(p.start + r);
        pc = ldg4(p.cells + cur);
    }
    sh_basis<DEG>(ray.dx, ray.dy, ray.dz, sh);

    float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f, t0 = 0.0f;
    uint32_t n = 0, nrec = 0;
    uint32_t chunk = kTapeNoChunk;
    // the step loop, instantiated for the ranked scan and (warps holding a ray it is not proven for) the exact one
    if (MODE == kScanFast && has_ray && needs_exact_scan(ray.dx, ray.dy, ray.dz))
        *p.exact_flag = 1u;
    for (uint32_t k = 0;; ++k) {
        if ((k % kTapeChunk) == 0) { // the warp enters a new chunk of steps
            uint32_t c = kTapeNoChunk;
            if (lane == 0) {
                c = atomicAdd(tape.ctrl + CURSOR, 1u);
                if (c >= tape.capacity || k / kTapeChunk >= tape.table_stride) {
                    atomicExch(tape.ctrl + 1, 1u);
                    c = kTapeNoChunk;
                } else {
                    tape.table[(uint64_t)gwarp * tape.table_stride + k / kTapeChunk] = c;
                }
            }
            chunk = __shfl_sync(FULL, c, 0);
        }
        if (!done) {
            n++;
            if (n > p.max_steps) {
                done = true;
            } else {
                uint32_t begin, nf;
                fa.row(cur, begin, nf);
                float t1 = __int_as_float(0x7f800000);
                uint32_t face = kNone;
                if (MODE == kScanPerRay && needs_exact_scan(ray.dx, ray.dy, ray.dz))
                    fa.template scan<true>(begin, nf, pc.x, pc.y, pc.z, ray, t1, face);
                else
                    fa.template scan<MODE == kScanExactTwin>(begin, nf, pc.x, pc.y, pc.z, ray, t1, face);
                if (face == kNone) {
                    done = true;
                } else {
                    if (chunk != kTapeNoChunk) // streaming store: the tape is written once, read once
                        __stcs(tape.pool + ((uint64_t)chunk * kTapeChunk + (k % kTapeChunk)) * 32 + lane,
                               make_uint2(cur, __float_as_uint(t1)));
                    nrec++;
                    uint32_t nxt = fa.neighbour(begin, face);
                    float4 pn = ldg4(p.cells + nxt);
                    if (t1 > t0) {
                        // composite_cell() and forward_kernel's quantile loop, written out (as is the epilogue
                        // below): shared, they move this kernel's register allocation and so its SASS.  Keep
                        // these copies in step with forward_kernel.
                        float s = pc.w;
                        float r_ = 0.0f, g_ = 0.0f, b_ = 0.0f;
                        if (s > 1e-6f)
                            sh_to_rgb<DEG>(p.sh_rows + (uint64_t)cur * sh_row(DEG), sh, r_, g_, b_);
                        float delta = fmaxf(__fsub_rn(t1, t0), 0.0f);
                        float alpha = 1.0f - expf(-s * delta);
                        float w = __fmul_rn(T, alpha);
                        if (p.contrib) {
                            if (p.out_half)
                                atomicAdd(reinterpret_cast<__half *>(p.contrib) + cur, __float2half_rn(w));
                            else
                                atomicAdd(reinterpret_cast<float *>(p.contrib) + cur, w);
                        }
                        cr = __fmaf_rn(w, r_, cr);
                        cg = __fmaf_rn(w, g_, cg);
                        cb = __fmaf_rn(w, b_, cb);
                        float Tn = __fmul_rn(T, __fsub_rn(1.0f, alpha));
                        while (qi < Q && Tn < cq) {
                            p.qdepth[(uint64_t)r * Q + qi] = __fadd_rn(t0, __fdiv_rn(logf(__fdiv_rn(T, cq)), s));
                            p.qidx[(uint64_t)r * Q + qi] = cur;
                            qi++;
                            if (qi < Q)
                                cq = __ldg(qv + qi);
                        }
                        T = Tn;
                        done = !(T > p.weight_threshold);
                    }
                    t0 = fmaxf(t0, t1);
                    cur = nxt;
                    pc = pn;
                }
            }
        }
        if (!__any_sync(FULL, !done))
            break;
    }
    if (!has_ray)
        return;
    tape.per_ray[r] = make_uint2(nrec, cur);
    // forward_kernel's epilogue, written out (see the cell step above)
    while (qi < Q) {
        p.qdepth[(uint64_t)r * Q + qi] = -1.0f;
        p.qidx[(uint64_t)r * Q + qi] = kNone;
        qi++;
    }
    float a = __fsub_rn(1.0f, T);
    if (p.out_half) {
        __half2 lo = __floats2half2_rn(cr, cg), hi = __floats2half2_rn(cb, a);
        uint2 v;
        v.x = *reinterpret_cast<uint32_t *>(&lo);
        v.y = *reinterpret_cast<uint32_t *>(&hi);
        reinterpret_cast<uint2 *>(p.rgba)[r] = v;
    } else {
        reinterpret_cast<float4 *>(p.rgba)[r] = make_float4(cr, cg, cb, a);
    }
    if (p.nint)
        p.nint[r] = n;
}

// ------------------------------------------------------------------ backward
struct BackwardParams {
    const float4 *cells;
    const float *sh_rows;
    const float *rays;
    const uint32_t *start;
    const float *quantiles;
    const uint32_t *qidx;
    const void *rgba;      // saved forward output [R][4]
    const void *rgba_grad; // [R][4]
    const float *depth_grad;
    const void *ray_error; // [R] or null
    void *point_error;     // [N] or null
    float *acc;            // [N][grad_row] fp32 accumulator
    uint32_t num_rays;
    uint32_t num_q;
    uint32_t image_width;
    uint32_t blocks_x;
    float weight_threshold;
    uint32_t max_steps;
    int io_half;
};

// Loads this thread's ray and upstream gradients (pipeline.cu:156-207).
template <int DEG>
__device__ __forceinline__ void backward_ray_setup(const BackwardParams &p, uint32_t r, RayGeom &ray,
                                                   float *sh, BackwardRay &st) {
    load_ray(p.rays, r, ray);
    sh_basis<DEG>(ray.dx, ray.dy, ray.dz, sh);
    st.err = 0.0f;
    if (p.io_half) {
        const __half *o = reinterpret_cast<const __half *>(p.rgba) + 4 * (uint64_t)r;
        const __half *gg = reinterpret_cast<const __half *>(p.rgba_grad) + 4 * (uint64_t)r;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            st.out[c] = __half2float(o[c]);
            st.g[c] = __half2float(gg[c]);
        }
        if (p.ray_error)
            st.err = __half2float(reinterpret_cast<const __half *>(p.ray_error)[r]);
    } else {
        float4 o = __ldg(reinterpret_cast<const float4 *>(p.rgba) + r);
        float4 gg = __ldg(reinterpret_cast<const float4 *>(p.rgba_grad) + r);
        st.out[0] = o.x; st.out[1] = o.y; st.out[2] = o.z; st.out[3] = o.w;
        st.g[0] = gg.x; st.g[1] = gg.y; st.g[2] = gg.z; st.g[3] = gg.w;
        if (p.ray_error)
            st.err = __ldg(reinterpret_cast<const float *>(p.ray_error) + r);
    }
    st.init();
    st.Q = p.quantiles ? p.num_q : 0u;
    st.qv = p.quantiles + (uint64_t)r * p.num_q;
    st.dg = p.depth_grad + (uint64_t)r * p.num_q;
    st.cq = st.Q ? __ldg(st.qv) : 0.0f;
    for (uint32_t i = 0; i < st.Q; ++i) { // pipeline.cu:196-207
        uint32_t pi = __ldg(p.qidx + (uint64_t)r * st.Q + i);
        if (pi != kNone)
            st.cdg = __fadd_rn(st.cdg, __fdiv_rn(__ldg(st.dg + i), ldg4(p.cells + pi).w));
    }
}

// Output of the RAY instantiations of the backward kernels: ray_grad[R][6] = dL/d(origin, direction as passed
// in), every ray written (no atomics).  A separate, trailing kernel parameter so that BackwardParams and the
// parameters after it keep their layout in the default instantiations.
struct RayGradOut {
    float *ray_grad;
    int scrub; // zero non-finite entries
};

// ray_grad[r] from the walk's sums: the colour's direction term sum_k G_k grad Y_k(d) is added, and the unit
// direction's gradient g is taken back through d = d_in / |d_in|: (g - d (d.g)) / |d_in|, with |d_in| the fp32
// norm normalize_dir() divides by
template <int DEG>
__device__ __forceinline__ void ray_grad_store(const BackwardParams &p, const RayGradOut &rg, uint32_t r,
                                               const RayGeom &ray, const RayAcc &ra, const float *G) {
    float gx = ra.gdx, gy = ra.gdy, gz = ra.gdz;
    sh_basis_grad<DEG>(ray.dx, ray.dy, ray.dz, G, gx, gy, gz);
    const float *rp = p.rays + 6 * (uint64_t)r;
    const float x = __ldg(rp + 3), y = __ldg(rp + 4), z = __ldg(rp + 5);
    const float norm = __fsqrt_rn(__fmaf_rn(x, x, __fmaf_rn(y, y, __fmul_rn(z, z))));
    const float dg = __fmaf_rn(ray.dx, gx, __fmaf_rn(ray.dy, gy, __fmul_rn(ray.dz, gz)));
    float v[6] = {ra.gox, ra.goy, ra.goz, __fdiv_rn(__fmaf_rn(-ray.dx, dg, gx), norm),
                  __fdiv_rn(__fmaf_rn(-ray.dy, dg, gy), norm), __fdiv_rn(__fmaf_rn(-ray.dz, dg, gz), norm)};
    float *out = rg.ray_grad + 6 * (uint64_t)r;
#pragma unroll
    for (int i = 0; i < 6; ++i)
        out[i] = (rg.scrub && !isfinite(v[i])) ? 0.0f : v[i];
}

__device__ __forceinline__ void add_point_error(const BackwardParams &p, uint32_t cell, float v) {
    if (p.io_half)
        atomicAdd(reinterpret_cast<__half *>(p.point_error) + cell, __float2half_rn(v));
    else
        atomicAdd(reinterpret_cast<float *>(p.point_error) + cell, v);
}

// one gradient row as 128-bit reductions (write_rgb_grad_to_sh, sh_utils.cuh:85-92, plus the
// density slot); a row whose three channel gradients are all zero adds nothing and is skipped
template <int DEG>
__device__ __forceinline__ void reduce_row_direct(float *row, const float *sh, const float dL_drgb[3],
                                                  float dL_ds) {
    constexpr int SR = sh_row(DEG);
    if (dL_drgb[0] != 0.0f || dL_drgb[1] != 0.0f || dL_drgb[2] != 0.0f) {
#pragma unroll
        for (int i = 0; i < SR; i += 4) {
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
                v[k] = (i + k < 3 * sh_dim(DEG)) ? __fmul_rn(sh[(i + k) / 3], dL_drgb[(i + k) % 3]) : 0.0f;
            red_add_v4(row + i, v[0], v[1], v[2], v[3]);
        }
    }
    red_add_v4(row + SR, dL_ds, 0.0f, 0.0f, 0.0f);
}

// ---- backward, direct: every lane reduces its own rows straight to HBM
// RAY: also writes ray_grad (RayGradOut)
template <int DEG, typename Faces, bool RAY>
__global__ void __launch_bounds__(kBlock) backward_kernel(const BackwardParams p, const Faces fa,
                                                          const RayGradOut rg) {
    uint32_t r;
    if (!thread_ray(p.num_rays, p.image_width, p.blocks_x, r))
        return;
    constexpr int GR = grad_row(DEG);
    constexpr int SR = sh_row(DEG);
    RayGeom ray;
    float sh[sh_dim(DEG)];
    BackwardRay st;
    backward_ray_setup<DEG>(p, r, ray, sh, st);
    RayAcc ra;
    float G[sh_dim(DEG)];
    if (RAY) {
        ra.init();
#pragma unroll
        for (int k = 0; k < sh_dim(DEG); ++k)
            G[k] = 0.0f;
    }

    auto cell_fn = [&](uint32_t cell, const float4 &pc, float t0, float t1, const float4 &pn, uint32_t nxt) -> bool {
        float rgb[3] = {0.0f, 0.0f, 0.0f};
        if (pc.w > 1e-6f)
            sh_to_rgb<DEG>(p.sh_rows + (uint64_t)cell * SR, sh, rgb[0], rgb[1], rgb[2]);
        float dL_drgb[3], dL_ds, w, fx, fy, fz;
        bool flush;
        uint32_t flush_idx;
        bool go = st.template cell<RAY>(cell, pc, nxt, pn, p.cells, t0, t1, rgb, ray, p.weight_threshold, dL_drgb,
                                        dL_ds, w, flush, flush_idx, fx, fy, fz, ra);
        if (RAY)
            sh_grad_contract<DEG>(p.sh_rows + (uint64_t)cell * SR, dL_drgb, G);
        if (p.point_error)
            add_point_error(p, cell, __fmul_rn(w, st.err));
        if (flush)
            red_add_v4(p.acc + (uint64_t)flush_idx * GR + SR, 0.0f, fx, fy, fz);
        reduce_row_direct<DEG>(p.acc + (uint64_t)cell * GR, sh, dL_drgb, dL_ds);
        return go;
    };
    walk(fa, p.cells, ray, __ldg(p.start + r), p.max_steps, cell_fn);
    if (RAY)
        ray_grad_store<DEG>(p, rg, r, ray, ra, G);
}

// ---- backward, warp-aggregated
// Same mathematics; what changes is how the per-cell gradient rows reach HBM.  Neighbouring
// rays of an 8x4 tile cross mostly the same cells, a few iterations apart (one ray clips a
// sliver cell the other misses and they drift out of lock-step), so instead of 13 x 128-bit
// reductions per lane per step the warp keeps a small direct-mapped cache of gradient rows in
// shared memory:
//   * a composited step's row is held in registers until the lane's next composited step, which
//     finishes that cell's position gradient (BackwardRay::cell flushes it one cell late); then
//     the lane writes the row (SH products, density grad, position grad) to its own staging row
//     in shared memory, so the position gradient needs no reduction of its own;
//   * lanes are grouped by cell (MATCH.ANY); a lane in a group of fewer than MIN_GROUP lanes
//     sends its staged row to HBM as one bulk reduction (cp.reduce.async.bulk: the TMA unit reads
//     the row, so the LSU issues no request per 16 bytes), and waits for that read to finish only
//     when it next rewrites the row, a step later;
//   * the warp sums the staged rows of a larger group "transposed" --
//     lane j owns elements 2j, 2j+1 of the row -- so the shared-memory update needs no atomics
//     and has no bank conflicts, and adds the sum to the cell's cache row;
//   * a cache row is written to HBM (13 lanes x one RED.128) only when its slot is claimed by
//     another cell, or when the warp's rays are finished.
// MIN_GROUP: smallest same-cell lane group routed through the cache (smaller groups send one
// bulk reduction per lane, which costs fewer issue slots than one serial cache round per group,
// at the price of more L2 atomic traffic).
// REPLAY = true: the steps come from the forward's tape of (cell, t1) instead of re-scanning
// faces.  When a tape is offered the host launches both instantiations back to back; each looks
// at the tape's overflow flag first and exactly one of them does the work (the other returns at
// once), so a pool overflow needs no host round trip.  (Prefetching the next cell's SH row into
// L1 or L2 as soon as the cell is known was tried and is no faster.)
// RAY: also writes ray_grad (RayGradOut), in both the replay and the re-walk instantiation.
template <int DEG, typename Faces, int SLOTS, int MIN_GROUP, int MIN_BLOCKS, bool REPLAY, bool RAY>
__global__ void __launch_bounds__(kBlock, MIN_BLOCKS * 128 / kBlock)
    backward_cached_kernel(const BackwardParams p, const Faces fa, const Tape tape, const RayGradOut rg) {
    if (tape.pool != nullptr) {
        const bool overflowed = tape.ctrl[1] != 0u;
        if (REPLAY == overflowed) // replay kernel on an overflowed tape / re-walk kernel on a good one
            return;
    }
    constexpr int GR = grad_row(DEG);
    constexpr int SR = sh_row(DEG);
    constexpr int HALF_ROW = GR / 2; // lanes that own two row elements each
    constexpr unsigned FULL = 0xffffffffu;
    static_assert(HALF_ROW <= 32, "row too wide for one warp pass");
    static_assert((SLOTS & (SLOTS - 1)) == 0, "SLOTS must be a power of two");
    static_assert(GR % 4 == 0 && SR % 4 == 0, "stage rows and bulk reductions need 16-byte multiples");

#ifdef RFB_EMU
    float *smem = rfb_emu_dynamic_smem();
#else
    extern __shared__ __align__(16) float smem[];
#endif
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int WARP_FLOATS = (32 * GR + SLOTS * GR + SLOTS + 3) & ~3; // keeps every warp's rows 16-byte aligned
    float *stage = smem + warp * WARP_FLOATS;                          // [32][GR]
    float *cache = stage + 32 * GR;                                    // [SLOTS][GR]
    uint32_t *tags = reinterpret_cast<uint32_t *>(cache + SLOTS * GR); // [SLOTS]
    for (int i = lane; i < SLOTS; i += 32)
        tags[i] = kNone;
    __syncwarp();

    constexpr bool replay = REPLAY;
    const uint32_t tile = (replay && tape.order) ? tape.order[blockIdx.x] : blockIdx.x; // longest tiles first
    uint32_t r;
    bool done = !thread_ray(p.num_rays, p.image_width, p.blocks_x, r, tile);
    const bool has_ray = !done;
    RayGeom ray = {0.f, 0.f, 0.f, 0.f, 0.f, 1.f};
    float sh[sh_dim(DEG)];
    BackwardRay st;
    uint32_t cur = 0;
    float4 pc = make_float4(0.f, 0.f, 0.f, 0.f);
    const uint32_t gwarp = tile * (kBlock / 32) + warp;
    uint32_t nrec = 0, last_cell = 0;
    uint2 rec = make_uint2(0u, 0u); // record of the step about to be processed (replay)
    if (!done) {
        backward_ray_setup<DEG>(p, r, ray, sh, st);
        cur = __ldg(p.start + r);
        pc = ldg4(p.cells + cur);
        if (replay) {
            uint2 pr = tape.per_ray[r];
            nrec = pr.x;
            last_cell = pr.y;
            done = nrec == 0;
        }
    } else {
#pragma unroll
        for (int i = 0; i < sh_dim(DEG); ++i)
            sh[i] = 0.0f;
    }
    float t0 = 0.0f;
    uint32_t n = 0;
    // replay pipeline: records k and k+1 are kept in registers and record k+2 is requested
    // while step k is processed, so the streamed tape read is never waited for.  (Also
    // prefetching the cell gather one step ahead costs 8 more registers, spills, and is slower.)
    uint32_t chunk_ahead = 0; // chunk id (warp-uniform) of tape row k + 2
    uint2 recB = make_uint2(0u, 0u);
    auto tape_row = [&](uint32_t chunk_id, uint32_t j) -> uint2 {
        // record j of this lane; past the end: the cell the forward stopped in
        return j < nrec ? __ldcs(tape.pool + ((uint64_t)chunk_id * kTapeChunk + (j % kTapeChunk)) * 32 + lane)
                        : make_uint2(last_cell, 0u);
    };
    if (replay) {
        chunk_ahead = tape.table[(uint64_t)gwarp * tape.table_stride]; // rows 0..31
        if (!done) {
            rec = tape_row(chunk_ahead, 0);
            recB = tape_row(chunk_ahead, 1);
        }
    }

    RayAcc ra;
    float G[sh_dim(DEG)];
    if (RAY) {
        ra.init();
#pragma unroll
        for (int k = 0; k < sh_dim(DEG); ++k)
            G[k] = 0.0f;
    }

    // the row of this lane's last composited cell, held until the lane's next composited step has finished that
    // cell's position gradient (BackwardRay::cell flushes it one cell late), so that the row and its position
    // gradient leave together; a ray's last row leaves with zero position slots once the ray is done
    uint32_t p_cell = kNone;
    float p_ds = 0.0f;
    float p_drgb[3] = {0.0f, 0.0f, 0.0f};

    for (uint32_t k = 0;; ++k) {
        bool c_valid = false; // this lane has a row for cell c_cell this iteration
        uint32_t c_cell = kNone;
        float dL_ds = 0.0f;
        float dL_drgb[3] = {0.0f, 0.0f, 0.0f};
        float fx = 0.0f, fy = 0.0f, fz = 0.0f; // c_cell's position gradient

        // one step of the ray: (cur, t1, nxt) from the tape, or from scanning the cell's faces
        bool step = false;
        float t1 = __int_as_float(0x7f800000);
        uint32_t nxt = 0;
        if (replay) {
            if (((k + 2) % kTapeChunk) == 0)
                chunk_ahead = tape.table[(uint64_t)gwarp * tape.table_stride + (k + 2) / kTapeChunk];
            if (!done) {
                uint2 recC = tape_row(chunk_ahead, k + 2);
                t1 = __uint_as_float(rec.y);
                nxt = recB.x;
                rec = recB;
                recB = recC;
                step = true;
            }
        } else if (!done) {
            n++;
            if (n > p.max_steps) {
                done = true;
            } else {
                uint32_t begin, nf;
                fa.row(cur, begin, nf);
                uint32_t face = kNone;
                if (needs_exact_scan(ray.dx, ray.dy, ray.dz)) // re-walk is the fallback path: tested per step
                    fa.template scan<true>(begin, nf, pc.x, pc.y, pc.z, ray, t1, face);
                else
                    fa.template scan<false>(begin, nf, pc.x, pc.y, pc.z, ray, t1, face);
                if (face == kNone) {
                    done = true;
                } else {
                    nxt = fa.neighbour(begin, face);
                    step = true;
                }
            }
        }
        if (step) {
            float4 pn = ldg4(p.cells + nxt);
            if (t1 > t0) {
                float rgb[3] = {0.0f, 0.0f, 0.0f};
                if (pc.w > 1e-6f)
                    sh_to_rgb<DEG>(p.sh_rows + (uint64_t)cur * SR, sh, rgb[0], rgb[1], rgb[2]);
                float w, n_ds, n_drgb[3];
                bool flush;
                uint32_t flush_idx;
                bool go = st.template cell<RAY>(cur, pc, nxt, pn, p.cells, t0, t1, rgb, ray, p.weight_threshold,
                                                n_drgb, n_ds, w, flush, flush_idx, fx, fy, fz, ra);
                if (RAY)
                    sh_grad_contract<DEG>(p.sh_rows + (uint64_t)cur * SR, n_drgb, G);
                if (p.point_error)
                    add_point_error(p, cur, __fmul_rn(w, st.err));
                // every composited step sets st.prev, so flush == (p_cell != kNone) and flush_idx == p_cell:
                // the held row leaves now, carrying its finished position gradient
                c_valid = flush;
                c_cell = p_cell;
                dL_ds = p_ds;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    dL_drgb[c] = p_drgb[c];
                    p_drgb[c] = n_drgb[c];
                }
                p_cell = cur;
                p_ds = n_ds;
                done = !go;
            }
            t0 = fmaxf(t0, t1);
            cur = nxt;
            pc = pn;
            if (replay && k + 1 >= nrec)
                done = true;
        }
        if (!c_valid && done && p_cell != kNone) {
            // the ray is done: its last composited cell's row leaves with zero position slots (that cell's
            // position gradient is never finished: quirk A.5.1)
            c_valid = true;
            c_cell = p_cell;
            dL_ds = p_ds;
#pragma unroll
            for (int c = 0; c < 3; ++c)
                dL_drgb[c] = p_drgb[c];
            fx = fy = fz = 0.0f;
            p_cell = kNone;
        }

        // ---- warp-collective phase: route this iteration's rows
        unsigned grp = __match_any_sync(FULL, c_valid ? c_cell : (0x80000000u | lane));
        bool single = c_valid && __popc(grp) < MIN_GROUP;
        bool staged = c_valid && !single;
        if (c_valid) {
            bulk_wait_read(); // this lane's previous bulk reduction has finished reading its stage row
            float4 *srow = reinterpret_cast<float4 *>(stage + lane * GR);
#pragma unroll
            for (int i = 0; i < SR; i += 4) {
                float v[4];
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    v[k] = (i + k < 3 * sh_dim(DEG)) ? __fmul_rn(sh[(i + k) / 3], dL_drgb[(i + k) % 3]) : 0.0f;
                srow[i / 4] = make_float4(v[0], v[1], v[2], v[3]);
            }
            srow[SR / 4] = make_float4(dL_ds, fx, fy, fz);
        }
        if (single) {
            // the whole row as one bulk reduction; a row whose three channel gradients are all zero sends
            // its density slot only
            const uint32_t off = (dL_drgb[0] != 0.0f || dL_drgb[1] != 0.0f || dL_drgb[2] != 0.0f) ? 0 : SR;
            fence_proxy_async_smem();
            bulk_red_add_f32(p.acc + (uint64_t)c_cell * GR + off, stage + lane * GR + off, (GR - off) * 4);
        }
        unsigned todo = __ballot_sync(FULL, staged);
        if (todo) {
            __syncwarp();
            while (todo) {
                int leader = __ffs(todo) - 1;
                unsigned gmask = __shfl_sync(FULL, grp, leader);
                uint32_t lc = __shfl_sync(FULL, c_cell, leader);
                todo &= ~gmask;
                float a0 = 0.0f, a1 = 0.0f;
                if (lane < HALF_ROW) {
                    // four staged rows per round: the loads are issued together so their
                    // shared-memory latency overlaps (groups have >= MIN_GROUP members)
                    const float *col = stage + 2 * lane;
                    unsigned m = gmask;
                    while (m) {
                        int s0 = __ffs(m) - 1;
                        m &= m - 1;
                        int s1 = m ? __ffs(m) - 1 : -1;
                        m &= m - 1;
                        int s2 = m ? __ffs(m) - 1 : -1;
                        m &= m - 1;
                        int s3 = m ? __ffs(m) - 1 : -1;
                        m &= m - 1;
                        float2 v0 = *reinterpret_cast<const float2 *>(col + s0 * GR);
                        float2 v1 = s1 >= 0 ? *reinterpret_cast<const float2 *>(col + s1 * GR) : make_float2(0.f, 0.f);
                        float2 v2 = s2 >= 0 ? *reinterpret_cast<const float2 *>(col + s2 * GR) : make_float2(0.f, 0.f);
                        float2 v3 = s3 >= 0 ? *reinterpret_cast<const float2 *>(col + s3 * GR) : make_float2(0.f, 0.f);
                        a0 += (v0.x + v1.x) + (v2.x + v3.x);
                        a1 += (v0.y + v1.y) + (v2.y + v3.y);
                    }
                }
                uint32_t slot = (lc * 2654435761u) >> (32 - __builtin_ctz(SLOTS));
                uint32_t tag = tags[slot];
                __syncwarp();
                float2 *crow = reinterpret_cast<float2 *>(cache + slot * GR + 2 * lane);
                if (tag == lc) {
                    if (lane < HALF_ROW) {
                        float2 c = *crow;
                        c.x += a0;
                        c.y += a1;
                        *crow = c;
                    }
                } else {
                    if (tag != kNone && lane < GR / 4) {
                        float4 v = *reinterpret_cast<const float4 *>(cache + slot * GR + 4 * lane);
                        red_add_v4(p.acc + (uint64_t)tag * GR + 4 * lane, v.x, v.y, v.z, v.w);
                    }
                    __syncwarp();
                    if (lane < HALF_ROW)
                        *crow = make_float2(a0, a1);
                    if (lane == 0)
                        tags[slot] = lc;
                }
                __syncwarp();
            }
        }
        if (!__any_sync(FULL, !done || p_cell != kNone))
            break;
    }

    // drain the cache
    __syncwarp();
    for (int slot = 0; slot < SLOTS; ++slot) {
        uint32_t tag = tags[slot];
        if (tag != kNone && lane < GR / 4) {
            float4 v = *reinterpret_cast<const float4 *>(cache + slot * GR + 4 * lane);
            red_add_v4(p.acc + (uint64_t)tag * GR + 4 * lane, v.x, v.y, v.z, v.w);
        }
    }
    bulk_wait_read(); // shared memory must outlive the bulk reductions' reads
    if (RAY && has_ray)
        ray_grad_store<DEG>(p, rg, r, ray, ra, G);
}

// accumulator -> reference-layout gradient outputs (+ optional finite scrub): flat over the output elements
// (consecutive threads, consecutive elements: the odd-length [N][A] rows leave fully coalesced), row length a
// compile-time constant, four elements per thread in flight.
template <typename AttrT, int DEG>
__global__ void __launch_bounds__(256) finalize_grads_kernel(const float *__restrict__ acc, uint32_t num_points,
                                                             float *__restrict__ points_grad,
                                                             AttrT *__restrict__ attr_grad, int scrub) {
    constexpr uint32_t A = attr_dim(DEG), SR = sh_row(DEG), GR = grad_row(DEG);
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)num_points * A;
#pragma unroll 4
    for (uint64_t e = gid; e < total; e += stride) {
        const uint64_t i = e / A;
        const uint32_t s = (uint32_t)(e % A);
        AttrT o = (AttrT)acc[i * GR + (s < A - 1 ? s : SR)];
        if (scrub && !isfinite((float)o))
            o = (AttrT)0.0f;
        attr_grad[e] = o;
    }
    const uint64_t total3 = (uint64_t)num_points * 3;
    for (uint64_t e = gid; e < total3; e += stride) {
        float g = acc[(e / 3) * GR + SR + 1 + (uint32_t)(e % 3)];
        if (scrub && !isfinite(g))
            g = 0.0f;
        points_grad[e] = g;
    }
}

// accumulator -> gradients of the model's PARAMETERS (the backward of get_trace_data fused in): the attribute
// gradient is rounded to the attribute dtype and scrubbed exactly like attr_grad above, then split into
// att_dc / att_sh and chained through activation_scale * softplus(density, beta=10).  Flat streaming form.
template <typename AttrT, int DEG>
__global__ void __launch_bounds__(256) finalize_params_kernel(const float *__restrict__ acc,
                                                              const float *__restrict__ density,
                                                              float activation_scale, uint32_t num_points,
                                                              float *__restrict__ points_grad,
                                                              float *__restrict__ att_dc_grad,
                                                              float *__restrict__ att_sh_grad,
                                                              float *__restrict__ density_grad, int scrub) {
    constexpr uint32_t A = attr_dim(DEG), SR = sh_row(DEG), GR = grad_row(DEG), REST = A - 4;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x, gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)num_points * A;
#pragma unroll 4
    for (uint64_t e = gid; e < total; e += stride) {
        const uint64_t i = e / A;
        const uint32_t s = (uint32_t)(e % A);
        AttrT o = (AttrT)acc[i * GR + (s < A - 1 ? s : SR)];
        if (scrub && !isfinite((float)o))
            o = (AttrT)0.0f;
        const float g = (float)o;
        if (s < 3)
            att_dc_grad[3 * i + s] = g;
        else if (s < A - 1)
            att_sh_grad[i * REST + (s - 3)] = g;
        else
            density_grad[i] = softplus_beta10_backward(g * activation_scale, density[i]);
    }
    const uint64_t total3 = (uint64_t)num_points * 3;
    for (uint64_t e = gid; e < total3; e += stride) {
        float g = acc[(e / 3) * GR + SR + 1 + (uint32_t)(e % 3)];
        if (scrub && !isfinite(g))
            g = 0.0f;
        points_grad[e] = g;
    }
}

// ------------------------------------------------------------------ multi-GPU: fused reduce + finalize
// The one exchange step of the ray-sharded path (SURVEY.md §8e): every rank holds a partial gradient
// accumulator [N][grad_row]; every rank needs the summed gradients in the reference layout.  Instead of
// ncclAllReduce -> finalize_grads_kernel (two passes over 218 MB per rank at 1 M points plus the collective's
// own staging), ONE kernel per rank works directly on peer-mapped memory over NVLink / NVSwitch:
//   * rank r owns the row blocks b = r, r + W, r + 2W, ... (kPeerRows rows each);
//   * for a block it loads the rows of ALL W accumulators (one local, W - 1 peer loads of 16 bytes per
//     thread, all in flight together), sums them in rank order (so every rank would compute the same bits),
//   * applies the finalize epilogue (reference layout [N][A] + [N][3], optional non-finite scrub, fp16
//     rounding once), staged through shared memory so that the unaligned 49-float rows leave as aligned
//     16-byte (fp16: 8-byte) stores,
//   * and stores the finished block into EVERY rank's output arrays (W - 1 peer stores per thread).
// Per rank: (W-1)/W of the accumulator comes in over NVLink and (W-1)/W of the outputs goes out, both directions
// at once; no intermediate buffer, no second pass.  The caller brackets the launch with cross-GPU barriers
// (all accumulators complete / all stores landed): radfoam_b200/sharded.py uses the symmetric-memory signal pads.
constexpr int kMaxPeers = 16;
constexpr int kPeerRows = 16; // rows per block: 16 * A floats is a whole number of 16-byte vectors for every A

struct PeerReduceParams {
    const float *acc[kMaxPeers];
    void *attr_grad[kMaxPeers];
    float *points_grad[kMaxPeers];
    uint32_t world, num_points, first_block, block_stride;
    int scrub;
    uint32_t rank;
    int debug_mode; // measurement only (RFB_PEER_DEBUG): 1 = store to the own rank only, 2 = load the own accumulator only
    // NVSwitch multicast addresses of the same three arrays (all null: plain peer loads / stores).  With them a
    // rank pulls only its own share through its link (the switch sums the W copies) and pushes it once (the
    // switch replicates it): (W-1)/W of the NVLink traffic of the peer-pointer form disappears.
    const float *mc_acc;
    void *mc_attr_grad;
    float *mc_points_grad;
};

// WORLD > 0: the number of ranks as a compile-time constant (2, 4, 8: exactly that many loads per thread in
// flight and no more registers than that needs, so more CTAs fit an SM); WORLD == 0: any world up to kMaxPeers.
template <int DEG, typename AttrT, int WORLD>
__global__ void __launch_bounds__(256) reduce_finalize_peers_kernel(const PeerReduceParams p) {
    constexpr int GR = grad_row(DEG), SR = sh_row(DEG), A = attr_dim(DEG);
    constexpr int ROW_VECS = GR / 4;                 // float4 per accumulator row
    constexpr int IN_VECS = kPeerRows * ROW_VECS;    // float4 loads per block (<= 208)
    constexpr int ATTR_VECS = kPeerRows * A / 4;     // 4-element stores of the attribute block
    constexpr int PTS_VECS = kPeerRows * 3 / 4;      // float4 stores of the points block
    static_assert(IN_VECS <= 256 && ATTR_VECS + PTS_VECS <= 256, "one pass per block");
    static_assert((kPeerRows * A) % 4 == 0 && (kPeerRows * 3) % 4 == 0, "blocks are whole vectors");
    __shared__ __align__(16) float rows[kPeerRows * GR];
    const uint32_t num_blocks = (p.num_points + kPeerRows - 1) / kPeerRows;
    const uint32_t t = threadIdx.x;
    for (uint32_t b = p.first_block + blockIdx.x * p.block_stride; b < num_blocks; b += gridDim.x * p.block_stride) {
        const uint32_t row0 = b * kPeerRows;
        const uint32_t nrows = min((uint32_t)kPeerRows, p.num_points - row0);
        if (t < nrows * ROW_VECS) {
            const uint64_t off = (uint64_t)row0 * GR + 4ull * t;
            if (p.mc_acc) {
                *reinterpret_cast<float4 *>(rows + 4 * t) = multimem_ld_reduce_add_v4(p.mc_acc + off);
            } else {
            constexpr int SLOTS = WORLD > 0 ? WORLD : kMaxPeers;
            const int world = WORLD > 0 ? WORLD : (int)p.world;
            float4 v[SLOTS];
#pragma unroll
            for (int w = 0; w < SLOTS; ++w)
                if (w < world)
                    v[w] = *reinterpret_cast<const float4 *>(p.acc[p.debug_mode == 2 ? p.rank : w] + off);
            float4 s = v[0];
#pragma unroll
            for (int w = 1; w < SLOTS; ++w)
                if (w < world) {
                    s.x += v[w].x;
                    s.y += v[w].y;
                    s.z += v[w].z;
                    s.w += v[w].w;
                }
            *reinterpret_cast<float4 *>(rows + 4 * t) = s;
            }
        }
        __syncthreads();
        const bool full = nrows == kPeerRows;
        const bool multicast = p.mc_acc != nullptr && full; // the ragged last block goes peer by peer
        if (t < ATTR_VECS) {
            // four consecutive elements of the block's [rows][A] output
            AttrT o[4];
            bool live[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t e = 4 * t + k, r = e / A, c = e % A;
                live[k] = r < nrows;
                float x = live[k] ? rows[r * GR + (c < A - 1 ? c : SR)] : 0.0f;
                AttrT a = (AttrT)x;
                if (p.scrub && !isfinite((float)a))
                    a = (AttrT)0.0f;
                o[k] = a;
            }
            const uint64_t e0 = (uint64_t)row0 * A + 4ull * t;
            if (multicast) {
                AttrT *dst = reinterpret_cast<AttrT *>(p.mc_attr_grad) + e0;
                if (sizeof(AttrT) == 4)
                    multimem_st_v4(reinterpret_cast<float *>(dst), *reinterpret_cast<const float4 *>(o));
                else
                    multimem_st_v2(dst, *reinterpret_cast<const float2 *>(o));
            } else
            for (uint32_t w = 0; w < p.world; ++w) {
                AttrT *dst = reinterpret_cast<AttrT *>(p.attr_grad[p.debug_mode == 1 ? p.rank : w]) + e0;
                if (full) {
                    if (sizeof(AttrT) == 4)
                        *reinterpret_cast<float4 *>(dst) = *reinterpret_cast<const float4 *>(o);
                    else
                        *reinterpret_cast<uint2 *>(dst) = *reinterpret_cast<const uint2 *>(o);
                } else {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (live[k])
                            dst[k] = o[k];
                }
            }
        } else if (t < ATTR_VECS + PTS_VECS) {
            const uint32_t u = t - ATTR_VECS;
            float o[4];
            bool live[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t e = 4 * u + k, r = e / 3, c = e % 3;
                live[k] = r < nrows;
                float x = live[k] ? rows[r * GR + SR + 1 + c] : 0.0f;
                if (p.scrub && !isfinite(x))
                    x = 0.0f;
                o[k] = x;
            }
            const uint64_t e0 = (uint64_t)row0 * 3 + 4ull * u;
            if (multicast)
                multimem_st_v4(p.mc_points_grad + e0, *reinterpret_cast<const float4 *>(o));
            else
            for (uint32_t w = 0; w < p.world; ++w) {
                float *dst = p.points_grad[p.debug_mode == 1 ? p.rank : w] + e0;
                if (full) {
                    *reinterpret_cast<float4 *>(dst) = *reinterpret_cast<const float4 *>(o);
                } else {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (live[k])
                            dst[k] = o[k];
                }
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ entry cell (SURVEY.md §8f.1)
// Nearest point of each query = the Voronoi cell that contains it = the cell a ray from that origin starts
// in (what scene.py:224-234 gets from radfoam.nn over the AABB tree, aabb_tree.cu:343-415, after a
// torch.unique over all ray origins).  Ray origins are camera positions: one per frame, a few hundred per
// training batch.  So the exact brute force is the cheap thing here, if it is tiled: U queries x N points
// distance evaluations, 12 N bytes of traffic in total (not per query), no tree to build or keep current
// while the points move every step.
//   nearest_points_kernel: a CTA streams its share of the points through shared memory in tiles; its 256
//     threads are Uc query lanes x S sub-slices (Uc = min(256, next power of two of U)), so every shared-
//     memory read is a broadcast (or conflict-free) and U = 1 keeps all lanes busy as well; per thread a
//     running (distance, index) minimum, merged by one 64-bit atomicMin on the packed key -- distance bits
//     (non-negative floats order like integers) above the index, i.e. exactly "smallest distance, lowest
//     index among equals".  Distances in the x0 + (x1 + x2) fma order.  A query without any comparable
//     distance (NaN) keeps the all-ones key, whose low word is kNone.
//   U comes from the host or, for the fused start-point path below, from device memory (no host sync).
constexpr int kNNTile = 1024;

__global__ void __launch_bounds__(256) nearest_points_kernel(const float *__restrict__ points, uint32_t num_points,
                                                             const float *__restrict__ queries,
                                                             uint32_t num_queries_host,
                                                             const uint32_t *__restrict__ num_queries_dev,
                                                             unsigned long long *__restrict__ best) {
    __shared__ float4 tile[kNNTile];
    const uint32_t U = num_queries_dev ? *num_queries_dev : num_queries_host;
    if (U == 0)
        return;
    uint32_t Uc = 1;
    while (Uc < U && Uc < 256u)
        Uc <<= 1;
    const uint32_t S = 256u / Uc, ql = threadIdx.x % Uc, sub = threadIdx.x / Uc;
    for (uint32_t q0 = 0; q0 < U; q0 += Uc) {
        const uint32_t q = q0 + ql;
        const bool live = q < U;
        float qx = 0.0f, qy = 0.0f, qz = 0.0f;
        if (live) {
            qx = queries[3 * (uint64_t)q];
            qy = queries[3 * (uint64_t)q + 1];
            qz = queries[3 * (uint64_t)q + 2];
        }
        float best_d = __int_as_float(0x7f800000);
        uint32_t best_i = kNone;
        for (uint64_t t0 = (uint64_t)blockIdx.x * kNNTile; t0 < num_points; t0 += (uint64_t)gridDim.x * kNNTile) {
            __syncthreads();
            const uint32_t cnt = (uint32_t)(num_points - t0 < (uint64_t)kNNTile ? num_points - t0 : kNNTile);
            for (uint32_t i = threadIdx.x; i < cnt; i += 256u)
                tile[i] = make_float4(points[3 * (t0 + i)], points[3 * (t0 + i) + 1], points[3 * (t0 + i) + 2], 0.0f);
            __syncthreads();
            if (live)
                for (uint32_t i = sub; i < cnt; i += S) {
                    const float4 pt = tile[i];
                    const float dx = pt.x - qx, dy = pt.y - qy, dz = pt.z - qz;
                    const float d2 = __fmaf_rn(dx, dx, __fmaf_rn(dy, dy, __fmul_rn(dz, dz)));
                    if (d2 < best_d) { // strict: the lowest index among this thread's equals stays
                        best_d = d2;
                        best_i = (uint32_t)t0 + i;
                    }
                }
        }
        if (live && best_i != kNone)
            atomicMin(best + q, ((unsigned long long)__float_as_uint(best_d) << 32) | best_i);
    }
}

__global__ void nearest_points_finish_kernel(const unsigned long long *__restrict__ best, uint32_t num_queries,
                                             uint32_t *__restrict__ indices) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < num_queries)
        indices[q] = (uint32_t)best[q]; // all-ones (never updated) -> kNone
}

// Start cell of every ray without a sort and without a host round trip (mirror of get_starting_point,
// scene.py:224-234): (1) the distinct ray origins are found with an open-addressing hash set keyed on the
// origin's bits; a table entry is just the index (+1) of the ray that claimed it, whose origin later arrivals
// compare with, so nothing has to be published before it is read.  Entries are read before they are CASed, so
// the 2 M rays of one camera cost a handful of atomics, not 2 M.  The claimer appends its origin to a dense
// query list.  (2) nearest_points_kernel over that list, its length read from device memory.  (3) every ray
// looks its start cell up through its table slot.  The table has >= 2 R entries, so it cannot fill up.
__global__ void origin_slots_kernel(const float *__restrict__ rays, uint32_t num_rays, uint32_t *table,
                                    uint32_t mask, uint32_t *__restrict__ slot_of_ray,
                                    uint32_t *__restrict__ query_of_slot, float *__restrict__ queries,
                                    uint32_t *num_queries) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= num_rays)
        return;
    const uint32_t *bits = reinterpret_cast<const uint32_t *>(rays);
    const uint32_t ox = bits[6 * (uint64_t)r], oy = bits[6 * (uint64_t)r + 1], oz = bits[6 * (uint64_t)r + 2];
    uint32_t h = (ox * 0x9E3779B1u) ^ (oy * 0x85EBCA77u) ^ (oz * 0xC2B2AE3Du);
    h ^= h >> 15;
    for (h &= mask;; h = (h + 1u) & mask) {
        uint32_t owner = *reinterpret_cast<volatile uint32_t *>(table + h);
        if (owner == 0u) {
            owner = atomicCAS(table + h, 0u, r + 1u);
            if (owner == 0u) { // claimed: this ray's origin becomes a query
                const uint32_t qn = atomicAdd(num_queries, 1u);
                query_of_slot[h] = qn;
                queries[3 * (uint64_t)qn] = __uint_as_float(ox);
                queries[3 * (uint64_t)qn + 1] = __uint_as_float(oy);
                queries[3 * (uint64_t)qn + 2] = __uint_as_float(oz);
                slot_of_ray[r] = h;
                return;
            }
        }
        const uint64_t o = (uint64_t)(owner - 1u) * 6;
        if (bits[o] == ox && bits[o + 1] == oy && bits[o + 2] == oz) {
            slot_of_ray[r] = h;
            return;
        }
    }
}

__global__ void start_points_scatter_kernel(const uint32_t *__restrict__ slot_of_ray, uint32_t num_rays,
                                            const uint32_t *__restrict__ query_of_slot,
                                            const unsigned long long *__restrict__ best,
                                            uint32_t *__restrict__ start) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < num_rays)
        start[r] = (uint32_t)best[query_of_slot[slot_of_ray[r]]];
}

// ------------------------------------------------------------------ point location by walking the adjacency graph
// The CSR adjacency the tracer takes is the Delaunay graph of the points, and on a Delaunay graph a greedy walk
// reaches the nearest site: when s is not the nearest point of q, the segment s -> q leaves the Voronoi cell of s
// through a face shared with a Delaunay neighbour j, and beyond that face j is strictly closer to q than s.  So
// every query costs a handful of row scans (about 15.5 distances each) from a nearby seed, with no tree to build
// or keep current while the points move.
//   Order: (d2, index) packed into one 64-bit key -- distance bits above the index, exactly "smaller distance,
//   lower index among equals" (rfb_nearest_point's rule); NaN distances count as +inf.  d2 in the x0 + (x1 + x2)
//   fma order of nearest_points_kernel.  A step moves to the smallest key of the row and is taken only if that
//   key is smaller than the current one, so the walk terminates on any adjacency (the key strictly decreases).
//   Seed: the hint when it names a point, else the nearest of a fixed strided sample of the points (spatially
//   sorted points make a strided sample an even cover of the scene; unsorted points only make the walks longer).
//   The sample streams through shared memory in tiles, every thread of the CTA reading the same entry.
constexpr uint32_t kLocateTile = 1024;

struct LocateParams {
    const float *points;
    const uint32_t *adj, *off;
    const float *queries;
    const uint32_t *hints; // nullptr: every seed from the sample
    uint32_t num_points, num_queries;
    uint32_t sample, stride; // seed sample: points[k * stride], k < sample
};

__device__ __forceinline__ float query_d2(float px, float py, float pz, float qx, float qy, float qz) {
    const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
    return __fmaf_rn(dx, dx, __fmaf_rn(dy, dy, __fmul_rn(dz, dz)));
}

__device__ __forceinline__ unsigned long long locate_key(float d2, uint32_t i) {
    const uint32_t bits = d2 != d2 ? 0x7f800000u : __float_as_uint(d2); // d2 >= +0: the bits order like the floats
    return ((unsigned long long)bits << 32) | i;
}

__device__ __forceinline__ unsigned long long point_key(const float *__restrict__ points, uint32_t j, float qx,
                                                        float qy, float qz) {
    const uint64_t b = 3 * (uint64_t)j;
    return locate_key(query_d2(__ldg(points + b), __ldg(points + b + 1), __ldg(points + b + 2), qx, qy, qz), j);
}

// The greedy walk from `s`: the key of the local minimum it ends in.
__device__ __forceinline__ unsigned long long walk_to_nearest(const LocateParams &p, uint32_t s, float qx, float qy,
                                                              float qz) {
    unsigned long long key = point_key(p.points, s, qx, qy, qz);
    for (;;) {
        unsigned long long best = key;
        const uint32_t end = __ldg(p.off + s + 1);
        for (uint32_t e = __ldg(p.off + s); e < end; ++e) {
            const unsigned long long k = point_key(p.points, __ldg(p.adj + e), qx, qy, qz);
            best = k < best ? k : best;
        }
        if (best == key)
            return key;
        key = best;
        s = (uint32_t)best;
    }
}

// Cell of query q: UINT32_MAX for q >= num_queries, for a NaN coordinate, and when even the cell found is at a
// non-finite distance (rfb_nearest_point finds no point then either).  Every thread of the CTA must call it: the
// seed search synchronises.
__device__ __forceinline__ uint32_t locate_point(const LocateParams &p, uint32_t q) {
    __shared__ float4 tile[kLocateTile];
    __shared__ int seeds_wanted;
    const bool live = q < p.num_queries;
    float qx = 0.0f, qy = 0.0f, qz = 0.0f;
    uint32_t seed = kNone;
    if (live) {
        qx = __ldg(p.queries + 3 * (uint64_t)q);
        qy = __ldg(p.queries + 3 * (uint64_t)q + 1);
        qz = __ldg(p.queries + 3 * (uint64_t)q + 2);
        if (p.hints) {
            const uint32_t h = __ldg(p.hints + q);
            seed = h < p.num_points ? h : kNone;
        }
    }
    const bool nan = qx != qx || qy != qy || qz != qz;
    const bool need = live && !nan && seed == kNone;
    if (threadIdx.x == 0)
        seeds_wanted = 0;
    __syncthreads();
    if (need)
        seeds_wanted = 1;
    __syncthreads();
    if (seeds_wanted) {
        float best_d = __int_as_float(0x7f800000);
        uint32_t best_i = 0; // no sample point at a finite distance: start from point 0
        for (uint32_t t0 = 0; t0 < p.sample; t0 += kLocateTile) {
            const uint32_t cnt = p.sample - t0 < kLocateTile ? p.sample - t0 : kLocateTile;
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
                const uint64_t j = 3 * ((uint64_t)(t0 + i) * p.stride);
                tile[i] = make_float4(__ldg(p.points + j), __ldg(p.points + j + 1), __ldg(p.points + j + 2), 0.0f);
            }
            __syncthreads();
            if (need)
                for (uint32_t i = 0; i < cnt; ++i) {
                    const float4 pt = tile[i];
                    const float d2 = query_d2(pt.x, pt.y, pt.z, qx, qy, qz);
                    if (d2 < best_d) { // strict, indices ascending: the lowest index among equals stays
                        best_d = d2;
                        best_i = (t0 + i) * p.stride;
                    }
                }
        }
        if (need)
            seed = best_i;
    }
    if (!live || nan)
        return kNone;
    const unsigned long long key = walk_to_nearest(p, seed, qx, qy, qz);
    return (key >> 32) >= 0x7f800000ull ? kNone : (uint32_t)key;
}

__global__ void __launch_bounds__(256) locate_points_kernel(const LocateParams p, uint32_t *__restrict__ indices) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t cell = locate_point(p, q);
    if (q < p.num_queries)
        indices[q] = cell;
}

// ------------------------------------------------------------------ field sampling
// The field at a point is its cell's attribute row: density = the last column, and the colour seen along a unit
// direction d = max(0, 0.5 + sum_k Y_k(d) c_k) with the tracer's own basis and FFMA chain (sh_basis,
// sh_coeffs_to_rgb), read from the caller's attributes -- the same floats the tracer's SH mirror holds -- so that
// it is the colour the tracer composites for that cell along a ray with direction d.  A query without a cell
// (UINT32_MAX) gets NaN.
template <int DEG, typename AttrT>
__global__ void __launch_bounds__(256) sample_field_kernel(const LocateParams p, const AttrT *__restrict__ attrs,
                                                           const float *__restrict__ dirs,
                                                           uint32_t *__restrict__ cells, AttrT *__restrict__ density,
                                                           AttrT *__restrict__ rgb) {
    constexpr int A = attr_dim(DEG), NC = 3 * sh_dim(DEG);
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t cell = locate_point(p, q);
    if (q >= p.num_queries)
        return;
    cells[q] = cell;
    const float nan = __int_as_float(0x7fc00000);
    if (cell == kNone) {
        density[q] = (AttrT)nan;
        if (rgb)
            rgb[3 * (uint64_t)q] = rgb[3 * (uint64_t)q + 1] = rgb[3 * (uint64_t)q + 2] = (AttrT)nan;
        return;
    }
    const AttrT *row = attrs + (uint64_t)cell * A;
    density[q] = row[A - 1];
    if (!rgb)
        return;
    float dx = __ldg(dirs + 3 * (uint64_t)q), dy = __ldg(dirs + 3 * (uint64_t)q + 1),
          dz = __ldg(dirs + 3 * (uint64_t)q + 2);
    normalize_dir(dx, dy, dz);
    float sh[sh_dim(DEG)];
    sh_basis<DEG>(dx, dy, dz, sh);
    float v[NC];
#pragma unroll
    for (int i = 0; i < NC; ++i)
        v[i] = (float)row[i];
    float r, g, b;
    sh_coeffs_to_rgb<DEG>(v, sh, r, g, b);
    rgb[3 * (uint64_t)q] = (AttrT)r;
    rgb[3 * (uint64_t)q + 1] = (AttrT)g;
    rgb[3 * (uint64_t)q + 2] = (AttrT)b;
}

// Backward of the sampling: acc[cell][3k + c] += Y_k(d) * dL/drgb_c (0 where the forward's rgb_c is 0, the
// tracer's ReLU mask) and acc[cell][A - 1] += dL/ddensity, in fp32.  Grid sampling puts many queries in one cell,
// so a warp first sums the rows of its lanes that share a cell: every lane stages its row in shared memory, the
// lanes of a group split the columns between them, and each column of a group reaches L2 as ONE atomic.
constexpr int kSampleBwdBlock = 128;

template <int DEG, typename AttrT>
__global__ void __launch_bounds__(kSampleBwdBlock) sample_field_backward_kernel(
    const uint32_t *__restrict__ cells, uint32_t num_queries, uint32_t num_points, const float *__restrict__ dirs,
    const AttrT *__restrict__ rgb, const AttrT *__restrict__ rgb_grad, const AttrT *__restrict__ density_grad,
    float *__restrict__ acc) {
    constexpr int A = attr_dim(DEG), NC = 3 * sh_dim(DEG);
    __shared__ float rows[kSampleBwdBlock / 32][32][A];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t cell = q < num_queries ? __ldg(cells + q) : kNone;
    if (cell >= num_points)
        cell = kNone; // a query that found no cell has no gradient
    if (cell != kNone) {
        float *row = rows[warp][lane];
        if (rgb_grad) {
            float dx = __ldg(dirs + 3 * (uint64_t)q), dy = __ldg(dirs + 3 * (uint64_t)q + 1),
                  dz = __ldg(dirs + 3 * (uint64_t)q + 2);
            normalize_dir(dx, dy, dz);
            float sh[sh_dim(DEG)];
            sh_basis<DEG>(dx, dy, dz, sh);
            float g[3];
#pragma unroll
            for (int c = 0; c < 3; ++c)
                g[c] = (float)rgb[3 * (uint64_t)q + c] == 0.0f ? 0.0f : (float)rgb_grad[3 * (uint64_t)q + c];
#pragma unroll
            for (int i = 0; i < NC; ++i)
                row[i] = __fmul_rn(sh[i / 3], g[i % 3]);
        } else {
#pragma unroll
            for (int i = 0; i < NC; ++i)
                row[i] = 0.0f;
        }
        row[A - 1] = density_grad ? (float)density_grad[q] : 0.0f;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, cell);
    __syncwarp();
    if (cell == kNone)
        return;
    const int size = __popc(peers), rank = __popc(peers & ((1u << lane) - 1u));
    for (int c = rank; c < A; c += size) {
        float s = 0.0f;
        for (unsigned m = peers; m; m &= m - 1u)
            s = __fadd_rn(s, rows[warp][__ffs(m) - 1][c]);
        if (s != 0.0f)
            atomicAdd(acc + (uint64_t)cell * A + c, s);
    }
}

// attribute_grad = the fp32 accumulator rounded once to the attribute dtype
__global__ void __launch_bounds__(256) round_to_half_kernel(const float *__restrict__ acc, uint64_t n,
                                                            __half *__restrict__ out) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = __float2half_rn(acc[i]);
}

// ------------------------------------------------------------------ farthest neighbour (SURVEY.md §8f.4)
// Per cell: the adjacent point farthest from it and half the mean neighbour distance ("cell radius"),
// what the densification pass reads (scene.py:434-461; reference kernel triangulation_ops.cu:9-44).
// Arithmetic as the reference's SASS has it: d = q - p, |d|^2 = fma(dx,dx, fma(dy,dy, dz*dz)), IEEE sqrt and
// divide, strict '>' first-max from 0, and `sum += 0.5 * dist` evaluated in fp64 and rounded back to fp32 every
// iteration.  That last step needs no fp64: 0.5*dist is exact and rounding an exact sum to 53 then to 24 bits
// equals rounding it to 24 bits directly whenever 53 >= 2*24 + 2 (double rounding is innocuous for +), so
// fmaf(dist, 0.5f, sum) is bit-identical and frees the kernel from the F2F/DFMA pipe the reference's form binds
// on.  Shape: one thread per row, four faces in flight; 8 lanes per row with the serial chain replayed by shuffle,
// the same over a float4 point mirror, and a thread per row over the mirror were built and were slower.
__device__ __forceinline__ float neighbour_distance(const float *__restrict__ points, uint64_t j, float px,
                                                    float py, float pz) {
    const float dx = __fsub_rn(points[3 * j], px), dy = __fsub_rn(points[3 * j + 1], py),
                dz = __fsub_rn(points[3 * j + 2], pz);
    return __fsqrt_rn(__fmaf_rn(dx, dx, __fmaf_rn(dy, dy, __fmul_rn(dz, dz))));
}

__global__ void __launch_bounds__(256) farthest_neighbor_kernel(const float *__restrict__ points,
                                                                const uint32_t *__restrict__ adjacency,
                                                                const uint32_t *__restrict__ offsets,
                                                                uint32_t num_points,
                                                                uint32_t *__restrict__ indices,
                                                                float *__restrict__ cell_radius) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_points)
        return;
    const float px = points[3 * i], py = points[3 * i + 1], pz = points[3 * i + 2];
    const uint32_t begin = offsets[i], num_faces = offsets[i + 1] - begin;
    float sum = 0.0f, farthest = 0.0f;
    uint32_t farthest_idx = kNone;
#pragma unroll 4
    for (uint32_t f = 0; f < num_faces; ++f) {
        const uint32_t j = adjacency[begin + f];
        const float dist = neighbour_distance(points, j, px, py, pz);
        sum = __fmaf_rn(dist, 0.5f, sum);
        if (dist > farthest) {
            farthest = dist;
            farthest_idx = j;
        }
    }
    indices[i] = farthest_idx;
    cell_radius[i] = __fdiv_rn(sum, __uint2float_rn(num_faces)); // 0/0 = NaN for an empty row, as upstream
}

// ------------------------------------------------------------------ benchmark
struct CameraParams {
    float position[3], forward[3], right[3], up[3];
    float fov;
    uint32_t width, height;
    int model;
};

// cast_ray (camera.h:56-85).  The packed RGBA8 output is held to byte equality with the reference's kernel, so
// the arithmetic is pinned to the association of its SASS (cuobjdump of oracle/_ref, benchmark<float,0>):
//   aspect = w / h, x = i / w, y = j / h                       IEEE divisions
//   u = fma(x, 2, -1) * aspect;  v = 1 - (y + y)
//   pinhole: s = 1 / tanf(fov * 0.5);  d_k = fma(v, up_k, fma(s, forward_k, u * right_k))
//   fisheye: theta = atan2f(v, u);  phi = sqrtf(fma(u, u, v * v)) * fov, clamped to pi - 1e-6 with mask 0;
//            a = sinf(phi) * cosf(theta), b = sinf(phi) * sinf(theta)
//            d_k = fma(cosf(phi), forward_k, fma(b, up_k, a * right_k))
//   d /= sqrtf(fma(d0, d0, fma(d1, d1, d2 * d2)))  when that is > 0;  d *= mask
// tanf / atan2f / sinf / cosf are the same libdevice routines the reference calls.
__device__ __forceinline__ void cast_ray(const CameraParams &c, int i, int j, RayGeom &ray) {
    const float aspect = __fdiv_rn((float)c.width, (float)c.height);
    const float x = __fdiv_rn((float)i, (float)c.width);
    const float y = __fdiv_rn((float)j, (float)c.height);
    const float u = __fmul_rn(__fmaf_rn(x, 2.0f, -1.0f), aspect);
    const float v = __fsub_rn(1.0f, __fadd_rn(y, y));
    float mask = 1.0f;
    float d[3];
    if (c.model == 0) {
        const float s = __fdiv_rn(1.0f, tanf(__fmul_rn(c.fov, 0.5f)));
#pragma unroll
        for (int k = 0; k < 3; ++k)
            d[k] = __fmaf_rn(v, c.up[k], __fmaf_rn(s, c.forward[k], __fmul_rn(u, c.right[k])));
    } else {
        const float theta = atan2f(v, u);
        float phi = __fmul_rn(__fsqrt_rn(__fmaf_rn(u, u, __fmul_rn(v, v))), c.fov);
        if (phi >= 3.14159265358979323846f) {
            phi = 3.14159265358979323846f - 1e-6f;
            mask = 0.0f;
        }
        const float sp = sinf(phi);
        const float a = __fmul_rn(sp, cosf(theta)), b = __fmul_rn(sp, sinf(theta));
        const float cp = cosf(phi);
#pragma unroll
        for (int k = 0; k < 3; ++k)
            d[k] = __fmaf_rn(cp, c.forward[k], __fmaf_rn(b, c.up[k], __fmul_rn(a, c.right[k])));
    }
    float n2 = __fmaf_rn(d[0], d[0], __fmaf_rn(d[1], d[1], __fmul_rn(d[2], d[2])));
    if (n2 > 0.0f) {
        float n = __fsqrt_rn(n2);
        d[0] = __fdiv_rn(d[0], n);
        d[1] = __fdiv_rn(d[1], n);
        d[2] = __fdiv_rn(d[2], n);
    }
    ray.ox = c.position[0];
    ray.oy = c.position[1];
    ray.oz = c.position[2];
    ray.dx = __fmul_rn(d[0], mask);
    ray.dy = __fmul_rn(d[1], mask);
    ray.dz = __fmul_rn(d[2], mask);
}

// make_rgba8 (tracing_utils.cuh:105-115): clamp, truncate
__device__ __forceinline__ uint32_t pack_rgba8(float r, float g, float b, float a) {
    r = fmaxf(0.0f, fminf(1.0f, r));
    g = fmaxf(0.0f, fminf(1.0f, g));
    b = fmaxf(0.0f, fminf(1.0f, b));
    a = fmaxf(0.0f, fminf(1.0f, a));
    int ri = (int)__fmul_rn(r, 255.0f), gi = (int)__fmul_rn(g, 255.0f), bi = (int)__fmul_rn(b, 255.0f),
        ai = (int)__fmul_rn(a, 255.0f);
    return ((uint32_t)ai << 24) | ((uint32_t)bi << 16) | ((uint32_t)gi << 8) | (uint32_t)ri;
}

struct BenchmarkParams {
    const float4 *cells;
    const float *sh_rows;
    const uint32_t *start; // one element
    uint32_t *out;
    CameraParams cam;
    uint32_t blocks_x;
    float weight_threshold;
    uint32_t max_steps;
    uint32_t *exact_flag;
};

template <int DEG, typename Faces, int MODE>
__global__ void __launch_bounds__(kBlock) benchmark_kernel(const BenchmarkParams p, const Faces fa) {
    if (MODE == kScanExactTwin && *p.exact_flag == 0u)
        return;
    uint32_t r;
    if (!thread_ray(p.cam.width * p.cam.height, p.cam.width, p.blocks_x, r))
        return;
    uint32_t pi = r % p.cam.width, pj = r / p.cam.width;
    RayGeom ray;
    cast_ray(p.cam, (int)pi, (int)pj, ray);
    float nrm = __fsqrt_rn(__fmaf_rn(ray.dx, ray.dx, __fmaf_rn(ray.dy, ray.dy, __fmul_rn(ray.dz, ray.dz))));
    if (nrm < 0.1f) {
        p.out[r] = 0;
        return;
    }
    float sh[sh_dim(DEG)];
    sh_basis<DEG>(ray.dx, ray.dy, ray.dz, sh);
    float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
    auto cell_fn = [&](uint32_t cell, const float4 &pc, float t0, float t1, const float4 &, uint32_t) -> bool {
        T = composite_cell<DEG>(p.sh_rows, sh, cell, pc.w, t0, t1, T, cr, cg, cb, [](float) {});
        return T > p.weight_threshold;
    };
    if (MODE == kScanFast && needs_exact_scan(ray.dx, ray.dy, ray.dz))
        *p.exact_flag = 1u;
    walk<MODE == kScanExactTwin>(fa, p.cells, ray, __ldg(p.start), p.max_steps, cell_fn);
    p.out[r] = pack_rgba8(cr, cg, cb, 1.0f);
}

// ------------------------------------------------------------------ visualization
// Pipeline::trace_visualization (pipeline.h:102-115, kernel pipeline.cu:345-470): the benchmark frame's walk
// plus a quantile depth and the step count, and one of four outputs chosen by a uniform runtime branch.
enum VisMode { kVisRGB = 0, kVisDepth = 1, kVisAlpha = 2, kVisIntersections = 3 };

// CMapTable (typing.h:143-146): caller-owned device tables, indexed by colour map; data[m] is float[sizes[m]][3]
struct CMapTable {
    const float *const *data;
    const int *sizes;
};

struct VisualizationParams {
    const float4 *cells;
    const float *sh_rows;
    CameraParams cam;
    uint32_t start;
    uint32_t blocks_x;
    float weight_threshold;
    uint32_t max_steps;
    int mode;
    int color_map;
    float bg[3];
    uint32_t checker_bg;
    float max_depth;
    float depth_quantile;
    CMapTable cmap;
    uint32_t *exact_flag;
};

// The frame goes to a surface (what the reference writes: surf2Dwrite at byte column 4x, trap on out-of-range) or
// to a linear uint32[height][width] buffer; both in the surface's bottom-up row order.
#ifdef RFB_EMU
// The CPU kernel-logic emulator has no surfaces: there the handle is the address of an RfbEmuSurface, and a store
// outside it aborts where the device's default boundary mode traps.
struct RfbEmuSurface {
    void *data;
    uint64_t pitch; // bytes per row
    uint32_t width_bytes, height;
};
#endif
struct SurfaceOut {
    cudaSurfaceObject_t surf;
    __device__ __forceinline__ void store(uint32_t x, uint32_t y, uint32_t v) const {
#ifdef RFB_EMU
        const RfbEmuSurface *s = reinterpret_cast<const RfbEmuSurface *>(surf);
        if ((uint64_t)4u * x + 4u > s->width_bytes || y >= s->height)
            abort();
        memcpy(static_cast<char *>(s->data) + (uint64_t)y * s->pitch + 4u * (uint64_t)x, &v, 4);
#else
        surf2Dwrite(v, surf, (int)(4u * x), (int)y);
#endif
    }
};
struct LinearOut {
    uint32_t *out;
    uint32_t width;
    __device__ __forceinline__ void store(uint32_t x, uint32_t y, uint32_t v) const {
        out[(uint64_t)y * width + x] = v;
    }
};

// cvt.rzi.s32.f32, with its rules for NaN (-> 0) and out-of-range values (saturation at INT_MIN / INT_MAX) written
// out, so that the same source means the same thing where a plain cast would be undefined (the CPU emulator).
__device__ __forceinline__ int f2i_rz_sat(float x) {
    if (x != x)
        return 0;
    if (x >= 2147483648.0f)
        return 2147483647;
    if (x < -2147483648.0f)
        return (int)0x80000000u;
    return (int)x;
}

// The .SAT modifier: clamp to [+0, 1], NaN -> +0.
__device__ __forceinline__ float sat_unit(float x) { return x > 0.0f ? (x < 1.0f ? x : 1.0f) : 0.0f; }

// The reference's clamps fold into the .SAT of the instruction that makes the value (FFMA.SAT / FADD.SAT in its
// SASS, visualization<float,0,128>), so a NaN channel becomes 0, not the 255 std::min/std::max would give.
// r, g, b are already in [0, 1].
__device__ __forceinline__ uint32_t pack_unit_rgb8(float r, float g, float b) {
    const uint32_t ri = (uint32_t)(int)__fmul_rn(r, 255.0f);
    const uint32_t gi = (uint32_t)(int)__fmul_rn(g, 255.0f);
    const uint32_t bi = (uint32_t)(int)__fmul_rn(b, 255.0f);
    return 0xff000000u | (bi << 16) | (gi << 8) | ri;
}

// colormap (tracing_utils.cuh:117-130), association read from the reference's SASS (visualization<float,0,128>):
//   p = (float)(L - 1) * v;  i0 = cvt.rzi.s32(p)  (NaN -> 0, saturating at INT_MIN / INT_MAX);  t = p - (float)i0
//   i1 = i0 + 1 (32-bit wrap);  both clamped to [0, L - 1]
//   c_k = sat(fma(1 - t, table[i0]_k, t * table[i1]_k))
__device__ __forceinline__ uint32_t colormap_rgba8(float v, int map, const CMapTable &cm) {
    const int last = cm.sizes[map] - 1;
    const float *vals = cm.data[map];
    const float pos = __fmul_rn((float)last, v);
    const int i0 = f2i_rz_sat(pos);
    const int i1 = (int)((uint32_t)i0 + 1u);
    const float t = __fsub_rn(pos, (float)i0);
    const float u = __fsub_rn(1.0f, t);
    const float *a = vals + 3 * (int64_t)max(0, min(i0, last));
    const float *b = vals + 3 * (int64_t)max(0, min(i1, last));
    return pack_unit_rgb8(sat_unit(__fmaf_rn(u, a[0], __fmul_rn(t, b[0]))),
                          sat_unit(__fmaf_rn(u, a[1], __fmul_rn(t, b[1]))),
                          sat_unit(__fmaf_rn(u, a[2], __fmul_rn(t, b[2]))));
}

template <int DEG, typename Faces, int MODE, typename Out>
__global__ void __launch_bounds__(kBlock) visualization_kernel(const VisualizationParams p, const Faces fa,
                                                               const Out out) {
    if (MODE == kScanExactTwin && *p.exact_flag == 0u)
        return;
    uint32_t r;
    if (!thread_ray(p.cam.width * p.cam.height, p.cam.width, p.blocks_x, r))
        return;
    const uint32_t pi = r % p.cam.width, pj = r / p.cam.width;
    const uint32_t row = p.cam.height - 1u - pj;
    RayGeom ray;
    cast_ray(p.cam, (int)pi, (int)pj, ray);
    float nrm = __fsqrt_rn(__fmaf_rn(ray.dx, ray.dx, __fmaf_rn(ray.dy, ray.dy, __fmul_rn(ray.dz, ray.dz))));
    if (nrm < 0.1f) {
        out.store(pi, row, 0u);
        return;
    }
    float sh[sh_dim(DEG)];
    sh_basis<DEG>(ray.dx, ray.dy, ray.dz, sh);
    const float q = p.depth_quantile;
    float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
    float depth = 0.0f;
    bool passed = false;
    auto cell_fn = [&](uint32_t cell, const float4 &pc, float t0, float t1, const float4 &, uint32_t) -> bool {
        const float s = pc.w;
        const float Tn = composite_cell<DEG>(p.sh_rows, sh, cell, s, t0, t1, T, cr, cg, cb, [](float) {});
        if (!passed && Tn < q) { // the forward's quantile depth, first quantile only
            depth = __fadd_rn(t0, __fdiv_rn(logf(__fdiv_rn(T, q)), s));
            passed = true;
        }
        T = Tn;
        return T > p.weight_threshold;
    };
    if (MODE == kScanFast && needs_exact_scan(ray.dx, ray.dy, ray.dz))
        *p.exact_flag = 1u;
    const uint32_t n = walk<MODE == kScanExactTwin>(fa, p.cells, ray, p.start, p.max_steps, cell_fn);

    uint32_t v;
    if (p.mode == kVisRGB) {
        float bg0 = p.bg[0], bg1 = p.bg[1], bg2 = p.bg[2];
        if (p.checker_bg) // 20-pixel checker: 0.3 where the two square parities agree, else 0.5
            bg0 = bg1 = bg2 = (((pi / 20u) ^ (pj / 20u)) & 1u) ? 0.5f : 0.3f;
        v = pack_unit_rgb8(sat_unit(__fmaf_rn(T, bg0, cr)), sat_unit(__fmaf_rn(T, bg1, cg)),
                           sat_unit(__fmaf_rn(T, bg2, cb)));
    } else if (p.mode == kVisDepth) {
        v = colormap_rgba8(__fdiv_rn(depth, p.max_depth), p.color_map, p.cmap);
    } else if (p.mode == kVisAlpha) {
        const float a = sat_unit(__fsub_rn(1.0f, T));
        v = pack_unit_rgb8(a, a, a);
    } else {
        v = colormap_rgba8(__fdiv_rn(__uint2float_rn(n - 1u), __uint2float_rn(p.max_steps)), p.color_map, p.cmap);
    }
    out.store(pi, row, v);
}

// ------------------------------------------------------------------ surface extraction (rfb_surface_count / _write)
// Cell C_i = box ∩ { x : (p_k - p_i).x <= (p_k - p_i).(p_i + p_k)/2 } over the neighbours k of row i with p_k != p_i:
// the region the walk treats as cell i.  For CSR entry e = (i, j) with inside[i], !inside[j] and p_j != p_i the
// polygon F_e = C_i ∩ plane_e, vertices counter-clockwise seen from j.  Geometry in fp64, rounded once to fp32.
// Both passes run a warp per row (the row's entries on its lanes; rows that are not inside leave at once) and get
// every polygon from surface_polygon, so the write pass reproduces the count pass's vertex counts exactly.
constexpr int kSurfaceMaxVerts = 32; // a polygon that needs more fails the call (kernel-local ping-pong buffers)
constexpr int kSurfaceBlock = 256;   // 8 rows per CTA
constexpr int kScanBlock = 256, kScanItems = 4, kScanTile = kScanBlock * kScanItems;

struct SurfaceParams {
    const float *points;
    const uint32_t *adj;
    const uint32_t *off;
    const uint8_t *inside;
    uint32_t num_points, num_entries;
    float lo[3], hi[3];
};

// Keeps the part of `in` (n vertices) where (x - m).nrm <= 0, vertex order preserved (Sutherland-Hodgman).  A new
// vertex is made only where an edge crosses the plane strictly, so a vertex on the plane is never doubled.  Returns
// the vertex count, or -1 when it would exceed MaxVerts.  NaN distances drop their vertices.
template <int MaxVerts = kSurfaceMaxVerts>
__device__ __forceinline__ int clip_polygon(const double (*in)[3], int n, double (*out)[3], const double *nrm,
                                            const double *m) {
    if (n == 0)
        return 0;
    auto dist = [&](const double *v) { return (v[0] - m[0]) * nrm[0] + (v[1] - m[1]) * nrm[1] + (v[2] - m[2]) * nrm[2]; };
    int k = 0;
    const double *prev = in[n - 1];
    double dp = dist(prev);
    for (int a = 0; a < n; ++a) {
        const double *cur = in[a];
        const double dc = dist(cur);
        if ((dp < 0.0 && dc > 0.0) || (dp > 0.0 && dc < 0.0)) {
            if (k == MaxVerts)
                return -1;
            const double t = dp / (dp - dc);
            for (int c = 0; c < 3; ++c)
                out[k][c] = prev[c] + t * (cur[c] - prev[c]);
            ++k;
        }
        if (dc <= 0.0) {
            if (k == MaxVerts)
                return -1;
            for (int c = 0; c < 3; ++c)
                out[k][c] = cur[c];
            ++k;
        }
        prev = cur;
        dp = dc;
    }
    return k;
}

__device__ __forceinline__ void load_point(const float *__restrict__ points, uint32_t i, float *q) {
    q[0] = __ldg(points + 3 * (uint64_t)i);
    q[1] = __ldg(points + 3 * (uint64_t)i + 1);
    q[2] = __ldg(points + 3 * (uint64_t)i + 2);
}

__device__ __forceinline__ bool same_point(const float *a, const float *b) {
    return a[0] == b[0] && a[1] == b[1] && a[2] == b[2];
}

// F_e for entry e of row i into `out` (kSurfaceMaxVerts vertices): its vertex count when the polygon is emitted, 0
// when it is not (filter, or fewer than 3 vertices), -1 when it needs more than kSurfaceMaxVerts vertices.
__device__ __forceinline__ int surface_polygon(const SurfaceParams &p, uint32_t i, uint32_t e,
                                               double (*out)[3]) {
    const uint32_t j = __ldg(p.adj + e);
    if (j >= p.num_points || p.inside[j])
        return 0;
    float pi[3], pj[3];
    load_point(p.points, i, pi);
    load_point(p.points, j, pj);
    if (same_point(pi, pj))
        return 0;
    double buf[kSurfaceMaxVerts][3];
    double nrm[3], m[3];
    for (int c = 0; c < 3; ++c) {
        nrm[c] = (double)pj[c] - (double)pi[c];
        m[c] = 0.5 * ((double)pi[c] + (double)pj[c]);
    }
    // plane ∩ a square around the midpoint that covers the box: half-width twice the box's half-diagonal plus the
    // midpoint's distance from the box centre, in an orthonormal (u, v) with u x v = nrm / |nrm|
    double r2 = 0.0, h2 = 0.0;
    for (int c = 0; c < 3; ++c) {
        const double lo = p.lo[c], hi = p.hi[c], mid = 0.5 * (lo + hi);
        r2 += (m[c] - mid) * (m[c] - mid);
        h2 += 0.25 * (hi - lo) * (hi - lo);
    }
    const double R = 2.0 * (sqrt(r2) + sqrt(h2));
    const double ax = fabs(nrm[0]), ay = fabs(nrm[1]), az = fabs(nrm[2]);
    const int a = ax <= ay && ax <= az ? 0 : (ay <= az ? 1 : 2); // nrm x (axis of its smallest component)
    double u[3] = {0.0, 0.0, 0.0};
    u[(a + 1) % 3] = nrm[(a + 2) % 3];
    u[(a + 2) % 3] = -nrm[(a + 1) % 3];
    const double un = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
    const double nn = sqrt(nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2]);
    for (int c = 0; c < 3; ++c)
        u[c] /= un;
    const double v[3] = {(nrm[1] * u[2] - nrm[2] * u[1]) / nn, (nrm[2] * u[0] - nrm[0] * u[2]) / nn,
                         (nrm[0] * u[1] - nrm[1] * u[0]) / nn};
    const double su[4] = {1.0, -1.0, -1.0, 1.0}, sv[4] = {1.0, 1.0, -1.0, -1.0};
    for (int k = 0; k < 4; ++k)
        for (int c = 0; c < 3; ++c)
            out[k][c] = m[c] + R * (su[k] * u[c] + sv[k] * v[c]);
    int n = 4;
    double(*cur)[3] = out, (*nxt)[3] = buf;
    auto clip = [&](const double *pn, const double *pm) {
        n = clip_polygon(cur, n, nxt, pn, pm);
        double(*t)[3] = cur;
        cur = nxt;
        nxt = t;
    };
    for (int c = 0; c < 6 && n > 0; ++c) { // the box: x_c <= hi_c, -x_c <= -lo_c
        double bn[3] = {0.0, 0.0, 0.0}, bm[3] = {0.0, 0.0, 0.0};
        bn[c % 3] = c < 3 ? 1.0 : -1.0;
        bm[c % 3] = c < 3 ? p.hi[c % 3] : p.lo[c % 3];
        clip(bn, bm);
    }
    const uint32_t end = min(__ldg(p.off + i + 1), p.num_entries);
    for (uint32_t k = __ldg(p.off + i); k < end && n > 0; ++k) {
        const uint32_t q = __ldg(p.adj + k);
        if (k == e || q >= p.num_points)
            continue;
        float pk[3];
        load_point(p.points, q, pk);
        if (same_point(pk, pi) || same_point(pk, pj)) // no plane; or plane_e itself, which F_e lies on
            continue;
        double kn[3], km[3];
        for (int c = 0; c < 3; ++c) {
            kn[c] = (double)pk[c] - (double)pi[c];
            km[c] = 0.5 * ((double)pi[c] + (double)pk[c]);
        }
        clip(kn, km);
    }
    if (n < 0)
        return -1;
    if (n < 3)
        return 0;
    if (cur != out)
        for (int k = 0; k < n; ++k)
            for (int c = 0; c < 3; ++c)
                out[k][c] = cur[k][c];
    return n;
}

// Count pass: vcount[e] = vertices of F_e (0 when not emitted), pcount[e] = 1 when emitted; totals[2] counts the
// polygons that exceeded kSurfaceMaxVerts (they are counted as not emitted).  Every entry of a row in [off[i],
// min(off[i+1], E)) is written.
__global__ void __launch_bounds__(kSurfaceBlock) surface_count_kernel(const SurfaceParams p,
                                                                      unsigned long long *__restrict__ vcount,
                                                                      uint32_t *__restrict__ pcount,
                                                                      unsigned long long *__restrict__ totals) {
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= p.num_points)
        return;
    const uint32_t i = (uint32_t)row, lane = threadIdx.x & 31u;
    const bool in_i = p.inside[i] != 0;
    const uint32_t end = min(__ldg(p.off + i + 1), p.num_entries);
    for (uint32_t e = __ldg(p.off + i) + lane; e < end; e += 32) {
        int n = 0;
        if (in_i) {
            double verts[kSurfaceMaxVerts][3];
            n = surface_polygon(p, i, e, verts);
        }
        if (n < 0)
            atomicAdd(totals + 2, 1ull);
        vcount[e] = n > 0 ? (unsigned long long)n : 0ull;
        pcount[e] = n > 0 ? 1u : 0u;
    }
}

// Exclusive scan of one (u64, u32) pair per thread over the CTA (warp shuffles, then one warp over the warp
// totals); *tv / *tc = the CTA's totals.  Ends with a barrier, so the shared state can be reused right away.
__device__ __forceinline__ void cta_exclusive_scan(unsigned long long &v, uint32_t &c, unsigned long long &tv,
                                                   uint32_t &tc) {
    __shared__ unsigned long long warp_v[32];
    __shared__ uint32_t warp_c[32];
    __shared__ unsigned long long total_v;
    __shared__ uint32_t total_c;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    unsigned long long iv = v;
    uint32_t ic = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long sv = __shfl_up_sync(0xffffffffu, iv, o);
        const uint32_t sc = __shfl_up_sync(0xffffffffu, ic, o);
        if ((int)lane >= o) {
            iv += sv;
            ic += sc;
        }
    }
    if (lane == 31) {
        warp_v[warp] = iv;
        warp_c[warp] = ic;
    }
    __syncthreads();
    if (warp == 0) {
        const unsigned long long x = lane < nwarps ? warp_v[lane] : 0ull;
        const uint32_t y = lane < nwarps ? warp_c[lane] : 0u;
        unsigned long long sx = x;
        uint32_t sy = y;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long a = __shfl_up_sync(0xffffffffu, sx, o);
            const uint32_t b = __shfl_up_sync(0xffffffffu, sy, o);
            if ((int)lane >= o) {
                sx += a;
                sy += b;
            }
        }
        if (lane < nwarps) {
            warp_v[lane] = sx - x;
            warp_c[lane] = sy - y;
        }
        if (lane == 31) {
            total_v = sx;
            total_c = sy;
        }
    }
    __syncthreads();
    v = iv - v + warp_v[warp];
    c = ic - c + warp_c[warp];
    tv = total_v;
    tc = total_c;
    __syncthreads();
}

// Scan step 1: per tile of kScanTile entries (kScanItems consecutive ones per thread), the sums.
__global__ void __launch_bounds__(kScanBlock) scan_tile_sums_kernel(const unsigned long long *__restrict__ v,
                                                                    const uint32_t *__restrict__ c, uint32_t n,
                                                                    unsigned long long *__restrict__ tile_v,
                                                                    uint32_t *__restrict__ tile_c) {
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    unsigned long long sv = 0;
    uint32_t sc = 0;
    for (int k = 0; k < kScanItems; ++k)
        if (base + k < n) {
            sv += v[base + k];
            sc += c[base + k];
        }
    unsigned long long tv;
    uint32_t tc;
    cta_exclusive_scan(sv, sc, tv, tc);
    if (threadIdx.x == 0) {
        tile_v[blockIdx.x] = tv;
        tile_c[blockIdx.x] = tc;
    }
}

// Scan step 2 (one CTA): the tile sums become exclusive tile prefixes; the grand totals go to v[n], c[n] and
// totals[0..1].
__global__ void __launch_bounds__(kScanBlock) scan_tile_prefix_kernel(unsigned long long *__restrict__ tile_v,
                                                                      uint32_t *__restrict__ tile_c, uint32_t tiles,
                                                                      unsigned long long *__restrict__ v,
                                                                      uint32_t *__restrict__ c, uint32_t n,
                                                                      unsigned long long *__restrict__ totals) {
    unsigned long long carry_v = 0;
    uint32_t carry_c = 0;
    for (uint32_t t0 = 0; t0 < tiles; t0 += kScanBlock) {
        const uint32_t t = t0 + threadIdx.x;
        unsigned long long x = t < tiles ? tile_v[t] : 0ull;
        uint32_t y = t < tiles ? tile_c[t] : 0u;
        unsigned long long tv;
        uint32_t tc;
        cta_exclusive_scan(x, y, tv, tc);
        if (t < tiles) {
            tile_v[t] = carry_v + x;
            tile_c[t] = carry_c + y;
        }
        carry_v += tv;
        carry_c += tc;
    }
    if (threadIdx.x == 0) {
        v[n] = carry_v;
        c[n] = carry_c;
        totals[0] = carry_v;
        totals[1] = carry_c;
    }
}

// Scan step 3: each tile's exclusive scan plus its tile prefix, in place.
__global__ void __launch_bounds__(kScanBlock) scan_add_back_kernel(unsigned long long *__restrict__ v,
                                                                   uint32_t *__restrict__ c, uint32_t n,
                                                                   const unsigned long long *__restrict__ tile_v,
                                                                   const uint32_t *__restrict__ tile_c) {
    const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    unsigned long long xv[kScanItems], sv = 0;
    uint32_t xc[kScanItems], sc = 0;
    for (int k = 0; k < kScanItems; ++k) {
        const bool ok = base + k < n;
        xv[k] = ok ? v[base + k] : 0ull;
        xc[k] = ok ? c[base + k] : 0u;
        sv += xv[k];
        sc += xc[k];
    }
    unsigned long long tv;
    uint32_t tc;
    cta_exclusive_scan(sv, sc, tv, tc);
    sv += tile_v[blockIdx.x];
    sc += tile_c[blockIdx.x];
    for (int k = 0; k < kScanItems; ++k)
        if (base + k < n) {
            v[base + k] = sv;
            c[base + k] = sc;
            sv += xv[k];
            sc += xc[k];
        }
}

// Write pass: the polygon of entry e goes to vertices [voff[e], voff[e+1]) and polygon slot poff[e] -- only when the
// count pass emitted it (poff[e+1] - poff[e] == 1) and it has exactly the counted vertex run, so nothing is ever
// written outside the counted output.  rgb = the colour of cell i along normalize(p_i - p_j), computed as
// sample_field_kernel computes it for that direction.
template <int DEG, typename AttrT>
__global__ void __launch_bounds__(kSurfaceBlock) surface_write_kernel(
    const SurfaceParams p, const AttrT *__restrict__ attrs, const unsigned long long *__restrict__ voff,
    const uint32_t *__restrict__ poff, const unsigned long long *__restrict__ totals, float *__restrict__ vertices,
    long long *__restrict__ offsets, uint32_t *__restrict__ cells, AttrT *__restrict__ rgb) {
    constexpr int A = attr_dim(DEG), NC = 3 * sh_dim(DEG);
    const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row == 0 && threadIdx.x == 0)
        offsets[totals[1]] = (long long)totals[0];
    if (row >= p.num_points)
        return;
    const uint32_t i = (uint32_t)row, lane = threadIdx.x & 31u;
    if (!p.inside[i])
        return;
    const uint32_t end = min(__ldg(p.off + i + 1), p.num_entries);
    for (uint32_t e = __ldg(p.off + i) + lane; e < end; e += 32) {
        const uint32_t slot = poff[e];
        if (poff[e + 1] - slot != 1u)
            continue;
        const unsigned long long v0 = voff[e], count = voff[e + 1] - v0;
        double verts[kSurfaceMaxVerts][3];
        const int n = surface_polygon(p, i, e, verts);
        if (n <= 0 || (unsigned long long)n != count)
            continue;
        for (int k = 0; k < n; ++k)
            for (int c = 0; c < 3; ++c)
                vertices[3 * (v0 + k) + c] = __double2float_rn(verts[k][c]);
        const uint32_t j = __ldg(p.adj + e);
        offsets[slot] = (long long)v0;
        cells[2 * (uint64_t)slot] = i;
        cells[2 * (uint64_t)slot + 1] = j;
        float pi[3], pj[3];
        load_point(p.points, i, pi);
        load_point(p.points, j, pj);
        float dx = __fsub_rn(pi[0], pj[0]), dy = __fsub_rn(pi[1], pj[1]), dz = __fsub_rn(pi[2], pj[2]);
        normalize_dir(dx, dy, dz);
        float sh[sh_dim(DEG)];
        sh_basis<DEG>(dx, dy, dz, sh);
        const AttrT *arow = attrs + (uint64_t)i * A;
        float cv[NC];
#pragma unroll
        for (int k = 0; k < NC; ++k)
            cv[k] = (float)arow[k];
        float r, g, b;
        sh_coeffs_to_rgb<DEG>(cv, sh, r, g, b);
        rgb[3 * (uint64_t)slot] = (AttrT)r;
        rgb[3 * (uint64_t)slot + 1] = (AttrT)g;
        rgb[3 * (uint64_t)slot + 2] = (AttrT)b;
    }
}

} // namespace rfb
