// Device-side building blocks of the H100 foam tracer (sm_90a).
//
// Behavioural spec: SURVEY.md Appendix A, i.e. radfoam's
//   src/tracing/tracing_utils.cuh:8-103  (cell walk, intersection gradient)
//   src/tracing/sh_utils.cuh:8-92        (SH basis, SH -> rgb, rgb-grad -> SH)
//   src/tracing/pipeline.cu:14-343       (forward / backward cell functors)
// Nothing here is shared with the reference's code; the arithmetic that decides
// the integer traversal is pinned with non-contractable intrinsics in the
// association the reference's own SASS uses (see walk_face()).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rfb {

constexpr uint32_t kNone = 0xFFFFFFFFu;
// Threads per CTA in the ray kernels.  A CTA's registers / shared memory are only released when its LAST
// warp finishes, and ray lengths vary widely (mean 97 cells, max 257 on the bench frame), so smaller CTAs
// keep the SM fuller in the kernel's tail; RFB_KBLOCK (32 / 64 / 128) is a build-time knob so that the
// choice is measured (tests/tools/kblock_bench.py).
#ifndef RFB_KBLOCK
#define RFB_KBLOCK 128
#endif
constexpr int kBlock = RFB_KBLOCK;
static_assert(kBlock == 32 || kBlock == 64 || kBlock == 128, "RFB_KBLOCK must be 32, 64 or 128");
// a CTA covers kTileW x kTileH pixels: warps of 8x4 pixels, two side by side when there are at least two
constexpr int kWarpsX = kBlock >= 64 ? 2 : 1;
constexpr int kWarpsY = kBlock / 32 / kWarpsX;
constexpr int kTileW = 8 * kWarpsX, kTileH = 4 * kWarpsY;

__host__ __device__ constexpr int sh_dim(int deg) { return (deg + 1) * (deg + 1); }
// floats per row of the internal SH mirror (3*sh_dim padded to a multiple of 4)
__host__ __device__ constexpr int sh_row(int deg) { return (3 * sh_dim(deg) + 3) & ~3; }
// floats per row of the gradient accumulator: [SH row][density, gx, gy, gz]
__host__ __device__ constexpr int grad_row(int deg) { return sh_row(deg) + 4; }
__host__ __device__ constexpr int attr_dim(int deg) { return 1 + 3 * sh_dim(deg); }

// Padded face rows: row i starts at padded_begin() -- a multiple of 4 slots (32-byte
// aligned) -- and holds nf real faces followed by ZERO faces up to the next multiple of 4
// (a zero face has dp == 0, which never wins), so the scan works on whole 4-face chunks
// without index masking.  Closed form, no prefix scan: with a = off_i + 3 i,
// ceil4(a + nf + 3) >= ceil4(a) + ceil4(nf), so rows never overlap; at most 3 slack slots
// per row stay unused (never written, never read).
__host__ __device__ __forceinline__ uint32_t padded_begin(uint32_t off_i, uint32_t i) {
    return (off_i + 3u * i + 3u) & ~3u;
}
__host__ __device__ __forceinline__ uint64_t padded_slots(uint32_t num_points, uint32_t num_edges) {
    return (uint64_t)num_edges + 3ull * num_points + 8ull;
}

// ---------------------------------------------------------------- loads
__device__ __forceinline__ float4 ldg4(const float4 *p) { return __ldg(p); }
__device__ __forceinline__ uint4 ldg4(const uint4 *p) { return __ldg(p); }
__device__ __forceinline__ uint2 ldg2(const uint2 *p) { return __ldg(p); }

// 16-byte fire-and-forget reduction (sm_90+): one L2 atomic transaction for four
// consecutive floats instead of four scalar REDs.
__device__ __forceinline__ void red_add_v4(float *addr, float a, float b, float c, float d) {
#ifdef RFB_EMU // tests/emu: kernel-logic emulation on the CPU (test infrastructure)
    rfb_emu_red_add_v4(addr, a, b, c, d);
#else
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b),
                 "f"(c), "f"(d)
                 : "memory");
#endif
}

// Bulk reduction (sm_90): the TMA unit reads `bytes` (a multiple of 16, both addresses 16-byte aligned) of shared
// memory at `src` and adds them as f32 into global memory at `dst`, so the LSU issues no request per 16 bytes and
// L2 receives whole sectors.  Each call is its own bulk group of the calling thread.  Shared-memory writes to `src`
// must be made visible to the async proxy first (fence_proxy_async_smem), and `src` may be rewritten only after
// bulk_wait_read.
__device__ __forceinline__ void bulk_red_add_f32(float *dst, const float *src, uint32_t bytes) {
#ifdef RFB_EMU // element by element with the emulator's atomics, done at issue (the hardware's order is unspecified)
    for (uint32_t i = 0; i < bytes / 4; ++i)
        atomicAdd(dst + i, src[i]);
#else
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;\n\t"
                 "cp.async.bulk.commit_group;" ::"l"(dst),
                 "r"(static_cast<uint32_t>(__cvta_generic_to_shared(src))), "r"(bytes)
                 : "memory");
#endif
}
__device__ __forceinline__ void fence_proxy_async_smem() {
#ifndef RFB_EMU
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
// waits until every bulk operation this thread issued has finished reading its shared-memory source
__device__ __forceinline__ void bulk_wait_read() {
#ifndef RFB_EMU
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
#endif
}

// NVSwitch multicast (NVLS): one load returns the SUM of the word at the same offset of every GPU's copy -- the
// switch does the reduction --, one store writes all copies.  `p` is an address in the multicast mapping of a
// symmetric allocation.
__device__ __forceinline__ float4 multimem_ld_reduce_add_v4(const float *p) {
#ifdef RFB_EMU
    return rfb_emu_multimem_ld_reduce_v4(p);
#else
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
#endif
}
__device__ __forceinline__ void multimem_st_v4(float *p, float4 v) {
#ifdef RFB_EMU
    rfb_emu_multimem_st(p, &v, 16);
#else
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
#endif
}
__device__ __forceinline__ void multimem_st_v2(void *p, float2 v) {
#ifdef RFB_EMU
    rfb_emu_multimem_st(p, &v, 8);
#else
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
#endif
}

// ---------------------------------------------------------------- SH basis
// Real SH basis of the (unit) direction (sh_coefficients<deg>(), sh_utils.cuh:34-70), with the multiply-add
// association PINNED to what nvcc makes of the reference's source in its kernels (read from oracle/_ref's SASS):
//   degree 2 (every square used at most twice, so the products are fused into the sums):
//     2zz - xx - yy = fma(-y, y, fma(-x, x, fma(z, z, z*z)));   xx - yy = fma(x, x, -(y*y))
//   degree 3 (the squares are shared by seven terms, so they are rounded products):
//     2zz - xx - yy = ((zz + zz) - xx) - yy;   xx - yy a plain difference;   3xx - yy = fma(xx, 3, -yy);
//     xx - 3yy = fma(yy, -3, xx);   4zz - xx - yy = fma(zz, 4, -xx) - yy;
//     2zz - 3xx - 3yy = fma(yy, -3, fma(xx, -3, zz + zz));   c*u*(...) = (c*u)*(...);   c*xy*z = (c*xy)*z
// Left to the compiler, the fusion depends on the surrounding kernel: round 2's warp-aggregated backward rounded
// y*y where the forward had fused it, the two bases differed in the last bit, and with it the backward's recomputed
// colour sum -- invisible at the default weight threshold, but with threshold 0 the late cells' gradients are
// (saved colour - recomputed colour) / T and became rounding residue (1e-6 where the reference has 1e-14;
// found by tests/test_gpu_fuzz.py).
template <int DEG>
__device__ __forceinline__ void sh_basis(float x, float y, float z, float *sh) {
    constexpr float C0 = 0.28209479177387814f;
    constexpr float C1 = 0.4886025119029199f;
    sh[0] = C0;
    if (DEG > 0) {
        sh[1] = __fmul_rn(-C1, y);
        sh[2] = __fmul_rn(C1, z);
        sh[3] = __fmul_rn(-C1, x);
    }
    if (DEG == 2) {
        sh[4] = __fmul_rn(1.0925484305920792f, __fmul_rn(x, y));
        sh[5] = __fmul_rn(-1.0925484305920792f, __fmul_rn(y, z));
        sh[6] = __fmul_rn(0.31539156525252005f, __fmaf_rn(-y, y, __fmaf_rn(-x, x, __fmaf_rn(z, z, __fmul_rn(z, z)))));
        sh[7] = __fmul_rn(-1.0925484305920792f, __fmul_rn(x, z));
        sh[8] = __fmul_rn(0.5462742152960396f, __fmaf_rn(x, x, -__fmul_rn(y, y)));
    }
    if (DEG > 2) {
        const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
        const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
        const float zz2 = __fadd_rn(zz, zz);
        const float xx_yy = __fsub_rn(xx, yy);
        const float zz4_xx_yy = __fsub_rn(__fmaf_rn(zz, 4.0f, -xx), yy);
        sh[4] = __fmul_rn(1.0925484305920792f, xy);
        sh[5] = __fmul_rn(-1.0925484305920792f, yz);
        sh[6] = __fmul_rn(0.31539156525252005f, __fsub_rn(__fsub_rn(zz2, xx), yy));
        sh[7] = __fmul_rn(-1.0925484305920792f, xz);
        sh[8] = __fmul_rn(0.5462742152960396f, xx_yy);
        sh[9] = __fmul_rn(__fmul_rn(-0.5900435899266435f, y), __fmaf_rn(xx, 3.0f, -yy));
        sh[10] = __fmul_rn(__fmul_rn(2.890611442640554f, xy), z);
        sh[11] = __fmul_rn(__fmul_rn(-0.4570457994644658f, y), zz4_xx_yy);
        sh[12] = __fmul_rn(__fmul_rn(0.3731763325901154f, z), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2)));
        sh[13] = __fmul_rn(__fmul_rn(-0.4570457994644658f, x), zz4_xx_yy);
        sh[14] = __fmul_rn(__fmul_rn(1.445305721320277f, z), xx_yy);
        sh[15] = __fmul_rn(__fmul_rn(-0.5900435899266435f, x), __fmaf_rn(yy, -3.0f, xx));
    }
}

// rgb = max(0, 0.5 + sum_k Y_k * c_k) per channel, accumulated k ascending in one
// FFMA chain per channel (load_sh_as_rgb, sh_utils.cuh:72-83), from the 3*sh_dim
// channel-interleaved coefficients `v`.
template <int DEG>
__device__ __forceinline__ void sh_coeffs_to_rgb(const float *v, const float *sh, float &r, float &g, float &b) {
    float rgb[3] = {0.5f, 0.5f, 0.5f};
#pragma unroll
    for (int i = 0; i < 3 * sh_dim(DEG); ++i)
        rgb[i % 3] = __fmaf_rn(sh[i / 3], v[i], rgb[i % 3]);
    // cwiseMax(0): (x < 0) ? 0 : x  (NaN stays NaN, as in the reference build)
    r = (rgb[0] < 0.0f) ? 0.0f : rgb[0];
    g = (rgb[1] < 0.0f) ? 0.0f : rgb[1];
    b = (rgb[2] < 0.0f) ? 0.0f : rgb[2];
}

// sh_coeffs_to_rgb of one row of the internal SH mirror: `row` is 16-byte aligned
// [3*sh_dim floats, channel-interleaved][pad].
template <int DEG>
__device__ __forceinline__ void sh_to_rgb(const float *__restrict__ row, const float *sh,
                                          float &r, float &g, float &b) {
    constexpr int NV = sh_row(DEG) / 4;
    float v[NV * 4];
    const float4 *row4 = reinterpret_cast<const float4 *>(row);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        float4 q = ldg4(row4 + i);
        v[4 * i + 0] = q.x;
        v[4 * i + 1] = q.y;
        v[4 * i + 2] = q.z;
        v[4 * i + 3] = q.w;
    }
    sh_coeffs_to_rgb<DEG>(v, sh, r, g, b);
}

// ---------------------------------------------------------------- the walk
struct RayGeom {
    float ox, oy, oz; // origin
    float dx, dy, dz; // unit direction
};

// The ranked face scan flushes subnormals (MUFU.RCP), so a front face whose dp = o.d is a positive subnormal
// would drop out of the ranking while the reference still divides by it.  Face offsets are fp16 values
// (|o_i| >= 2^-24 or 0), so every nonzero partial sum of dp is a multiple of 2^-34 * 2^-23 * min|d_i| over the
// nonzero d_i: with all nonzero |d_i| >= 2^-60 a nonzero dp is >= 2^-117, never subnormal.  Rays with a smaller
// nonzero direction component (pathological input) must take the exact scan on every step instead.  Any test or
// flag for that INSIDE the step loop of the recording forward costs time (a flag register, a second loop
// instantiation selected per warp, a per-step test were each measured slower), so the
// hot kernels come as twins: the fast one (ranked scan) raises a device flag when it meets such a ray and the
// exact one, launched right behind it, re-does the launch only if the flag is up (ScanMode).  Kernels off the
// hot path choose per ray (walk()).
enum ScanMode { kScanFast = 0, kScanExactTwin = 1, kScanPerRay = 2 };
__device__ __forceinline__ bool needs_exact_scan(float dx, float dy, float dz) {
    const float kTiny = 8.673617379884035e-19f; // 2^-60
    const float ax = fabsf(dx), ay = fabsf(dy), az = fabsf(dz);
    return (ax != 0.0f && ax < kTiny) || (ay != 0.0f && ay < kTiny) || (az != 0.0f && az < kTiny);
}

// ray.direction /= ray.direction.norm()  (pipeline.cu:39-40): squared norm in the
// x0 + (x1 + x2) order with the two fusions nvcc applies, IEEE sqrt and division.
__device__ __forceinline__ void normalize_dir(float &x, float &y, float &z) {
    float n2 = __fmaf_rn(x, x, __fmaf_rn(y, y, __fmul_rn(z, z)));
    float n = __fsqrt_rn(n2);
    x = __fdiv_rn(x, n);
    y = __fdiv_rn(y, n);
    z = __fdiv_rn(z, n);
}

// ray r of a [R][6] (origin, direction) array, its direction normalised
__device__ __forceinline__ void load_ray(const float *rays, uint32_t r, RayGeom &ray) {
    const float *rp = rays + 6 * (uint64_t)r;
    ray.ox = __ldg(rp + 0);
    ray.oy = __ldg(rp + 1);
    ray.oz = __ldg(rp + 2);
    ray.dx = __ldg(rp + 3);
    ray.dy = __ldg(rp + 4);
    ray.dz = __ldg(rp + 5);
    normalize_dir(ray.dx, ray.dy, ray.dz);
}

// One bisector-plane test (tracing_utils.cuh:52-65).  `h` is one face record:
// (dx, dy, dz, 0) in fp16 = RN_half(neighbour - cell point).  Association as in
// the reference's SASS (SURVEY.md Appendix D, re-read from oracle/_ref):
//   f   = fma(o, 0.5, P)            per component
//   dp  = fma(ox, dx, fma(oy, dy, oz*dz))
//   num = fma(ox, fx-rx, fma(oy, fy-ry, oz*(fz-rz)))
//   t   = num / dp   (IEEE)
__device__ __forceinline__ void walk_face(uint2 h, float px, float py, float pz,
                                          const RayGeom &ray, float &t, float &dp) {
    __half2 hxy = *reinterpret_cast<__half2 *>(&h.x);
    __half2 hzw = *reinterpret_cast<__half2 *>(&h.y);
    float ox = __low2float(hxy), oy = __high2float(hxy), oz = __low2float(hzw);
    float fx = __fmaf_rn(ox, 0.5f, px);
    float fy = __fmaf_rn(oy, 0.5f, py);
    float fz = __fmaf_rn(oz, 0.5f, pz);
    dp = __fmaf_rn(ox, ray.dx, __fmaf_rn(oy, ray.dy, __fmul_rn(oz, ray.dz)));
    float num = __fmaf_rn(ox, __fsub_rn(fx, ray.ox),
                          __fmaf_rn(oy, __fsub_rn(fy, ray.oy), __fmul_rn(oz, __fsub_rn(fz, ray.oz))));
    t = __fdiv_rn(num, dp);
}

// MUFU.RCP: 1-ulp reciprocal (inputs/outputs flushed), used only to RANK faces; the value
// that is kept, t1, always comes from the IEEE division.
__device__ __forceinline__ float rcp_approx(float x) {
#ifdef RFB_EMU
    return rfb_emu_rcp_approx(x);
#else
    float r;
    // volatile: keeps the MUFU unconditional so the ranking loop stays branch-free
    asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#endif
}

// Same plane test without the division: returns num and dp.
__device__ __forceinline__ void walk_face_parts(uint2 h, float px, float py, float pz,
                                                const RayGeom &ray, float &num, float &dp) {
    __half2 hxy = *reinterpret_cast<__half2 *>(&h.x);
    __half2 hzw = *reinterpret_cast<__half2 *>(&h.y);
    float ox = __low2float(hxy), oy = __high2float(hxy), oz = __low2float(hzw);
    float fx = __fmaf_rn(ox, 0.5f, px);
    float fy = __fmaf_rn(oy, 0.5f, py);
    float fz = __fmaf_rn(oz, 0.5f, pz);
    dp = __fmaf_rn(ox, ray.dx, __fmaf_rn(oy, ray.dy, __fmul_rn(oz, ray.dz)));
    num = __fmaf_rn(ox, __fsub_rn(fx, ray.ox),
                    __fmaf_rn(oy, __fsub_rn(fy, ray.oy), __fmul_rn(oz, __fsub_rn(fz, ray.oz))));
}

// Scene view the walk reads: this library's padded face mirror.  Rows start at
// padded_begin() (a multiple of 4 slots => 32-byte aligned), so two faces arrive per 128-bit
// load; the neighbour index of a face sits at the same slot of `nbr`.  Pad slots hold zero
// faces (dp == 0 never wins).  trace_benchmark's caller-built half4[E] offsets
// (pipeline.h:117-126) are copied into the same layout by build_faces_from_diff_kernel.
struct PaddedFaces {
    const uint2 *faces;
    const uint32_t *nbr;
    const uint32_t *off;
    __device__ __forceinline__ void row(uint32_t cell, uint32_t &begin, uint32_t &nf) const {
        uint32_t a = __ldg(off + cell), b = __ldg(off + cell + 1);
        begin = padded_begin(a, cell);
        nf = b - a;
    }
    // Exact scan: first minimum of t = num / dp (IEEE) over faces with dp > 0, strict `<`,
    // array order -- literally the reference's loop (zero pad faces have dp == 0).
    __device__ __forceinline__ void scan_exact(uint32_t begin, uint32_t nf, float px, float py,
                                               float pz, const RayGeom &ray, float &t1,
                                               uint32_t &face) const {
        const uint4 *p = reinterpret_cast<const uint4 *>(faces + begin);
        for (uint32_t f = 0; f < nf; f += 4) {
            uint4 a = ldg4(p + (f >> 1));
            uint4 b = ldg4(p + (f >> 1) + 1);
            float t, dp;
            walk_face(make_uint2(a.x, a.y), px, py, pz, ray, t, dp);
            if (dp > 0.0f && t < t1) { t1 = t; face = f; }
            walk_face(make_uint2(a.z, a.w), px, py, pz, ray, t, dp);
            if (dp > 0.0f && t < t1) { t1 = t; face = f + 1; }
            walk_face(make_uint2(b.x, b.y), px, py, pz, ray, t, dp);
            if (dp > 0.0f && t < t1) { t1 = t; face = f + 2; }
            walk_face(make_uint2(b.z, b.w), px, py, pz, ray, t, dp);
            if (dp > 0.0f && t < t1) { t1 = t; face = f + 3; }
        }
    }
    // Fast scan with the same result.  Faces are RANKED by q = num * rcp(dp) (2 instructions
    // instead of the ~10 of an IEEE division); q is within 2^-22 relative of the exact quotient,
    // so if the runner-up's q clears the best q by more than 2^-19 relative, the exact
    // quotients are ordered the same way and no exact tie exists: the winner is the
    // reference's winner and t1 is its IEEE quotient.  Otherwise (near-ties, non-finite or
    // flushed values: rare) the row is rescanned exactly.
    // EXACT_ONLY: the instantiation for rays the ranking is not proven for (needs_exact_scan()).
    template <bool EXACT_ONLY = false>
    __device__ __forceinline__ void scan(uint32_t begin, uint32_t nf, float px, float py, float pz,
                                         const RayGeom &ray, float &t1, uint32_t &face) const {
        const float kInf = __int_as_float(0x7f800000);
        if (EXACT_ONLY) {
            scan_exact(begin, nf, px, py, pz, ray, t1, face);
            return;
        }
        const uint4 *p = reinterpret_cast<const uint4 *>(faces + begin);
        float best = kInf, second = kInf; // invariant: best <= second
        uint32_t bf = kNone;
        for (uint32_t f = 0; f < nf; f += 4) {
            uint4 a = ldg4(p + (f >> 1));
            uint4 b = ldg4(p + (f >> 1) + 1);
            uint2 rec[4] = {make_uint2(a.x, a.y), make_uint2(a.z, a.w), make_uint2(b.x, b.y),
                            make_uint2(b.z, b.w)};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float num, dp;
                walk_face_parts(rec[k], px, py, pz, ray, num, dp);
                float q = num * rcp_approx(dp);
                q = (dp > 0.0f) ? q : kInf;
                bf = (q < best) ? f + k : bf;
                // runner-up: min(second, max(best, q)); a NaN q collapses it onto best, which
                // only sends the row to the exact rescan
                second = fminf(second, fmaxf(best, q));
                best = fminf(best, q);
            }
        }
        if (best == kInf) {
            // nothing ranked: normally the ray is leaving through an unbounded hull cell (no
            // face with dp > 0 -> the reference finds no face either).  A cheap dp-only pass
            // confirms that; only a front face whose quotient overflowed needs the exact scan.
            bool any_front = false;
            for (uint32_t f = 0; f < nf; f += 4) {
                uint4 a = ldg4(p + (f >> 1));
                uint4 b = ldg4(p + (f >> 1) + 1);
                uint2 rec[4] = {make_uint2(a.x, a.y), make_uint2(a.z, a.w), make_uint2(b.x, b.y),
                                make_uint2(b.z, b.w)};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    __half2 hxy = *reinterpret_cast<__half2 *>(&rec[k].x);
                    __half2 hzw = *reinterpret_cast<__half2 *>(&rec[k].y);
                    float dp = __fmaf_rn(__low2float(hxy), ray.dx,
                                         __fmaf_rn(__high2float(hxy), ray.dy,
                                                   __fmul_rn(__low2float(hzw), ray.dz)));
                    any_front |= dp > 0.0f;
                }
            }
            if (!any_front)
                return; // face stays kNone, t1 stays +inf
            scan_exact(begin, nf, px, py, pz, ray, t1, face);
            return;
        }
        // 2^-19 relative clearance; |second| is capped at 4|best| because beyond that the gap
        // itself dwarfs any rounding (and so that a lone candidate, second == +inf, is clear)
        float ab = fabsf(best);
        float margin = 1.9073486e-06f * fmaxf(ab, fminf(fabsf(second), 4.0f * ab + 1e-30f)) + 1e-35f;
        bool clear = (second - best) > margin; // false for NaN / no ranked face (inf - inf)
        if (clear && fabsf(best) < 1e30f) {
            // the winner's IEEE quotient: re-evaluate that one face exactly
            float t, dp;
            walk_face(ldg2(faces + begin + bf), px, py, pz, ray, t, dp);
            t1 = t;
            face = bf;
        } else {
            scan_exact(begin, nf, px, py, pz, ray, t1, face);
        }
    }
    __device__ __forceinline__ uint32_t neighbour(uint32_t begin, uint32_t face) const {
        return __ldg(nbr + begin + face);
    }
};

// The per-ray cell walk (trace<>, tracing_utils.cuh:8-89).  cells[i] =
// (point.xyz, density).  `cell_fn(cell, density, t0, t1, P, Pnext)` is called
// for every cell with t1 > t0 and returns false to stop.  Returns n = cells
// entered (max_steps + 1 when the budget ran out).
template <bool EXACT_ONLY, typename Faces, typename CellFn>
__device__ __forceinline__ uint32_t walk(const Faces &fa, const float4 *__restrict__ cells,
                                         const RayGeom &ray, uint32_t start, uint32_t max_steps,
                                         CellFn &&cell_fn) {
    float t0 = 0.0f;
    uint32_t n = 0;
    uint32_t cur = start;
    float4 pc = ldg4(cells + cur);
    for (;;) {
        n++;
        if (n > max_steps)
            break;
        uint32_t begin, nf;
        fa.row(cur, begin, nf);
        float t1 = __int_as_float(0x7f800000);
        uint32_t face = kNone;
        fa.template scan<EXACT_ONLY>(begin, nf, pc.x, pc.y, pc.z, ray, t1, face);
        if (face == kNone)
            break;
        uint32_t nxt = fa.neighbour(begin, face);
        float4 pn = ldg4(cells + nxt);
        if (t1 > t0) {
            if (!cell_fn(cur, pc, t0, t1, pn))
                break;
        }
        t0 = fmaxf(t0, t1);
        cur = nxt;
        pc = pn;
    }
    return n;
}

// d t / d p of the ray / bisector(p, q) intersection (cell_intersection_grad,
// tracing_utils.cuh:91-103), from the fp32 points.  Gradient sums over rays cancel heavily
// (terms 1e3x the result), so one differently-fused multiply-add shows up at 1e-4 of the
// result; the association is therefore pinned to the reference's SASS:
//   n = q - p;  a = fma(p + q, 0.5, -o);  dp = fma(nx,dx, fma(ny,dy, nz*dz))
//   num = fma(nx,ax, fma(ny,ay, nz*az));  g_i = fma(num, d_i, dp * (o_i - p_i)) / (dp * dp)
__device__ __forceinline__ void isect_grad(float px, float py, float pz, float qx, float qy,
                                           float qz, const RayGeom &ray, float &gx, float &gy,
                                           float &gz) {
    float nx = __fsub_rn(qx, px), ny = __fsub_rn(qy, py), nz = __fsub_rn(qz, pz);
    float ax = __fmaf_rn(__fadd_rn(px, qx), 0.5f, -ray.ox);
    float ay = __fmaf_rn(__fadd_rn(py, qy), 0.5f, -ray.oy);
    float az = __fmaf_rn(__fadd_rn(pz, qz), 0.5f, -ray.oz);
    float dp = __fmaf_rn(nx, ray.dx, __fmaf_rn(ny, ray.dy, __fmul_rn(nz, ray.dz)));
    float num = __fmaf_rn(nx, ax, __fmaf_rn(ny, ay, __fmul_rn(nz, az)));
    float inv = __fmul_rn(dp, dp);
    gx = __fdiv_rn(__fmaf_rn(num, ray.dx, __fmul_rn(dp, __fsub_rn(ray.ox, px))), inv);
    gy = __fdiv_rn(__fmaf_rn(num, ray.dy, __fmul_rn(dp, __fsub_rn(ray.oy, py))), inv);
    gz = __fdiv_rn(__fmaf_rn(num, ray.dz, __fmul_rn(dp, __fsub_rn(ray.oz, pz))), inv);
}

// Both directions of one bisector at once: gp = d t / d p and gq = d t / d q for the plane
// between p and q.  Swapping the roles of p and q negates n, dp and num exactly (negation
// commutes with rounding) and leaves a and dp*dp unchanged, so the second gradient reuses them:
//   gq_i = -( fma(num, d_i, dp * (o_i - q_i)) / (dp*dp) )
// bit-identical to isect_grad(q, p, ...), at roughly half its cost.
// The plane's n = q - p, dp = n.d and num = ((p + q)/2 - o).n are returned as well (the ray gradient's
// dt/do = -n/dp and dt/dd = -(num/dp) n/dp reuse them).
__device__ __forceinline__ void isect_grad_pair(float px, float py, float pz, float qx, float qy,
                                                float qz, const RayGeom &ray, float &gpx, float &gpy,
                                                float &gpz, float &gqx, float &gqy, float &gqz, float &nx,
                                                float &ny, float &nz, float &dp, float &num) {
    nx = __fsub_rn(qx, px), ny = __fsub_rn(qy, py), nz = __fsub_rn(qz, pz);
    float ax = __fmaf_rn(__fadd_rn(px, qx), 0.5f, -ray.ox);
    float ay = __fmaf_rn(__fadd_rn(py, qy), 0.5f, -ray.oy);
    float az = __fmaf_rn(__fadd_rn(pz, qz), 0.5f, -ray.oz);
    dp = __fmaf_rn(nx, ray.dx, __fmaf_rn(ny, ray.dy, __fmul_rn(nz, ray.dz)));
    num = __fmaf_rn(nx, ax, __fmaf_rn(ny, ay, __fmul_rn(nz, az)));
    float inv = __fmul_rn(dp, dp);
    gpx = __fdiv_rn(__fmaf_rn(num, ray.dx, __fmul_rn(dp, __fsub_rn(ray.ox, px))), inv);
    gpy = __fdiv_rn(__fmaf_rn(num, ray.dy, __fmul_rn(dp, __fsub_rn(ray.oy, py))), inv);
    gpz = __fdiv_rn(__fmaf_rn(num, ray.dz, __fmul_rn(dp, __fsub_rn(ray.oz, pz))), inv);
    gqx = -__fdiv_rn(__fmaf_rn(num, ray.dx, __fmul_rn(dp, __fsub_rn(ray.ox, qx))), inv);
    gqy = -__fdiv_rn(__fmaf_rn(num, ray.dy, __fmul_rn(dp, __fsub_rn(ray.oy, qy))), inv);
    gqz = -__fdiv_rn(__fmaf_rn(num, ray.dz, __fmul_rn(dp, __fsub_rn(ray.oz, qz))), inv);
}

// Per-ray sums of the ray gradient dL/d(origin, direction) (the RAY instantiations of the backward kernels;
// DESIGN.md §2).  The walk's cell sequence is held fixed: a composited cell's t1 lies on its exit plane
// (cur, next) and its t0 on the exit plane of the previous composited cell, both planes of the fp32 points, with
// dt/do = -n/dp and dt/dd = -(num/dp) n/dp (d the unit direction).  The colour's dependence on the direction
// is summed separately, as G_k = sum over cells and channels of dL/drgb_c * a[cell, 3k+c] (ray_grad_store()).
struct RayAcc {
    float gox, goy, goz; // dL/do
    float gdx, gdy, gdz; // dL/dd (unit direction) through the planes
    float jx, jy, jz;    // exit plane of the previous composited cell: -n/dp ...
    float jt;            // ... and num/dp
    __device__ __forceinline__ void init() {
        gox = goy = goz = gdx = gdy = gdz = 0.0f;
        jx = jy = jz = jt = 0.0f;
    }
    // dL/dt * (dt/do, dt/dd) of the plane (jx, jy, jz, jt)
    __device__ __forceinline__ void add(float dL_dt, float px, float py, float pz, float pt) {
        gox = __fmaf_rn(dL_dt, px, gox);
        goy = __fmaf_rn(dL_dt, py, goy);
        goz = __fmaf_rn(dL_dt, pz, goz);
        const float s = __fmul_rn(dL_dt, pt);
        gdx = __fmaf_rn(s, px, gdx);
        gdy = __fmaf_rn(s, py, gdy);
        gdz = __fmaf_rn(s, pz, gdz);
    }
};

// G_k += sum_c dL/drgb_c * a[3k+c] for one cell's SH row (the row sh_to_rgb read; L1-resident by now)
template <int DEG>
__device__ __forceinline__ void sh_grad_contract(const float *__restrict__ row, const float dL_drgb[3],
                                                 float *G) {
    if (dL_drgb[0] == 0.0f && dL_drgb[1] == 0.0f && dL_drgb[2] == 0.0f)
        return;
    constexpr int NV = sh_row(DEG) / 4;
    float v[NV * 4];
    const float4 *row4 = reinterpret_cast<const float4 *>(row);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        float4 q = ldg4(row4 + i);
        v[4 * i + 0] = q.x;
        v[4 * i + 1] = q.y;
        v[4 * i + 2] = q.z;
        v[4 * i + 3] = q.w;
    }
#pragma unroll
    for (int k = 0; k < sh_dim(DEG); ++k)
        G[k] = __fmaf_rn(dL_drgb[2], v[3 * k + 2],
                         __fmaf_rn(dL_drgb[1], v[3 * k + 1], __fmaf_rn(dL_drgb[0], v[3 * k], G[k])));
}

// (gx, gy, gz) += sum_k G_k grad Y_k(x, y, z): the gradient of the real SH basis of sh_basis() (same constants).
// Every operation is an explicit intrinsic, so that all kernels that inline this round it the same way (ray_grad
// is bit-identical across the direct, re-walk and replay backward).
template <int DEG>
__device__ __forceinline__ void sh_basis_grad(float x, float y, float z, const float *G, float &gx, float &gy,
                                              float &gz) {
    // g += c * m
    auto acc = [](float &g, float c, float m) { g = __fmaf_rn(c, m, g); };
    constexpr float C1 = 0.4886025119029199f;
    if (DEG > 0) {
        acc(gy, -C1, G[1]);
        acc(gz, C1, G[2]);
        acc(gx, -C1, G[3]);
    }
    if (DEG > 1) {
        // Y4 = A xy, Y5 = -A yz, Y6 = B (2zz - xx - yy), Y7 = -A xz, Y8 = C (xx - yy)
        constexpr float A = 1.0925484305920792f, B2 = 2.0f * 0.31539156525252005f, C2 = 2.0f * 0.5462742152960396f;
        const float g4 = __fmul_rn(A, G[4]), g5 = __fmul_rn(A, G[5]), g6 = __fmul_rn(B2, G[6]),
                    g7 = __fmul_rn(A, G[7]), g8 = __fmul_rn(C2, G[8]);
        acc(gx, g4, y);
        acc(gy, g4, x);
        acc(gy, -g5, z);
        acc(gz, -g5, y);
        acc(gx, -g6, x);
        acc(gy, -g6, y);
        acc(gz, __fmul_rn(2.0f, g6), z);
        acc(gx, -g7, z);
        acc(gz, -g7, x);
        acc(gx, g8, x);
        acc(gy, -g8, y);
    }
    if (DEG > 2) {
        const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
        const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
        const float g9 = __fmul_rn(-0.5900435899266435f, G[9]), g10 = __fmul_rn(2.890611442640554f, G[10]),
                    g11 = __fmul_rn(-0.4570457994644658f, G[11]), g12 = __fmul_rn(0.3731763325901154f, G[12]),
                    g13 = __fmul_rn(-0.4570457994644658f, G[13]), g14 = __fmul_rn(1.445305721320277f, G[14]),
                    g15 = __fmul_rn(-0.5900435899266435f, G[15]);
        // Y9 = c9 y (3xx - yy)
        acc(gx, __fmul_rn(6.0f, g9), xy);
        acc(gy, __fmul_rn(3.0f, g9), __fsub_rn(xx, yy));
        // Y10 = c10 xyz
        acc(gx, g10, yz);
        acc(gy, g10, xz);
        acc(gz, g10, xy);
        // Y11 = c11 y (4zz - xx - yy)
        acc(gx, __fmul_rn(-2.0f, g11), xy);
        acc(gy, g11, __fsub_rn(__fsub_rn(__fmul_rn(4.0f, zz), xx), __fmul_rn(3.0f, yy)));
        acc(gz, __fmul_rn(8.0f, g11), yz);
        // Y12 = c12 z (2zz - 3xx - 3yy)
        acc(gx, __fmul_rn(-6.0f, g12), xz);
        acc(gy, __fmul_rn(-6.0f, g12), yz);
        acc(gz, __fmul_rn(3.0f, g12), __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), xx), yy));
        // Y13 = c13 x (4zz - xx - yy)
        acc(gx, g13, __fsub_rn(__fsub_rn(__fmul_rn(4.0f, zz), __fmul_rn(3.0f, xx)), yy));
        acc(gy, __fmul_rn(-2.0f, g13), xy);
        acc(gz, __fmul_rn(8.0f, g13), xz);
        // Y14 = c14 z (xx - yy)
        acc(gx, __fmul_rn(2.0f, g14), xz);
        acc(gy, __fmul_rn(-2.0f, g14), yz);
        acc(gz, g14, __fsub_rn(xx, yy));
        // Y15 = c15 x (xx - 3yy)
        acc(gx, __fmul_rn(3.0f, g15), __fsub_rn(xx, yy));
        acc(gy, __fmul_rn(-6.0f, g15), xy);
    }
}

// One composited cell of the forward-style kernels (forward cell functor, pipeline.cu:66-85): the cell's colour (its
// SH row is read only above density 1e-6), alpha, the weight w = T alpha and the colour sums, in the association
// every forward-style kernel pins.  `on_weight(w)` runs between the weight and the colour sums (the forward's
// `contrib` atomics sit there).  Returns the transmittance behind the cell; T itself is left to the caller.
template <int DEG, typename OnWeight>
__device__ __forceinline__ float composite_cell(const float *__restrict__ sh_rows, const float *sh, uint32_t cell,
                                                float s, float t0, float t1, float T, float &cr, float &cg,
                                                float &cb, OnWeight &&on_weight) {
    float r_ = 0.0f, g_ = 0.0f, b_ = 0.0f;
    if (s > 1e-6f)
        sh_to_rgb<DEG>(sh_rows + (uint64_t)cell * sh_row(DEG), sh, r_, g_, b_);
    float delta = fmaxf(__fsub_rn(t1, t0), 0.0f);
    float alpha = 1.0f - expf(-s * delta);
    float w = __fmul_rn(T, alpha);
    on_weight(w);
    cr = __fmaf_rn(w, r_, cr);
    cg = __fmaf_rn(w, g_, cg);
    cb = __fmaf_rn(w, b_, cb);
    return __fmul_rn(T, __fsub_rn(1.0f, alpha));
}

// Per-ray state of the backward pass and the analytic gradients of one composited cell
// (backward cell functor, pipeline.cu:219-331; SURVEY.md Appendix A.4/A.5, quirks kept).
// Shared by both backward kernels; every multiply-add is pinned to the reference's SASS
// association for the reason given at isect_grad().
struct BackwardRay {
    float out[4];   // saved forward rgba
    float g[4];     // dL/drgba
    float k_alpha;  // (1 - rgba.a) * dL/da, constant per ray
    float err;
    uint32_t Q, qi;
    const float *qv, *dg;
    float cq, cdg;
    float T, cr, cg, cb;
    uint32_t prev;
    float ppx, ppy, ppz; // prev_point (zero before the first composited cell: quirk A.5.2)
    float pgx, pgy, pgz; // prev_point_grad
    float cgx, cgy, cgz; // current_point_grad

    __device__ __forceinline__ void init() {
        T = 1.0f;
        cr = cg = cb = 0.0f;
        prev = kNone;
        ppx = ppy = ppz = 0.0f;
        pgx = pgy = pgz = 0.0f;
        cgx = cgy = cgz = 0.0f;
        qi = 0;
        cdg = 0.0f;
        k_alpha = __fmul_rn(__fsub_rn(1.0f, out[3]), g[3]);
    }

    // Gradients of one cell.  Outputs: dL/drgb (ReLU-masked), dL/dsigma, and -- when
    // `flush` -- the finished position gradient (fx,fy,fz) of point `flush_idx` (the
    // previous composited cell: gradients are flushed one cell late, quirk A.5.1).
    // Returns whether the ray continues.  RAY: also adds the cell's plane terms of the ray gradient to `ra`.
    template <bool RAY>
    __device__ __forceinline__ bool cell(uint32_t cur, const float4 &pc, const float4 &pn,
                                         float t0, float t1, const float rgb[3],
                                         const RayGeom &ray, float weight_threshold,
                                         float dL_drgb[3], float &dL_ds, float &w_out, bool &flush,
                                         uint32_t &flush_idx, float &fx_, float &fy_, float &fz_, RayAcc &ra) {
        const float s = pc.w;
        float delta = fmaxf(__fsub_rn(t1, t0), 0.0f);
        float alpha = 1.0f - expf(__fmul_rn(s, -delta));
        float oma = __fsub_rn(1.0f, alpha);
        float omae = __fadd_rn(oma, 1e-6f);
        float denom = __fmul_rn(omae, T);
        float w = __fmul_rn(alpha, T);
        w_out = w;
        cr = __fmaf_rn(w, rgb[0], cr);
        cg = __fmaf_rn(w, rgb[1], cg);
        cb = __fmaf_rn(w, rgb[2], cb);
        float rest0 = __fdiv_rn(__fsub_rn(out[0], cr), denom);
        float rest1 = __fdiv_rn(__fsub_rn(out[1], cg), denom);
        float rest2 = __fdiv_rn(__fsub_rn(out[2], cb), denom);
        float dot = __fmaf_rn(g[0], __fsub_rn(rgb[0], rest0),
                              __fmaf_rn(g[1], __fsub_rn(rgb[1], rest1),
                                        __fmul_rn(g[2], __fsub_rn(rgb[2], rest2))));
        float dL_dalpha = __fmaf_rn(dot, T, __fdiv_rn(k_alpha, omae));
        float Tn = __fmul_rn(oma, T);
        dL_ds = __fmul_rn(dL_dalpha, __fmul_rn(delta, oma));
        float dL_dt0 = 0.0f;
        float ray_dt0 = 0.0f; // RAY: sum of the depth gradients of the quantiles this cell fires (d depth / d t0 = 1)
        while (qi < Q && Tn < cq) {
            const float dgq = __ldg(dg + qi);
            if (RAY)
                ray_dt0 = __fadd_rn(ray_dt0, dgq);
            float gq = __fdiv_rn(dgq, s);
            dL_dt0 = __fadd_rn(gq, dL_dt0);
            float m = __fmul_rn(logf(__fdiv_rn(T, cq)), gq);
            dL_ds = __fsub_rn(dL_ds, __fdiv_rn(m, s));
            cdg = __fsub_rn(cdg, gq);
            qi++;
            if (qi < Q)
                cq = __ldg(qv + qi);
        }
        float dL_dd = __fmul_rn(dL_dalpha, (delta > 0.0f) ? __fmul_rn(s, oma) : 0.0f);
        if (qi < Q) {
            dL_ds = __fmaf_rn(cdg, -delta, dL_ds);
            dL_dd = __fmaf_rn(cdg, -s, dL_dd);
        }
        dL_dt0 = __fsub_rn(dL_dt0, dL_dd);
        const float dL_dt1 = dL_dd;

        // position gradients through t0 / t1 (pipeline.cu:284-313)
        float ax, ay, az, bx, by, bz, ex, ey, ez, nx, ny, nz;
        // entry plane (prev | cur): e = dt0/dcur, a = dt0/dprev; exit plane (cur | next):
        // b = dt1/dcur, n = dt1/dnext.  Before the first composited cell prev_point is the
        // origin (quirk A.5.2) and dt0/dprev is defined as zero (pipeline.cu:284-289).
        float pnx, pny, pnz, pdp, pnum; // planes (cur | prev) and (cur | next)
        isect_grad_pair(pc.x, pc.y, pc.z, ppx, ppy, ppz, ray, ex, ey, ez, ax, ay, az, pnx, pny, pnz, pdp, pnum);
        if (prev == kNone)
            ax = ay = az = 0.0f;
        isect_grad_pair(pc.x, pc.y, pc.z, pn.x, pn.y, pn.z, ray, bx, by, bz, nx, ny, nz, pnx, pny, pnz, pdp, pnum);
        if (RAY) {
            // t0 lies on the previous composited cell's exit plane (the constant 0 before the first one), t1 on
            // this cell's; dL/dt0 takes the depth gradients themselves, not the point gradient's gd / sigma
            if (prev != kNone)
                ra.add(__fsub_rn(ray_dt0, dL_dd), ra.jx, ra.jy, ra.jz, ra.jt);
            ra.jx = -__fdiv_rn(pnx, pdp);
            ra.jy = -__fdiv_rn(pny, pdp);
            ra.jz = -__fdiv_rn(pnz, pdp);
            ra.jt = __fdiv_rn(pnum, pdp);
            ra.add(dL_dt1, ra.jx, ra.jy, ra.jz, ra.jt);
        }
        pgx = __fmaf_rn(dL_dt0, ax, pgx);
        pgy = __fmaf_rn(dL_dt0, ay, pgy);
        pgz = __fmaf_rn(dL_dt0, az, pgz);
        cgx = __fadd_rn(cgx, __fmaf_rn(dL_dt0, ex, __fmul_rn(dL_dt1, bx)));
        cgy = __fadd_rn(cgy, __fmaf_rn(dL_dt0, ey, __fmul_rn(dL_dt1, by)));
        cgz = __fadd_rn(cgz, __fmaf_rn(dL_dt0, ez, __fmul_rn(dL_dt1, bz)));
        flush = prev != kNone;
        flush_idx = prev;
        fx_ = pgx; fy_ = pgy; fz_ = pgz;
        ppx = pc.x; ppy = pc.y; ppz = pc.z;
        prev = cur;
        pgx = cgx; pgy = cgy; pgz = cgz;
        cgx = __fmul_rn(dL_dt1, nx);
        cgy = __fmul_rn(dL_dt1, ny);
        cgz = __fmul_rn(dL_dt1, nz);

        T = Tn;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float v = __fmul_rn(g[c], w);
            dL_drgb[c] = (rgb[c] == 0.0f) ? 0.0f : v;
        }
        return T > weight_threshold;
    }
};

// the walk, with the scan variant chosen per ray (one-thread-per-ray kernels)
template <typename Faces, typename CellFn>
__device__ __forceinline__ uint32_t walk(const Faces &fa, const float4 *__restrict__ cells,
                                         const RayGeom &ray, uint32_t start, uint32_t max_steps,
                                         CellFn &&cell_fn) {
    if (needs_exact_scan(ray.dx, ray.dy, ray.dz))
        return walk<true>(fa, cells, ray, start, max_steps, cell_fn);
    return walk<false>(fa, cells, ray, start, max_steps, cell_fn);
}

// ray index of this thread.  image_width == 0: linear.  Otherwise the rays are a
// row-major image; a CTA covers a kTileW x kTileH pixel block (16x8 at 128 threads) and each
// warp an 8x4 tile, so the lanes of a warp sit in the same or adjacent cells.
// `block` is the tile this CTA works on: blockIdx.x, or a scheduled order of the tiles (backward replay).
__device__ __forceinline__ bool thread_ray(uint32_t num_rays, uint32_t image_width,
                                           uint32_t blocks_x, uint32_t &ray_idx, uint32_t block) {
    if (image_width == 0) {
        ray_idx = block * kBlock + threadIdx.x;
        return ray_idx < num_rays;
    }
    uint32_t bx = block % blocks_x, by = block / blocks_x;
    uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t x = bx * kTileW + (warp % kWarpsX) * 8 + (lane & 7);
    uint32_t y = by * kTileH + (warp / kWarpsX) * 4 + (lane >> 3);
    uint32_t height = num_rays / image_width;
    ray_idx = y * image_width + x;
    return x < image_width && y < height;
}
__device__ __forceinline__ bool thread_ray(uint32_t num_rays, uint32_t image_width,
                                           uint32_t blocks_x, uint32_t &ray_idx) {
    return thread_ray(num_rays, image_width, blocks_x, ray_idx, blockIdx.x);
}

} // namespace rfb
