/*
 * vis_oracle.c -- CPU restatement of the reference's visualization kernel (src/tracing/pipeline.cu:345-470,
 * colormap src/tracing/tracing_utils.cuh:117-130).  TEST INFRASTRUCTURE ONLY.
 *
 * It builds on the CPU restatement of the tracer: oracle/radfoam_oracle.c is compiled into the same library
 * (included, not copied), so the ray generation, SH colour and cell walk are exactly the ones the other oracle
 * tests check.  Built on first use by tests/vis_oracle.py with the flags of oracle/Makefile.
 */
#include "../oracle/radfoam_oracle.c"

/* float -> int as the device's cvt.rzi.s32.f32 does it: truncation, NaN -> 0, saturation at INT_MIN / INT_MAX
 * (a C cast is undefined behaviour for all three). */
static int f2i_rz(float x) {
    if (x != x)
        return 0;
    if (x >= 2147483648.0f)
        return 2147483647;
    if (x < -2147483648.0f)
        return (int)0x80000000u;
    return (int)x;
}

/* the .SAT the reference's SASS folds its clamps into: [+0, 1], NaN -> +0 */
static float sat(float x) { return x > 0.0f ? (x < 1.0f ? x : 1.0f) : 0.0f; }

static uint32_t pack_unit_rgb8(float r, float g, float b) {
    uint32_t ri = (uint32_t)f2i_rz(r * 255.0f), gi = (uint32_t)f2i_rz(g * 255.0f), bi = (uint32_t)f2i_rz(b * 255.0f);
    return 0xff000000u | (bi << 16) | (gi << 8) | ri;
}

/* colormap, src/tracing/tracing_utils.cuh:117-130, in the association of the reference's SASS:
 * p = (float)(L-1) * v; i0 = rzi(p); t = p - (float)i0; i1 = i0 + 1 with 32-bit wrap; both clamped to [0, L-1];
 * c = sat(fma(1 - t, table[i0], t * table[i1])). */
static uint32_t colormap_rgba8(float v, const float *table, int len) {
    int last = len - 1;
    float p = (float)last * v;
    int i0 = f2i_rz(p);
    int i1 = (int)((uint32_t)i0 + 1u);
    float t = p - (float)i0, u = 1.0f - t;
    i0 = i0 < last ? i0 : last;
    i0 = i0 > 0 ? i0 : 0;
    i1 = i1 < last ? i1 : last;
    i1 = i1 > 0 ? i1 : 0;
    const float *a = table + 3 * (size_t)i0, *b = table + 3 * (size_t)i1;
    return pack_unit_rgb8(sat(fmaf(u, a[0], t * b[0])), sat(fmaf(u, a[1], t * b[1])), sat(fmaf(u, a[2], t * b[2])));
}

/* visualization kernel + Pipeline::trace_visualization, src/tracing/pipeline.cu:345-470, 703-736: the benchmark walk
 * plus the first-quantile depth and the number of cells entered; mode 0 RGB, 1 depth, 2 alpha, 3 intersections.
 * cmap_tables[m] is float[cmap_sizes[m]][3] (host memory here).  Pixel (i, j) goes to row height-1-j of the
 * u32[height][width] output, as on the reference's surface. */
int rfo_trace_visualization(int sh_degree, int attr_is_half, float weight_threshold,
                            uint32_t max_intersections, int mode, int color_map, const float *bg_color,
                            int checker_bg, float max_depth, float depth_quantile,
                            const float *const *cmap_tables, const int32_t *cmap_sizes, const float *points,
                            const void *attributes, const uint32_t *adj, const uint32_t *off,
                            const uint16_t *adjacent_diff, const float *cam_position,
                            const float *cam_forward, const float *cam_right, const float *cam_up, float fov,
                            uint32_t width, uint32_t height, int model, uint32_t start_point,
                            uint32_t *output_rgba, int num_threads) {
    if (sh_degree < 0 || sh_degree > 3 || mode < 0 || mode > 3 || color_map < 0 || color_map > 3)
        return 1;
    if ((mode == 1 || mode == 3) && (!cmap_tables || !cmap_sizes))
        return 1;
    int sh_dim = (sh_degree + 1) * (sh_degree + 1);
    const half_t *diff = (const half_t *)adjacent_diff;
    int parallel = num_threads != 1;
#ifdef _OPENMP
    if (num_threads > 0)
        omp_set_num_threads(num_threads);
#endif
#pragma omp parallel for schedule(dynamic, 256) if (parallel)
    for (int64_t idx = 0; idx < (int64_t)width * height; ++idx) {
        int pi = (int)(idx % width), pj = (int)(idx / width);
        size_t dst = (size_t)(height - 1 - (uint32_t)pj) * width + (size_t)pi;
        float o[3], d[3];
        cast_ray(cam_position, cam_forward, cam_right, cam_up, fov, width, height, model, pi, pj, o, d);
        float nrm = sqrtf(fmaf(d[0], d[0], fmaf(d[1], d[1], d[2] * d[2])));
        if (nrm < 0.1f) {
            output_rgba[dst] = 0;
            continue;
        }
        float sh[16];
        sh_coefficients(sh_degree, d, sh);
        float T = 1.0f, acc[3] = {0, 0, 0}, depth = 0.0f;
        int passed = 0;
        float t0 = 0.0f;
        uint32_t n = 0, cur = start_point;
        float P[3] = {points[3 * (size_t)cur], points[3 * (size_t)cur + 1], points[3 * (size_t)cur + 2]};
        for (;;) {
            n++;
            if (n > max_intersections)
                break;
            uint32_t b = off[cur], nf = off[cur + 1] - b;
            float t1;
            uint32_t face = scan_faces(diff, b, nf, P, o, d, &t1);
            if (face == RF_NONE)
                break;
            uint32_t nxt = adj[b + face];
            if (t1 > t0) {
                float rgb[3], s;
                load_attributes(sh_dim, sh, attributes, attr_is_half, cur, rgb, &s);
                float delta = fmaxf(t1 - t0, 0.0f);
                float alpha = 1.0f - expf(-s * delta);
                float w = T * alpha;
                for (int c = 0; c < 3; ++c)
                    acc[c] = fmaf(w, rgb[c], acc[c]);
                float Tn = T * (1.0f - alpha);
                if (!passed && Tn < depth_quantile) {
                    depth = t0 + logf(T / depth_quantile) / s;
                    passed = 1;
                }
                T = Tn;
                if (!(T > weight_threshold))
                    break;
            }
            t0 = fmaxf(t0, t1);
            cur = nxt;
            P[0] = points[3 * (size_t)nxt];
            P[1] = points[3 * (size_t)nxt + 1];
            P[2] = points[3 * (size_t)nxt + 2];
        }
        uint32_t out;
        if (mode == 0) {
            float bg[3] = {bg_color[0], bg_color[1], bg_color[2]};
            if (checker_bg)
                bg[0] = bg[1] = bg[2] = (((uint32_t)pi / 20u) ^ ((uint32_t)pj / 20u)) & 1u ? 0.5f : 0.3f;
            out = pack_unit_rgb8(sat(fmaf(T, bg[0], acc[0])), sat(fmaf(T, bg[1], acc[1])), sat(fmaf(T, bg[2], acc[2])));
        } else if (mode == 1) {
            out = colormap_rgba8(depth / max_depth, cmap_tables[color_map], cmap_sizes[color_map]);
        } else if (mode == 2) {
            float a = sat(1.0f - T);
            out = pack_unit_rgb8(a, a, a);
        } else {
            out = colormap_rgba8((float)(n - 1u) / (float)max_intersections, cmap_tables[color_map],
                                 cmap_sizes[color_map]);
        }
        output_rgba[dst] = out;
    }
    return 0;
}

