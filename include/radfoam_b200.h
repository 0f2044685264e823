/*
 * radfoam_b200.h -- C ABI of the B200-native drop-in for radfoam's src/tracing
 * hot path (the differentiable Voronoi ray tracer).
 *
 * Every entry point replaces one piece of the reference's native interface
 * (paths relative to the radfoam tree):
 *
 *   rfb_create_pipeline      <- radfoam::create_pipeline            src/tracing/pipeline.h:133 (impl pipeline.cu:776-805)
 *   rfb_attribute_dim/type   <- Pipeline::attribute_dim/_type       src/tracing/pipeline.h:128-130
 *   rfb_prefetch_adjacent_diff <- radfoam::prefetch_adjacent_diff   src/tracing/pipeline.h:50-56
 *   rfb_trace_forward        <- Pipeline::trace_forward             src/tracing/pipeline.h:62-78
 *   rfb_trace_backward       <- Pipeline::trace_backward            src/tracing/pipeline.h:80-100
 *   rfb_trace_benchmark      <- Pipeline::trace_benchmark           src/tracing/pipeline.h:117-126
 *   rfb_trace_visualization <- Pipeline::trace_visualization src/tracing/pipeline.h:102-115
 *   rfb_locate_points        <- radfoam::nn over the AABB tree  src/aabb_tree/aabb_tree.cu:343-415 (any number of queries)
 *   rfb_sample_field(_backward)  (new) the field at arbitrary points and its attribute gradient
 *
 * The reference interface is a C++ vtable taking raw device pointers (Eigen
 * types appear only as reinterpret_casts of packed floats); this header
 * flattens the same argument lists to POD so any FFI (ctypes, pybind11, cgo...)
 * can bind it.  All array arguments are DEVICE pointers on the current CUDA
 * device; `stream` is a cudaStream_t passed as void* (NULL = legacy default
 * stream, which is what the reference launches on, common_kernels.cuh:34-39).
 *
 * Conventions:
 *   - every function returns 0 on success, nonzero on failure; the message of
 *     the last failure on the calling thread is rfb_last_error()  (the
 *     reference throws std::runtime_error, cuda_helpers.h:12-30).
 *   - layouts are the reference's: points[N][3] f32; attributes[N][A] row-major
 *     (A = 1 + 3*(deg+1)^2: SH coefficients interleaved RGB then density,
 *     sh_utils.cuh:78-80, pipeline.cu:49) in f32 or f16; point_adjacency[E] u32
 *     and point_adjacency_offsets[N+1] u32 (CSR, rows ascending,
 *     delaunay.cu:146-226); rays[R][6] f32 = origin, direction (camera.h:7-10);
 *     start_point_index[R] u32; depth_quantiles[R][Q] f32.
 *   - outputs are the reference's: ray_rgba[R][4] (attr dtype),
 *     quantile_depths[R][Q] f32, quantile_point_indices[R][Q] u32,
 *     num_intersections[R] u32, point_contribution[N] (attr dtype, caller
 *     zero-initialises), points_grad[N][3] f32, attribute_grad[N][A] (attr
 *     dtype), point_error[N] (attr dtype, caller zero-initialises).
 *     Unlike the reference, points_grad / attribute_grad are fully
 *     OVERWRITTEN by rfb_trace_backward (no caller zero-fill needed; a
 *     zero-filled buffer gives the same result).  ray_grad[R][6] f32 =
 *     dL/d(origin, direction as passed in) is opt-in (RFB_FLAG_RAY_GRAD):
 *     with the flag it is fully overwritten; without it, it is never
 *     written, like the reference kernel (pipeline.cu:132-343).
 *   - the pipeline object owns only its own scratch (cached, re-laid-out
 *     mirrors of the scene and the fp32 gradient accumulator); it never frees
 *     or retains caller memory beyond a call.
 */
#ifndef RADFOAM_B200_H
#define RADFOAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RFB_ABI_VERSION 1

/* radfoam::ScalarType subset accepted by create_pipeline (src/utils/typing.h:22-29) */
enum { RFB_FLOAT32 = 0, RFB_FLOAT16 = 1 };

/* radfoam::CameraModel, src/tracing/camera.h:12-15 */
enum { RFB_PINHOLE = 0, RFB_FISHEYE = 1 };

/* radfoam::TraceSettings, src/tracing/pipeline.h:10-20 */
typedef struct rfb_trace_settings {
    float weight_threshold;     /* default 0.001f */
    uint32_t max_intersections; /* default 1024   */
} rfb_trace_settings;

/* radfoam::Camera, src/tracing/camera.h:17-34 (CVec3f = 3 packed floats) */
typedef struct rfb_camera {
    float position[3];
    float forward[3];
    float right[3];
    float up[3];
    float fov;
    uint32_t width;
    uint32_t height;
    int32_t model; /* RFB_PINHOLE / RFB_FISHEYE */
} rfb_camera;

/* Optional per-call hints; NULL means all-zero (always safe, never changes results). */
typedef struct rfb_launch_opts {
    /* Nonzero: identifies the contents of (points, attributes, adjacency).  When
     * two consecutive calls on one pipeline pass the same nonzero value and the
     * same device pointers / sizes, the re-laid-out scene mirrors (the
     * reference's adjacent_diff among them, which it rebuilds on every call,
     * pipeline.cu:613-620, 667-674) are reused instead of rebuilt.  0 = rebuild. */
    uint64_t scene_version;
    /*   PRECONDITIONS of a nonzero scene_version (the library cannot verify them cheaply):
     *     - the caller MUST pass a new value whenever it has written to points, attributes,
     *       point_adjacency or point_adjacency_offsets since the last call with the old value
     *       (in-place optimizer updates included) -- otherwise stale mirrors are traced, silently;
     *     - the four device pointers MUST stay allocated and unmoved for as long as a value is
     *       reused (the cache key is pointer + size + version, not contents);
     *     - a pipeline MUST NOT be used from two streams at once; consecutive calls on different
     *       streams are ordered by the library (events on the mirrors and on the tape).
     *   Setting the environment variable RFB_DEBUG=1 makes every cache hit re-checksum points and
     *   attributes on the device (synchronising) and fail with a message when they changed under
     *   an unchanged version.  scene_version == 0 is always safe: nothing is cached. */
    /* Nonzero: rays form a row-major image of this width (R % width == 0); rays
     * are then assigned to warps as 8x4 pixel tiles for cell coherence.
     * 0 = rays are an unordered batch (linear assignment).  Results are
     * identical either way (up to fp32 summation order of the scatter-adds). */
    uint32_t image_width;
    uint32_t flags; /* RFB_FLAG_* */
} rfb_launch_opts;

/* zero non-finite gradient entries in the backward epilogue (what
 * radfoam_model/render.py:98-99 does in two extra passes after the call) */
#define RFB_FLAG_SCRUB_NONFINITE 1u
/* trace_forward: also record the walk tape -- (cell, t1) per ray and visited cell, 8 bytes --
 * so that the backward of the same step can replay it instead of re-scanning faces (the
 * reference's backward re-walks every ray, pipeline.cu:132-343).  Needs a nonzero scene_version. */
#define RFB_FLAG_RECORD_TAPE 2u
/* trace_backward: the caller vouches that rays / start points / quantiles / settings / scene are
 * those of this pipeline's last recording forward; the library additionally checks pointers,
 * sizes, settings and scene_version and silently re-walks when anything differs.  Results are
 * identical either way.  PRECONDITION: the CONTENTS of rays and start_point_index MUST be
 * unchanged since that forward (the library compares the pointers, not the data).  If the tape's
 * memory cannot be allocated the forward simply does not record and the backward re-walks. */
#define RFB_FLAG_USE_TAPE 4u
/* trace_backward: also compute ray_grad[r] = dL/d(origin, direction as passed in, before renormalisation),
 * with the walk's cell sequence held fixed (DESIGN.md §2).  ray_grad is fully overwritten and MUST NOT be NULL;
 * RFB_FLAG_SCRUB_NONFINITE zeroes its non-finite entries too.  Every other output is the same with or without
 * it.  (rfb_trace_backward_accumulate_rays takes ray_grad directly instead of this flag.) */
#define RFB_FLAG_RAY_GRAD 8u

typedef struct rfb_pipeline rfb_pipeline;

const char *rfb_last_error(void);
int rfb_abi_version(void);

/* sh_degree in {0,1,2,3}, attr_dtype in {RFB_FLOAT32, RFB_FLOAT16}; anything else
 * fails ("Unsupported SH degree" / "Unsupported attribute type", pipeline.cu:776-805). */
int rfb_create_pipeline(int sh_degree, int attr_dtype, rfb_pipeline **out);
void rfb_destroy_pipeline(rfb_pipeline *pipeline);
uint32_t rfb_attribute_dim(const rfb_pipeline *pipeline);
int rfb_attribute_type(const rfb_pipeline *pipeline);

/* adjacent_diff[e] = half4(RN(points[adj[e]] - points[i]), 0) for e in row i;
 * adjacent_diff has room for point_adjacency_size half4 (8-byte) entries. */
int rfb_prefetch_adjacent_diff(const float *points, uint32_t num_points,
                               uint32_t point_adjacency_size,
                               const uint32_t *point_adjacency,
                               const uint32_t *point_adjacency_offsets,
                               void *adjacent_diff, void *stream);

/* Entry cell of each query point = index of its nearest point (exact: smallest distance, ties -> lowest index;
 * UINT32_MAX for a query with NaN coordinates).  Stands in for radfoam::nn over the AABB tree
 * (src/aabb_tree/aabb_tree.h:18-27) for the one use the tracer has for it: the start cell of a camera
 * (radfoam_model/scene.py:224-234).  A tiled brute force: U x N distance evaluations, 12 N bytes of traffic in
 * total; meant for camera counts (1 .. a few thousand queries).  points[N][3], queries[M][3] f32, indices[M]
 * u32, all device pointers.  For many distinct queries rfb_locate_points is the scalable lookup. */
int rfb_nearest_point(const float *points, uint32_t num_points, const float *queries,
                      uint32_t num_queries, uint32_t *indices, void *stream);

/* RadFoamScene.get_starting_point (radfoam_model/scene.py:224-234) in one call, without its torch.unique
 * sort over all rays and without a host round trip: start_point_index[r] = nearest point of the origin of
 * rays[r] (rays[R][6] f32).  Distinct origins are found with a device-side hash set, each is looked up once.
 * Cost O(R + U N) for U distinct origins. */
int rfb_start_points(const float *points, uint32_t num_points, const float *rays,
                     uint32_t num_rays, uint32_t *start_point_index, void *stream);

/* Per point i: indices[i] = the adjacent point farthest from it (first maximum in row order; UINT32_MAX when
 * the row is empty or every neighbour coincides with it), cell_radius[i] = sum(0.5*|p_j - p_i|) / num_faces
 * (NaN for an empty row).  Replaces radfoam::farthest_neighbor (src/delaunay/triangulation_ops.h:8-15, kernel
 * triangulation_ops.cu:9-44; pybind farthest_neighbor, torch_bindings/triangulation_bindings.cpp:184-216), the
 * CSR pass the densification step runs before sampling new points (radfoam_model/scene.py:434-461).
 * Bit-identical outputs.  points[N][3] f32, CSR as for the tracer, indices[N] u32, cell_radius[N] f32. */
int rfb_farthest_neighbor(const float *points, uint32_t num_points,
                          const uint32_t *point_adjacency,
                          const uint32_t *point_adjacency_offsets,
                          uint32_t *indices, float *cell_radius, void *stream);

/* Cell of any number of query points, found by walking the adjacency graph (radfoam::nn over the AABB tree,
 * src/aabb_tree/aabb_tree.cu:343-415, answers the same question).  From a seed cell s the walk scans row s of the
 * CSR and moves to the neighbour smallest in the order (d2, index) -- d2 = fma(dx,dx, fma(dy,dy, dz*dz)) in fp32,
 * as rfb_nearest_point computes it, ties to the lower index -- and stops when no neighbour is smaller than s.
 * Seeds: hints[m] when it is < num_points; when it is not, or hints is NULL, the library's seed (the nearest of a
 * fixed strided sample of the points).  Cost: the walk's row scans (about 15.5 distances each) per query, instead
 * of rfb_nearest_point's N.  Contract:
 *   - indices[m] is always a local minimum of (d2, index) over the adjacency graph (empty rows are legal: the
 *     walk stops there);
 *   - when the adjacency is the Delaunay graph of `points`, it is the nearest point as rfb_nearest_point defines
 *     it, except for queries whose best and second-best distances are within fp32 rounding of each other;
 *   - when the points have moved since the adjacency was built (a stale triangulation) only the local-minimum
 *     property holds (a stale AABB tree promises no more);
 *   - a query with a NaN coordinate, or whose cell is at a non-finite distance, yields UINT32_MAX.
 * No host synchronisation, no allocation; safe under CUDA-graph capture.  points[N][3], queries[M][3] f32,
 * CSR as for the tracer, hints[M] / indices[M] u32, all device pointers. */
int rfb_locate_points(const float *points, uint32_t num_points,
                      const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets,
                      const float *queries, uint32_t num_queries,
                      const uint32_t *hints, uint32_t *indices, void *stream);

/* The field at M query points: cells[m] = rfb_locate_points' cell (same seeds, same contract),
 * density[m] = attributes[cell][A-1] and, when directions[M][3] is given (renormalised in the kernel, as ray
 * directions are), rgb[m][3] = max(0, 0.5 + sum_k Y_k(dir) c_k): the colour the tracer composites for that cell
 * along a ray with that direction, bit for bit (same SH basis and FFMA chain).  directions and rgb are both given
 * or both NULL.  density and rgb are in the pipeline's attribute dtype; a query without a cell (UINT32_MAX) gets
 * NaN.  Reads only its arguments: no pipeline state (scene mirrors, walk tape, accumulator) is used or changed. */
int rfb_sample_field(rfb_pipeline *pipeline, const float *points, uint32_t num_points, const void *attributes,
                     const uint32_t *point_adjacency, const uint32_t *point_adjacency_offsets,
                     const float *queries, uint32_t num_queries, const uint32_t *hints,
                     const float *directions, uint32_t *cells, void *density, void *rgb, void *stream);

/* Backward of rfb_sample_field with respect to the attributes: attribute_grad[N][A] (attr dtype) is fully
 * overwritten with sum over queries m in cell i of  Y_k(dir_m) dL/drgb_m[c]  at column 3k+c (0 where the forward's
 * rgb_m[c] is 0, the clamp) and dL/ddensity_m at column A-1.  Summed in fp32, rounded once to the attribute dtype.
 * rgb_grad[M][3] / density_grad[M] (attr dtype) may each be NULL (no gradient); rgb_grad needs directions and the
 * forward's rgb.  Queries whose cell is not a point (UINT32_MAX) contribute nothing.  The gradients with respect to
 * points and queries are zero almost everywhere (the field is piecewise constant) and are not formed; those with
 * respect to the directions are not computed.  Uses stream-ordered scratch for fp16, never the pipeline's
 * accumulator: a recorded walk tape or accumulated trace gradients stay as they were. */
int rfb_sample_field_backward(rfb_pipeline *pipeline, uint32_t num_points, uint32_t num_queries,
                              const uint32_t *cells, const float *directions, const void *rgb,
                              const void *rgb_grad, const void *density_grad, void *attribute_grad,
                              void *stream);

int rfb_trace_forward(rfb_pipeline *pipeline, const rfb_trace_settings *settings,
                      uint32_t num_points, const float *points,
                      const void *attributes, uint32_t point_adjacency_size,
                      const uint32_t *point_adjacency,
                      const uint32_t *point_adjacency_offsets, uint32_t num_rays,
                      const float *rays, const uint32_t *start_point_index,
                      uint32_t num_depth_quantiles, const float *depth_quantiles,
                      void *ray_rgba, float *quantile_depths,
                      uint32_t *quantile_point_indices,
                      uint32_t *num_intersections, void *point_contribution,
                      const rfb_launch_opts *opts, void *stream);

int rfb_trace_backward(rfb_pipeline *pipeline, const rfb_trace_settings *settings,
                       uint32_t num_points, const float *points,
                       const void *attributes, uint32_t point_adjacency_size,
                       const uint32_t *point_adjacency,
                       const uint32_t *point_adjacency_offsets, uint32_t num_rays,
                       const float *rays, const uint32_t *start_point_index,
                       uint32_t num_depth_quantiles, const float *depth_quantiles,
                       const uint32_t *quantile_point_indices,
                       const void *ray_rgba, const void *ray_rgba_grad,
                       const float *depth_grad, const void *ray_error,
                       float *ray_grad, float *points_grad, void *attribute_grad,
                       void *point_error, const rfb_launch_opts *opts,
                       void *stream);

/* ---- split backward for ray-sharded multi-GPU use (SURVEY.md §8e) ----
 * rfb_trace_backward == accumulate (zeroes then fills the pipeline's fp32
 * accumulator [N][rfb_grad_row_floats]) + finalize (writes the reference-layout
 * outputs).  A data-parallel caller all-reduces the accumulator between them. */
int rfb_trace_backward_accumulate(
    rfb_pipeline *pipeline, const rfb_trace_settings *settings,
    uint32_t num_points, const float *points, const void *attributes,
    uint32_t point_adjacency_size, const uint32_t *point_adjacency,
    const uint32_t *point_adjacency_offsets, uint32_t num_rays,
    const float *rays, const uint32_t *start_point_index,
    uint32_t num_depth_quantiles, const float *depth_quantiles,
    const uint32_t *quantile_point_indices, const void *ray_rgba,
    const void *ray_rgba_grad, const float *depth_grad, const void *ray_error,
    void *point_error, const rfb_launch_opts *opts, void *stream);
/* rfb_trace_backward_accumulate that also writes ray_grad[R][6] (see RFB_FLAG_RAY_GRAD; NULL = not wanted,
 * which is rfb_trace_backward_accumulate).  RFB_FLAG_SCRUB_NONFINITE in opts->flags zeroes its non-finite
 * entries; the accumulator itself is never scrubbed (finalize does that). */
int rfb_trace_backward_accumulate_rays(
    rfb_pipeline *pipeline, const rfb_trace_settings *settings,
    uint32_t num_points, const float *points, const void *attributes,
    uint32_t point_adjacency_size, const uint32_t *point_adjacency,
    const uint32_t *point_adjacency_offsets, uint32_t num_rays,
    const float *rays, const uint32_t *start_point_index,
    uint32_t num_depth_quantiles, const float *depth_quantiles,
    const uint32_t *quantile_point_indices, const void *ray_rgba,
    const void *ray_rgba_grad, const float *depth_grad, const void *ray_error,
    void *point_error, float *ray_grad, const rfb_launch_opts *opts, void *stream);
/* device pointer + element count of the fp32 accumulator of the last accumulate */
int rfb_grad_accumulator(rfb_pipeline *pipeline, float **ptr, uint64_t *num_floats);
uint32_t rfb_grad_row_floats(const rfb_pipeline *pipeline);
int rfb_trace_backward_finalize(rfb_pipeline *pipeline, uint32_t num_points,
                                float *points_grad, void *attribute_grad,
                                uint32_t flags, void *stream);

/* ---- parameter-form scene: RadFoamScene.get_trace_data (radfoam_model/scene.py:202-217) fused in ----
 * The reference builds  attributes = cat(att_dc, att_sh, activation_scale * softplus(density, beta=10)).to(dtype)
 * with torch ops before every trace and splits attr_grad back through them afterwards (3-5 passes over [N][A]).
 * While a parameter-form scene is bound, the `attributes` argument of rfb_trace_forward /
 * rfb_trace_backward_accumulate is ignored (may be NULL): the re-layout kernel reads the three parameter
 * arrays (f32: att_dc[N][3], att_sh[N][A-4], density[N] pre-activation) directly, and
 * rfb_trace_backward_finalize_params writes the gradients of the PARAMETERS (attribute gradient rounded to the
 * pipeline's attr dtype and scrubbed like attribute_grad, then chained through cat and softplus).  The same
 * scene_version contract applies (bump it when the parameters are written).  rfb_trace_backward (the fused
 * accumulate+finalize) is not available while bound. */
typedef struct rfb_scene_params {
    const float *att_dc;
    const float *att_sh;
    const float *density;
    float activation_scale;
} rfb_scene_params;
int rfb_bind_scene_params(rfb_pipeline *pipeline, const rfb_scene_params *params /* NULL: unbind */);
int rfb_trace_backward_finalize_params(rfb_pipeline *pipeline, uint32_t num_points, float *points_grad,
                                       float *att_dc_grad, float *att_sh_grad, float *density_grad,
                                       uint32_t flags, void *stream);

/* ---- fused cross-GPU reduction + finalize over peer-mapped memory (NVLink / NVSwitch) ----
 * rfb_set_grad_accumulator: make rfb_trace_backward_accumulate scatter into caller-provided device memory
 * (16-byte aligned, >= num_points * rfb_grad_row_floats() floats; e.g. a symmetric / IPC-mapped allocation
 * that the other GPUs of the box can address) instead of the pipeline's own buffer.  NULL restores the
 * internal buffer.  The memory stays the caller's; accumulate zero-fills it first, as it does its own.
 *
 * rfb_reduce_finalize_peers: rank `rank` of `world` (<= 16) sums its share of the rows (blocks of 16 rows
 * dealt round-robin) over ALL ranks' accumulators peer_acc[0..world) -- device pointers addressable from the
 * current device, peer_acc[rank] being this rank's own -- in rank order, applies the finalize epilogue
 * (reference layout, RFB_FLAG_SCRUB_NONFINITE) and stores the finished rows into every rank's
 * peer_attribute_grad[w] ([N][A], attr dtype) and peer_points_grad[w] ([N][3] f32).  After ALL ranks have run
 * it every rank holds the complete gradients, bit-identical across ranks.  The CALLER provides the two
 * cross-GPU barriers: every rank's accumulate must have finished before any rank starts, and every rank must
 * have finished before the outputs are read or an accumulator is written again.
 *
 * `multicast` (optional, NULL = none): NVSwitch multicast addresses of the same three arrays (one mapping that
 * reaches every rank's copy; e.g. torch symmetric memory's multicast_ptr + the array's offset).  With it a rank
 * reads its share with multimem.ld_reduce -- the switch returns the sum over all ranks -- and writes it with
 * multimem.st -- the switch replicates it --, so only 1/world of the arrays crosses each GPU's link in each
 * direction instead of (world-1)/world.  The sum is then formed by the switch (order unspecified, fp32);
 * every rank still receives identical bits. */
typedef struct rfb_multicast {
    const float *acc;
    void *attribute_grad;
    float *points_grad;
} rfb_multicast;
int rfb_set_grad_accumulator(rfb_pipeline *pipeline, float *ptr, uint64_t num_floats);
int rfb_reduce_finalize_peers(rfb_pipeline *pipeline, uint32_t world, uint32_t rank,
                              uint32_t num_points, const float *const *peer_acc,
                              void *const *peer_attribute_grad,
                              float *const *peer_points_grad,
                              const rfb_multicast *multicast, uint32_t flags,
                              void *stream);

/* forward-only render with in-kernel ray generation (camera.h:56-85) and RGBA8
 * packing (tracing_utils.cuh:105-115).  adjacent_diff is the caller-built
 * half4[E] array exactly as the reference takes it (benchmark.py:41-54);
 * start_point_index points at ONE u32; output_rgba is u32[width*height]. */
int rfb_trace_benchmark(rfb_pipeline *pipeline, const rfb_trace_settings *settings,
                        uint32_t num_points, const float *points,
                        const void *attributes,
                        const uint32_t *point_adjacency,
                        const uint32_t *point_adjacency_offsets,
                        const void *adjacent_diff, const rfb_camera *camera,
                        const uint32_t *start_point_index, uint32_t *output_rgba,
                        const rfb_launch_opts *opts, void *stream);

/* radfoam::VisualizationMode, src/tracing/pipeline.h:22-27 */
enum { RFB_VIS_RGB = 0, RFB_VIS_DEPTH = 1, RFB_VIS_ALPHA = 2, RFB_VIS_INTERSECTIONS = 3 };

/* radfoam::ColorMap, src/utils/typing.h:136-141 (an index into rfb_cmap_table) */
enum { RFB_CMAP_GRAY = 0, RFB_CMAP_VIRIDIS = 1, RFB_CMAP_INFERNO = 2, RFB_CMAP_TURBO = 3 };

/* radfoam::VisualizationSettings, src/tracing/pipeline.h:29-47 (defaults: RGB, Turbo,
 * bg (1, 1, 1), no checker, max_depth 10, depth_quantile 0.5) */
typedef struct rfb_visualization_settings {
    int32_t mode;      /* RFB_VIS_* */
    int32_t color_map; /* RFB_CMAP_*: the table used by the depth and intersections modes */
    float bg_color[3]; /* RGB mode: background seen through the remaining transmittance */
    uint32_t checker_bg; /* nonzero: a 20-pixel 0.3 / 0.5 grey checker instead of bg_color */
    float max_depth;      /* depth mode: the depth mapped to the end of the colour map */
    float depth_quantile; /* depth mode: the depth where transmittance first drops below this */
} rfb_visualization_settings;

/* radfoam::CMapTable, src/utils/typing.h:143-146.  Both arrays are DEVICE memory owned by the caller:
 * data[m] points at sizes[m] >= 1 RGB entries (float[sizes[m]][3]) of colour map m, for m in RFB_CMAP_*.
 * The library ships no colour-map data. */
typedef struct rfb_cmap_table {
    const float *const *data;
    const int32_t *sizes;
} rfb_cmap_table;

/* Preview render with in-kernel ray generation, as rfb_trace_benchmark, but with the settings' output
 * (RFB_VIS_RGB: colour over a background; RFB_VIS_DEPTH: colormap(depth / max_depth); RFB_VIS_ALPHA: 1 - T;
 * RFB_VIS_INTERSECTIONS: colormap((cells entered - 1) / max_intersections)) written as RGBA8 words to a 2-D
 * surface: pixel (i, j) goes to byte column 4 i of row height - 1 - j (bottom-up, for GL).  output_surface is a
 * cudaSurfaceObject_t of at least width x height 4-byte texels.  start_index is the entry cell, by value;
 * num_tets is accepted and ignored, as in the reference.  cmap_table may be NULL for the RGB and alpha modes. */
int rfb_trace_visualization(rfb_pipeline *pipeline, const rfb_trace_settings *settings,
                            const rfb_visualization_settings *vis_settings,
                            const rfb_camera *camera, const rfb_cmap_table *cmap_table,
                            uint32_t num_points, uint32_t num_tets, const float *points,
                            const void *attributes, const uint32_t *point_adjacency,
                            const uint32_t *point_adjacency_offsets,
                            const void *adjacent_diff, uint32_t start_index,
                            uint64_t output_surface, const rfb_launch_opts *opts,
                            void *stream);

/* rfb_trace_visualization into a linear buffer: output_rgba is u32[height][width] in the surface's row order
 * (the frame equals a 2-D copy of the surface rfb_trace_visualization would fill). */
int rfb_trace_visualization_rgba8(rfb_pipeline *pipeline, const rfb_trace_settings *settings,
                                  const rfb_visualization_settings *vis_settings,
                                  const rfb_camera *camera, const rfb_cmap_table *cmap_table,
                                  uint32_t num_points, uint32_t num_tets, const float *points,
                                  const void *attributes, const uint32_t *point_adjacency,
                                  const uint32_t *point_adjacency_offsets,
                                  const void *adjacent_diff, uint32_t start_index,
                                  uint32_t *output_rgba, const rfb_launch_opts *opts,
                                  void *stream);

/* kernels launched by this library (all threads of the process) since the last reset
 * (bench.py reports it as gpu_launches) */
uint64_t rfb_launch_count(void);
void rfb_reset_launch_count(void);

/* cudaMalloc / cudaFree calls this library has made since it was loaded (its scratch buffers are grow-only:
 * both stay constant in steady state; bench.py reports the delta over its timed loops) */
void rfb_device_alloc_counts(uint64_t *allocs, uint64_t *frees);

/* drop cached scene mirrors (next call rebuilds) */
void rfb_invalidate_cache(rfb_pipeline *pipeline);

/* State of the walk tape of the last recording forward (waits for that forward): pool capacity
 * and chunks requested (8 KB each: 32 steps x 32 rays x 8 bytes), and whether the pool overflowed
 * (then the backward re-walks and the pool is enlarged for the next recording). */
int rfb_tape_status(rfb_pipeline *pipeline, uint32_t *capacity_chunks, uint32_t *used_chunks,
                    uint32_t *overflowed);

/* Live kernel timing for roofline reporting: when enabled, CUDA events are recorded on the
 * launching stream right around the forward / backward ray kernel of every call.
 * rfb_last_kernel_ms(which = 0 forward, 1 backward) waits for and returns the duration of the
 * most recent one. */
void rfb_set_profiling(rfb_pipeline *pipeline, int enabled);
int rfb_last_kernel_ms(rfb_pipeline *pipeline, int which, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* RADFOAM_B200_H */
