// C-ABI shim around the reference's Pipeline::trace_visualization (src/tracing/pipeline.h:102-115) — TEST
// INFRASTRUCTURE ONLY.
//
// Built by oracle/ref_vis.mk into oracle/_ref/libradfoam_ref_vis.so and linked against oracle/_ref/libradfoam_ref.so,
// which holds the reference's own tracing TU (pipeline.cu, compiled where it lies, unmodified).  The reference
// renders into a CUDA surface; this shim creates one on a cudaArray per call, lets the reference's kernel fill it
// and copies it out row by row (the surface's own bottom-up order) into a linear device buffer.
#include <cuda_runtime.h>

#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>

#include "tracing/pipeline.h"

namespace {

thread_local std::string g_last_error;

std::shared_ptr<radfoam::Pipeline> get_pipeline(int sh_degree, int attr_is_half) {
    static std::mutex m;
    static std::map<int, std::shared_ptr<radfoam::Pipeline>> cache;
    std::lock_guard<std::mutex> lock(m);
    int key = sh_degree * 2 + (attr_is_half ? 1 : 0);
    auto it = cache.find(key);
    if (it != cache.end())
        return it->second;
    auto p = radfoam::create_pipeline(sh_degree, attr_is_half ? radfoam::Float16 : radfoam::Float32);
    cache[key] = p;
    return p;
}

void check(cudaError_t e) {
    if (e != cudaSuccess)
        throw std::runtime_error(cudaGetErrorString(e));
}

} // namespace

extern "C" {

const char *rfrefvis_last_error() { return g_last_error.c_str(); }

// cmap_data / cmap_sizes: the device arrays of a CMapTable (src/utils/typing.h:143-146).
// output_rgba: u32[height][width], device.
int rfrefvis_trace_visualization(int sh_degree, int attr_is_half, float weight_threshold,
                                 uint32_t max_intersections, int mode, int color_map, const float *bg_color,
                                 int checker_bg, float max_depth, float depth_quantile, const void *cmap_data,
                                 const void *cmap_sizes, uint32_t num_points, const float *points,
                                 const void *attributes, const uint32_t *point_adjacency,
                                 const uint32_t *point_adjacency_offsets, const void *adjacent_diff,
                                 const float *cam_position, const float *cam_forward, const float *cam_right,
                                 const float *cam_up, float fov, uint32_t width, uint32_t height, int model,
                                 uint32_t start_index, uint32_t *output_rgba) {
    cudaArray_t array = nullptr;
    cudaSurfaceObject_t surf = 0;
    try {
        radfoam::TraceSettings s;
        s.weight_threshold = weight_threshold;
        s.max_intersections = max_intersections;
        radfoam::VisualizationSettings vis = radfoam::default_visualization_settings();
        vis.mode = static_cast<radfoam::VisualizationMode>(mode);
        vis.color_map = static_cast<radfoam::ColorMap>(color_map);
        vis.bg_color = radfoam::Vec3f(bg_color[0], bg_color[1], bg_color[2]);
        vis.checker_bg = checker_bg != 0;
        vis.max_depth = max_depth;
        vis.depth_quantile = depth_quantile;
        radfoam::CMapTable cmap;
        cmap.data = reinterpret_cast<const float *const *>(cmap_data);
        cmap.sizes = reinterpret_cast<const int *>(cmap_sizes);
        radfoam::Camera camera;
        camera.position = radfoam::Vec3f(cam_position);
        camera.forward = radfoam::Vec3f(cam_forward);
        camera.right = radfoam::Vec3f(cam_right);
        camera.up = radfoam::Vec3f(cam_up);
        camera.fov = fov;
        camera.width = width;
        camera.height = height;
        camera.model = model == 0 ? radfoam::Pinhole : radfoam::Fisheye;

        cudaChannelFormatDesc fmt = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);
        check(cudaMallocArray(&array, &fmt, width, height, cudaArraySurfaceLoadStore));
        cudaResourceDesc res = {};
        res.resType = cudaResourceTypeArray;
        res.res.array.array = array;
        check(cudaCreateSurfaceObject(&surf, &res));
        get_pipeline(sh_degree, attr_is_half)
            ->trace_visualization(s, vis, camera, cmap, num_points, 0, points, attributes, point_adjacency,
                                  point_adjacency_offsets, adjacent_diff, start_index, (uint64_t)surf, nullptr);
        check(cudaGetLastError());
        check(cudaMemcpy2DFromArray(output_rgba, 4 * (size_t)width, array, 0, 0, 4 * (size_t)width, height,
                                    cudaMemcpyDeviceToDevice));
        cudaDestroySurfaceObject(surf);
        cudaFreeArray(array);
        return 0;
    } catch (const std::exception &e) {
        g_last_error = e.what();
        if (surf)
            cudaDestroySurfaceObject(surf);
        if (array)
            cudaFreeArray(array);
        return 1;
    }
}

} // extern "C"
