// ORACLE: a C entry to the reference's depth renderer (local_sensing/src/depth_render.cu, compiled unmodified by depth.mk) — test
// infrastructure only. One handle per scene cloud; ref_depth_render is DepthRender::render_pose: the double[16] camera-from-world matrix
// (row-major) in, the width x height int32 depth image in mm out (999999 where nothing is seen). Exceptions become a non-zero return.
#include "depth_render.cuh"
#include <exception>

extern "C" void *ref_depth_create(float fx, float fy, float cx, float cy, int width, int height, const float *xyz, int n) {
    try {
        DepthRender *r = new DepthRender();
        r->set_para(fx, fy, cx, cy, width, height);
        std::vector<float> cloud(xyz, xyz + 3 * (size_t)n);
        r->set_data(cloud);
        return r;
    } catch (const std::exception &) { return nullptr; }
}

extern "C" int ref_depth_render(void *h, const double *transformation, int *out) {
    try {
        static_cast<DepthRender *>(h)->render_pose(const_cast<double *>(transformation), out);
        return cudaDeviceSynchronize() == cudaSuccess ? 0 : 1;
    } catch (const std::exception &) { return 1; }
}

extern "C" void ref_depth_destroy(void *h) { delete static_cast<DepthRender *>(h); }
