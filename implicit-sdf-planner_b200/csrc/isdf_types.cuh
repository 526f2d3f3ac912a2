// Device-visible parameter blocks shared by the kernels and the C-ABI layer.
#pragma once
#include "isdf_math.cuh"
#include "isdf_shapes.cuh"

namespace isdf {

// Occupancy as one BIT per voxel, z fastest: word (ix*Y + iy)*Zw + (iz >> 5), bit iz & 31. A 512^3 map is 16 MiB
// (L2-resident on H100: 50 MB of L2) instead of the reference's 1 GiB of doubles (GridMap3D.h:215); a 14-voxel z-run of a
// pose window is one or two 32-bit loads + a funnel shift.
struct DevGrid {
    const uint32_t *bits;
    int X, Y, Z, Zw;
    double bmin[3], bmax[3];
    double res;
};

struct DevCfg {
    FlatParams fp;
    double vmax2, omgmax2, thetamax;
    double wv, wp, womg, wtheta;
    double mu;        // smoothingEps
    double safety;    // safety_hor
    double half_bd;   // kernel_size * occupancy_resolution / 2
    int K;            // integralIntervs
    int flags;
};

// growable device buffer (host-side helper)
template <typename T>
struct DevBuf {
    T *p = nullptr; size_t n = 0;
    cudaError_t ensure(size_t cnt) {
        if (cnt <= n) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; n = 0;
        cudaError_t e = cudaMalloc((void **)&p, cnt * sizeof(T));
        if (e == cudaSuccess) n = cnt;
        return e;
    }
    cudaError_t upload(const T *h, size_t cnt, cudaStream_t st) {
        cudaError_t e = ensure(cnt);
        if (e != cudaSuccess) return e;
        return cudaMemcpyAsync(p, h, cnt * sizeof(T), cudaMemcpyHostToDevice, st);
    }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

// function-local scratch buffer: released on EVERY exit path (the CU_TRY early returns of the query entry points included)
template <typename T>
struct ScopedDevBuf : DevBuf<T> {
    ScopedDevBuf() = default;
    ScopedDevBuf(const ScopedDevBuf &) = delete;
    ScopedDevBuf &operator=(const ScopedDevBuf &) = delete;
    ~ScopedDevBuf() { this->release(); }
};

constexpr int PARTIAL_STRIDE = 20;  // per sample / per point: 18 gradC entries (axis*6+k), gradT term, cost term

}  // namespace isdf
