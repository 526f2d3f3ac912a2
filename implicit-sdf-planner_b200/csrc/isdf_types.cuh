// Device-visible parameter blocks shared by the kernels and the C-ABI layer.
#pragma once
#include "isdf_math.cuh"
#include "isdf_shapes.cuh"
#include <utility>

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

// Growable buffer (host-side helper) that owns its allocation: device memory (DevBuf) or pinned host memory (PinnedBuf, staging for
// one-copy transfers). ensure / upload only grow, and growing discards the contents. Move-only; `buf = {}` frees it.
template <typename T, bool PINNED>
struct OwnedBuf {
    T *p = nullptr; size_t n = 0;
    OwnedBuf() = default;
    OwnedBuf(OwnedBuf &&o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
    OwnedBuf &operator=(OwnedBuf &&o) noexcept { std::swap(p, o.p); std::swap(n, o.n); return *this; }
    ~OwnedBuf() { if (p) PINNED ? cudaFreeHost(p) : cudaFree(p); }
    cudaError_t ensure(size_t cnt) {
        if (cnt <= n) return cudaSuccess;
        *this = OwnedBuf();
        cudaError_t e = PINNED ? cudaMallocHost((void **)&p, cnt * sizeof(T)) : cudaMalloc((void **)&p, cnt * sizeof(T));
        if (e == cudaSuccess) n = cnt;
        return e;
    }
    cudaError_t upload(const T *h, size_t cnt, cudaStream_t st) {
        cudaError_t e = ensure(cnt);
        if (e != cudaSuccess) return e;
        return cudaMemcpyAsync(p, h, cnt * sizeof(T), cudaMemcpyHostToDevice, st);
    }
};
template <typename T> using DevBuf = OwnedBuf<T, false>;
template <typename T> using PinnedBuf = OwnedBuf<T, true>;

constexpr int PARTIAL_STRIDE = 20;  // per sample / per point: 18 gradC entries (axis*6+k), gradT term, cost term

}  // namespace isdf
