// Occupancy-map kernels: packing a dense grid into the bit grid (DevGrid), building it from a point cloud (the reference's
// PCSmapManager::rcvGlobalMapHandler, PCSmap_manager.cpp:111-181) and reading it back. Included by isdf_api.cu, whose unit is compiled
// with -fmad=false: the cloud index below is FP64 subtraction and IEEE division only, so it rounds exactly like the reference's x86-64 build.
#pragma once
#include "isdf_types.cuh"

namespace isdf {

// ---- dense grid -> bits ------------------------------------------------------------------------------------------
// sources of k_pack_bits: "voxel i is occupied"
template <typename T>
struct NonZero {
    const T *p;
    __device__ __forceinline__ bool operator()(size_t i) const { return p[i] != (T)0; }
};
struct CountAtLeast {   // point counts of the cloud path, sta_threshold > 1
    const uint32_t *cnt;
    uint32_t thr;
    __device__ __forceinline__ bool operator()(size_t i) const { return cnt[i] >= thr; }
};
struct AllSet {         // sta_threshold <= 0: count >= threshold holds for every voxel
    __device__ __forceinline__ bool operator()(size_t) const { return true; }
};

template <typename Src>
__global__ void k_pack_bits(const Src src, uint32_t *bits, int rows, int Z, int Zw) {
    // one warp per 32-voxel word: ballot of "voxel occupied"; bits past Z in a row's last word stay 0
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long nwords = (long long)rows * Zw;
    if (gw >= nwords) return;
    const int row = (int)(gw / Zw), w = (int)(gw - (long long)row * Zw);
    const int z = w * 32 + lane;
    const bool o = (z < Z) && src((size_t)row * Z + z);
    const unsigned b = __ballot_sync(0xffffffffu, o);
    if (lane == 0) bits[gw] = b;
}

// ---- bits -> dense grid (readback), rows [row0, row0 + nrows) of X*Y ------------------------------------------
template <typename T>
__global__ void k_unpack_bits(const uint32_t *bits, T *out, long long row0, int nrows, int Z, int Zw) {
    const long long total = (long long)nrows * Z;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / Z;
        const int z = (int)(i - r * Z);
        out[i] = (T)((bits[(row0 + r) * Zw + (z >> 5)] >> (z & 31)) & 1u);
    }
}

// popcount of the bit grid (padding bits are 0); an integer sum, so the same in any order
__global__ void k_popcount(const uint32_t *bits, long long nwords, unsigned long long *out) {
    unsigned long long s = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (long long)gridDim.x * blockDim.x) s += __popc(bits[i]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// ---- point cloud -> bits ---------------------------------------------------------------------------------------
// float -> uint32 preserving order (negative floats reversed below the positives), so integer min / max give the float extrema
__host__ __device__ __forceinline__ uint32_t float_to_ordered(uint32_t u) { return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__host__ __device__ __forceinline__ uint32_t ordered_to_float(uint32_t o) { return (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o; }

// record i of a cloud: x, y, z float32 at byte offsets 0, 4, 8; false if any coordinate is NaN or Inf
__device__ __forceinline__ bool cloud_point(const char *pts, long long i, int stride, float &x, float &y, float &z) {
    const float *p = reinterpret_cast<const float *>(pts + i * (long long)stride);
    x = __ldg(p); y = __ldg(p + 1); z = __ldg(p + 2);
    return isfinite(x) && isfinite(y) && isfinite(z);
}

// ext[0..2] = ordered min of x, y, z; ext[3..5] = ordered max; ext[6] = records skipped (non-finite). n < 2^32, so ext[6] cannot wrap.
__global__ void __launch_bounds__(256) k_cloud_bounds(const char *pts, long long n, int stride, uint32_t *ext) {
    uint32_t mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u}, skipped = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float c[3];
        if (!cloud_point(pts, i, stride, c[0], c[1], c[2])) { skipped++; continue; }
        for (int a = 0; a < 3; a++) {
            const uint32_t o = float_to_ordered(__float_as_uint(c[a]));
            mn[a] = min(mn[a], o); mx[a] = max(mx[a], o);
        }
    }
    for (int a = 0; a < 3; a++) { mn[a] = __reduce_min_sync(0xffffffffu, mn[a]); mx[a] = __reduce_max_sync(0xffffffffu, mx[a]); }
    skipped = __reduce_add_sync(0xffffffffu, skipped);
    __shared__ uint32_t s[7];
    if (threadIdx.x < 7) s[threadIdx.x] = threadIdx.x < 3 ? 0xffffffffu : 0u;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
        for (int a = 0; a < 3; a++) { atomicMin(&s[a], mn[a]); atomicMax(&s[3 + a], mx[a]); }
        if (skipped) atomicAdd(&s[6], skipped);
    }
    __syncthreads();
    if (threadIdx.x < 3) atomicMin(&ext[threadIdx.x], s[threadIdx.x]);
    else if (threadIdx.x < 6) atomicMax(&ext[threadIdx.x], s[threadIdx.x]);
    else if (threadIdx.x == 6 && s[6]) atomicAdd(&ext[6], s[6]);
}

struct CloudFrame {
    double bmin[3], bmax[3], res;
    int X, Y, Z, Zw;
};

// GridMap3D::getGridIndex (Gridmap3D.cpp:135-175) for a point inside the bounds (the caller has checked isInMap), with its clamps as
// written: "iy < 0" and "iz < 0" reset ix, not iy / iz (quirk Q6; unreachable since every coordinate is >= bmin). The cloud path and the
// ESDF queries (isdf_esdf.cuh) share it.
__device__ __forceinline__ void grid_index(const CloudFrame &F, double x, double y, double z, int &ix, int &iy, int &iz) {
    const double dx = x - F.bmin[0], dy = y - F.bmin[1], dz = z - F.bmin[2];
    ix = (int)floor(dx / F.res); iy = (int)floor(dy / F.res); iz = (int)floor(dz / F.res);
    if (ix < 0) ix = 0;
    if (ix >= F.X) ix = F.X - 1;
    if (iy < 0) ix = 0;
    if (iy >= F.Y) iy = F.Y - 1;
    if (iz < 0) ix = 0;
    if (iz >= F.Z) iz = F.Z - 1;
}
// a cloud record (isInMap holds for every finite record)
__device__ __forceinline__ void cloud_index(const CloudFrame &F, float x, float y, float z, int &ix, int &iy, int &iz) {
    grid_index(F, (double)x, (double)y, (double)z, ix, iy, iz);
}

// sta_threshold == 1: set the voxel's bit directly, for the finite records inside [bmin, bmax] (isInMap; every finite record of the cloud
// that set the frame is inside it). Lanes of a warp that hit the same 32-bit word (neighbouring records of a spatially coherent cloud) OR
// their bits together first (__match_any_sync), and the group's leader skips the atomic when a plain load already shows every bit set. The
// loop trip count is warp-uniform so that every lane takes part in the match. cnt (may be NULL): {inside, outside, non-finite, bits this
// launch set}; each bit's 0 -> 1 transition is seen by exactly one atomicOr, so the last count is exact in any order.
enum { FUSE_USED, FUSE_OUTSIDE, FUSE_SKIPPED, FUSE_ADDED };
__global__ void __launch_bounds__(256) k_cloud_mark(const char *pts, long long n, int stride, const CloudFrame F, uint32_t *bits,
                                                    unsigned long long *cnt) {
    __shared__ uint32_t sbit[256];
    const int lane = threadIdx.x & 31;
    uint32_t *wbit = sbit + (threadIdx.x & ~31);
    const long long wstride = (long long)gridDim.x * blockDim.x;
    unsigned long long c[4] = {0, 0, 0, 0};
    for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += wstride) {
        const long long i = base + lane;
        uint32_t word = 0xffffffffu, bit = 0;   // X*Y*Zw < 2^31 words, so 0xffffffff names no word
        float x, y, z;
        if (i < n) {
            if (!cloud_point(pts, i, stride, x, y, z)) c[FUSE_SKIPPED]++;
            else if (!((double)x >= F.bmin[0] && (double)x <= F.bmax[0] && (double)y >= F.bmin[1] && (double)y <= F.bmax[1] &&
                       (double)z >= F.bmin[2] && (double)z <= F.bmax[2])) c[FUSE_OUTSIDE]++;
            else {
                int ix, iy, iz;
                cloud_index(F, x, y, z, ix, iy, iz);
                word = (uint32_t)(((long long)ix * F.Y + iy) * F.Zw + (iz >> 5));
                bit = 1u << (iz & 31);
                c[FUSE_USED]++;
            }
        }
        const unsigned peers = __match_any_sync(0xffffffffu, word);
        wbit[lane] = bit;
        __syncwarp();
        if (word != 0xffffffffu && lane == __ffs(peers) - 1) {
            uint32_t acc = 0;
            for (unsigned m = peers; m; m &= m - 1) acc |= wbit[__ffs(m) - 1];
            if ((bits[word] & acc) != acc) c[FUSE_ADDED] += __popc(acc & ~atomicOr(&bits[word], acc));
        }
        __syncwarp();
    }
    if (!cnt) return;
    for (int k = 0; k < 4; k++) {
        unsigned long long v = c[k];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && v) atomicAdd(&cnt[k], v);
    }
}

// sta_threshold > 1: per-voxel point counts (n < 2^32 records, so a count cannot wrap)
__global__ void __launch_bounds__(256) k_cloud_count(const char *pts, long long n, int stride, const CloudFrame F, uint32_t *cnt) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float x, y, z;
        if (!cloud_point(pts, i, stride, x, y, z)) continue;
        int ix, iy, iz;
        cloud_index(F, x, y, z, ix, iy, iz);
        atomicAdd(&cnt[((size_t)ix * F.Y + iy) * F.Z + iz], 1u);
    }
}

}  // namespace isdf
