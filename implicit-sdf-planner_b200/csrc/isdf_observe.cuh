// Known space (include/isdf.h, DESIGN §3.22): which voxels a depth image has proven empty, the boxes a caller asserts are free, and the
// blocked grid (occupied | not known) the clearance family reads under ISDF_UNKNOWN_OCCUPIED.
//   k_obs_mip     : one level of each image's min-mip (cell (i, j) of level l: the minimum over the 2 x 2 cells below it, clipped)
//   k_obs_voxels  : one thread per (pose, voxel) of the map inside the pose's horizon box: the four-part rule, atomicOr into the known bits
//   k_known_boxes : one thread per voxel of a box's index range: its cube inside the box
//   k_blocked     : one thread per word: occ | (~known & the row's valid bits)
// Compiled only into isdf_sense_tu.cu with -fmad=false, so that the FP64 corner arithmetic rounds operation by operation and a numpy
// restatement (tests/observe_oracle.py) reproduces every decision.
#pragma once
#include "isdf_sense.cuh"

namespace isdf {

// the padded closed cube of voxel index i on one axis (include/isdf.h: known space)
__device__ __forceinline__ void voxel_span(double bmin, double res, int i, double &lo, double &hi) {
    const double pad = 1e-12 * (fabs(bmin) + (double)(i + 1) * res);
    lo = (bmin + (double)i * res) - pad;
    hi = (bmin + (double)(i + 1) * res) + pad;
}

__global__ void __launch_bounds__(256) k_obs_mip(const int32_t *src, int sw, int sh, int32_t *dst, int dw, int dh, int P) {
    const long long n = (long long)P * dw * dh, ssz = (long long)sw * sh, dsz = (long long)dw * dh;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(t / dsz);
        const long long k = t - p * dsz;
        const int j = (int)(k / dw), i = (int)(k - (long long)j * dw);
        const int32_t *s = src + p * ssz;
        int m = s[(long long)(2 * j) * sw + 2 * i];
        if (2 * i + 1 < sw) m = min(m, s[(long long)(2 * j) * sw + 2 * i + 1]);
        if (2 * j + 1 < sh) {
            m = min(m, s[(long long)(2 * j + 1) * sw + 2 * i]);
            if (2 * i + 1 < sw) m = min(m, s[(long long)(2 * j + 1) * sw + 2 * i + 1]);
        }
        dst[t] = m;
    }
}

constexpr int OBS_LEVELS = 32;
struct ObsArgs {
    const SensePose *poses; int P;
    const int32_t *img, *mip;              // level 0: the chunk's images; levels >= 1: the mip, level l of image p at off[l] + p w[l] h[l]
    long long off[OBS_LEVELS]; int w[OBS_LEVELS], h[OBS_LEVELS]; int nlev;
    double bmin[3], res; int X, Y, Z, Zw;
    int D;                                 // voxels per axis of a pose's horizon box
    double horizon, fx, fy, cx, cy;        // fx .. cy: the render's FP32 parameters
    uint32_t *known;
    unsigned long long *cnt;               // {voxels tested, voxels added}
};

// rules 2, 1 and 3 for voxel (ix, iy, iz) seen from pose P (include/isdf.h), operation order as written there; shared by isdf_map_observe
// and isdf_view_gain. fx .. cy: the render's FP32 parameters. On success the pixel rectangle x0 .. x1, y0 .. y1, the corners' largest camera
// depth zmax and the depth margin e2 (E_2) that rule 4 needs.
struct ObsView { int x0, x1, y0, y1; double zmax, e2; };
__device__ __forceinline__ bool obs_in_view(const double bmin[3], double res, double horizon, double fx, double fy, double cx, double cy, int W,
                                            int H, const SensePose &P, int ix, int iy, int iz, ObsView &o) {
    double lo[3], hi[3];
    voxel_span(bmin[0], res, ix, lo[0], hi[0]);
    voxel_span(bmin[1], res, iy, lo[1], hi[1]);
    voxel_span(bmin[2], res, iz, lo[2], hi[2]);
    // 2. every corner within the horizon of the body position
    for (int k = 0; k < 8; k++) {
        const double d0 = ((k & 1) ? hi[0] : lo[0]) - P.body[0], d1 = ((k & 2) ? hi[1] : lo[1]) - P.body[1], d2 = ((k & 4) ? hi[2] : lo[2]) - P.body[2];
        if (!(sqrt((d0 * d0 + d1 * d1) + d2 * d2) <= horizon)) return false;
    }
    double M = 0.0;
    for (int a = 0; a < 3; a++) M = fmax(M, fmax(fabs(lo[a]), fabs(hi[a])));
    double E[3];
    for (int i = 0; i < 3; i++) {
        const double r0 = P.r[3 * i], r1 = P.r[3 * i + 1], r2 = P.r[3 * i + 2];
        E[i] = 1e-6 * (((fabs(r0) + fabs(r1)) + fabs(r2)) * M + fabs((double)P.t[i])) + 1e-30;
        if (!(E[i] < 1e24)) return false;
    }
    // camera coordinates of the corners: ((r0 x + r1 y) + r2 z) + t
    double zmin = INFINITY, zmax = -INFINITY, umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY, a = 0.0, b = 0.0;
    double cz[8], cx8[8], cy8[8];
    for (int k = 0; k < 8; k++) {
        const double X = (k & 1) ? hi[0] : lo[0], Y = (k & 2) ? hi[1] : lo[1], Zc = (k & 4) ? hi[2] : lo[2];
        double c[3];
        for (int i = 0; i < 3; i++) c[i] = (((double)P.r[3 * i] * X + (double)P.r[3 * i + 1] * Y) + (double)P.r[3 * i + 2] * Zc) + (double)P.t[i];
        cx8[k] = c[0]; cy8[k] = c[1]; cz[k] = c[2];
        zmin = fmin(zmin, c[2]); zmax = fmax(zmax, c[2]);
    }
    // 1. in front of the camera by the transform's margin
    if (!(zmin > E[2])) return false;
    for (int k = 0; k < 8; k++) {
        const double qx = cx8[k] / cz[k], qy = cy8[k] / cz[k];
        const double u = qx * fx + cx, v = qy * fy + cy;
        umin = fmin(umin, u); umax = fmax(umax, u); vmin = fmin(vmin, v); vmax = fmax(vmax, v);
        a = fmax(a, fabs(qx)); b = fmax(b, fabs(qy));
    }
    // 3. the pixel rectangle, widened by the projection's rounding, inside the image
    const double zl = zmin - E[2];
    const double dqx = (E[0] + a * E[2]) / zl, dqy = (E[1] + b * E[2]) / zl;
    const double eu = (fx * dqx + 1.2e-7 * ((a + dqx) * fx + fabs(cx))) + 1e-9 * (1.0 + (a * fx + fabs(cx)));
    const double ev = (fy * dqy + 1.2e-7 * ((b + dqy) * fy + fabs(cy))) + 1e-9 * (1.0 + (b * fy + fabs(cy)));
    const double fx0 = floor((umin - eu) + 0.5), fx1 = floor((umax + eu) + 0.5);
    const double fy0 = floor((vmin - ev) + 0.5), fy1 = floor((vmax + ev) + 0.5);
    if (!(fx0 >= 0.0 && fx1 <= (double)(W - 1) && fy0 >= 0.0 && fy1 <= (double)(H - 1))) return false;
    o.x0 = (int)fx0; o.x1 = (int)fx1; o.y0 = (int)fy0; o.y1 = (int)fy1;
    o.zmax = zmax; o.e2 = E[2];
    return true;
}

// the four-part rule for voxel (ix, iy, iz) and pose P (include/isdf.h): rules 2, 1, 3, then 4 on the image's min-mip
__device__ bool obs_voxel(const ObsArgs &A, const SensePose &P, int p, int ix, int iy, int iz) {
    ObsView o;
    if (!obs_in_view(A.bmin, A.res, A.horizon, A.fx, A.fy, A.cx, A.cy, A.w[0], A.h[0], P, ix, iy, iz, o)) return false;
    const int x0 = o.x0, x1 = o.x1, y0 = o.y0, y1 = o.y1;
    // 4. the rectangle's minimum depth (from the mip) beyond the corners' depth plus dist_mm's rounding and the transform's error
    int l = 0;
    while ((x1 >> l) - (x0 >> l) > 1 || (y1 >> l) - (y0 >> l) > 1) l++;
    const int i0 = x0 >> l, i1 = x1 >> l, j0 = y0 >> l, j1 = y1 >> l, w = A.w[l];
    const int32_t *m = l == 0 ? A.img + (long long)p * w * A.h[0] : A.mip + A.off[l] + (long long)p * w * A.h[l];
    const int dmin = min(min(m[(long long)j0 * w + i0], m[(long long)j0 * w + i1]), min(m[(long long)j1 * w + i0], m[(long long)j1 * w + i1]));
    const double d = (1000.0 * o.e2 + 0.5) + 1.2e-7 * (1000.0 * (o.zmax + o.e2) + 1.0);
    return (double)dmin > 1000.0 * o.zmax + d;
}

__device__ __forceinline__ void warp_add(unsigned long long *cnt, unsigned long long v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(cnt, v);
}

// the first voxel index of pose P's horizon box on axis a (one voxel of slack on each side; every voxel the rule can mark lies inside)
__device__ __forceinline__ int obs_box_lo(const ObsArgs &A, const SensePose &P, int a) {
    return (int)fmax(-2147483000.0, fmin(2147483000.0, floor(((P.body[a] - A.horizon) - A.bmin[a]) / A.res) - 1.0));
}

__global__ void __launch_bounds__(256) k_obs_voxels(const ObsArgs A) {
    const long long D = A.D, D3 = D * D * D, n = (long long)A.P * D3;
    const long long stride = (long long)gridDim.x * blockDim.x;
    unsigned long long tested = 0, added = 0;
    // trip count warp-uniform, so that every lane takes part in the reductions
    for (long long base = blockIdx.x * (long long)blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
        const long long t = base + (threadIdx.x & 31);
        if (t >= n) continue;
        const int p = (int)(t / D3);
        const long long k = t - p * D3;
        const SensePose &P = A.poses[p];
        const int ix = obs_box_lo(A, P, 0) + (int)(k / (D * D)), iy = obs_box_lo(A, P, 1) + (int)((k / D) % D), iz = obs_box_lo(A, P, 2) + (int)(k % D);
        if (ix < 0 || ix >= A.X || iy < 0 || iy >= A.Y || iz < 0 || iz >= A.Z) continue;
        tested++;
        if (!obs_voxel(A, P, p, ix, iy, iz)) continue;
        uint32_t *word = A.known + ((long long)ix * A.Y + iy) * A.Zw + (iz >> 5);
        const uint32_t bit = 1u << (iz & 31);
        if (!(*word & bit) && !(atomicOr(word, bit) & bit)) added++;   // bits only grow: a stale read only costs the atomic
    }
    warp_add(A.cnt, tested);
    warp_add(A.cnt + 1, added);
}

// voxels whose cube (unpadded: bmin + i res .. bmin + (i + 1) res) lies inside the closed box [lo, hi], over the index range i0 + [0, n)
// (the host's loose bound)
__global__ void __launch_bounds__(256) k_known_boxes(DevGrid G, uint32_t *known, double lx, double ly, double lz, double hx, double hy, double hz,
                                                     int i0x, int i0y, int i0z, int nx, int ny, int nz) {
    const long long n = (long long)nx * ny * nz;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const int ix = i0x + (int)(t / ((long long)ny * nz)), iy = i0y + (int)((t / nz) % ny), iz = i0z + (int)(t % nz);
        const int id[3] = {ix, iy, iz};
        double lo[3], hi[3];
        for (int a = 0; a < 3; a++) { lo[a] = G.bmin[a] + (double)id[a] * G.res; hi[a] = G.bmin[a] + (double)(id[a] + 1) * G.res; }
        if (lo[0] >= lx && hi[0] <= hx && lo[1] >= ly && hi[1] <= hy && lo[2] >= lz && hi[2] <= hz)
            atomicOr(known + ((long long)ix * G.Y + iy) * G.Zw + (iz >> 5), 1u << (iz & 31));
    }
}

// blocked = occ | (~known & valid bits); known NULL: nothing known
__global__ void __launch_bounds__(256) k_blocked(const uint32_t *occ, const uint32_t *known, uint32_t *out, long long nwords, int Z, int Zw) {
    const int tail = Z & 31;
    const uint32_t last = tail ? (1u << tail) - 1u : 0xffffffffu;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nwords; i += (long long)gridDim.x * blockDim.x) {
        const uint32_t valid = (int)(i % Zw) == Zw - 1 ? last : 0xffffffffu;
        out[i] = occ[i] | (~(known ? known[i] : 0u) & valid);
    }
}

}  // namespace isdf
