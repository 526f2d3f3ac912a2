// View gain (include/isdf.h, DESIGN §3.25): how many unknown voxels a rig of cameras would observe from a pose.
//   k_sense_poses : per (camera, pose), the render's camera-from-world (isdf_sense.cuh), camera c of pose p at c P + p
//   k_view_gain   : grid (CTAs per pose, poses): every CTA's voxels belong to one pose's horizon box; per voxel, cheapest test first: in the
//                   map, neither occupied nor known (two bit reads), in view of some camera (rules 2, 1, 3 of isdf_map_observe through
//                   obs_in_view), then the integer line from the pose's voxel over the occupancy words. One integer atomicAdd per CTA.
// Compiled only into isdf_sense_tu.cu with -fmad=false, so that the in-view decisions are isdf_map_observe's to the bit.
#pragma once
#include "isdf_observe.cuh"

namespace isdf {

struct ViewArgs {
    const SensePose *poses; int P, ncam;   // P poses of the chunk, ncam cameras: pose p of camera c at poses[c P + p]
    const ViewCam *cams;                   // ncam: each camera's horizon, FP32-rounded intrinsics and image size
    const uint8_t *want;                   // P (may be NULL: all): poses with want[p] == 0 are skipped (their gain left as it is)
    double bmin[3], res; int X, Y, Z, Zw;
    int D;                                 // voxels per axis of a pose's box, from the largest horizon
    double hmax;
    const uint32_t *occ, *known;           // known NULL: nothing known
    unsigned long long *gain;              // P: the chunk's counts (added to)
};

__device__ __forceinline__ bool view_bit(const uint32_t *g, const ViewArgs &A, int x, int y, int z) {
    return (__ldg(g + ((long long)x * A.Y + y) * A.Zw + (z >> 5)) >> (z & 31)) & 1u;
}
__device__ __forceinline__ int view_floordiv(int a, int b) {   // b > 0
    const int q = a / b;
    return (a % b < 0) ? q - 1 : q;
}
__device__ __forceinline__ int view_index(double x, double bmin, double res) {
    return (int)fmax(-2147483000.0, fmin(2147483000.0, floor((x - bmin) / res)));
}

// (c): no occupied voxel strictly between the pose's voxel s and v on the integer line s + floor((2 k d + m) / (2 m)), k = 1 .. m - 1
__device__ bool view_line_clear(const ViewArgs &A, const int s[3], int ix, int iy, int iz) {
    const int d0 = ix - s[0], d1 = iy - s[1], d2 = iz - s[2];
    const int m = max(max(abs(d0), abs(d1)), abs(d2));
    for (int k = 1; k < m; k++) {
        const int x = s[0] + view_floordiv(2 * k * d0 + m, 2 * m), y = s[1] + view_floordiv(2 * k * d1 + m, 2 * m),
                  z = s[2] + view_floordiv(2 * k * d2 + m, 2 * m);
        if (x < 0 || x >= A.X || y < 0 || y >= A.Y || z < 0 || z >= A.Z) continue;   // outside the map: free
        if (view_bit(A.occ, A, x, y, z)) return false;
    }
    return true;
}

__global__ void __launch_bounds__(256) k_view_gain(const __grid_constant__ ViewArgs A) {
    __shared__ unsigned long long part[8];
    const int p = blockIdx.y;
    if (A.want && !A.want[p]) return;   // uniform over the CTA
    const SensePose &P0 = A.poses[p];
    int lo[3], s[3];
    for (int a = 0; a < 3; a++) {
        lo[a] = (int)fmax(-2147483000.0, fmin(2147483000.0, floor(((P0.body[a] - A.hmax) - A.bmin[a]) / A.res) - 1.0));
        s[a] = view_index(P0.body[a], A.bmin[a], A.res);
    }
    const long long D = A.D, D3 = D * D * D;
    unsigned long long cnt = 0;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < D3; t += (long long)gridDim.x * blockDim.x) {
        const int ix = lo[0] + (int)(t / (D * D)), iy = lo[1] + (int)((t / D) % D), iz = lo[2] + (int)(t % D);
        if (ix < 0 || ix >= A.X || iy < 0 || iy >= A.Y || iz < 0 || iz >= A.Z) continue;
        if (view_bit(A.occ, A, ix, iy, iz) || (A.known && view_bit(A.known, A, ix, iy, iz))) continue;
        bool seen = false;
        for (int c = 0; c < A.ncam && !seen; c++) {
            const ViewCam &K = A.cams[c];
            ObsView o;
            seen = obs_in_view(A.bmin, A.res, K.horizon, K.fx, K.fy, K.cx, K.cy, K.w, K.h, A.poses[(long long)c * A.P + p], ix, iy, iz, o);
        }
        if (seen && view_line_clear(A, s, ix, iy, iz)) cnt++;
    }
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long sum = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) sum += part[w];
        if (sum) atomicAdd(A.gain + p, sum);
    }
}

}  // namespace isdf
