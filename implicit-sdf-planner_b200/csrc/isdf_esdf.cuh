// Euclidean distance field of the occupancy map: GridMap3D::generateESDF3d (Gridmap3D.cpp:361-525) and its trilinear queries
// getSDFValue / getSDFValueWithGrad (GridMap3D.h:114-193). Included by isdf_api.cu, whose unit is compiled with -fmad=false: the
// queries are FP64 add / mul / div / sqrt only, so they round exactly like the reference's x86-64 build.
//
// The reference's field is the exact integer Euclidean distance transform: at every voxel grid_esdf = res * sqrt((double)d2), d2 the
// squared voxel distance to the nearest occupied voxel (grid_map_buffer_neg: to the nearest free voxel), res * sqrt(DBL_MAX) when the
// map has no such voxel. Its FP64 parabola envelope only ever holds exact integers below 2^53 or DBL_MAX, so any exact integer transform
// followed by res * sqrt((double)d2) gives the same bits. Here the transform is integer throughout (DESIGN §3.15):
//   pass z   k_esdf_z      one warp per (x, y) line of the bit grid: nearest set / clear bit along z by word-level clz / ffs, both fields
//   pass y   k_esdf_line   one thread per (x, z) line, lanes on consecutive z: Meijster's lower envelope with int64 comparisons, in place
//   pass x   k_esdf_line   one thread per (y, z) line, the same
// d2 is stored as uint32 (ESDF_NONE = no site); field values are formed only when read (k_esdf_expand, k_esdf_query).
#pragma once
#include "isdf_types.cuh"
#include "isdf_map.cuh"
#include <cfloat>

namespace isdf {

constexpr uint32_t ESDF_NONE = 0xffffffffu;   // no site in the line (after pass x: in the map)
// fillESDF computes q * q in int (Gridmap3D.cpp:537-544): beyond 46341 voxels on an axis the reference overflows. With this limit and
// X * Y * ceil(Z / 32) < 2^31 every d2 stays below 2^32 - 1 (the largest, 46341 x 31 x 46341, gives 2 * 46340^2 + 30^2 = 4 294 792 100),
// and every stack index and separator fits 16 bits.
constexpr int ESDF_AXIS_MAX = 46341;
enum { ESDF_POSITIVE = 0, ESDF_NEGATIVE = 1, ESDF_SIGNED = 2 };

// ---- pass z ------------------------------------------------------------------------------------------------------
// site bits of word w of a row: occupied voxels for the positive field, free voxels (bits below Z only) for the negative one
__device__ __forceinline__ uint32_t esdf_sites(const uint32_t *row, int w, int Zw, int Z, bool neg) {
    if (w >= Zw) return 0u;
    const uint32_t b = row[w];
    if (!neg) return b;
    const int rem = Z - 32 * w;
    return ~b & (rem >= 32 ? 0xffffffffu : ((1u << rem) - 1u));
}

// One warp per row, 32 words (1024 voxels) per chunk, lane = word. Per word: the last site before it (a forward max-scan with a carry
// across chunks) and the first site after it (a backward min-scan, with the first site past the chunk found by a look-ahead that is kept
// until the chunk end passes it, so a row is read at most twice). Then lane = voxel, one word of the chunk at a time: coalesced writes.
__global__ void __launch_bounds__(256) k_esdf_z(const uint32_t *bits, long long rows, int Z, int Zw, uint32_t *pos, uint32_t *neg) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += nwarps) {
        const uint32_t *row = bits + r * Zw;
        for (int f = 0; f < 2; f++) {
            uint32_t *out = (f ? neg : pos) + r * Z;
            int carry = -1;              // last site before the chunk (-1: none)
            int ahead = -1;              // first site past an earlier chunk (INT_MAX: none); -1: not looked up yet
            for (int w0 = 0; w0 < Zw; w0 += 32) {
                const int w = w0 + lane;
                const uint32_t s = esdf_sites(row, w, Zw, Z, f);
                const int last = s ? 32 * w + 31 - __clz(s) : -1;
                const int first = s ? 32 * w + __ffs(s) - 1 : INT_MAX;
                // exclusive scans within the chunk
                int L = last, R = first;
                for (int o = 1; o < 32; o <<= 1) {
                    const int l2 = __shfl_up_sync(0xffffffffu, L, o), r2 = __shfl_down_sync(0xffffffffu, R, o);
                    if (lane >= o) L = max(L, l2);
                    if (lane + o < 32) R = min(R, r2);
                }
                L = __shfl_up_sync(0xffffffffu, L, 1); R = __shfl_down_sync(0xffffffffu, R, 1);
                if (lane == 0) L = -1;
                if (lane == 31) R = INT_MAX;
                L = max(L, carry);
                const int chunk_end = 32 * (w0 + 32);   // first voxel past the chunk
                if (ahead != INT_MAX && ahead < chunk_end) {
                    ahead = INT_MAX;
                    for (int v0 = w0 + 32; v0 < Zw; v0 += 32) {
                        const uint32_t t = esdf_sites(row, v0 + lane, Zw, Z, f);
                        const unsigned any = __ballot_sync(0xffffffffu, t != 0u);
                        if (any) {
                            const int src = __ffs(any) - 1;
                            const uint32_t tw = __shfl_sync(0xffffffffu, t, src);
                            ahead = 32 * (v0 + src) + __ffs(tw) - 1;
                            break;
                        }
                    }
                }
                R = min(R, ahead);
                const int chunk_last = (int)__reduce_max_sync(0xffffffffu, (unsigned)(last + 1)) - 1;   // -1: no site in the chunk
                carry = max(carry, chunk_last);
                const int nw = min(32, Zw - w0);
                for (int j = 0; j < nw; j++) {
                    const uint32_t sj = __shfl_sync(0xffffffffu, s, j);
                    const int Lj = __shfl_sync(0xffffffffu, L, j), Rj = __shfl_sync(0xffffffffu, R, j);
                    const int z = 32 * (w0 + j) + lane;
                    if (z >= Z) continue;   // the row's last word only; no shuffle follows in this iteration
                    const uint32_t below = sj & (0xffffffffu >> (31 - lane)), above = sj & (0xffffffffu << lane);
                    const int left = below ? 32 * (w0 + j) + 31 - __clz(below) : Lj;
                    const int right = above ? 32 * (w0 + j) + __ffs(above) - 1 : Rj;
                    uint32_t d2 = ESDF_NONE;
                    if (left >= 0) d2 = (uint32_t)(z - left) * (uint32_t)(z - left);
                    if (right != INT_MAX) d2 = min(d2, (uint32_t)(right - z) * (uint32_t)(right - z));
                    out[z] = d2;
                }
            }
        }
    }
}

// ---- passes y and x -------------------------------------------------------------------------------------------
// Line l of field f (l < nlines) has m voxels at base + u * stride, base = (l / Z) * outer + l % Z: pass y takes outer = Y Z,
// stride = Z; pass x outer = Z, stride = Y Z. Consecutive threads take consecutive z, so every field access is coalesced.
// Meijster's envelope (exact integer separators, floor division) over the line's finite values, in place: the stack holds each
// envelope site's index, the first voxel it wins and its value, so the backward write needs nothing the forward pass overwrote.
// G threads (G <= nlines, so the stack, G * m entries of 8 bytes, is at most 8 bytes per voxel) take lines t, t + G, ... of both
// fields. Thread t's stack entry k lies at stack[k * G + t]: lanes at equal depth touch adjacent entries.
struct EsdfLines {
    uint32_t *f[2];
    long long nlines, outer, stride;
    int m, Z;
};

__global__ void __launch_bounds__(256) k_esdf_line(const EsdfLines P, long long G, uint2 *stack) {
    const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t0 >= G) return;
    uint2 *stk = stack + t0;
    const int m = P.m;
    for (long long l2 = t0; l2 < 2 * P.nlines; l2 += G) {
        const int f = l2 >= P.nlines;
        const long long l = l2 - (f ? P.nlines : 0);
        uint32_t *line = (f ? P.f[1] : P.f[0]) + (l / P.Z) * P.outer + (l % P.Z);
        int q = -1;
        int ts = 0, tt = 0;        // top of the stack: site, first voxel it wins
        uint32_t tg = 0;           //                   its value
        for (int u = 0; u < m; u++) {
            const uint32_t g = line[(long long)u * P.stride];
            if (g == ESDF_NONE) continue;
            // pop while the top site loses to u at the top's first voxel
            while (q >= 0) {
                const long long a = (long long)(tt - ts) * (tt - ts) + tg, b = (long long)(tt - u) * (tt - u) + g;
                if (a <= b) break;
                if (--q >= 0) { const uint2 e = stk[q * G]; ts = e.x & 0xffff; tt = e.x >> 16; tg = e.y; }
            }
            if (q < 0) {
                q = 0; ts = u; tt = 0; tg = g;
                stk[0] = make_uint2((uint32_t)u, g);
            } else {
                // u wins from w = 1 + floor((u^2 - s^2 + g(u) - g(s)) / (2 (u - s))) on
                const long long num = (long long)u * u - (long long)ts * ts + (long long)g - (long long)tg, den = 2ll * (u - ts);
                const long long w = 1 + (num >= 0 ? num / den : -((-num + den - 1) / den));
                if (w < m) {
                    q++; ts = u; tt = (int)w; tg = g;
                    stk[q * G] = make_uint2((uint32_t)u | ((uint32_t)w << 16), g);
                }
            }
        }
        if (q < 0) continue;        // no site: the line already holds ESDF_NONE everywhere
        for (int u = m - 1; u >= 0; u--) {
            line[(long long)u * P.stride] = (uint32_t)((unsigned long long)(u - ts) * (u - ts) + tg);
            if (u == tt && --q >= 0) { const uint2 e = stk[q * G]; ts = e.x & 0xffff; tt = e.x >> 16; tg = e.y; }
        }
    }
}

// ---- reading the field ----------------------------------------------------------------------------------------
// grid_resolution * std::sqrt(val) (Gridmap3D.cpp:397, 474), val = DBL_MAX where the reference's envelope saw no site
__device__ __forceinline__ double esdf_dist(uint32_t d2, double res) { return res * sqrt(d2 == ESDF_NONE ? DBL_MAX : (double)d2); }

// the value of one voxel of a field; SIGNED is the reference's combine step (Gridmap3D.cpp:513-522) with the positive distance where it
// adds grid_map (DESIGN §6)
__device__ __forceinline__ double esdf_value(const uint32_t *pos, const uint32_t *neg, int field, double res, long long i) {
    if (field == ESDF_POSITIVE) return esdf_dist(pos[i], res);
    if (field == ESDF_NEGATIVE) return esdf_dist(neg[i], res);
    double v = esdf_dist(pos[i], res);
    const double n = esdf_dist(neg[i], res);
    if (n > 0.0) v += (-n + res);
    return v;
}

__global__ void k_esdf_expand(const uint32_t *pos, const uint32_t *neg, int field, double res, long long i0, long long cnt, double *out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (long long)gridDim.x * blockDim.x)
        out[i] = esdf_value(pos, neg, field, res, i0 + i);
}

struct EsdfView {
    const uint32_t *pos, *neg;
    int X, Y, Z;
    double bmin[3], bmax[3], res;
};

// getSDFValue (grad == nullptr) / getSDFValueWithGrad (GridMap3D.h:114-193), operation for operation:
//   pos_m = pos_w - 0.5 * res; idx = getGridIndex(pos_m), (0, 0, 0) when pos_m is outside [bmin, bmax] (Gridmap3D.cpp:135-140);
//   diff = (pos_w - getGridCubeCenter(idx)) * (1 / res); corner values through getGridSDFValue(Vector3i), 0 past the top index
//   (the isInMap(getGridCubeCenter(...)) test before it is dead: its 0 is overwritten). A point with a non-finite coordinate gives NaN.
__global__ void k_esdf_query(const EsdfView V, int field, const double *pts, long long n, double *dist, double *grad) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const double p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
        if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) {
            const double nan = __longlong_as_double(0x7ff8000000000000ll);
            dist[i] = nan;
            if (grad) grad[3 * i] = grad[3 * i + 1] = grad[3 * i + 2] = nan;
            continue;
        }
        const double h = 0.5 * V.res;
        const double pm[3] = {p[0] - h, p[1] - h, p[2] - h};
        int idx[3] = {0, 0, 0};
        bool in = true;
        for (int a = 0; a < 3; a++) in = in && !(pm[a] < V.bmin[a]) && !(pm[a] > V.bmax[a]);
        if (in) {
            CloudFrame F;
            for (int a = 0; a < 3; a++) F.bmin[a] = V.bmin[a];
            F.res = V.res; F.X = V.X; F.Y = V.Y; F.Z = V.Z; F.Zw = 0;
            grid_index(F, pm[0], pm[1], pm[2], idx[0], idx[1], idx[2]);
        }
        const double inv = 1.0 / V.res;
        double diff[3];
        for (int a = 0; a < 3; a++) diff[a] = (p[a] - ((idx[a] + 0.5) * V.res + V.bmin[a])) * inv;
        double v[2][2][2];
        for (int x = 0; x < 2; x++)
            for (int y = 0; y < 2; y++)
                for (int z = 0; z < 2; z++) {
                    const int jx = idx[0] + x, jy = idx[1] + y, jz = idx[2] + z;
                    v[x][y][z] = (jx < V.X && jy < V.Y && jz < V.Z)
                                     ? esdf_value(V.pos, V.neg, field, V.res, ((long long)jx * V.Y + jy) * V.Z + jz) : 0.0;
                }
        const double v00 = (1 - diff[0]) * v[0][0][0] + diff[0] * v[1][0][0];
        const double v01 = (1 - diff[0]) * v[0][0][1] + diff[0] * v[1][0][1];
        const double v10 = (1 - diff[0]) * v[0][1][0] + diff[0] * v[1][1][0];
        const double v11 = (1 - diff[0]) * v[0][1][1] + diff[0] * v[1][1][1];
        const double v0 = (1 - diff[1]) * v00 + diff[1] * v10;
        const double v1 = (1 - diff[1]) * v01 + diff[1] * v11;
        dist[i] = (1 - diff[2]) * v0 + diff[2] * v1;
        if (grad) {
            const double g2 = (v1 - v0) * inv;
            const double g1 = ((1 - diff[2]) * (v10 - v00) + diff[2] * (v11 - v01)) * inv;
            double g0 = (1 - diff[2]) * (1 - diff[1]) * (v[1][0][0] - v[0][0][0]);
            g0 += (1 - diff[2]) * diff[1] * (v[1][1][0] - v[0][1][0]);
            g0 += diff[2] * (1 - diff[1]) * (v[1][0][1] - v[0][0][1]);
            g0 += diff[2] * diff[1] * (v[1][1][1] - v[0][1][1]);
            g0 *= inv;
            grad[3 * i] = g0; grad[3 * i + 1] = g1; grad[3 * i + 2] = g2;
        }
    }
}

}  // namespace isdf
