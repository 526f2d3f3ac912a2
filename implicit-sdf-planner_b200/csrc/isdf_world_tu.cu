// Translation unit of the world generators (isdf_world.cuh): the host programs of globalmap_gene's maps, mockamap's draws and permutation,
// and the emission, Perlin selection and box kernels. Compiled with -fmad=false, so the FP64 coordinate and noise arithmetic rounds
// operation by operation as the reference's g++ build.
#include "isdf_world.cuh"
#include <cub/block/block_scan.cuh>
#include <cub/block/block_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <random>

namespace isdf {
namespace {

constexpr long long LOOP_CAP = 1ll << 31;            // steps of one reference loop
constexpr long long POINT_CAP = 1ll << 59;           // 16-byte records below 2^63 bytes
constexpr int TILE_THREADS = 256, TILE_ITEMS = 16, TILE = TILE_THREADS * TILE_ITEMS;

// ================================================= globalmap_gene: the host walk ==================================================
// Walks mapGene(map_id) as the reference runs it, recording each wall and road as a segment (its lists and its stream offset) instead of
// its points, and drawing on the host only the values that steer the program (map 2's trees, the cubes of maps 4 and 11).
struct Walker {
    WorldPlan &P;
    const double res;
    std::string err;
    int stream = 0;
    unsigned long long draw = 0;   // draws taken from the current stream
    long long points = 0;
    uint32_t win[GLIBC_DEG] = {}; unsigned long long win_at = ~0ull; int win_stream = -1;

    Walker(WorldPlan &P_, double res_) : P(P_), res(res_) {}

    int rand() {
        if (win_stream != stream || draw < win_at || draw >= win_at + GLIBC_DEG) {
            glibc_window(P.base.data() + GLIBC_DEG * stream, P.tab.data(), draw, win);
            win_at = draw; win_stream = stream;
        }
        return (int)(win[draw++ - win_at] >> 1);
    }
    void srand() { stream = 1; draw = 0; }

    // for (t = start; t < end; t += res): the list of t, appended to the coordinates; its offset, or -1 (err set)
    int list(double start, double end, int *count) {
        const double est = (end - start) / res;
        if (!(est < (double)LOOP_CAP)) { err = "a generator loop would take more than 2^31 steps"; return -1; }
        const int off = (int)P.coord.size();
        long long c = 0;
        for (double t = start; t < end; t += res) {
            if (++c >= LOOP_CAP) { err = "a generator loop would take more than 2^31 steps"; return -1; }
            P.coord.push_back(t);
        }
        *count = (int)c;
        return off;
    }
    bool add(WorldSeg s) {
        if (!err.empty()) return false;
        if (P.coord.size() >= (size_t)INT32_MAX) { err = "coordinate lists beyond 2^31 entries"; return false; }
        s.npts = (long long)s.n[0] * s.n[1];
        if (s.n[2] && s.npts > POINT_CAP / s.n[2]) { err = "the cloud would exceed 2^63 bytes"; return false; }
        s.npts *= s.n[2];
        if (points > POINT_CAP - s.npts) { err = "the cloud would exceed 2^63 bytes"; return false; }
        s.point0 = points; s.stream = stream; s.draw0 = draw;
        points += s.npts;
        if (s.kind != WSEG_POINT) draw += 3ull * (unsigned long long)s.npts;
        if (s.npts) P.seg.push_back(s);
        return true;
    }
    // geneWall(ori_x, ori_y, length, width, height): t_z from 0
    void wall(double ox, double oy, double l, double w, double h) { wall_z(ox, oy, 0.0, h, l, w); }
    // geneWall(ori_x, ori_y, ori_z, length, width, height)
    void wall(double ox, double oy, double oz, double l, double w, double h) { wall_z(ox, oy, oz, h + oz, l, w); }
    void wall_z(double ox, double oy, double z0, double z1, double l, double w) {
        if (!err.empty()) return;
        WorldSeg s{}; s.kind = WSEG_WALL;
        if ((s.off[0] = list(z0, z1, &s.n[0])) < 0) return;
        if ((s.off[1] = list(oy, oy + w, &s.n[1])) < 0) return;
        if ((s.off[2] = list(ox, ox + l, &s.n[2])) < 0) return;
        add(s);
    }
    // geneRoad(start, end, width): Eigen's norm as sqrt((x^2 + y^2) + z^2) and normalize as division by the same square root
    void road(const double sp[3], const double ep[3], double width) {
        if (!err.empty()) return;
        const double dir[3] = {ep[0] - sp[0], ep[1] - sp[1], ep[2] - sp[2]};
        const double length = std::sqrt((dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2]);
        const double t_step = res / length, k_step = res / width;
        double ex[3] = {-dir[1], dir[0], 0};
        const double en = std::sqrt((ex[0] * ex[0] + ex[1] * ex[1]) + ex[2] * ex[2]);
        if (en > 0) for (double &e : ex) e /= en;
        for (double &e : ex) e *= width;
        WorldSeg s{}; s.kind = WSEG_ROAD; s.n[0] = 1;
        s.off[1] = (int)P.coord.size();
        long long c = 0;
        if (!(1.0 / t_step < (double)LOOP_CAP) || !(1.0 / k_step < (double)LOOP_CAP)) { err = "a generator loop would take more than 2^31 steps"; return; }
        for (double t = 0; t <= 1; t += t_step) {
            if (++c >= LOOP_CAP) { err = "a generator loop would take more than 2^31 steps"; return; }
            for (int a = 0; a < 3; a++) P.coord.push_back(sp[a] + t * dir[a]);
        }
        s.n[1] = (int)c;
        s.off[2] = (int)P.coord.size(); c = 0;
        for (double k = -0.5; k <= 0.5; k += k_step) {
            if (++c >= LOOP_CAP) { err = "a generator loop would take more than 2^31 steps"; return; }
            for (int a = 0; a < 3; a++) P.coord.push_back(k * ex[a]);
        }
        s.n[2] = (int)c;
        add(s);
    }
    void point(double x, double y, double z) {
        WorldSeg s{}; s.kind = WSEG_POINT; s.n[0] = s.n[1] = s.n[2] = 1; s.off[0] = (int)P.coord.size();
        P.coord.push_back(x); P.coord.push_back(y); P.coord.push_back(z);
        add(s);
    }
};

// mapGene(id) of globalmap_gene.cpp, restated call for call
void map_program(Walker &W, int id, const double init[3]) {
    const double res = W.res;
    W.wall(0, 0, 0.2, 0.2, 3.0);
    switch (id) {
    case 1:
        W.wall(50, 20, 15.0, 0.2, 0.2, 3.0);
        W.wall(25.0, 0.0, 2.0, 10.0, 5.0);
        W.wall(25.0, 0.0, 7.0, 2.0, 10.0, 5.0);
        break;
    case 2: {
        W.wall(100, 100, 0.2, 0.2, 3.0);
        int tree_number = 20;
        while (tree_number-- && W.err.empty()) {
            const double x = (W.rand() % 3000) / 50.0, y = (W.rand() % 3000) / 50.0;
            if (std::sqrt((x - init[0]) * (x - init[0]) + (y - init[1]) * (y - init[1])) < 0.09) { tree_number++; continue; }
            W.wall(x, y, 5, 5, 20);
        }
        break;
    }
    case 3:
        W.wall(50, 50, 15.0, 0.2, 0.2, 3.0);
        W.wall(10.0, 0.0, 2.0, 2.0, 14.0); W.wall(10.0, 10.0, 2.0, 2.0, 14.0); W.wall(10.0, 2.0, 2.0, 8.0, 3.0);
        W.wall(10.0, 2.0, 12.0, 2.0, 8.0, 2.0); W.wall(10.0, 5.0, 3.0, 2.0, 5.0, 5.5); W.wall(10.0, 10.0, 2.0, 40.0, 15.0);
        W.wall(20.0, 0.0, 2.0, 2.0, 14.0); W.wall(20.0, 10.0, 2.0, 2.0, 14.0); W.wall(20.0, 2.0, 2.0, 8.0, 5.0);
        W.wall(20.0, 2.0, 14.0, 2.0, 8.0, 0.0); W.wall(20.0, 5.0, 5.0, 2.0, 5.0, 5.5); W.wall(20.0, 10.0, 2.0, 40.0, 15.0);
        W.wall(10.0, 0.0, 13.0, 2.0, 50.0, 5.0); W.wall(20.0, 0.0, 13.0, 2.0, 50.0, 5.0);
        break;
    case 4: case 11: {
        W.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        W.srand();
        const int num = id == 4 ? 250 : 300, lo = id == 4 ? 50 : 15;
        for (int i = 0; i < num && W.err.empty(); i++) {
            const double x = (W.rand() % 450 + lo) / 10, y = (W.rand() % 450 + lo) / 10, z = (W.rand() % 250 + 50) / 10;   // int division
            const double len = 1.5 * res;
            W.wall(x, y, z, len, len, len);
        }
        break;
    }
    case 5:
        W.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        W.wall(30, 0, 2.0, 50, 15.0); W.wall(30, 0, 18.0, 2.0, 50, 16.0);
        break;
    case 6: W.wall(60, 60, 35.0, 0.2, 0.2, 3.0); break;
    case 7:
        W.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        W.wall(30, 0, 1.1, 60.0, 8.0); W.wall(30, 0, 5.0, 1.1, 25.0, 7.0); W.wall(30, 35.0, 5.0, 1.1, 25.0, 7.0);
        W.wall(30, 0.0, 12.0, 1.1, 21.0, 9.0); W.wall(30, 39.0, 12.0, 1.1, 21.0, 9.0);
        W.wall(30, 0.0, 21.0, 1.1, 60.0, 4.0); W.wall(30, 28.0, 14.0, 1.1, 4.0, 2.0);
        break;
    case 8:
        W.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        W.point(30, 30, 2.0);
        break;
    case 9:
        W.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        for (double h = -60; h < 30 && W.err.empty(); h += 0.5) {
            if (h > 0.0 && h < 5.5) continue;
            double spt[3] = {0, 20, h}, ept[3];
            std::memcpy(ept, spt, sizeof spt); ept[2] += 45; ept[0] = 50;
            if (h < 0) { spt[0] -= h; spt[2] = 0; std::memcpy(ept, spt, sizeof spt); ept[2] += 45; ept[0] = 50; }
            W.road(spt, ept, 0.5);
        }
        break;
    case 10:
        W.wall(50, 50, 15.0, 0.2, 0.2, 3.0);
        W.wall(10.0, 0.0, 2.0, 50.0, 35.0); W.wall(25.0, 0.0, 2.0, 50.0, 35.0); W.wall(40.0, 0.0, 2.0, 50.0, 35.0);
        W.wall(10.0, 49.0, 30.0, 1.0, 35.0);
        W.wall(0.0, 0.0, -1.0, 50.0, 50.0, 1.0);
        break;
    }
}

// one thread per chunk: binary-search its segment, jump the stream to its first draw, then emit its points with their draws in sequence
__global__ void __launch_bounds__(128) k_world_emit(const WorldSeg *seg, int nseg, long long nchunks, const double *coord,
                                                    const uint32_t *base, const uint32_t *tab, long long cap, float *out) {
    __shared__ double s_add[20];   // (v / 250.0, v / 800.0) for v = rand() % 10
    if (threadIdx.x < 10) { s_add[threadIdx.x] = threadIdx.x / 250.0; s_add[10 + threadIdx.x] = threadIdx.x / 800.0; }
    __syncthreads();
    const long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    int lo = 0, hi = nseg - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (seg[mid].chunk0 <= c) lo = mid; else hi = mid - 1; }
    const WorldSeg S = seg[lo];
    const long long p0 = (c - S.chunk0) * WORLD_CHUNK, np = min((long long)WORLD_CHUNK, S.npts - p0);
    const bool vec = ((uintptr_t)out & 15) == 0;
    auto store = [&](long long p, double x, double y, double z) {
        if (p >= cap) return;
        if (vec) reinterpret_cast<float4 *>(out)[p] = make_float4((float)x, (float)y, (float)z, 1.0f);
        else { out[4 * p] = (float)x; out[4 * p + 1] = (float)y; out[4 * p + 2] = (float)z; out[4 * p + 3] = 1.0f; }
    };
    if (S.kind == WSEG_POINT) { store(S.point0, coord[S.off[0]], coord[S.off[0] + 1], coord[S.off[0] + 2]); return; }
    uint32_t w[GLIBC_DEG];
    glibc_window(base + GLIBC_DEG * S.stream, tab, S.draw0 + 3ull * (unsigned long long)p0, w);
    const int n1 = S.n[1], n2 = S.n[2];
    long long q = p0 / n2;
    int i2 = (int)(p0 - q * n2), i1 = (int)(q % n1), i0 = (int)(q / n1);
    const double *L0 = coord + S.off[0], *L1 = coord + S.off[1], *L2 = coord + S.off[2];
    const bool road = S.kind == WSEG_ROAD;
    for (long long b = 0; b < np; b += GLIBC_DEG) {
#pragma unroll
        for (int k = 0; k < GLIBC_DEG; k++) {
            uint32_t v[3];
#pragma unroll
            for (int a = 0; a < 3; a++) {
                const int d = 3 * k + a;
                if (d && d % GLIBC_DEG == 0) glibc_advance(w);
                v[a] = (w[d % GLIBC_DEG] >> 1) % 10u;
            }
            if (b + k < np) {
                double x, y, z;
                if (road) {
                    const double *pv = L1 + 3 * i1, *ke = L2 + 3 * i2;
                    x = pv[0] + ke[0]; y = pv[1] + ke[1]; z = pv[2] + ke[2];
                } else {
                    x = L2[i2]; y = L1[i1]; z = L0[i0];
                }
                store(S.point0 + p0 + b + k, x + s_add[v[0]], y + s_add[v[1]], z + s_add[10 + v[2]]);
                if (++i2 == n2) { i2 = 0; if (++i1 == n1) { i1 = 0; i0++; } }
            }
        }
        glibc_advance(w);
    }
}

// ================================================= Perlin (maps.cpp perlin3D, perlinnoise.cpp) ===================================
__device__ __forceinline__ double pn_fade(double t) { return t * t * t * (t * (t * 6 - 15) + 10); }
__device__ __forceinline__ double pn_lerp(double t, double a, double b) { return a + t * (b - a); }
__device__ __forceinline__ double pn_grad(int hash, double x, double y, double z) {
    const int h = hash & 15;
    const double u = h < 8 ? x : y, v = h < 4 ? y : h == 12 || h == 14 ? x : z;
    return ((h & 1) == 0 ? u : -u) + ((h & 2) == 0 ? v : -v);
}
__device__ double pn_noise(const int *p, double x, double y, double z) {
    const int X = (int)floor(x) & 255, Y = (int)floor(y) & 255, Z = (int)floor(z) & 255;
    x -= floor(x); y -= floor(y); z -= floor(z);
    const double u = pn_fade(x), v = pn_fade(y), w = pn_fade(z);
    const int A = p[X] + Y, AA = p[A] + Z, AB = p[A + 1] + Z, B = p[X + 1] + Y, BA = p[B] + Z, BB = p[B + 1] + Z;
    const double res = pn_lerp(w, pn_lerp(v, pn_lerp(u, pn_grad(p[AA], x, y, z), pn_grad(p[BA], x - 1, y, z)),
                                          pn_lerp(u, pn_grad(p[AB], x, y - 1, z), pn_grad(p[BB], x - 1, y - 1, z))),
                               pn_lerp(v, pn_lerp(u, pn_grad(p[AA + 1], x, y, z - 1), pn_grad(p[BA + 1], x - 1, y, z - 1)),
                                          pn_lerp(u, pn_grad(p[AB + 1], x, y - 1, z - 1), pn_grad(p[BB + 1], x - 1, y - 1, z - 1))));
    return (res + 1.0) / 2.0;
}
// order-preserving key of a double (-0 taken as +0; the noise is never NaN)
__device__ __forceinline__ unsigned long long key_of(double d) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(d + 0.0);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}

struct PerlinArgs { int X, Y, Z, fractal; double complexity, attenuation, scale; long long n; };

__global__ void __launch_bounds__(256) k_world_noise(const int *perm, PerlinArgs A, unsigned long long *key) {
    __shared__ int p[512];
    for (int i = threadIdx.x; i < 512; i += blockDim.x) p[i] = perm[i];
    __syncthreads();
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < A.n; v += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(v % A.Z);
        const long long q = v / A.Z;
        const int j = (int)(q % A.Y), i = (int)(q / A.Y);
        double tnoise = 0;
        for (int it = 1; it <= A.fractal; ++it) {
            const int dfv = 1 << it;   // pow(2, it), exact
            const double ta = A.attenuation / it;
            tnoise += ta * pn_noise(p, (dfv * i) * A.complexity, (dfv * j) * A.complexity, (dfv * k) * A.complexity);
        }
        key[v] = key_of(tnoise);
    }
}

// one radix-select pass: the histogram of digit `shift` among the keys whose higher digits equal sel[0]'s
__global__ void __launch_bounds__(256) k_world_hist(const unsigned long long *key, long long n, const unsigned long long *sel, int shift,
                                                    unsigned int *hist) {
    __shared__ unsigned int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long prefix = sel[0], mask = shift == 56 ? 0ull : ~0ull << (shift + 8);
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
        const unsigned long long k = key[v];
        if ((k & mask) == prefix) atomicAdd(&h[(k >> shift) & 255], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}
// the digit holding the sel[1]-th smallest among the candidates; resets the histogram for the next pass
__global__ void k_world_pick(unsigned int *hist, unsigned long long *sel, int shift) {
    if (threadIdx.x == 0) {
        unsigned long long k = sel[1], below = 0;
        int d = 0;
        for (; d < 255; d++) {
            if (k < below + hist[d]) break;
            below += hist[d];
        }
        sel[0] |= (unsigned long long)d << shift;
        sel[1] = k - below;
    }
    __syncthreads();
    hist[threadIdx.x] = 0;
}

__global__ void __launch_bounds__(TILE_THREADS) k_world_tile_count(const unsigned long long *key, long long n, const unsigned long long *sel,
                                                                  long long *cnt) {
    using BR = cub::BlockReduce<int, TILE_THREADS>;
    __shared__ typename BR::TempStorage tmp;
    const unsigned long long thr = sel[0];
    const long long t0 = blockIdx.x * (long long)TILE;
    int c = 0;
    for (int e = 0; e < TILE_ITEMS; e++) {
        const long long v = t0 + e * TILE_THREADS + threadIdx.x;
        c += v < n && key[v] > thr;
    }
    const int tot = BR(tmp).Sum(c);
    if (threadIdx.x == 0) cnt[blockIdx.x] = tot;
}
// the tile's voxels above the threshold at their ranks (thread t holds voxels t0 + 16 t .. + 15, so ranks follow voxel order)
__global__ void __launch_bounds__(TILE_THREADS) k_world_perlin_write(const unsigned long long *key, PerlinArgs A, const unsigned long long *sel,
                                                                    const long long *off, long long cap, float *out) {
    using BS = cub::BlockScan<int, TILE_THREADS>;
    __shared__ typename BS::TempStorage tmp;
    const unsigned long long thr = sel[0];
    const long long v0 = blockIdx.x * (long long)TILE + (long long)threadIdx.x * TILE_ITEMS;
    unsigned flags = 0;
    int c = 0;
    for (int e = 0; e < TILE_ITEMS; e++) {
        const long long v = v0 + e;
        if (v < A.n && key[v] > thr) { flags |= 1u << e; c++; }
    }
    int ex;
    BS(tmp).ExclusiveSum(c, ex);
    long long r = off[blockIdx.x] + ex;
    const bool vec = ((uintptr_t)out & 15) == 0;
    const double hx = A.X / (2 * A.scale), hy = A.Y / (2 * A.scale);
    for (int e = 0; e < TILE_ITEMS; e++) {
        if (!((flags >> e) & 1u)) continue;
        const long long v = v0 + e;
        if (r < cap) {
            const int k = (int)(v % A.Z);
            const long long q = v / A.Z;
            const int j = (int)(q % A.Y), i = (int)(q / A.Y);
            const float x = (float)(i / A.scale - hx), y = (float)(j / A.scale - hy), z = (float)(k / A.scale);
            if (vec) reinterpret_cast<float4 *>(out)[r] = make_float4(x, y, z, 1.0f);
            else { out[4 * r] = x; out[4 * r + 1] = y; out[4 * r + 2] = z; out[4 * r + 3] = 1.0f; }
        }
        r++;
    }
}

// ================================================= boxes (maps.cpp randomMapGenerate) ============================================
// one block per box: its (r, s, t) voxels in tiles of the block, the shell's ranks by a block scan
__global__ void __launch_bounds__(256) k_world_boxes(const WorldBox *box, double res, long long cap, float *out) {
    using BS = cub::BlockScan<int, 256>;
    __shared__ typename BS::TempStorage tmp;
    const WorldBox B = box[blockIdx.x];
    const int nr = B.rh - B.rl;
    if (nr <= 0 || B.hei <= 0) return;
    const long long nv = (long long)nr * nr * B.hei;
    const bool vec = ((uintptr_t)out & 15) == 0;
    long long base = B.point0;
    for (long long t0 = 0; t0 < nv; t0 += blockDim.x) {
        const long long v = t0 + threadIdx.x;
        int r = 0, s = 0, t = 0, f = 0;
        if (v < nv) {
            t = (int)(v % B.hei);
            const long long q = v / B.hei;
            s = B.rl + (int)(q % nr); r = B.rl + (int)(q / nr);
            f = r == B.rl || r == B.rh - 1 || s == B.rl || s == B.rh - 1 || t == 0 || t == B.hei - 1;
        }
        int ex, tot;
        BS(tmp).ExclusiveSum(f, ex, tot);
        __syncthreads();
        const long long p = base + ex;
        if (f && p < cap) {
            const float x = (float)(B.x + r * res), y = (float)(B.y + s * res), z = (float)(t * res);
            if (vec) reinterpret_cast<float4 *>(out)[p] = make_float4(x, y, z, 1.0f);
            else { out[4 * p] = x; out[4 * p + 1] = y; out[4 * p + 2] = z; out[4 * p + 3] = 1.0f; }
        }
        base += tot;
    }
}

int bad(std::string *msg, const char *m) { *msg = m; return ISDF_ERR_INVALID; }

int plan_globalmap(const isdf_world_params &p, WorldPlan &P, std::string *msg) {
    if (p.map_id < 1 || p.map_id > 11) return bad(msg, "map_id must be in 1..11");
    if (!std::isfinite(p.cloud_resolution) || !(p.cloud_resolution > 0)) return bad(msg, "cloud_resolution must be positive and finite");
    for (double v : p.init) if (!std::isfinite(v)) return bad(msg, "init must be finite");
    P.tab.resize(64 * GLIBC_DEG); glibc_jump_table(P.tab.data());
    P.base.resize(2 * GLIBC_DEG); glibc_base(p.rand_seed, P.base.data()); glibc_base(p.srand_seed, P.base.data() + GLIBC_DEG);
    Walker W(P, p.cloud_resolution);
    map_program(W, p.map_id, p.init);
    if (!W.err.empty()) { *msg = W.err; return ISDF_ERR_INVALID; }
    P.n = W.points; P.n_exact = true;
    for (WorldSeg &s : P.seg) { s.chunk0 = P.nchunks; P.nchunks += (s.npts + WORLD_CHUNK - 1) / WORLD_CHUNK; }
    return 0;
}

int check_sizes(const isdf_world_params &p, std::string *msg) {
    if (p.size[0] < 1 || p.size[1] < 1 || p.size[2] < 1) return bad(msg, "sizes must be positive");
    if ((long long)p.size[0] * p.size[1] * p.size[2] >= (1ll << 31)) return bad(msg, "size[0] size[1] size[2] must be below 2^31 voxels");
    if (!std::isfinite(p.scale) || !(p.scale > 0)) return bad(msg, "scale must be positive and finite");
    return 0;
}

int plan_perlin(const isdf_world_params &p, WorldPlan &P, std::string *msg) {
    if (int rc = check_sizes(p, msg)) return rc;
    if (!std::isfinite(p.complexity) || !std::isfinite(p.fill) || !std::isfinite(p.attenuation))
        return bad(msg, "complexity, fill and attenuation must be finite");
    if (p.fractal < 1) return bad(msg, "fractal must be >= 1");
    const double m = (double)std::max(p.size[0], std::max(p.size[1], p.size[2]));
    if (p.fractal > 30 || std::ldexp(m, p.fractal) >= 2147483648.0 || std::ldexp(m, p.fractal) * std::fabs(p.complexity) >= 2147483648.0)
        return bad(msg, "2^fractal max(size) and 2^fractal max(size) |complexity| must be below 2^31");
    const long long n = (long long)p.size[0] * p.size[1] * p.size[2];
    const double d = (double)(uint32_t)n * (1 - p.fill);   // info.cloud->width (uint32_t) * (1 - fill)
    if (!(d > -1.0 && d < (double)n)) return bad(msg, "tpos = (int)(X Y Z (1 - fill)) is outside [0, X Y Z)");
    P.tpos = (int)d;
    P.perm.resize(256);
    std::iota(P.perm.begin(), P.perm.end(), 0);
    std::default_random_engine engine((unsigned int)p.seed);
    std::shuffle(P.perm.begin(), P.perm.end(), engine);
    P.perm.insert(P.perm.end(), P.perm.begin(), P.perm.end());
    P.n = n; P.n_exact = false;
    return 0;
}

int plan_boxes(const isdf_world_params &p, WorldPlan &P, std::string *msg) {
    if (int rc = check_sizes(p, msg)) return rc;
    if (p.obstacle_number < 0) return bad(msg, "obstacle_number must be >= 0");
    if (!std::isfinite(p.width_min) || !std::isfinite(p.width_max) || p.width_min > p.width_max)
        return bad(msg, "widths must be finite with width_min <= width_max");
    const double S = p.scale, res = 1 / S;
    std::default_random_engine eng((int)p.seed);   // BasicInfo::seed is an int
    std::uniform_real_distribution<double> rx(-p.size[0] / (2 * S), p.size[0] / (2 * S)), ry(-p.size[1] / (2 * S), p.size[1] / (2 * S)),
        rw(p.width_min, p.width_max), rh(0, p.size[2] / S);
    long long pts = 0;
    for (int i = 0; i < p.obstacle_number; i++) {
        const double x = rx(eng), y = ry(eng), w = rw(eng), h = rh(eng);
        const double wn = std::ceil(w / res), hn = std::ceil(h / res);
        if (!(std::fabs(wn) < 1e6 && std::fabs(hn) < 1e6)) return bad(msg, "a box's shell product can reach 2^31 (box too large)");
        const int widNum = (int)wn, heiNum = (int)hn;
        WorldBox B{x, y, pts, -widNum / 2, widNum / 2, heiNum};
        const long long nr = B.rh - B.rl;
        const double W = (double)std::max(nr - 1, 0ll), H = (double)std::max(heiNum - 1, 0);
        if (W * W * W * W * H * H >= 2147483648.0) return bad(msg, "a box's shell product can reach 2^31 (box too large)");
        long long cnt = 0;
        if (nr > 0 && heiNum > 0) {
            const long long inner = std::max(nr - 2, 0ll) * std::max(nr - 2, 0ll);
            cnt = (nr * nr - inner) * heiNum + inner * std::min(heiNum, 2);
        }
        pts += cnt;
        P.box.push_back(B);
    }
    P.box_res = res; P.n = pts; P.n_exact = true;
    return 0;
}

size_t align_up(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

int world_plan(const isdf_world_params &p, WorldPlan &P, std::string *msg) {
    P = WorldPlan();
    P.p = p; P.kind = p.kind;
    if (p.reserved_[0] || p.reserved_[1]) return bad(msg, "reserved_ must be 0");
    switch (p.kind) {
    case ISDF_WORLD_GLOBALMAP: return plan_globalmap(p, P, msg);
    case ISDF_WORLD_PERLIN: return plan_perlin(p, P, msg);
    case ISDF_WORLD_BOXES: return plan_boxes(p, P, msg);
    default: return bad(msg, "unknown world kind");
    }
}

#define W_TRY(x) do { const cudaError_t e_ = (x); if (e_ != cudaSuccess) return e_; } while (0)

cudaError_t world_emit(WorldScratch &W, const WorldPlan &P, long long cap, float *d_points, long long *n, cudaStream_t st, int *launches) {
    if (P.kind == ISDF_WORLD_GLOBALMAP) {
        *n = P.n;
        if (P.seg.empty() || cap == 0) return cudaSuccess;
        const size_t b_seg = P.seg.size() * sizeof(WorldSeg), b_coord = P.coord.size() * sizeof(double);
        const size_t o_coord = align_up(b_seg), o_base = o_coord + align_up(b_coord), o_tab = o_base + align_up(P.base.size() * 4);
        const size_t total = o_tab + P.tab.size() * 4;
        std::vector<char> h(total);
        std::memcpy(h.data(), P.seg.data(), b_seg); std::memcpy(h.data() + o_coord, P.coord.data(), b_coord);
        std::memcpy(h.data() + o_base, P.base.data(), P.base.size() * 4); std::memcpy(h.data() + o_tab, P.tab.data(), P.tab.size() * 4);
        W_TRY(W.d_prog.upload(h.data(), total, st));
        const long long blocks = (P.nchunks + 127) / 128;
        k_world_emit<<<(unsigned)blocks, 128, 0, st>>>((const WorldSeg *)W.d_prog.p, (int)P.seg.size(), P.nchunks, (const double *)(W.d_prog.p + o_coord),
                                                  (const uint32_t *)(W.d_prog.p + o_base), (const uint32_t *)(W.d_prog.p + o_tab), cap, d_points);
        ++*launches;
        return cudaGetLastError();
    }
    if (P.kind == ISDF_WORLD_BOXES) {
        *n = P.n;
        if (P.box.empty() || cap == 0) return cudaSuccess;
        W_TRY(W.d_prog.upload((const char *)P.box.data(), P.box.size() * sizeof(WorldBox), st));
        k_world_boxes<<<(unsigned)P.box.size(), 256, 0, st>>>((const WorldBox *)W.d_prog.p, P.box_res, cap, d_points);
        ++*launches;
        return cudaGetLastError();
    }
    // Perlin: keys, 8 radix-select passes, tile counts, their scan, the ordered write, one read of the count
    const isdf_world_params &p = P.p;
    PerlinArgs A{p.size[0], p.size[1], p.size[2], p.fractal, p.complexity, p.attenuation, p.scale, P.n};
    const long long tiles = (P.n + TILE - 1) / TILE;
    W_TRY(W.d_prog.upload((const char *)P.perm.data(), P.perm.size() * sizeof(int32_t), st));
    W_TRY(W.d_key.ensure((size_t)P.n)); W_TRY(W.d_hist.ensure(256)); W_TRY(W.d_sel.ensure(2)); W_TRY(W.d_tile.ensure(2 * (size_t)tiles + 1));   // offsets (tiles + 1), then the counts
    W_TRY(W.h_n.ensure(2));
    W.h_n.p[0] = 0; W.h_n.p[1] = P.tpos;
    W_TRY(cudaMemcpyAsync(W.d_sel.p, W.h_n.p, 16, cudaMemcpyHostToDevice, st));
    W_TRY(cudaMemsetAsync(W.d_hist.p, 0, 256 * sizeof(unsigned), st));
    const unsigned grid = (unsigned)std::min<long long>((P.n + 255) / 256, 132 * 16);
    k_world_noise<<<grid, 256, 0, st>>>((const int *)W.d_prog.p, A, W.d_key.p);
    ++*launches;
    for (int shift = 56; shift >= 0; shift -= 8) {
        k_world_hist<<<grid, 256, 0, st>>>(W.d_key.p, P.n, W.d_sel.p, shift, W.d_hist.p);
        k_world_pick<<<1, 256, 0, st>>>(W.d_hist.p, W.d_sel.p, shift);
        *launches += 2;
    }
    long long *d_cnt = W.d_tile.p + tiles + 1;
    k_world_tile_count<<<(unsigned)tiles, TILE_THREADS, 0, st>>>(W.d_key.p, P.n, W.d_sel.p, d_cnt);
    ++*launches;
    W_TRY(cudaMemsetAsync(W.d_tile.p, 0, sizeof(long long), st));
    size_t tmp = 0;
    W_TRY(cub::DeviceScan::InclusiveSum(nullptr, tmp, d_cnt, W.d_tile.p + 1, (int)tiles, st));
    W_TRY(W.d_tmp.ensure(tmp));
    W_TRY(cub::DeviceScan::InclusiveSum(W.d_tmp.p, tmp, d_cnt, W.d_tile.p + 1, (int)tiles, st));
    ++*launches;
    if (cap > 0) {
        k_world_perlin_write<<<(unsigned)tiles, TILE_THREADS, 0, st>>>(W.d_key.p, A, W.d_sel.p, W.d_tile.p, cap, d_points);
        ++*launches;
    }
    W_TRY(cudaGetLastError());
    W_TRY(cudaMemcpyAsync(W.h_n.p, W.d_tile.p + tiles, 8, cudaMemcpyDeviceToHost, st));
    W_TRY(cudaStreamSynchronize(st));
    *n = W.h_n.p[0];
    return cudaSuccess;
}

}  // namespace isdf

// diagnostics (not in include/isdf.h): glibc rand() after srand(seed) at each of n stream offsets, by the jump-ahead the generators use
extern "C" int isdf_dbg_world_rand(uint32_t seed, const uint64_t *offsets, int64_t n, int32_t *out) {
    using namespace isdf;
    if (!offsets || !out || n < 0) return ISDF_ERR_INVALID;
    std::vector<uint32_t> tab(64 * GLIBC_DEG), base(GLIBC_DEG);
    glibc_jump_table(tab.data()); glibc_base(seed, base.data());
    uint32_t w[GLIBC_DEG];
    for (int64_t i = 0; i < n; i++) {
        glibc_window(base.data(), tab.data(), offsets[i], w);
        out[i] = (int32_t)(w[0] >> 1);
    }
    return 0;
}
