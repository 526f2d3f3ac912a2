// World generators (include/isdf.h, DESIGN §3.19): the reference's globalmap_gene maps 1-11 and mockamap's Perlin and box worlds, point
// for point.
//   glibc_*          : glibc's TYPE_3 rand() stream with jump-ahead. u_m = r_{m+3} obeys u_m = u_{m-3} + u_{m-31} (mod 2^32) for every
//                      m >= 31, so u_m = sum_i c_i u_i with c = x^m mod (x^31 - x^28 - 1) over Z/2^32; draw k is u_{k+341} >> 1. One
//                      __host__ __device__ body: the host draws map 2's trees and the cubes of maps 4 and 11, the device its chunk starts.
//   k_world_emit     : one thread per chunk of WORLD_CHUNK points of one segment (a wall, a road or map 8's point): the chunk's start
//                      window by jump-ahead, then its draws in sequence, each point from its segment's coordinate lists
//   k_world_noise / k_world_hist / k_world_pick : Perlin: the noise of every voxel as an order-preserving 64-bit key, then an exact
//                      k-th smallest by radix select (8 passes of 8 bits), no sort
//   k_world_tile_count / k_world_perlin_write   : the voxels above the threshold, compacted in (i, j, k) order from the stored keys
//   k_world_boxes    : one block per box, its shell in (r, s, t) order
// Compiled only into isdf_world_tu.cu with -fmad=false: the FP64 noise and coordinates round operation by operation as the reference's
// g++ build (no -march, so no FMA).
#pragma once
#include "../../include/isdf.h"
#include "isdf_types.cuh"
#include <string>
#include <vector>

namespace isdf {

constexpr int WORLD_CHUNK = 31 * 32;   // points per emission thread: a whole number of 31-point blocks (93 draws, three windows)
constexpr int GLIBC_DEG = 31;
constexpr unsigned long long GLIBC_DISCARD = 310;   // srandom_r discards 10 x 31 outputs

// glibc srandom_r(seed) as u_0..u_30 = r_3..r_33 (r_31..r_33 = r_0..r_2)
__host__ __device__ inline void glibc_base(uint32_t seed, uint32_t u[GLIBC_DEG]) {
    if (seed == 0) seed = 1;
    int32_t r[GLIBC_DEG];
    int32_t word = (int32_t)seed;
    r[0] = word;
    for (int i = 1; i < GLIBC_DEG; i++) {
        const long long hi = word / 127773, lo = word % 127773;
        word = (int32_t)(16807 * lo - 2836 * hi);
        if (word < 0) word += 2147483647;
        r[i] = word;
    }
    for (int j = 0; j < 28; j++) u[j] = (uint32_t)r[j + 3];
    for (int j = 28; j < GLIBC_DEG; j++) u[j] = (uint32_t)r[j - 28];
}

// out = a b mod (x^31 - x^28 - 1), coefficients mod 2^32 (out may alias a or b)
__host__ __device__ inline void glibc_polymul(const uint32_t *a, const uint32_t *b, uint32_t *out) {
    uint32_t t[2 * GLIBC_DEG - 1];
#pragma unroll
    for (int k = 0; k < 2 * GLIBC_DEG - 1; k++) t[k] = 0;
#pragma unroll
    for (int i = 0; i < GLIBC_DEG; i++) {
        const uint32_t ai = a[i];
#pragma unroll
        for (int j = 0; j < GLIBC_DEG; j++) t[i + j] += ai * b[j];
    }
#pragma unroll
    for (int k = 2 * GLIBC_DEG - 2; k >= GLIBC_DEG; k--) { t[k - 3] += t[k]; t[k - GLIBC_DEG] += t[k]; }   // x^k = x^{k-3} + x^{k-31}
#pragma unroll
    for (int k = 0; k < GLIBC_DEG; k++) out[k] = t[k];
}

// c = x c mod (x^31 - x^28 - 1)
__host__ __device__ inline void glibc_mulx(uint32_t c[GLIBC_DEG]) {
    const uint32_t top = c[GLIBC_DEG - 1];
#pragma unroll
    for (int j = GLIBC_DEG - 1; j > 0; j--) c[j] = c[j - 1];
    c[0] = top;
    c[28] += top;
}

// tab[b] = x^(2^b) mod (x^31 - x^28 - 1), b = 0..63 (64 x 31 words)
inline void glibc_jump_table(uint32_t *tab) {
    for (int i = 0; i < GLIBC_DEG; i++) tab[i] = i == 1;
    for (int b = 1; b < 64; b++) glibc_polymul(tab + (b - 1) * GLIBC_DEG, tab + (b - 1) * GLIBC_DEG, tab + b * GLIBC_DEG);
}

// w[j] = u_{k + 341 + j}, j = 0..30: the window whose words >> 1 are draws k .. k + 30 of the stream with base u (tab: glibc_jump_table)
__host__ __device__ inline void glibc_window(const uint32_t *u, const uint32_t *tab, unsigned long long k, uint32_t w[GLIBC_DEG]) {
    const unsigned long long m = k + GLIBC_DISCARD + GLIBC_DEG;
    uint32_t c[GLIBC_DEG];
#pragma unroll
    for (int i = 0; i < GLIBC_DEG; i++) c[i] = i == 0;
    for (int b = 0; b < 64; b++)
        if ((m >> b) & 1ull) glibc_polymul(c, tab + b * GLIBC_DEG, c);
#pragma unroll
    for (int j = 0; j < GLIBC_DEG; j++) {
        uint32_t s = 0;
#pragma unroll
        for (int i = 0; i < GLIBC_DEG; i++) s += c[i] * u[i];
        w[j] = s;
        glibc_mulx(c);
    }
}

// the next 31 words of the stream in place: w[j] = u_{m+j} -> u_{m+31+j} = u_{m+28+j} + u_{m+j}
__host__ __device__ __forceinline__ void glibc_advance(uint32_t w[GLIBC_DEG]) {
#pragma unroll
    for (int j = 0; j < GLIBC_DEG; j++) w[j] += w[(j + 28) % GLIBC_DEG];
}

// one segment of a globalmap world: its points are (z outer, y, x inner) over its lists for a wall, (t outer, k inner) for a road
enum { WSEG_WALL = 0, WSEG_ROAD = 1, WSEG_POINT = 2 };
struct WorldSeg {
    long long point0, chunk0, npts;   // first point in the cloud, first emission chunk, points
    unsigned long long draw0;         // stream offset (draws after seeding) of its first draw
    int stream, kind;                 // base index (0: srand(rand_seed), 1: srand(srand_seed)); WSEG_*
    int n[3], off[3];                 // loop counts, outer to inner, and their lists' offsets in the coordinate array (doubles)
                                      // wall: z, y, x lists (1 double each); road: -, paver positions, k * expand (3 doubles each);
                                      // point: its x, y, z at off[0]
};

// one box of a box world: its shell in (r, s, t) order from point0
struct WorldBox {
    double x, y;
    long long point0;
    int rl, rh, hei;
};

// the host's program of one call: everything but the device work
struct WorldPlan {
    int kind = 0;
    long long n = 0;          // the cloud's size (globalmap, boxes), or the voxel count bounding it (Perlin)
    bool n_exact = false;
    // globalmap
    std::vector<WorldSeg> seg; std::vector<double> coord; std::vector<uint32_t> base, tab;   // base: 31 words per stream
    long long nchunks = 0;
    // Perlin
    std::vector<int32_t> perm;   // 512 entries
    long long tpos = 0;
    // boxes
    std::vector<WorldBox> box; double box_res = 0;
    isdf_world_params p{};
};

// the call's device scratch, owned by the context
struct WorldScratch {
    DevBuf<char> d_prog;                       // segments + coordinates + bases + jump table, or boxes, or the permutation
    DevBuf<unsigned long long> d_key;          // Perlin keys
    DevBuf<unsigned int> d_hist;               // 256 bins
    DevBuf<unsigned long long> d_sel;          // {prefix, k}
    DevBuf<long long> d_tile;                  // per-tile counts, then offsets (tiles + 1)
    DevBuf<char> d_tmp;                        // scan scratch
    DevBuf<float> d_out;                       // the host form's records
    PinnedBuf<long long> h_n;
};

// ---- host interface of the world translation unit (isdf_world_tu.cu) ----
// validates p and builds the host program; 0, or ISDF_ERR_INVALID with *msg
int world_plan(const isdf_world_params &p, WorldPlan &P, std::string *msg);
// runs the plan on st: min(n, cap) records into d_points (device), the size into *n (read back for Perlin only)
cudaError_t world_emit(WorldScratch &W, const WorldPlan &P, long long cap, float *d_points, long long *n, cudaStream_t st, int *launches);

}  // namespace isdf
