// Frontiers of known space and frontier goals (include/isdf.h, DESIGN §3.24).
//
// T_o is the front end's traversability over the occupancy grid, T_b the same over the blocked grid occ | ~known (both from the
// feasibility kernels of isdf_frontend.cuh in their traversability mode). F = T_b & dilate26(T_o & ~T_b): places where the robot fits
// with every kernel cell known free, next to places where it would fit if unseen space were free.
//   k_fr_frontier   one thread per 32-voxel word: the 26-dilation as word-parallel shifts along z and ORs over the 3 x 3 (x, y) rows,
//                   ANDed with T_b; the word's population count (for the list) and |T_b| (one atomic per warp)
//   (CUB scan)      list positions: word w's frontier voxels start at woff[w]; a voxel's position is woff[w] + popc of the lower bits,
//                   so the list is in ascending voxel index
//   k_fr_list       the list: voxel indices, and every voxel its own union-find parent
//   k_fr_hook       union-find over list positions: every voxel joins its (up to 13) frontier neighbours of smaller index; a root is
//                   only ever hooked under a smaller root (atomicCAS), so parents point down and each component's root is its smallest
//                   position, i.e. its smallest voxel index, whatever the order of the hooks
//   k_fr_flatten    parent = root; root flags for the cluster slots (CUB scan: slots in ascending root, i.e. ascending cluster id)
//   k_fr_accum      integer sums, sizes and index boxes per cluster (integer atomics: exact, order-free)
//   k_fr_table      the cluster records and each frontier voxel's cluster id
// Goals: the fields g_b from the starts over T_b (k_fp_relax* with trav = T_b, unweighted), then per pair
//   k_fg_score      atomicMin of the best score's bit pattern (a non-negative double) over the candidate list
//   k_fg_pick       atomicMin of the list position among the voxels with that score (the smallest voxel index)
//   k_fg_record     GOAL / FRONTIER / NONE and the record
// With a view rig (isdf_frontier_goals_view), between the size rule (k_fg_cand) and the selection: k_fg_view_poses puts a pose at every
// frontier voxel's cube centre, view_gain_run (isdf_view.cuh) counts the gains of the voxels the size rule kept, and k_fg_gain_cand clears
// the candidates whose gain is below min_gain.
#pragma once
#include "isdf_frontpath.cuh"

namespace isdf {

struct FrArgs {
    DevGrid grid;                  // dims, bmin, res of the map (grid.bits unused)
    const uint32_t *to, *tb;       // T_o and T_b, grid.bits' layout
    uint32_t *f;                   // F, grid.bits' layout
    int *cnt;                      // per word: |F| in the word (k_fr_frontier), then scanned into woff
    const int *woff;               // nword + 1: first list position of each word
    unsigned long long *ntb;       // |T_b|
    int n;                         // |F|
    long long *vox;                // n: voxel index
    int *parent;                   // n: union-find parent, then the root
    int *root;                     // n + 1: 1 at roots (k_fr_flatten), scanned into cluster slots (slot of root r = root[r])
    const int *slot;               // n + 1: the scan of root flags
    int nc;                        // clusters
    unsigned long long *sum;       // 3 per cluster: sums of the voxel indices per axis
    int *size, *box;               // per cluster: size; 6 per cluster: index box (min x, y, z, max x, y, z)
    int *croot;                    // per cluster: its root's list position
    long long *cid;                // n: each frontier voxel's cluster id (its root's voxel index)
    isdf_frontier_cluster *table;  // nc records
};

__device__ __forceinline__ uint32_t fr_word(const uint32_t *b, const DevGrid &G, int x, int y, int zw) {
    return (zw >= 0 && zw < G.Zw) ? __ldg(b + ((size_t)x * G.Y + y) * G.Zw + zw) : 0u;
}
// the bits of word (x, y, zw) of T_o & ~T_b, shifted by -1, 0, +1 along z and ORed (bit j: voxel 32 zw + j or a z-neighbour is in it)
__device__ __forceinline__ uint32_t fr_zdilate(const FrArgs &A, int x, int y, int zw) {
    const DevGrid &G = A.grid;
    const uint32_t w = fr_word(A.to, G, x, y, zw) & ~fr_word(A.tb, G, x, y, zw);
    const uint32_t wp = fr_word(A.to, G, x, y, zw - 1) & ~fr_word(A.tb, G, x, y, zw - 1);
    const uint32_t wn = fr_word(A.to, G, x, y, zw + 1) & ~fr_word(A.tb, G, x, y, zw + 1);
    return w | (w << 1) | (wp >> 31) | (w >> 1) | (wn << 31);
}

__global__ void __launch_bounds__(256) k_fr_frontier(const __grid_constant__ FrArgs A) {
    const DevGrid &G = A.grid;
    const long long nword = (long long)G.X * G.Y * G.Zw;
    const int tail = G.Z & 31;
    unsigned long long ntb = 0;
    for (long long wi = (long long)blockIdx.x * blockDim.x + threadIdx.x; wi < nword; wi += (long long)gridDim.x * blockDim.x) {
        const int zw = (int)(wi % G.Zw), y = (int)((wi / G.Zw) % G.Y), x = (int)(wi / ((long long)G.Zw * G.Y));
        const uint32_t valid = (zw == G.Zw - 1 && tail) ? ((1u << tail) - 1u) : 0xffffffffu;
        const uint32_t tb = __ldg(A.tb + wi) & valid;
        ntb += __popc(tb);
        uint32_t d = 0u;
        if (tb)
            for (int dx = -1; dx <= 1; dx++) {
                if (x + dx < 0 || x + dx >= G.X) continue;
                for (int dy = -1; dy <= 1; dy++) {
                    if (y + dy < 0 || y + dy >= G.Y) continue;
                    d |= fr_zdilate(A, x + dx, y + dy, zw);
                }
            }
        const uint32_t f = tb & d;
        A.f[wi] = f;
        A.cnt[wi] = __popc(f);
    }
    for (int o = 16; o; o >>= 1) ntb += __shfl_xor_sync(0xffffffffu, ntb, o);
    if ((threadIdx.x & 31) == 0 && ntb) atomicAdd(A.ntb, ntb);
}

__global__ void __launch_bounds__(256) k_fr_list(const __grid_constant__ FrArgs A) {
    const DevGrid &G = A.grid;
    const long long nword = (long long)G.X * G.Y * G.Zw;
    for (long long wi = (long long)blockIdx.x * blockDim.x + threadIdx.x; wi < nword; wi += (long long)gridDim.x * blockDim.x) {
        uint32_t f = A.f[wi];
        int pos = A.woff[wi];
        const long long base = (wi / G.Zw) * G.Z + 32ll * (wi % G.Zw);   // voxel index of the word's bit 0
        while (f) {
            const int j = __ffs((int)f) - 1;
            f &= f - 1;
            A.vox[pos] = base + j;
            A.parent[pos] = pos;
            pos++;
        }
    }
}

// the list position of frontier voxel (x, y, z), -1 when it is not one
__device__ __forceinline__ int fr_pos(const FrArgs &A, int x, int y, int z) {
    const DevGrid &G = A.grid;
    if (x < 0 || x >= G.X || y < 0 || y >= G.Y || z < 0 || z >= G.Z) return -1;
    const size_t w = ((size_t)x * G.Y + y) * G.Zw + (z >> 5);
    const uint32_t f = A.f[w], b = 1u << (z & 31);
    if (!(f & b)) return -1;
    return A.woff[w] + __popc(f & (b - 1u));
}
__device__ __forceinline__ int fr_find(const int *parent, int x) {
    for (int p; (p = __ldcg(parent + x)) != x;) x = p;
    return x;
}

__global__ void __launch_bounds__(256) k_fr_hook(const __grid_constant__ FrArgs A) {
    const DevGrid &G = A.grid;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += gridDim.x * blockDim.x) {
        const long long v = A.vox[i];
        const int z = (int)(v % G.Z), y = (int)((v / G.Z) % G.Y), x = (int)(v / ((long long)G.Z * G.Y));
        // the 13 neighbours of smaller voxel index: (dx, dy, dz) lexicographically negative
        for (int k = 0; k < 13; k++) {
            const int dx = k / 9 - 1, dy = (k / 3) % 3 - 1, dz = k % 3 - 1;
            const int j = fr_pos(A, x + dx, y + dy, z + dz);
            if (j < 0) continue;
            int a = i, b = j;
            while (true) {
                a = fr_find(A.parent, a); b = fr_find(A.parent, b);
                if (a == b) break;
                if (a < b) { const int t = a; a = b; b = t; }
                if (atomicCAS(A.parent + a, a, b) == a) break;
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_fr_flatten(const __grid_constant__ FrArgs A) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += gridDim.x * blockDim.x) {
        const int r = fr_find(A.parent, i);
        A.parent[i] = r;   // an ancestor: concurrent finds stay correct
        A.root[i] = r == i;
    }
}

__global__ void __launch_bounds__(256) k_fr_accum(const __grid_constant__ FrArgs A) {
    const DevGrid &G = A.grid;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += gridDim.x * blockDim.x) {
        const int r = A.parent[i], k = A.slot[r];
        const long long v = A.vox[i];
        const int id[3] = {(int)(v / ((long long)G.Z * G.Y)), (int)((v / G.Z) % G.Y), (int)(v % G.Z)};
        if (r == i) A.croot[k] = i;
        atomicAdd(A.size + k, 1);
        for (int a = 0; a < 3; a++) {
            atomicAdd(A.sum + 3 * (size_t)k + a, (unsigned long long)id[a]);
            atomicMin(A.box + 6 * (size_t)k + a, id[a]);
            atomicMax(A.box + 6 * (size_t)k + 3 + a, id[a]);
        }
        A.cid[i] = A.vox[r];
    }
}

__global__ void k_fr_table_init(const __grid_constant__ FrArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.nc) return;
    A.size[k] = 0;
    for (int a = 0; a < 3; a++) { A.sum[3 * (size_t)k + a] = 0ull; A.box[6 * (size_t)k + a] = 0x7fffffff; A.box[6 * (size_t)k + 3 + a] = -1; }
}

// centroid_a = bmin_a + ((double) sum_a / (double) size + 0.5) * res (the unit is compiled with -fmad=false)
__global__ void k_fr_table(const __grid_constant__ FrArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.nc) return;
    isdf_frontier_cluster c;
    c.id = A.vox[A.croot[k]];
    c.size = A.size[k];
    for (int a = 0; a < 3; a++) {
        c.bmin[a] = A.box[6 * (size_t)k + a];
        c.bmax[a] = A.box[6 * (size_t)k + 3 + a];
        c.centroid[a] = A.grid.bmin[a] + ((double)A.sum[3 * (size_t)k + a] / (double)A.size[k] + 0.5) * A.grid.res;
    }
    A.table[k] = c;
}

// ---- frontier goals ----
struct FgArgs {
    DevGrid grid;
    const unsigned long long *g;   // the chunk's fields (slice s at g + s*X*Y*Z)
    const long long *vox;          // the frontier list
    const uint8_t *cand;           // per list position: its cluster has at least min_cluster_voxels voxels
    int n;
    double goal_weight;
    int nt;                        // the chunk's pairs
    const int *pair;               // nt: pair index
    const int *slice;              // nt: the pair's field slice
    const double *goals;           // B x 3
    const int *tgt;                // B x 3: the goal voxels
    unsigned long long *best;      // B: the best score's bits (FP_INF: none)
    unsigned *pick;                // B: the list position picked among the best (0xffffffff: none)
    const isdf_frontier_cluster *table;
    const long long *cid;          // n: cluster ids
    const long long *gain;         // n: view gains (NULL without a rig: every record's gain 0)
    isdf_frontier_goal *out;       // B records
};

// the cube centre of voxel v on axis a: bmin + (i + 0.5) res, a FRONTIER record's point
__device__ __forceinline__ double fg_centre(const DevGrid &G, long long v, int a) {
    const int i = a == 0 ? (int)(v / ((long long)G.Z * G.Y)) : a == 1 ? (int)((v / G.Z) % G.Y) : (int)(v % G.Z);
    return (i + 0.5) * G.res + G.bmin[a];
}

// score(f) = g_b(f) + goal_weight * sqrt((dx*dx + dy*dy) + dz*dz), d = cube centre of f - goal; the bits of +inf when f is not a
// candidate or not reached
__device__ __forceinline__ unsigned long long fg_score(const FgArgs &A, const unsigned long long *g, const double *gl, int i) {
    if (!A.cand[i]) return FP_INF;
    const long long v = A.vox[i];
    const unsigned long long gv = g[v];
    if (gv == FP_INF) return FP_INF;
    const DevGrid &G = A.grid;
    const int id[3] = {(int)(v / ((long long)G.Z * G.Y)), (int)((v / G.Z) % G.Y), (int)(v % G.Z)};
    double d[3];
    for (int a = 0; a < 3; a++) d[a] = ((id[a] + 0.5) * G.res + G.bmin[a]) - gl[a];
    return (unsigned long long)__double_as_longlong(__longlong_as_double((long long)gv) + A.goal_weight * sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]));
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
    for (int o = 16; o; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
    return v;
}

// PICK = false: best[b] = the least score; PICK = true: pick[b] = the least list position whose score is best[b]. Every thread of a
// CTA runs the same number of loop trips (the warp reductions need whole warps).
template <bool PICK>
__global__ void __launch_bounds__(256) k_fg_select(const __grid_constant__ FgArgs A) {
    const DevGrid &G = A.grid;
    const long long nvox = (long long)G.X * G.Y * G.Z;
    for (int t = blockIdx.y; t < A.nt; t += gridDim.y) {
        const int b = A.pair[t];
        const unsigned long long *g = A.g + (size_t)A.slice[t] * nvox;
        const double *gl = A.goals + 3 * (size_t)b;
        const unsigned long long best = PICK ? A.best[b] : 0ull;
        const int stride = gridDim.x * blockDim.x;
        for (int i0 = blockIdx.x * blockDim.x; i0 < A.n; i0 += stride) {
            const int i = i0 + threadIdx.x;
            const unsigned long long s = i < A.n ? fg_score(A, g, gl, i) : FP_INF;
            if (!PICK) {
                const unsigned long long m = warp_min_u64(s);
                if ((threadIdx.x & 31) == 0 && m != FP_INF) atomicMin(A.best + b, m);
            } else {
                const unsigned p = __reduce_min_sync(0xffffffffu, s == best ? (unsigned)i : 0xffffffffu);
                if ((threadIdx.x & 31) == 0 && p != 0xffffffffu) atomicMin(A.pick + b, p);
            }
        }
    }
}

// the records of the chunk's pairs: GOAL when the field reaches the goal voxel, else FRONTIER at the pick, else NONE
__global__ void k_fg_record(const __grid_constant__ FgArgs A) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= A.nt) return;
    const DevGrid &G = A.grid;
    const int b = A.pair[t];
    const unsigned long long *g = A.g + (size_t)A.slice[t] * G.X * G.Y * G.Z;
    const int *tv = A.tgt + 3 * (size_t)b;
    const long long vt = ((long long)tv[0] * G.Y + tv[1]) * G.Z + tv[2];
    isdf_frontier_goal r;
    r.gain = 0;
    const double inf = __longlong_as_double((long long)FP_INF);
    if (g[vt] != FP_INF) {
        r.kind = ISDF_FRONTIER_GOAL; r.voxel = vt; r.cluster = -1;
        r.g = r.score = __longlong_as_double((long long)g[vt]);
        for (int a = 0; a < 3; a++) r.point[a] = A.goals[3 * (size_t)b + a];
    } else if (A.pick[b] != 0xffffffffu) {
        const int i = (int)A.pick[b];
        const long long v = A.vox[i];
        r.kind = ISDF_FRONTIER_FRONTIER; r.voxel = v; r.cluster = A.cid[i];
        r.g = __longlong_as_double((long long)g[v]);
        r.score = __longlong_as_double((long long)A.best[b]);
        for (int a = 0; a < 3; a++) r.point[a] = fg_centre(G, v, a);
        if (A.gain) r.gain = (int32_t)min(A.gain[i], 2147483647ll);
    } else {
        r.kind = ISDF_FRONTIER_NONE; r.voxel = -1; r.cluster = -1;
        r.g = r.score = inf;
        for (int a = 0; a < 3; a++) r.point[a] = A.goals[3 * (size_t)b + a];
    }
    A.out[b] = r;
}

// cand[i] = the cluster of list position i has at least min_voxels voxels
__global__ void k_fg_cand(int n, const int *parent, const int *slot, const int *size, int min_voxels, uint8_t *cand) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cand[i] = size[slot[parent[i]]] >= min_voxels;
}

// the view-gain poses of the frontier list: position i at f's cube centre, quaternion (1, 0, 0, 0), 7 doubles per pose
__global__ void k_fg_view_poses(const DevGrid G, int n, const long long *vox, double *pose) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double *o = pose + 7 * (size_t)i;
    for (int a = 0; a < 3; a++) o[a] = fg_centre(G, vox[i], a);
    o[3] = 1.0; o[4] = o[5] = o[6] = 0.0;
}

// the gain rule folded into the candidates: cand[i] = cand[i] and gain[i] >= min_gain
__global__ void k_fg_gain_cand(int n, const long long *gain, long long min_gain, uint8_t *cand) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cand[i] = cand[i] && gain[i] >= min_gain;
}

}  // namespace isdf
