// Front-end path search: the exact shortest 26-connected path over the attitude-feasible voxels, as a cost-to-come FIELD.
//
// Reference: AstarPathSearcher::AstarPathSearch / getPath / getastarSE3Path (front_end_Astar.hpp:197-402), a serial A* that calls
// checkKernelValue once per neighbour of every expanded node. A voxel can be entered iff it is in the map, not occupied and SOME attitude
// fits there (visit_kernels_by_distance tries every attitude), i.e. iff its feasibility mask is not zero: a property of the voxel alone.
// So the search is a shortest-path problem on a fixed graph, and its cost-to-come field is data-parallel.
//
// GPU mapping (S sources share one launch; grid.y is the source, and source s owns field slice g + s*X*Y*Z, its own pair of frontier bit
// sets and its own flag ring):
//   traversability  the feasibility kernels of isdf_frontend.cuh in their traversability output mode: one bit per voxel, grid.bits' layout
//   k_fp_init       g = +inf everywhere, g(source) = 0, the source in its frontier 0
//   k_fp_relax[_multi] one round of label-correcting relaxation: a thread per 32-voxel word of its source's current frontier; every frontier
//                   voxel u offers g(u) + w to its 26 neighbours with atomicMin on the bit pattern of the non-negative double
//                   (order-preserving, so the result does not depend on the order, nor on which sources share the launch); improved voxels
//                   form the next frontier. Rounds are launched in chunks; a CTA whose source's frontier is empty returns at once, and the
//                   host reads one aggregate flag (some source has a frontier) per chunk.
//   WEIGHTED        the relaxations and the walk are templated on the unknown-voxel surcharge (isdf_frontpath_params.unknown_weight):
//                   the weighted instances multiply the edge into a voxel that is not KNOWN by 1 + unknown_weight (fp_weight); weight 0
//                   launches the unweighted instances, whose code is the surcharge-free kernels' own
//   k_fp_walk       one warp per target: lane l tests offset l of the parent rule on the target's field slice, the first lane of the
//                   ballot is the parent. Pass 0 counts the path, pass 1 writes its voxel indices into scratch.
//   k_fp_place      one warp per path: from scratch to its place in pair order, with the cube centres
//   k_fp_node_masks the colliding-attitude set of every path node (frontend_colliding: the mask OR of isdf_frontend_check_batch)
//   k_fp_attitudes  one thread per target: the attitude chain along its path, frontend_visit from the father's attitude
#pragma once
#include "isdf_frontend.cuh"

namespace isdf {

constexpr unsigned long long FP_INF = 0x7ff0000000000000ull;   // +inf as a bit pattern: above every finite non-negative double
constexpr int FP_FLAG_RING = 4;                                  // flags[r % ring] != 0: round r has a frontier
constexpr long long FP_FIELD_BUDGET = 4ll << 30;                 // bytes of fields held at once when the caller sets no limit (max_fields 0)

struct PathArgs {
    DevGrid grid;
    const uint32_t *trav;        // traversability bits, grid.bits' layout
    unsigned long long *g;       // one field per source, X*Y*Z FP64 bit patterns each: source s at g + s*X*Y*Z, address ix*Y*Z + iy*Z + iz
    uint32_t *front;             // two frontier bit sets per source (even / odd rounds), grid.bits' layout: source s's at front + 2*s*X*Y*Zw
    uint32_t *front1;            // one source: its odd-round set (k_fp_relax)
    unsigned *flags;             // FP_FLAG_RING words per source
    unsigned *any;               // FP_FLAG_RING words: some source has a frontier in round r (the flags themselves for one source)
    unsigned *rounds;            // rounds in which some source had a frontier
    const int *src;              // 3 per source: the source voxels
    // targets and paths
    int nt;
    const int *tgt;              // nt x 3
    const int *tsrc;             // nt x 4: the target's source voxel and the slice of its field
    const int *pair;             // nt: the target's pair index (cost, found)
    int *len;                    // nt: path length in nodes (pass 0)
    const int *off;              // nt + 1: first node of each path (walk pass 1: in scratch; place and attitudes: in pair order)
    const int *soff;             // nt: first node of each path in scratch (place)
    int *scratch;                // 3 per node: the walk's voxel indices
    int *nodes;                  // 3 per node
    double *xyz;                 // 3 per node: cube centres
    double *rp;                  // 2 per node: roll, pitch
    double *cost;                // per pair
    uint8_t *found;              // per pair
    const uint32_t *colliding;   // 4 per node (k_fp_node_masks)
};

// the surcharge on unknown voxels, read by the WEIGHTED instances only. A parameter after the kernels' own, so that the unweighted
// instances keep the surcharge-free kernels' parameter offsets and code.
struct FpSurcharge {
    const uint32_t *known;       // the map's KNOWN bits, grid.bits' layout (NULL: nothing is known)
    double cw;                   // 1 + unknown_weight: the factor on an edge into a voxel that is not known
};

__device__ __forceinline__ bool fp_trav(const PathArgs &P, int x, int y, int z) {
    return (__ldg(P.trav + ((size_t)x * P.grid.Y + y) * P.grid.Zw + (z >> 5)) >> (z & 31)) & 1u;
}
// edge cost sqrt(i*i + j*j + k*k) of front_end_Astar.hpp:230 (IEEE sqrt: correctly rounded)
__device__ __forceinline__ double fp_edge(int n) { return sqrt((double)n); }
// the edge into v = (x, y, z): fp_edge, times cw when v is not known (one rounded product; the unit is compiled with -fmad=false, so the
// sum g(u) + w is not contracted either)
template <bool WEIGHTED>
__device__ __forceinline__ double fp_weight(const PathArgs &P, const FpSurcharge &U, int n, int x, int y, int z) {
    if (!WEIGHTED) return fp_edge(n);
    const bool known = U.known && ((__ldg(U.known + ((size_t)x * P.grid.Y + y) * P.grid.Zw + (z >> 5)) >> (z & 31)) & 1u);
    return fp_edge(n) * (known ? 1.0 : U.cw);
}

__global__ void k_fp_init(const __grid_constant__ PathArgs P) {
    const int s = blockIdx.y;
    const long long nvox = (long long)P.grid.X * P.grid.Y * P.grid.Z;
    const int sx = P.src[3 * s], sy = P.src[3 * s + 1], sz = P.src[3 * s + 2];
    const long long v0 = ((long long)sx * P.grid.Y + sy) * P.grid.Z + sz;
    unsigned long long *g = P.g + (size_t)s * nvox;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvox; v += (long long)gridDim.x * blockDim.x) {
        g[v] = (v == v0) ? 0ull : FP_INF;
        if (v == v0) {
            P.front[(size_t)2 * s * P.grid.X * P.grid.Y * P.grid.Zw + ((size_t)sx * P.grid.Y + sy) * P.grid.Zw + (sz >> 5)] = 1u << (sz & 31);
            P.flags[(size_t)s * FP_FLAG_RING] = 1u;
            P.any[0] = 1u;
        }
    }
}

// one source (S = 1): its flag ring is also the aggregate one (P.any == P.flags). WEIGHTED: the unknown-voxel surcharge (fp_weight).
// The weighted instances ask for one resident CTA (minBlocks 1): left to itself ptxas held them to 64 registers with 28 bytes of spills;
// with it they take 76 and spill nothing. minBlocks 0 leaves the unweighted instances' code exactly as it was (64 and 78 registers).
template <bool WEIGHTED>
__global__ void __launch_bounds__(256, WEIGHTED ? 1 : 0) k_fp_relax(const __grid_constant__ PathArgs P, int r, const FpSurcharge U) {
    // the flag of round r + 2 is cleared before anyone can set it (round r + 1 sets it); round r sets the flag of round r + 1
    if (blockIdx.x == 0 && threadIdx.x == 0) P.flags[(r + 2) % FP_FLAG_RING] = 0u;
    if (*(volatile unsigned *)(P.flags + r % FP_FLAG_RING) == 0u) return;
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(P.rounds, 1u);
    const DevGrid &G = P.grid;
    uint32_t *cur = (r & 1) ? P.front1 : P.front, *nxt = (r & 1) ? P.front : P.front1;
    const long long nword = (long long)G.X * G.Y * G.Zw;
    bool improved = false;
    for (long long wi = (long long)blockIdx.x * blockDim.x + threadIdx.x; wi < nword; wi += (long long)gridDim.x * blockDim.x) {
        uint32_t bits = cur[wi];
        if (!bits) continue;
        cur[wi] = 0u;   // this set becomes round r + 2's next frontier
        const int zw = (int)(wi % G.Zw), iy = (int)((wi / G.Zw) % G.Y), ix = (int)(wi / ((long long)G.Zw * G.Y));
        while (bits) {
            const int iz = 32 * zw + __ffs((int)bits) - 1;
            bits &= bits - 1;
            // a value read while another thread lowers it is still the cost of a path; the lowering thread re-queues u
            const double gu = __longlong_as_double((long long)__ldcg(P.g + ((size_t)ix * G.Y + iy) * G.Z + iz));
            for (int di = -1; di <= 1; di++) {
                const int x = ix + di;
                if (x < 0 || x >= G.X) continue;
                for (int dj = -1; dj <= 1; dj++) {
                    const int y = iy + dj;
                    if (y < 0 || y >= G.Y) continue;
                    for (int dk = -1; dk <= 1; dk++) {
                        const int z = iz + dk;
                        if (z < 0 || z >= G.Z || (di == 0 && dj == 0 && dk == 0) || !fp_trav(P, x, y, z)) continue;
                        const unsigned long long cand = (unsigned long long)__double_as_longlong(gu + fp_weight<WEIGHTED>(P, U, di * di + dj * dj + dk * dk, x, y, z));
                        unsigned long long *gv = P.g + ((size_t)x * G.Y + y) * G.Z + z;
                        if (cand >= __ldcg(gv)) continue;
                        if (cand < atomicMin(gv, cand)) {
                            atomicOr(nxt + ((size_t)x * G.Y + y) * G.Zw + (z >> 5), 1u << (z & 31));
                            improved = true;
                        }
                    }
                }
            }
        }
    }
    if (__any_sync(0xffffffffu, improved) && (threadIdx.x & 31) == 0) P.flags[(r + 1) % FP_FLAG_RING] = 1u;
}

// S > 1 (grid.y = S). One source keeps k_fp_relax above: this form needs the per-source offsets and the aggregate flag, and at S = 1 it
// took 553 ms against the single-source kernel's 530-536 ms for the bench_frontpath.py field at 512^3 on an H100 (78 registers against 64)
template <bool WEIGHTED>
__global__ void __launch_bounds__(256, WEIGHTED ? 1 : 0) k_fp_relax_multi(const __grid_constant__ PathArgs P, int r, const FpSurcharge U) {
    const int s = blockIdx.y;
    unsigned *flags = P.flags + (size_t)s * FP_FLAG_RING;
    // the flags of round r + 2 are cleared before anyone can set them (round r + 1 sets them); round r sets those of round r + 1
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        flags[(r + 2) % FP_FLAG_RING] = 0u;
        if (s == 0) {
            P.any[(r + 2) % FP_FLAG_RING] = 0u;
            if (*(volatile unsigned *)(P.any + r % FP_FLAG_RING)) atomicAdd(P.rounds, 1u);
        }
    }
    if (*(volatile unsigned *)(flags + r % FP_FLAG_RING) == 0u) return;
    const DevGrid &G = P.grid;
    const long long nword = (long long)G.X * G.Y * G.Zw;
    unsigned long long *g = P.g + (size_t)s * G.X * G.Y * G.Z;
    uint32_t *cur = P.front + (size_t)(2 * s + (r & 1)) * nword, *nxt = P.front + (size_t)(2 * s + 1 - (r & 1)) * nword;
    bool improved = false;
    for (long long wi = (long long)blockIdx.x * blockDim.x + threadIdx.x; wi < nword; wi += (long long)gridDim.x * blockDim.x) {
        uint32_t bits = cur[wi];
        if (!bits) continue;
        cur[wi] = 0u;   // this set becomes round r + 2's next frontier
        const int zw = (int)(wi % G.Zw), iy = (int)((wi / G.Zw) % G.Y), ix = (int)(wi / ((long long)G.Zw * G.Y));
        while (bits) {
            const int iz = 32 * zw + __ffs((int)bits) - 1;
            bits &= bits - 1;
            // a value read while another thread lowers it is still the cost of a path; the lowering thread re-queues u
            const double gu = __longlong_as_double((long long)__ldcg(g + ((size_t)ix * G.Y + iy) * G.Z + iz));
            for (int di = -1; di <= 1; di++) {
                const int x = ix + di;
                if (x < 0 || x >= G.X) continue;
                for (int dj = -1; dj <= 1; dj++) {
                    const int y = iy + dj;
                    if (y < 0 || y >= G.Y) continue;
                    for (int dk = -1; dk <= 1; dk++) {
                        const int z = iz + dk;
                        if (z < 0 || z >= G.Z || (di == 0 && dj == 0 && dk == 0) || !fp_trav(P, x, y, z)) continue;
                        const unsigned long long cand = (unsigned long long)__double_as_longlong(gu + fp_weight<WEIGHTED>(P, U, di * di + dj * dj + dk * dk, x, y, z));
                        unsigned long long *gv = g + ((size_t)x * G.Y + y) * G.Z + z;
                        if (cand >= __ldcg(gv)) continue;
                        if (cand < atomicMin(gv, cand)) {
                            atomicOr(nxt + ((size_t)x * G.Y + y) * G.Zw + (z >> 5), 1u << (z & 31));
                            improved = true;
                        }
                    }
                }
            }
        }
    }
    if (__any_sync(0xffffffffu, improved) && (threadIdx.x & 31) == 0) {
        flags[(r + 1) % FP_FLAG_RING] = 1u;
        P.any[(r + 1) % FP_FLAG_RING] = 1u;
    }
}

// parent rule on field g: among the 26 neighbours u of v with g(u) + w(u, v) == g(v), the first in the reference's offset order (i, j,
// k = -1..1, i outermost; lane = 9 (i + 1) + 3 (j + 1) + (k + 1)). w is v's edge weight: WEIGHTED reads the known bit of v, the node the
// walk steps from. The whole warp calls this.
template <bool WEIGHTED>
__device__ __forceinline__ bool fp_parent(const PathArgs &P, const FpSurcharge &U, const unsigned long long *g, int &x, int &y, int &z, int lane) {
    const DevGrid &G = P.grid;
    const double gv = __longlong_as_double((long long)g[((size_t)x * G.Y + y) * G.Z + z]);
    const int di = lane / 9 - 1, dj = (lane / 3) % 3 - 1, dk = lane % 3 - 1;
    const int ux = x + di, uy = y + dj, uz = z + dk;
    bool ok = false;
    if (lane < 27 && lane != 13 && ux >= 0 && ux < G.X && uy >= 0 && uy < G.Y && uz >= 0 && uz < G.Z) {
        const unsigned long long gu = g[((size_t)ux * G.Y + uy) * G.Z + uz];
        ok = gu != FP_INF && __longlong_as_double((long long)gu) + fp_weight<WEIGHTED>(P, U, di * di + dj * dj + dk * dk, x, y, z) == gv;
    }
    const unsigned b = __ballot_sync(0xffffffffu, ok);
    if (!b) return false;
    const int l = __ffs((int)b) - 1;
    x += l / 9 - 1; y += (l / 3) % 3 - 1; z += l % 3 - 1;
    return true;
}

template <bool WEIGHTED>
__global__ void __launch_bounds__(128) k_fp_walk(const __grid_constant__ PathArgs P, int pass, const FpSurcharge U) {
    const int t = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (t >= P.nt) return;   // whole warps
    const DevGrid &G = P.grid;
    const int *ts = P.tsrc + 4 * (size_t)t;
    const int sx = ts[0], sy = ts[1], sz = ts[2];
    const unsigned long long *g = P.g + (size_t)ts[3] * G.X * G.Y * G.Z;
    int x = P.tgt[3 * t], y = P.tgt[3 * t + 1], z = P.tgt[3 * t + 2];
    const unsigned long long gt = g[((size_t)x * G.Y + y) * G.Z + z];
    const bool found = gt != FP_INF;
    auto put = [&](int k, int px, int py, int pz) {
        if (lane != 0) return;
        int *n = P.scratch + 3 * (size_t)k;
        n[0] = px; n[1] = py; n[2] = pz;
    };
    if (!found) {   // no path: the target's start alone
        if (pass == 0) { if (lane == 0) { P.len[t] = 1; P.found[P.pair[t]] = 0; P.cost[P.pair[t]] = __longlong_as_double((long long)FP_INF); } }
        else put(P.off[t], sx, sy, sz);
        return;
    }
    // g strictly decreases along parents (every edge costs >= 1), so the walk ends at the source within X*Y*Z steps
    const long long cap = (long long)G.X * G.Y * G.Z;
    long long n = 1;
    const int last = (pass == 1) ? P.off[t + 1] - 1 : 0;
    if (pass == 1) put(last, x, y, z);
    while (!(x == sx && y == sy && z == sz) && n < cap) {
        if (!fp_parent<WEIGHTED>(P, U, g, x, y, z, lane)) break;
        if (pass == 1) put(last - (int)n, x, y, z);
        n++;
    }
    if (pass == 0 && lane == 0) { P.len[t] = (int)n; P.found[P.pair[t]] = 1; P.cost[P.pair[t]] = __longlong_as_double((long long)gt); }
}

// path b from scratch (soff[b]) to nodes[off[b]..] in pair order, with its cube centres (getGridCubeCenter, Gridmap3D.cpp:177-194)
__global__ void __launch_bounds__(128) k_fp_place(const __grid_constant__ PathArgs P) {
    const int b = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (b >= P.nt) return;
    const DevGrid &G = P.grid;
    const int a = P.off[b], n = P.off[b + 1] - a;
    const int *from = P.scratch + 3 * (size_t)P.soff[b];
    for (int k = lane; k < n; k += 32) {
        const int px = from[3 * k], py = from[3 * k + 1], pz = from[3 * k + 2];
        int *o = P.nodes + 3 * ((size_t)a + k);
        o[0] = px; o[1] = py; o[2] = pz;
        double *c = P.xyz + 3 * ((size_t)a + k);
        c[0] = (px + 0.5) * G.res + G.bmin[0]; c[1] = (py + 0.5) * G.res + G.bmin[1]; c[2] = (pz + 0.5) * G.res + G.bmin[2];
    }
}

// the colliding-attitude set of each of n path nodes (A.q_ind = the nodes, A.out = 4 words per node)
__global__ void __launch_bounds__(256) k_fp_node_masks(const __grid_constant__ FrontArgs A) {
    extern __shared__ __align__(16) uint32_t fe_sm[];
    frontend_stage_masks(A, fe_sm);
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= A.nq) return;
    uint32_t m[4];
    frontend_colliding(A, fe_sm, A.q_ind[3 * q], A.q_ind[3 * q + 1], A.q_ind[3 * q + 2], m);
    for (int k = 0; k < 4; k++) A.out[4 * (size_t)q + k] = m[k];
}

// node 0 level, node m + 1 = checkKernelValue(attitude of node m, node m + 1): isdf_frontend_check_batch applied as a chain
__global__ void k_fp_attitudes(const __grid_constant__ FrontArgs A, const __grid_constant__ PathArgs P) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.nt) return;
    const int a = P.off[t], b = P.off[t + 1];
    double fr = 0.0, fp = 0.0;
    P.rp[2 * (size_t)a] = 0.0; P.rp[2 * (size_t)a + 1] = 0.0;
    for (int k = a + 1; k < b; k++) {
        const uint32_t *c = P.colliding + 4 * (size_t)k;
        const uint32_t m[4] = {c[0], c[1], c[2], c[3]};
        double cr, cp;
        frontend_visit(A, m, fr, fp, cr, cp);
        P.rp[2 * (size_t)k] = cr; P.rp[2 * (size_t)k + 1] = cp;
        fr = cr; fp = cp;
    }
}

}  // namespace isdf
