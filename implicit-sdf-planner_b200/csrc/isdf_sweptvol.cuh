// Certified swept volume of one trajectory (isdf_swept_volume_*, include/isdf.h): SV(p) = min over t of sd(R(t)^T (p - x(t))) with a
// proven enclosure [lower, value], at caller points or at the nodes of a grid, and the surface {SV = 0} of a grid as a triangle mesh.
//
// Per point p (DESIGN §3.12 has the derivation): the certificate's initial intervals (K per piece) with their motion bounds D_a, D_b
// (cert_bound, isdf_certify.cuh). For a shape whose SDF is a signed Euclidean distance, sd_t(p) >= sd_e(p) - D_e on an interval, so
// lb = max(sd_a - D_a, sd_b - D_b) (cert_lb) bounds SV from below on it, and every evaluated sample bounds it from above.
//   sphere cull  an interval with max_e(|p - x(t_e)| - r_body - D_e) >= band (rounded down) cannot reach below band: dropped unevaluated;
//   rounds       level-synchronous: with hi as it stood at the round's start, an interval with lb < hi - tol is split at its midpoint
//                (the midpoint is evaluated) until max_depth or the point's sample budget (earlier intervals first); the rest are leaves.
//   result       value = hi (capped at band), lower = min(hi, min leaf lb), t* (earliest time attaining hi, -1 when hi == band),
//                decided = lower >= hi - tol.
//
// Mapping:
//   * k_sv_prep — the per-call pass: pose of every initial sample (the clearance scan's pose code), D_a / D_b of every initial interval,
//     piece start times. None of it depends on p.
//   * k_sv_bricks<FILL> — one warp per brick of SV_BRICK^3 grid nodes: the sphere cull with the brick's radius added (and a relative
//     slack that covers the node test's rounding), so a brick test that drops an interval implies every node's test drops it. Pass 0
//     counts, an exclusive scan gives offsets, pass 1 writes each brick's surviving interval indices in interval order.
//   * k_sv_refine<MODE> — persistent warps draw work items (bricks of a grid, or single points) from one counter. A brick without
//     candidates is written as band / decided with no SDF evaluation. Otherwise the warp runs each node: the exact per-node cull over the
//     brick's list (the same intervals, in the same order, as over all intervals: a node's result does not depend on its brick), then
//     the rounds with the interval lists in a per-warp global scratch. Analytic shapes: one lane per sample; exact-sign meshes: the warp
//     answers each sample cooperatively (mesh_sdf_grad_warp_lat). Which warp runs a node decides nothing: results depend only on p.
//   * marching tetrahedra — k_sv_mt_count (per node: crossed-edge mask and vertex count; per cell: triangle count), two exclusive scans,
//     k_sv_mt_emit (vertices and triangles at their scanned positions). No atomics decide a position.
// Vertex positions and node coordinates are written with __dadd_rn / __dmul_rn / __ddiv_rn: no contraction, so a NumPy restatement
// reproduces them bit for bit.
//
// Included by isdf_api.cu (argument block, launch interface) and isdf_clearance_tu.cu, which defines ISDF_CLEARANCE_TU and instantiates
// the kernels with the clearance scan's floating-point flags (the certificate's pose pad assumes that arithmetic).
#pragma once
#include "isdf_types.cuh"
#include "isdf_clearance.cuh"
#include "isdf_certify.cuh"

namespace isdf {

constexpr int SV_WARPS = 4;
constexpr int SV_THREADS = SV_WARPS * 32;
constexpr int SV_BRICK = 4;                // grid nodes per brick edge
constexpr int SV_SCAN_THREADS = 1024;

// an interval of the rounds: [ta, tb] of local time in `piece`, its sample times ta / tbs (tbs differs from tb only at a piece's last
// initial interval, as in the certificate), endpoint SDF values fa / fb and motion bounds Da / Db
struct SvolIv { double ta, tb, tbs, fa, fb, Da, Db; int piece, depth; };
static_assert(sizeof(SvolIv) == 64, "interval record");

struct SvolArgs {
    DevShape shape;
    FlatParams fp;
    double r_rot, r_body, band, tol;
    int N, K, max_depth, max_samples;
    const double *T, *C;           // N; 6N x 3 column-major
    double *toff;                  // N: trajectory time at which each piece starts
    double *pose;                  // N (K + 1) x 12: position, rows of R
    double *Dab;                   // N K x 2
    // nodes: a grid (pts == nullptr) or a point list
    double bmin[3], res;
    int X, Y, Z, BX, BY, BZ;
    const double *pts;             // npts x 3
    int npts;
    long long *boff;               // bricks + 1: candidate counts, then exclusive offsets (the last entry is the total)
    int *blist;                    // candidate interval indices of every brick, brick by brick
    double *value, *lower, *tstar; // per node / point (lower, tstar, decided may be null)
    uint8_t *decided;
    SvolIv *scratch;                 // per resident warp: scap records
    long long scap, split_at;      // split_at: start of the second list inside a warp's records
    int nwarps;
    int *cursor;
    unsigned long long *counters;  // {SDF evaluations, undecided nodes, deepest level, bricks culled}
};

// arguments of the marching-tetrahedra kernels
struct SvolMeshArgs {
    double bmin[3], res;
    int X, Y, Z;
    const double *value, *tstar;
    uint8_t *emask;                // per node: crossed edges (bit d: direction d)
    long long *voff, *foff;        // per node + 1: counts, then exclusive offsets
    double *V, *vtime;             // nV x 3, nV
    int32_t *F;                    // nF x 3
};

#ifdef ISDF_CLEARANCE_TU
// node coordinate bmin + (double) i * res without contraction
__device__ __forceinline__ double sv_coord(double bmin, double res, int i) { return __dadd_rn(bmin, __dmul_rn((double)i, res)); }

// ---- marching tetrahedra tables -------------------------------------------------------------------------------------------------
// edge directions of a node, by bits (x = 1, y = 2, z = 4): +x, +y, +z, +x+y, +x+z, +y+z, +x+y+z
static __device__ __constant__ const int SV_DIR_BITS[7] = {1, 2, 4, 3, 5, 6, 7};
static __device__ __constant__ const int SV_BITS_DIR[8] = {-1, 0, 1, 3, 2, 4, 5, 6};
// the 6 Kuhn tetrahedra {000, e_a, e_a + e_b, 111}, (a, b, c) in lexicographic order, as corner bits of v0..v3; orientation = the
// permutation's sign (det[e_a, e_a + e_b, 111] = det[e_a, e_b, e_c])
static __device__ __constant__ const int SV_TET[6][4] = {{0, 1, 3, 7}, {0, 1, 5, 7}, {0, 2, 3, 7}, {0, 2, 6, 7}, {0, 4, 5, 7}, {0, 4, 6, 7}};
static __device__ __constant__ const int SV_TET_POS[6] = {1, 0, 0, 1, 1, 0};
// an even permutation (i, j, k, l) of (0, 1, 2, 3) starting with i
static __device__ __constant__ const int SV_EVEN[4][4] = {{0, 1, 2, 3}, {1, 0, 3, 2}, {2, 3, 0, 1}, {3, 2, 1, 0}};

// ---- helpers -----------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sv_absdiff_rd(double a, double b) { return a >= b ? __dadd_rd(a, -b) : __dadd_rd(b, -a); }
// |p - x| rounded down
__device__ __forceinline__ double sv_dist_rd(double px, double py, double pz, const double *x) {
    const double dx = sv_absdiff_rd(px, x[0]), dy = sv_absdiff_rd(py, x[1]), dz = sv_absdiff_rd(pz, x[2]);
    return __dsqrt_rd(__dadd_rd(__dadd_rd(__dmul_rd(dx, dx), __dmul_rd(dy, dy)), __dmul_rd(dz, dz)));
}
// the sphere cull's bound of one endpoint: |p - x_e| - r_body - D_e, rounded down
__device__ __forceinline__ double sv_cull_bound(double px, double py, double pz, const double *x, double rb, double D) {
    return __dadd_rd(__dadd_rd(sv_dist_rd(px, py, pz, x), -rb), -D);
}

// the clearance scan's pose (piece_eval, flat_quat_only, quat_rot) of piece i at local time t: position, rows of R
__device__ __forceinline__ void sv_pose(const SvolArgs &A, int i, double t, double *out) {
    double cx[6], cy[6], cz[6];
#pragma unroll
    for (int k = 0; k < 6; k++) { cx[k] = __ldg(A.C + 6 * i + k); cy[k] = __ldg(A.C + 6 * A.N + 6 * i + k); cz[k] = __ldg(A.C + 12 * A.N + 6 * i + k); }
    PieceEval pe;
    piece_eval(cx, cy, cz, t, pe);
    const quat4 q = flat_quat_only(A.fp, pe.vel, pe.acc);
    const rot3 R = quat_rot(q);
    out[0] = pe.pos.x; out[1] = pe.pos.y; out[2] = pe.pos.z;
    out[3] = R.r0.x; out[4] = R.r0.y; out[5] = R.r0.z; out[6] = R.r1.x; out[7] = R.r1.y; out[8] = R.r1.z; out[9] = R.r2.x; out[10] = R.r2.y; out[11] = R.r2.z;
}

// body-frame query point of p at a pose
__device__ __forceinline__ d3 sv_body_point(const double *ps, d3 p) {
    rot3 R;
    R.r0 = mk3(ps[3], ps[4], ps[5]); R.r1 = mk3(ps[6], ps[7], ps[8]); R.r2 = mk3(ps[9], ps[10], ps[11]);
    return rot_applyT(R, p - mk3(ps[0], ps[1], ps[2]));
}

// (value, time) order of the upper bound: smaller value, then earlier time
__device__ __forceinline__ bool sv_key_less(double v, double t, double bv, double bt) { return v < bv || (v == bv && t < bt); }
__device__ __forceinline__ void sv_warp_keymin(double &v, double &t) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o), ot = __shfl_xor_sync(0xffffffffu, t, o);
        if (sv_key_less(ov, ot, v, t)) { v = ov; t = ot; }
    }
}

// SDF of the shape at p for the pose of every lane in `mask`: analytic shapes per lane; meshes one warp-cooperative query per lane
template <int MODE>
__device__ __forceinline__ double sv_sdf(const SvolArgs &A, d3 p, const double *ps, bool want, int lane, WideStack *stk) {
    double out = 0.0;
    if (MODE == 0) {
        if (want) out = shape_sdf_analytic(A.shape, sv_body_point(ps, p));
        return out;
    }
    unsigned m = __ballot_sync(0xffffffffu, want);
    while (m) {
        const int l = __ffs(m) - 1;
        m &= m - 1;
        double q[12];
#pragma unroll
        for (int k = 0; k < 12; k++) q[k] = __shfl_sync(0xffffffffu, ps[k], l);
        d3 g;
        const double s = mesh_sdf_grad_warp_lat(A.shape.mesh, sv_body_point(q, p), A.band, g, lane, stk);
        if (lane == l) out = s;
    }
    return out;
}

// ---- per-call pass ----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CERT_THREADS) k_sv_prep(const __grid_constant__ SvolArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x, K = A.K;
    if (k < A.N * (K + 1)) {   // samples: the certificate's initial samples, j * step
        const int i = k / (K + 1), j = k - i * (K + 1);
        sv_pose(A, i, j * (A.T[i] * (1.0 / K)), A.pose + 12 * (size_t)k);
    }
    if (k < A.N * K) {         // intervals: [j step, (j + 1) step], the last one ending at T_i
        const int i = k / K, j = k - i * K;
        const double step = A.T[i] * (1.0 / K), ta = j * step, tbs = (j + 1) * step, tb = (j + 1 == K) ? A.T[i] : tbs;
        A.Dab[2 * k] = cert_bound(A.fp, A.r_rot, A.band, A.C, A.N, i, ta, tb, ta);
        A.Dab[2 * k + 1] = cert_bound(A.fp, A.r_rot, A.band, A.C, A.N, i, ta, tb, tbs);
    }
    if (k == 0) {
        double t = 0.0;
        for (int q = 0; q < A.N; q++) { A.toff[q] = t; t += A.T[q]; }
    }
}

// ---- brick cull ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void sv_brick_range(const SvolArgs &A, int b, int lo[3], int hi[3]) {
    const int bz = b % A.BZ, by = (b / A.BZ) % A.BY, bx = b / (A.BZ * A.BY);
    lo[0] = bx * SV_BRICK; lo[1] = by * SV_BRICK; lo[2] = bz * SV_BRICK;
    hi[0] = min(lo[0] + SV_BRICK, A.X) - 1; hi[1] = min(lo[1] + SV_BRICK, A.Y) - 1; hi[2] = min(lo[2] + SV_BRICK, A.Z) - 1;
}

template <bool FILL>
__global__ void __launch_bounds__(SV_THREADS) k_sv_bricks(const __grid_constant__ SvolArgs A, int nbricks) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * SV_WARPS + (threadIdx.x >> 5);
    if (b >= nbricks) return;
    int lo[3], hi[3];
    sv_brick_range(A, b, lo, hi);
    double c[3], rho2 = 0.0;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double plo = sv_coord(A.bmin[a], A.res, lo[a]), phi = sv_coord(A.bmin[a], A.res, hi[a]);
        c[a] = 0.5 * (plo + phi);
        const double h = fmax(__dadd_ru(phi, -c[a]), __dadd_ru(c[a], -plo));
        rho2 = __dadd_ru(rho2, __dmul_ru(h, h));
    }
    const double rho = __dsqrt_ru(rho2), rb = __dadd_ru(A.r_body, rho);
    const int NK = A.N * A.K;
    long long pos = FILL ? A.boff[b] : 0;
    for (int base = 0; base < NK; base += 32) {
        const int q = base + lane;
        bool keep = false;
        if (q < NK) {
            const int i = q / A.K, s = q + i;   // sample index of the interval's first endpoint
            const double Da = A.Dab[2 * q], Db = A.Dab[2 * q + 1];
            const double *xa = A.pose + 12 * (size_t)s, *xb = xa + 12;
            const double da = sv_dist_rd(c[0], c[1], c[2], xa), db = sv_dist_rd(c[0], c[1], c[2], xb);
            // the node test rounds |p - x| - r_body - D_e down on its own: the slack keeps "brick drops" => "node drops"
            const double La = __dadd_rd(__dadd_rd(da, -rb), -Da), Lb = __dadd_rd(__dadd_rd(db, -rb), -Db);
            const double sa = 1e-12 * (da + rb + Da), sb = 1e-12 * (db + rb + Db);
            keep = !(fmax(La - sa, Lb - sb) >= A.band);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (FILL && keep) A.blist[pos + __popc(bal & ((1u << lane) - 1u))] = q;
        pos += __popc(bal);
    }
    if (!FILL && lane == 0) A.boff[b] = pos;
}

// ---- per-node refinement ----------------------------------------------------------------------------------------------------------
template <int MODE>
__device__ void sv_node(const SvolArgs &A, d3 p, const int *cand, long long ncand, SvolIv *cur, SvolIv *nxt, int lane, WideStack *stk, long long out_idx,
                        unsigned long long &nevals, int &undecided, int &deepest) {
    const unsigned lt = (1u << lane) - 1u;
    const int K = A.K;
    const double band = A.band;
    double hv = band, ht = INFINITY;   // this lane's best (value, time)
    int nk = 0;
    int cq = -2, ck = 0;               // the previous chunk's last lane: interval, kept
    double cfb = 0.0;
    // round 0: the exact sphere cull, then the endpoint values of the kept intervals (a sample shared by two kept intervals once)
    for (long long base = 0; base < ncand; base += 32) {
        const long long k = base + lane;
        const bool valid = k < ncand;
        const int q = valid ? (cand ? __ldg(cand + k) : (int)k) : -1;
        int i = 0, j = 0, s = 0;
        double Da = 0, Db = 0;
        bool kept = false;
        if (valid) {
            i = q / K; j = q - i * K; s = q + i;
            Da = A.Dab[2 * q]; Db = A.Dab[2 * q + 1];
            const double La = sv_cull_bound(p.x, p.y, p.z, A.pose + 12 * (size_t)s, A.r_body, Da);
            const double Lb = sv_cull_bound(p.x, p.y, p.z, A.pose + 12 * (size_t)(s + 1), A.r_body, Db);
            kept = !(fmax(La, Lb) >= band);
        }
        int pq = __shfl_up_sync(0xffffffffu, q, 1), pk = __shfl_up_sync(0xffffffffu, (int)kept, 1);
        if (lane == 0) { pq = cq; pk = ck; }
        const bool need_a = kept && !(pk && pq == q - 1 && j != 0);
        double psa[12], psb[12];
        if (kept) {
#pragma unroll
            for (int t = 0; t < 12; t++) { psa[t] = A.pose[12 * (size_t)s + t]; psb[t] = A.pose[12 * (size_t)(s + 1) + t]; }
        } else {
#pragma unroll
            for (int t = 0; t < 12; t++) { psa[t] = 0.0; psb[t] = 0.0; }
        }
        double fa = sv_sdf<MODE>(A, p, psa, need_a, lane, stk);
        const double fb = sv_sdf<MODE>(A, p, psb, kept, lane, stk);
        nevals += __popc(__ballot_sync(0xffffffffu, need_a)) + __popc(__ballot_sync(0xffffffffu, kept));
        double pfb = __shfl_up_sync(0xffffffffu, fb, 1);
        if (lane == 0) pfb = cfb;
        if (kept && !need_a) fa = pfb;
        double ta = 0, tb = 0, tbs = 0;
        if (kept) {
            const double step = A.T[i] * (1.0 / K);
            ta = j * step; tbs = (j + 1) * step; tb = (j + 1 == K) ? A.T[i] : tbs;
            const double t0 = A.toff[i];
            if (need_a && sv_key_less(fa, t0 + ta, hv, ht)) { hv = fa; ht = t0 + ta; }
            if (sv_key_less(fb, t0 + tbs, hv, ht)) { hv = fb; ht = t0 + tbs; }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, kept);
        if (kept) {
            SvolIv I;
            I.ta = ta; I.tb = tb; I.tbs = tbs; I.fa = fa; I.fb = fb; I.Da = Da; I.Db = Db; I.piece = i; I.depth = 0;
            cur[nk + __popc(bal & lt)] = I;
        }
        nk += __popc(bal);
        cq = __shfl_sync(0xffffffffu, q, 31); ck = __shfl_sync(0xffffffffu, (int)kept, 31); cfb = __shfl_sync(0xffffffffu, fb, 31);
    }
    sv_warp_keymin(hv, ht);
    // rounds: split what the round-start hi does not settle, earlier intervals first within the budget
    double lo_leaf = INFINITY;
    int used = 0, dep = 0, n = nk;
    while (n > 0) {
        __syncwarp();
        const double hi0 = hv;
        int nn = 0;
        for (int base = 0; base < n; base += 32) {
            const int k = base + lane;
            const bool valid = k < n;
            SvolIv I;
            bool wants = false;
            double lb = 0.0, m = 0.0;
            if (valid) {
                I = cur[k];
                lb = cert_lb(I.fa, I.fb, I.Da, I.Db);
                m = I.ta + 0.5 * (I.tb - I.ta);
                wants = lb < hi0 - A.tol && I.depth < A.max_depth && I.ta < m && m < I.tb;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, wants);
            const int rank = __popc(bal & lt), allowed = max(A.max_samples - used, 0);
            const bool split = wants && rank < allowed;
            if (valid && !split) { lo_leaf = fmin(lo_leaf, lb != lb ? -INFINITY : lb); dep = max(dep, I.depth); }
            double ps[12];
            if (split) sv_pose(A, I.piece, m, ps);
            else {
#pragma unroll
                for (int t = 0; t < 12; t++) ps[t] = 0.0;
            }
            const double fm = sv_sdf<MODE>(A, p, ps, split, lane, stk);
            if (split) {
                const double tm = A.toff[I.piece] + m;
                if (sv_key_less(fm, tm, hv, ht)) { hv = fm; ht = tm; }
                SvolIv L = I, R = I;
                L.tb = m; L.tbs = m; L.fb = fm; L.depth = I.depth + 1;
                R.ta = m; R.fa = fm; R.depth = I.depth + 1;
                L.Da = cert_bound(A.fp, A.r_rot, band, A.C, A.N, I.piece, L.ta, L.tb, L.ta);
                L.Db = cert_bound(A.fp, A.r_rot, band, A.C, A.N, I.piece, L.ta, L.tb, L.tbs);
                R.Da = cert_bound(A.fp, A.r_rot, band, A.C, A.N, I.piece, R.ta, R.tb, R.ta);
                R.Db = cert_bound(A.fp, A.r_rot, band, A.C, A.N, I.piece, R.ta, R.tb, R.tbs);
                nxt[2 * (nn + rank)] = L; nxt[2 * (nn + rank) + 1] = R;
            }
            const int took = min(__popc(bal), allowed);
            nn += took; used += took; nevals += took;
        }
        sv_warp_keymin(hv, ht);
        SvolIv *t = cur; cur = nxt; nxt = t;
        n = 2 * nn;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo_leaf = fmin(lo_leaf, __shfl_xor_sync(0xffffffffu, lo_leaf, o)); dep = max(dep, __shfl_xor_sync(0xffffffffu, dep, o)); }
    const double hi = fmin(hv, band), lo = fmin(hi, lo_leaf);
    const bool dec = lo >= hi - A.tol;
    if (lane == 0) {
        A.value[out_idx] = hi;
        if (A.lower) A.lower[out_idx] = lo;
        if (A.tstar) A.tstar[out_idx] = hi == band ? -1.0 : ht;
        if (A.decided) A.decided[out_idx] = dec ? 1 : 0;
    }
    undecided += dec ? 0 : 1;
    deepest = max(deepest, dep);
}

// MODE 0: analytic shape, 1: exact-sign mesh. Work items: the bricks of a grid, or single points.
template <int MODE>
__global__ void __launch_bounds__(SV_THREADS) k_sv_refine(const __grid_constant__ SvolArgs A, int nitems) {
    __shared__ WideStack stks[SV_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gw = blockIdx.x * SV_WARPS + warp;
    SvolIv *cur = A.scratch + gw * A.scap, *nxt = cur + A.split_at;
    unsigned long long nevals = 0;
    int undecided = 0, deepest = 0, culled = 0;
    for (;;) {
        int w = 0;
        if (lane == 0) w = atomicAdd(A.cursor, 1);
        w = __shfl_sync(0xffffffffu, w, 0);
        if (w >= nitems) break;
        if (!A.pts) {
            int lo[3], hi[3];
            sv_brick_range(A, w, lo, hi);
            const long long off = A.boff[w], cnt = A.boff[w + 1] - off;
            const int ny = hi[1] - lo[1] + 1, nz = hi[2] - lo[2] + 1, nb = (hi[0] - lo[0] + 1) * ny * nz;
            if (cnt == 0) {   // no interval reaches below band anywhere in the brick
                for (int u = lane; u < nb; u += 32) {
                    const int ix = lo[0] + u / (ny * nz), iy = lo[1] + (u / nz) % ny, iz = lo[2] + u % nz;
                    const long long a = ((long long)ix * A.Y + iy) * A.Z + iz;
                    A.value[a] = A.band;
                    if (A.lower) A.lower[a] = A.band;
                    if (A.tstar) A.tstar[a] = -1.0;
                    if (A.decided) A.decided[a] = 1;
                }
                culled++;
                continue;
            }
            for (int u = 0; u < nb; u++) {
                const int ix = lo[0] + u / (ny * nz), iy = lo[1] + (u / nz) % ny, iz = lo[2] + u % nz;
                const d3 p = mk3(sv_coord(A.bmin[0], A.res, ix), sv_coord(A.bmin[1], A.res, iy), sv_coord(A.bmin[2], A.res, iz));
                sv_node<MODE>(A, p, A.blist + off, cnt, cur, nxt, lane, &stks[warp], ((long long)ix * A.Y + iy) * A.Z + iz, nevals, undecided, deepest);
            }
        } else {
            const d3 p = mk3(A.pts[3 * (size_t)w], A.pts[3 * (size_t)w + 1], A.pts[3 * (size_t)w + 2]);
            sv_node<MODE>(A, p, nullptr, (long long)A.N * A.K, cur, nxt, lane, &stks[warp], w, nevals, undecided, deepest);
        }
    }
    if (lane == 0 && A.counters) {
        if (nevals) atomicAdd(A.counters, nevals);
        if (undecided) atomicAdd(A.counters + 1, (unsigned long long)undecided);
        if (deepest) atomicMax(A.counters + 2, (unsigned long long)deepest);
        if (culled) atomicAdd(A.counters + 3, (unsigned long long)culled);
    }
}

// ---- exclusive scan of n counts (n + 1 entries: the last one receives the total) -------------------------------------------------------
// exclusive scan over the SV_SCAN_THREADS (= 32 warps) threads of a block; every thread gets the block total
__device__ __forceinline__ long long sv_block_scan(long long v, long long &total) {
    __shared__ long long s_w[32];
    __shared__ long long s_tot;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_w[w] = x;
    __syncthreads();
    if (w == 0) {
        const long long y = s_w[lane];
        long long z = y;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const long long u = __shfl_up_sync(0xffffffffu, z, o); if (lane >= o) z += u; }
        s_w[lane] = z - y;
        if (lane == 31) s_tot = z;
    }
    __syncthreads();
    const long long r = s_w[w] + x - v;
    total = s_tot;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(SV_SCAN_THREADS) k_sv_scan_blocks(long long *a, long long n, long long *bsum) {
    const long long k = (long long)blockIdx.x * SV_SCAN_THREADS + threadIdx.x;
    const long long v = k < n ? a[k] : 0;
    long long total = 0;
    const long long r = sv_block_scan(v, total);
    if (k < n) a[k] = r;
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SV_SCAN_THREADS) k_sv_scan_top(long long *bsum, long long nb, long long *a, long long n) {
    long long run = 0;
    for (long long base = 0; base < nb; base += SV_SCAN_THREADS) {
        const long long k = base + threadIdx.x;
        const long long v = k < nb ? bsum[k] : 0;
        long long total = 0;
        const long long r = sv_block_scan(v, total);
        if (k < nb) bsum[k] = run + r;
        run += total;
    }
    if (threadIdx.x == 0) a[n] = run;
}
__global__ void __launch_bounds__(SV_SCAN_THREADS) k_sv_scan_add(long long *a, long long n, const long long *bsum) {
    const long long k = (long long)blockIdx.x * SV_SCAN_THREADS + threadIdx.x;
    if (k < n) a[k] += bsum[blockIdx.x];
}

// ---- marching tetrahedra --------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool sv_inside(double f) { return f < 0.0; }

// per node: crossed-edge mask and vertex count; triangles of the cell whose lowest corner is the node
__global__ void __launch_bounds__(256) k_sv_mt_count(const __grid_constant__ SvolMeshArgs M) {
    const long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x, n = (long long)M.X * M.Y * M.Z;
    if (a >= n) return;
    const int iz = (int)(a % M.Z), iy = (int)((a / M.Z) % M.Y), ix = (int)(a / ((long long)M.Y * M.Z));
    const bool in0 = sv_inside(M.value[a]);
    unsigned mask = 0;
    for (int d = 0; d < 7; d++) {
        const int b = SV_DIR_BITS[d], jx = ix + (b & 1), jy = iy + ((b >> 1) & 1), jz = iz + ((b >> 2) & 1);
        if (jx >= M.X || jy >= M.Y || jz >= M.Z) continue;
        if (sv_inside(M.value[((long long)jx * M.Y + jy) * M.Z + jz]) != in0) mask |= 1u << d;
    }
    M.emask[a] = (uint8_t)mask;
    M.voff[a] = __popc(mask);
    int nt = 0;
    if (ix + 1 < M.X && iy + 1 < M.Y && iz + 1 < M.Z) {
        unsigned cin = 0;
        for (int c = 0; c < 8; c++)
            if (sv_inside(M.value[((long long)(ix + (c & 1)) * M.Y + iy + ((c >> 1) & 1)) * M.Z + iz + ((c >> 2) & 1)])) cin |= 1u << c;
        for (int t = 0; t < 6; t++) {
            int k = 0;
            for (int v = 0; v < 4; v++) k += (cin >> SV_TET[t][v]) & 1;
            nt += (k == 1 || k == 3) ? 1 : (k == 2 ? 2 : 0);
        }
    }
    M.foff[a] = nt;
}

// vertex id of the tet edge between corners cu, cw (cw = cu + a direction) of the cell at (ix, iy, iz)
__device__ __forceinline__ int sv_edge_vertex(const SvolMeshArgs &M, int ix, int iy, int iz, int cu, int cw) {
    const long long a = ((long long)(ix + (cu & 1)) * M.Y + iy + ((cu >> 1) & 1)) * M.Z + iz + ((cu >> 2) & 1);
    const int d = SV_BITS_DIR[cw & ~cu];
    return (int)(M.voff[a] + __popc((unsigned)M.emask[a] & ((1u << d) - 1u)));
}

__global__ void __launch_bounds__(256) k_sv_mt_emit(const __grid_constant__ SvolMeshArgs M) {
    const long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x, n = (long long)M.X * M.Y * M.Z;
    if (a >= n) return;
    const int iz = (int)(a % M.Z), iy = (int)((a / M.Z) % M.Y), ix = (int)(a / ((long long)M.Y * M.Z));
    const unsigned mask = M.emask[a];
    long long v = M.voff[a];
    const double f0 = M.value[a];
    const double p0[3] = {sv_coord(M.bmin[0], M.res, ix), sv_coord(M.bmin[1], M.res, iy), sv_coord(M.bmin[2], M.res, iz)};
    for (int d = 0; d < 7; d++) {
        if (!((mask >> d) & 1u)) continue;
        const int b = SV_DIR_BITS[d], jx = ix + (b & 1), jy = iy + ((b >> 1) & 1), jz = iz + ((b >> 2) & 1);
        const long long a1 = ((long long)jx * M.Y + jy) * M.Z + jz;
        const double f1 = M.value[a1];
        const double p1[3] = {sv_coord(M.bmin[0], M.res, jx), sv_coord(M.bmin[1], M.res, jy), sv_coord(M.bmin[2], M.res, jz)};
        const double s = __ddiv_rn(f0, __dadd_rn(f0, -f1));
#pragma unroll
        for (int c = 0; c < 3; c++) M.V[3 * v + c] = __dadd_rn(p0[c], __dmul_rn(s, __dadd_rn(p1[c], -p0[c])));
        M.vtime[v] = fabs(f0) <= fabs(f1) ? M.tstar[a] : M.tstar[a1];
        v++;
    }
    if (ix + 1 >= M.X || iy + 1 >= M.Y || iz + 1 >= M.Z) return;
    long long f = M.foff[a];
    unsigned cin = 0;
    for (int c = 0; c < 8; c++)
        if (sv_inside(M.value[((long long)(ix + (c & 1)) * M.Y + iy + ((c >> 1) & 1)) * M.Z + iz + ((c >> 2) & 1)])) cin |= 1u << c;
    for (int t = 0; t < 6; t++) {
        const int *tv = SV_TET[t];
        int in = 0, k = 0;
        for (int q = 0; q < 4; q++) if ((cin >> tv[q]) & 1) { in |= 1 << q; k++; }
        if (k == 0 || k == 4) continue;
        // E(x, y): the vertex on the edge between tet vertices x and y (the lower one in the chain v0 < v1 < v2 < v3 is the edge's origin)
        auto E = [&](int x, int y) { return x < y ? sv_edge_vertex(M, ix, iy, iz, tv[x], tv[y]) : sv_edge_vertex(M, ix, iy, iz, tv[y], tv[x]); };
        int tri[2][3], nt;
        if (k == 1 || k == 3) {   // the isolated vertex i: the triangle of its three edges, normal away from i when i is inside
            int i = 0;
            for (int q = 0; q < 4; q++) if ((((in >> q) & 1) != 0) == (k == 1)) i = q;
            const int *e = SV_EVEN[i];
            tri[0][0] = E(i, e[1]); tri[0][1] = E(i, e[2]); tri[0][2] = E(i, e[3]);
            if (k == 3) { const int x = tri[0][1]; tri[0][1] = tri[0][2]; tri[0][2] = x; }
            nt = 1;
        } else {                  // inside {i, j}, outside {k, l} with (i, j, k, l) even: quad E(i,l) E(j,l) E(j,k) E(i,k), diagonal E(i,l)-E(j,k)
            int ins[2], outs[2], ni = 0, no = 0;
            for (int q = 0; q < 4; q++) { if ((in >> q) & 1) ins[ni++] = q; else outs[no++] = q; }
            int i = ins[0], j = ins[1], kk = outs[0], l = outs[1];
            const int perm[4] = {i, j, kk, l};
            int inv = 0;
            for (int x = 0; x < 4; x++) for (int y = x + 1; y < 4; y++) inv += perm[x] > perm[y];
            if (inv & 1) { const int x = kk; kk = l; l = x; }
            tri[0][0] = E(i, l); tri[0][1] = E(j, l); tri[0][2] = E(j, kk);
            tri[1][0] = E(i, l); tri[1][1] = E(j, kk); tri[1][2] = E(i, kk);
            nt = 2;
        }
        for (int q = 0; q < nt; q++) {
            if (!SV_TET_POS[t]) { const int x = tri[q][1]; tri[q][1] = tri[q][2]; tri[q][2] = x; }
            M.F[3 * f] = tri[q][0]; M.F[3 * f + 1] = tri[q][1]; M.F[3 * f + 2] = tri[q][2];
            f++;
        }
    }
}
#endif  // ISDF_CLEARANCE_TU

// ---- launch interface (isdf_clearance_tu.cu) --------------------------------------------------------------------------------------
cudaError_t sv_prep_launch(const SvolArgs &A, cudaStream_t st);
cudaError_t sv_bricks_launch(const SvolArgs &A, int nbricks, bool fill, cudaStream_t st);
// mode 0 analytic, 1 exact-sign mesh; grid = persistent CTAs
cudaError_t sv_refine_launch(const SvolArgs &A, int mode, int nitems, unsigned grid, cudaStream_t st);
// exclusive scan of a[0..n) in place, a[n] = total; bsum: (n + 1023) / 1024 scratch entries
cudaError_t sv_scan_launch(long long *a, long long n, long long *bsum, cudaStream_t st);
cudaError_t sv_mesh_count_launch(const SvolMeshArgs &M, cudaStream_t st);
cudaError_t sv_mesh_emit_launch(const SvolMeshArgs &M, cudaStream_t st);
// resident CTAs per SM of the refinement kernel (the smaller over the two modes)
cudaError_t sv_refine_resident_blocks(int *blocks);

}  // namespace isdf
