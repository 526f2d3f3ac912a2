// Trajectory clearance check (isdf_trajectory_clearance, include/isdf.h): for every pose sample of a trajectory, the smallest robot SDF
// over the occupied voxels near the pose, capped at `reach`, and the voxel that realises it; then a per-trajectory summary.
//
// Definition (normative; include/isdf.h states the same): piece i has K_c + 1 samples at local times j * step, step = T_i * (1 / K_c),
// posed exactly as the discrete path poses its samples (piece_eval, flat_quat_only, quat_rot). The candidates of a sample are the
// occupied voxels whose centre c satisfies |R^T (c - x)|_inf <= H, H = half_bd + reach (a strict > on any axis excludes, as hpp:800);
// voxels outside the map do not exist (no projInMap clamping). clear = min(reach, min over candidates of sdf(R^T (c - x))). The witness
// is the address ix*Y*Z + iy*Z + iz of the candidate realising the minimum when it is < reach, the smallest address among exact ties,
// else -1.
//
// Mapping:
//   * k_clearance_scan — persistent warps draw samples from one device counter. A warp computes its sample's pose once (shared memory),
//     bounds the world window by the exact AABB of the rotated H box (half-width H * sum_j |R_ij| per axis, widened by one voxel against
//     rounding: the per-voxel box test, not the window, decides), intersects it with the map and enumerates its occupied voxels from the
//     bit grid with rows as lanes (scan_window, isdf_discrete.cuh). The warp keeps a running best key (b, witness), b starting at reach.
//   * analytic shapes: every candidate gets the closed-form SDF (no distance-bound cull holds for them in general); each lane keeps its
//     own best key and one shuffle arg-min per sample combines them.
//   * exact-sign meshes (a true distance): branch and bound on b. Exact culls — the body-frame H box, the mesh AABB inflated by b (a
//     point outside the AABB is outside the mesh, sdf >= its distance to the box), the cell grid's bound d_c - ghd > b (outside the
//     grid: gpad > b) — queue the survivors; each survivor is re-tested against the current b and answered by the warp-cooperative
//     nearest-triangle search of isdf_mesh.cuh (candidate list, else 32-ary tree bounded by max(b, sign_radius)), sign from the
//     pseudonormal. Culls are strict (> b), so a candidate that TIES b is still answered and the (value, address) key decides.
//   * winding-sign meshes (s = 1 - 2 w, not a distance): every candidate in the H box is answered exactly (unbounded nearest triangle,
//     hierarchical winding number), as the discrete path does in that mode.
//   * k_clearance_summary — one CTA per trajectory: min / first attaining sample / first hit / count over its samples. Only minima and
//     integer counts are reduced, so the result does not depend on scheduling, and a trajectory's summary is the same bits whether it is
//     checked alone or inside a batch.
//
// Included by isdf_api.cu (argument block, launch interface) and isdf_clearance_tu.cu, which defines ISDF_CLEARANCE_TU and is the only
// translation unit that instantiates the kernels (FMA contraction on, like the discrete path).
#pragma once
#include "isdf_types.cuh"
#include "isdf_discrete.cuh"

namespace isdf {

constexpr int CLR_WARPS = 4;
constexpr int CLR_THREADS = CLR_WARPS * 32;
constexpr int CLR_SUM_THREADS = 256;

// one per trajectory; layout of isdf_clearance_summary (include/isdf.h)
struct ClrSummary {
    double min_clearance, t_min, first_hit;
    long long voxel_min;
    int piece_min, sample_min, colliding_samples, collision_free;
};
static_assert(sizeof(ClrSummary) == 48, "isdf_clearance_summary layout");

struct ClrArgs {
    DevGrid grid;
    DevShape shape;
    FlatParams fp;
    double half_bd;
    double reach, margin;
    int N, K, N0;                  // pieces, samples per piece K_c (K_c + 1 per piece), pieces per trajectory
    const double *T;               // N
    const double *C;               // 6N x 3 column-major
    double *clear;                 // N * (K + 1)
    long long *voxel;              // N * (K + 1)
    ClrSummary *summary;           // N / N0
    int *cursor;                   // persistent warps draw samples from this counter (zero on entry)
    unsigned long long *counters;  // may be null: {candidate pairs (box passed), exact mesh searches}
};

// key order of the running best: (value, address); address -1 = "no witness" (a candidate that only equals reach never wins)
__device__ __forceinline__ bool clr_better(double v, long long a, double bv, long long ba) { return v < bv || (v == bv && ba >= 0 && a < ba); }

// warp-wide arg-min of (value, address) keys; every lane returns the winner
__device__ __forceinline__ void clr_warp_argmin(double &v, long long &a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const long long oa = __shfl_xor_sync(0xffffffffu, a, o);
        if (ov < v || (ov == v && (unsigned long long)oa < (unsigned long long)a)) { v = ov; a = oa; }   // -1 sorts last among ties
    }
}

#ifdef ISDF_CLEARANCE_TU
struct ClrSurvivor { double px, py, pz; long long addr; uint32_t off, cnt, seed, pad; };   // cnt bit 31: cell centre inside
struct ClrWarpSmem {
    double pose[12];        // pos 0..2, R rows 3..11
    ClrSurvivor sv[64];
    WideStack stk;
};

// MODE 0: analytic shape, 1: exact-sign mesh, 2: winding-sign mesh
template <int MODE>
__global__ void __launch_bounds__(CLR_THREADS) k_clearance_scan(const __grid_constant__ ClrArgs A) {
    __shared__ ClrWarpSmem wsm[CLR_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;
    ClrWarpSmem &sm = wsm[warp];
    const DevGrid &G = A.grid;
    const DevMesh &Mh = A.shape.mesh;
    const int K = A.K, S = A.N * (K + 1);
    const double H = A.half_bd + A.reach;
    for (;;) {
        int s = 0;
        if (lane == 0) s = atomicAdd(A.cursor, 1);
        s = __shfl_sync(0xffffffffu, s, 0);
        if (s >= S) break;
        const int i = s / (K + 1), j = s - i * (K + 1);
        Window W;
        bool empty, finite;
        {   // pose (every lane computes the same values; lane 0 publishes them) and the world window of the rotated H box
            double cx[6], cy[6], cz[6];
#pragma unroll
            for (int k = 0; k < 6; k++) { cx[k] = __ldg(A.C + 6 * i + k); cy[k] = __ldg(A.C + 6 * A.N + 6 * i + k); cz[k] = __ldg(A.C + 12 * A.N + 6 * i + k); }
            const double step = __ldg(A.T + i) * (1.0 / K);
            PieceEval pe;
            piece_eval(cx, cy, cz, j * step, pe);
            const quat4 q = flat_quat_only(A.fp, pe.vel, pe.acc);
            const rot3 R = quat_rot(q);
            const d3 pos = pe.pos;
            if (lane == 0) {
                double *ps = sm.pose;
                ps[0] = pos.x; ps[1] = pos.y; ps[2] = pos.z;
                ps[3] = R.r0.x; ps[4] = R.r0.y; ps[5] = R.r0.z; ps[6] = R.r1.x; ps[7] = R.r1.y; ps[8] = R.r1.z; ps[9] = R.r2.x; ps[10] = R.r2.y; ps[11] = R.r2.z;
            }
            const double ex = H * (fabs(R.r0.x) + fabs(R.r0.y) + fabs(R.r0.z));
            const double ey = H * (fabs(R.r1.x) + fabs(R.r1.y) + fabs(R.r1.z));
            const double ez = H * (fabs(R.r2.x) + fabs(R.r2.y) + fabs(R.r2.z));
            // voxel centres (i + 0.5) res + bmin inside [x - e, x + e], one voxel of slack on each side (clamped before the int conversion)
            auto lo_idx = [&](double x, double e, int a, int n) { return (int)fmin(fmax(floor((x - e - G.bmin[a]) / G.res - 0.5) - 1.0, 0.0), (double)n); };
            auto hi_idx = [&](double x, double e, int a, int n) { return (int)fmax(fmin(ceil((x + e - G.bmin[a]) / G.res - 0.5) + 1.0, (double)n - 1.0), -1.0); };
            W.ix0 = lo_idx(pos.x, ex, 0, G.X); W.ix1 = hi_idx(pos.x, ex, 0, G.X);
            W.iy0 = lo_idx(pos.y, ey, 1, G.Y); W.iy1 = hi_idx(pos.y, ey, 1, G.Y);
            W.iz0 = lo_idx(pos.z, ez, 2, G.Z); W.iz1 = hi_idx(pos.z, ez, 2, G.Z);
            finite = isfinite(pos.x) && isfinite(pos.y) && isfinite(pos.z) && isfinite(ex) && isfinite(ey) && isfinite(ez);
            empty = !finite || W.ix0 > W.ix1 || W.iy0 > W.iy1 || W.iz0 > W.iz1;
        }
        __syncwarp();
        const d3 pos = mk3(sm.pose[0], sm.pose[1], sm.pose[2]);
        rot3 R; R.r0 = mk3(sm.pose[3], sm.pose[4], sm.pose[5]); R.r1 = mk3(sm.pose[6], sm.pose[7], sm.pose[8]); R.r2 = mk3(sm.pose[9], sm.pose[10], sm.pose[11]);
        double bv = A.reach;       // running best key (warp-uniform for meshes, per lane for analytic shapes)
        long long ba = -1;
        unsigned long long npairs = 0, nsearch = 0;
        int nsv = 0;

        // survivors of the mesh culls, in queue order: re-test against the current b, then the exact search (all lanes, same answer)
        auto answer_survivors = [&]() {
            for (int k = 0; k < nsv; k++) {
                const ClrSurvivor v = sm.sv[k];
                const d3 p = mk3(v.px, v.py, v.pz);
                const int cnt = (int)(v.cnt & 0x7fffffffu);
                double reach_q = 1e300;
                if (MODE == 1) {
                    if (p.x < Mh.blo[0] - bv || p.x > Mh.bhi[0] + bv || p.y < Mh.blo[1] - bv || p.y > Mh.bhi[1] + bv || p.z < Mh.blo[2] - bv ||
                        p.z > Mh.bhi[2] + bv)
                        continue;
                    // bounded search: nothing within the bound means sdf >= bound (outside) — the relative widening keeps exact ties answerable
                    if (Mh.sign_radius > 0.0) reach_q = fmax(bv, Mh.sign_radius) * (1.0 + 1e-12);
                }
                const bool has = cnt != 0 && lane < cnt;
                const int first_id = has ? (int)__ldg(Mh.cand + v.off + lane) : -1;
                const float first_lb = has ? __ldg(Mh.cand_lb + v.off + lane) : 0.0f;
                double d2; d3 c = mk3(0, 0, 0); int tri, feat;
                nsearch++;
                if (!mesh_search_rec(Mh, p, reach_q, lane, &sm.stk, cnt, v.off, first_id, first_lb, (int)v.seed, (v.cnt >> 31) != 0u, d2, c, tri, feat)) continue;
                d3 g;
                const double sdf = mesh_finish_t<MODE == 2>(Mh, p, p - c, d2, tri, feat, g);
                if (clr_better(sdf, v.addr, bv, ba)) { bv = sdf; ba = v.addr; }
            }
            nsv = 0;
            __syncwarp();
        };

        if (!empty) {
            scan_window(G, W, lane, [&](bool valid, int vx, int vy, int vz, int) {
                bool box = false;
                d3 prel = mk3(0, 0, 0);
                if (valid) {
                    prel = rot_applyT(R, voxel_centre(G, vx, vy, vz) - pos);
                    box = !(fabs(prel.x) > H || fabs(prel.y) > H || fabs(prel.z) > H);
                }
                npairs += __popc(__ballot_sync(0xffffffffu, box));
                const long long addr = ((long long)vx * G.Y + vy) * G.Z + vz;
                if (MODE == 0) {
                    if (box) {
                        const double sdf = shape_sdf_analytic(A.shape, prel);
                        if (clr_better(sdf, addr, bv, ba)) { bv = sdf; ba = addr; }
                    }
                    return;
                }
                bool pass = box;
                uint4 rec = make_uint4(0u, 0xffffffffu, 0u, 0u);   // {dist bits, seed, off, cnt}; seed 0xffffffff = outside the cell grid
                if (box) {
                    const int cxi = (int)floor((prel.x - Mh.glo[0]) * Mh.inv_gcell), cyi = (int)floor((prel.y - Mh.glo[1]) * Mh.inv_gcell),
                              czi = (int)floor((prel.z - Mh.glo[2]) * Mh.inv_gcell);
                    const bool in_grid = !(cxi < 0 || cyi < 0 || czi < 0 || cxi >= Mh.gdim[0] || cyi >= Mh.gdim[1] || czi >= Mh.gdim[2]);
                    if (in_grid) rec = __ldg(Mh.cell_rec + ((size_t)(cxi * Mh.gdim[1] + cyi) * Mh.gdim[2] + czi));
                    if (MODE == 1) {
                        if (prel.x < Mh.blo[0] - bv || prel.x > Mh.bhi[0] + bv || prel.y < Mh.blo[1] - bv || prel.y > Mh.bhi[1] + bv ||
                            prel.z < Mh.blo[2] - bv || prel.z > Mh.bhi[2] + bv)
                            pass = false;
                        else if (in_grid) pass = !((double)__uint_as_float(rec.x) - Mh.ghd > bv);
                        else pass = !(Mh.gpad > bv);
                    }
                }
                const unsigned bal = __ballot_sync(0xffffffffu, pass);
                if (pass) {
                    ClrSurvivor &v = sm.sv[nsv + __popc(bal & lt_mask)];
                    v.px = prel.x; v.py = prel.y; v.pz = prel.z; v.addr = addr; v.off = rec.z; v.seed = rec.y;
                    v.cnt = rec.w | ((rec.y != 0xffffffffu && __uint_as_float(rec.x) < 0.0f) ? 0x80000000u : 0u);
                }
                nsv += __popc(bal);
                __syncwarp();
                if (nsv >= 32) answer_survivors();
            });
            if (MODE != 0 && nsv > 0) answer_survivors();
        }
        if (MODE == 0) clr_warp_argmin(bv, ba);
        if (lane == 0) {
            A.clear[s] = !finite ? nan("") : (ba >= 0) ? bv : A.reach;   // a non-finite pose is never reported clear
            A.voxel[s] = ba;
            if (A.counters) {
                if (npairs) atomicAdd(A.counters, npairs);
                if (nsearch) atomicAdd(A.counters + 1, nsearch);
            }
        }
        __syncwarp();
    }
}

// One CTA per trajectory: samples reduced by minimum / first index / integer count — independent of the thread schedule.
__global__ void __launch_bounds__(CLR_SUM_THREADS) k_clearance_summary(const __grid_constant__ ClrArgs A) {
    __shared__ double s_v[CLR_SUM_THREADS];
    __shared__ int s_i[CLR_SUM_THREADS], s_h[CLR_SUM_THREADS], s_c[CLR_SUM_THREADS];
    const int b = blockIdx.x, K = A.K, N0 = A.N0;
    const int per = N0 * (K + 1), s0 = b * per;
    double mv = 1e300; int mi = 0x7fffffff, hi = 0x7fffffff, cnt = 0;
    for (int k = threadIdx.x; k < per; k += CLR_SUM_THREADS) {   // ascending k per thread: the first index of a tie is kept
        double v = A.clear[s0 + k];
        if (v != v) v = -INFINITY;                                // non-finite pose: reported as the minimum and as colliding
        if (v < mv) { mv = v; mi = k; }
        if (v < A.margin) { cnt++; if (k < hi) hi = k; }
    }
    s_v[threadIdx.x] = mv; s_i[threadIdx.x] = mi; s_h[threadIdx.x] = hi; s_c[threadIdx.x] = cnt;
    __syncthreads();
    for (int o = CLR_SUM_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            const double ov = s_v[threadIdx.x + o]; const int oi = s_i[threadIdx.x + o];
            if (ov < s_v[threadIdx.x] || (ov == s_v[threadIdx.x] && oi < s_i[threadIdx.x])) { s_v[threadIdx.x] = ov; s_i[threadIdx.x] = oi; }
            s_h[threadIdx.x] = min(s_h[threadIdx.x], s_h[threadIdx.x + o]);
            s_c[threadIdx.x] += s_c[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    // trajectory time of local sample k: T of the earlier pieces of the trajectory added in ascending order, plus j * step
    auto traj_time = [&](int k) {
        const int p = k / (K + 1), j = k - p * (K + 1);
        double t = 0.0;
        for (int q = 0; q < p; q++) t += A.T[b * N0 + q];
        return t + j * (A.T[b * N0 + p] * (1.0 / K));
    };
    ClrSummary r;
    const int m = s_i[0];
    r.min_clearance = s_v[0] == -INFINITY ? nan("") : s_v[0];
    r.piece_min = m / (K + 1);
    r.sample_min = m - r.piece_min * (K + 1);
    r.t_min = traj_time(m);
    r.voxel_min = A.voxel[s0 + m];
    r.colliding_samples = s_c[0];
    r.collision_free = s_c[0] == 0 ? 1 : 0;
    r.first_hit = s_c[0] == 0 ? -1.0 : traj_time(s_h[0]);
    A.summary[b] = r;
}
#endif  // ISDF_CLEARANCE_TU

// ---- launch interface of the clearance translation unit (isdf_clearance_tu.cu) --------------------------------------------------------
// mode: 0 analytic, 1 exact-sign mesh, 2 winding-sign mesh; grid = persistent CTAs
cudaError_t clearance_launch(const ClrArgs &A, int mode, unsigned grid, cudaStream_t st);
// resident CTAs per SM of the scan kernel (the smallest over the three modes)
cudaError_t clearance_resident_blocks(int *blocks);

}  // namespace isdf
