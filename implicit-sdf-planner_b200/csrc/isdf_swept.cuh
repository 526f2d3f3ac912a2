// Swept-volume collision term: addSaftyPenaOnSweptVolumeParallel (back_end_optimizer.hpp:557-649) and the SV-SDF query
// getSDFofSweptVolume<true>(p, t, g, set_ts=false) (sw_manager.hpp:710-747) with choiceTInit (:367-445),
// gradientDescent (:1000-1062), getSDFAtTimeStamp (:550-556), getSDF_DOTAtTimeStampOptimized (:593-662),
// getGradPrelAtTimeStamp (:566-572), Trajectory::locatePieceIdx / getPos_Vel_Acc_Jerk (trajectory.hpp:105-149, 545-570).
//
// GPU mapping — the reference runs one OpenMP thread per obstacle point through a long scalar search; here
//   k_sv_table : the coarse time grid t = 0, 0.2, ... (same running sum as the reference's for-loop) and the robot
//                pose at each coarse time are computed ONCE per evaluation and shared by every point (the reference
//                recomputes the pose per point per sample);
//   k_sv_points_cta<MESH>: one CTA (8 warps) per obstacle point. The threads split the coarse scan (in-range bitmap -> intervals
//                via bit scans) and each fine scan.
//                Mesh robots: every exact SDF value is a warp-cooperative closest-triangle search, the scans are pruned with the
//                body-frame cell grid's Lipschitz brackets and the warps evaluate the descent's step candidates in parallel
//                (details at the kernel).
//                Analytic shapes: warp 0 runs the sign descent SPECULATIVELY: in one pass the 32 lanes evaluate f(x), the six
//                finite-difference samples of the gradient and all 18 candidate steps x -/+ 0.02/2^d, so an outer iteration
//                costs one SDF latency instead of up to 9 + 7 dependent ones.
//                Accept/reject decisions replay the reference's sequential logic exactly (same comparisons, same
//                iteration accounting);
//   k_sv_reduce / k_sv_finish: deterministic per-piece reduction (fixed thread->point map, fixed trees) and the
//                gradT(j<i) prefix of hpp:642-645 as a suffix sum.
#pragma once
#include "isdf_types.cuh"
#include <cuda/barrier>
#include <cuda/ptx>
#include <vector>
#include <algorithm>

namespace isdf {

// Stage the MINCO block [C (18N doubles) | T (N doubles)] into shared memory with the TMA bulk-copy engine
// (cp.async.bulk global -> shared, completion on an mbarrier; SASS: UBLKCP) — one elected thread issues the copies,
// every thread waits on the barrier. Falls back to a cooperative loop when the 16-byte alignment rules do not hold.
__device__ __forceinline__ void stage_traj_block(double *sC, double *sT, const double *gC, const double *gT, int N,
                                                 cuda::barrier<cuda::thread_scope_block> *bar) {
    const bool tma_ok = ((reinterpret_cast<unsigned long long>(gC) & 15ull) == 0) && ((reinterpret_cast<unsigned long long>(gT) & 15ull) == 0) &&
                        ((N & 1) == 0);
    if (tma_ok) {
        if (threadIdx.x == 0) {
            init(bar, blockDim.x);
            cuda::ptx::fence_proxy_async(cuda::ptx::space_shared);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            cuda::memcpy_async(sC, gC, cuda::aligned_size_t<16>(sizeof(double) * 18 * (size_t)N), *bar);
            cuda::memcpy_async(sT, gT, cuda::aligned_size_t<16>(sizeof(double) * (size_t)N), *bar);
        }
        cuda::barrier<cuda::thread_scope_block>::arrival_token tok = bar->arrive();
        bar->wait(std::move(tok));
    } else {
        for (int k = threadIdx.x; k < 18 * N; k += blockDim.x) sC[k] = gC[k];
        for (int k = threadIdx.x; k < N; k += blockDim.x) sT[k] = gT[k];
        __syncthreads();
    }
}

constexpr int SV_MAX_COARSE = 1536;  // traj_duration < 300 s (updateTraj ignores longer ones, swm:291) at 0.2 s
constexpr int SV_FLAG_WORDS = SV_MAX_COARSE / 32;

struct TrajView { const double *T; const double *C; int N; };

// locatePieceIdx (trajectory.hpp:545-563): sequential subtraction, strict '>', clamps past the end
__device__ __forceinline__ int traj_locate(const TrajView &tr, double &t) {
    int idx = 0;
    const int N = tr.N;
    // eight pieces per trip: the durations are loaded together and the subtractions run ahead speculatively, so the dependent chain is
    // the eight subtractions themselves — same operations in the same order as the reference's loop, the first failing comparison wins
    while (idx + 8 <= N) {
        double d[8], s[8];
#pragma unroll
        for (int k = 0; k < 8; k++) d[k] = tr.T[idx + k];
        s[0] = t;
#pragma unroll
        for (int k = 1; k < 8; k++) s[k] = s[k - 1] - d[k - 1];
        int stop = 8;
        double tsel = s[7] - d[7];
#pragma unroll
        for (int k = 7; k >= 0; k--) if (!(s[k] > d[k])) { stop = k; tsel = s[k]; }
        t = tsel; idx += stop;
        if (stop < 8) return idx;
    }
    for (; idx < N; idx++) {
        const double dur = tr.T[idx];
        if (!(t > dur)) break;
        t -= dur;
    }
    if (idx == N) { idx--; t += tr.T[idx]; }
    return idx;
}

// Piece::getPos_Vel_Acc_Jerk (trajectory.hpp:105-149): running powers, integer factors multiplied first
__device__ __forceinline__ void traj_pvaj(const TrajView &tr, double tabs, d3 &p, d3 &v, d3 &a, d3 &j) {
    double t = tabs;
    const int i = traj_locate(tr, t);
    const double *cx = tr.C + 6 * i, *cy = tr.C + 6 * tr.N + 6 * i, *cz = tr.C + 12 * tr.N + 6 * i;
    double px = 0, py = 0, pz = 0, vx = 0, vy = 0, vz = 0, ax = 0, ay = 0, az = 0, jx = 0, jy = 0, jz = 0;
    double ptn = 1.0, vtn = 1.0, atn = 1.0, jtn = 1.0;
    int vn = 1, am = 1, an = 2, jl = 1, jm = 2, jn = 3;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        const double x = cx[k], y = cy[k], z = cz[k];
        px += ptn * x; py += ptn * y; pz += ptn * z; ptn *= t;
        if (k >= 1) { const double f = vn * vtn; vx += f * x; vy += f * y; vz += f * z; vtn *= t; vn++; }
        if (k >= 2) { const double f = (am * an) * atn; ax += f * x; ay += f * y; az += f * z; atn *= t; am++; an++; }
        if (k >= 3) { const double f = (jl * jm * jn) * jtn; jx += f * x; jy += f * y; jz += f * z; jtn *= t; jl++; jm++; jn++; }
    }
    p = mk3(px, py, pz); v = mk3(vx, vy, vz); a = mk3(ax, ay, az); j = mk3(jx, jy, jz);
}

struct SvArgs {
    DevCfg cfg;
    DevShape shape;
    int N;
    const double *T, *C;
    int P;
    const double *pts;
    double *tstar, *sdf, *grel;   // per point (in/out, out, out)
    double *times;                // coarse time grid
    double *poses;                // 12 per coarse time: x(3), R rows(9)
    int *meta;                    // [0] = number of coarse samples
    double *state;                // [0] = traj_duration (persists across evaluations like the SweptVolumeManager member)
    double *partial;              // P x PARTIAL_STRIDE
    int *piece;                   // P (piece of t*, -1 = no contribution)
    double *piece_gdt, *piece_cost;  // N each
    double *out;                  // 19N+1
    unsigned long long *counter;  // reference-equivalent SDF evaluation count
    double *count_out;            // host entry point only: the count (bit pattern) lands behind the result vector, one D2H copy fetches both
    int rank, world;
    const double *g_t, *g_s, *g_g;  // tier-T1: given t*, sdf*, g_rel (null = search)
    // longest-first schedule of the point CTAs: work[pk] = cycles point pk took in this evaluation; order = this rank's points sorted by
    // the previous evaluation's work (null: natural order). A launch is a few waves of CTAs and ends with its slowest point — started
    // first, that point overlaps the others instead of trailing them. Results do not depend on the order (per-point outputs).
    unsigned *work;
    int *order;
    int use_order;
};

// ---- k_sv_table ---------------------------------------------------------------------------------------------------
constexpr int SV_TABLE_THREADS = 256;
constexpr int SV_TABLE_CTAS = SV_MAX_COARSE / SV_TABLE_THREADS;
// CTA bx computes the poses of coarse samples [256 bx, 256 bx + 256). The coarse time grid is a chain of repeated additions
// (choiceTInit's loop variable, swm:392): thread 0 of every CTA walks the whole chain (a few microseconds) and keeps its own slice.
__device__ __forceinline__ void sv_table_body(const SvArgs &A, const int bx) {
    extern __shared__ __align__(16) double smem[];
    double *sC = smem, *sT = smem + 18 * A.N;
#pragma nv_diag_suppress static_var_with_dynamic_init
    __shared__ cuda::barrier<cuda::thread_scope_block> bar;
    stage_traj_block(sC, sT, A.C, A.T, A.N, &bar);
    __shared__ int s_nc;
    __shared__ double s_times[SV_TABLE_THREADS];
    const int k0 = bx * SV_TABLE_THREADS;
    if (threadIdx.x == 0) {
        double td = 0.0;
        for (int k = 0; k < A.N; k++) td += sT[k];         // getTotalDuration (trajectory.hpp:457-466)
        const double dur = (td < 3 * 1e2) ? td : A.state[0];   // updateTraj (swm:287-296): longer trajectories keep the previous duration
        int nc = 0;
        for (double t = 0; t < dur && nc < SV_MAX_COARSE; t += 0.2) {   // choiceTInit's coarse loop (swm:392)
            if (nc >= k0 && nc < k0 + SV_TABLE_THREADS) s_times[nc - k0] = t;
            nc++;
        }
        s_nc = nc;
        if (bx == 0) { A.meta[0] = nc; if (td < 3 * 1e2) A.state[0] = td; }
    }
    __syncthreads();
    const TrajView tr = {sT, sC, A.N};
    const int k = k0 + (int)threadIdx.x;
    if (k < s_nc) {
        const double t = s_times[threadIdx.x];
        A.times[k] = t;
        d3 x, v, a, j;
        traj_pvaj(tr, t, x, v, a, j);
        const rot3 R = quat_rot(flat_quat_only(A.cfg.fp, v, a));
        double *o = A.poses + 12 * (size_t)k;
        o[0] = x.x; o[1] = x.y; o[2] = x.z;
        o[3] = R.r0.x; o[4] = R.r0.y; o[5] = R.r0.z; o[6] = R.r1.x; o[7] = R.r1.y; o[8] = R.r1.z; o[9] = R.r2.x; o[10] = R.r2.y; o[11] = R.r2.z;
    }
}

// ---- helpers for k_sv_points_cta --------------------------------------------------------------------------------
// Cell-grid bracket of the mesh SDF at a body-frame point: the SDF is 1-Lipschitz, so every point of a cell lies within
// ghd of the cell centre's signed distance. Outside the grid only the lower bound gpad is known.
__device__ __forceinline__ void mesh_bracket(const DevMesh &M, d3 prel, double &lo, double &hi) {
    lo = -1e300; hi = 1e300;
    if (M.gdim[0] <= 0) return;
    const int cell = mesh_cell_index(M, prel);
    if (cell < 0) { lo = M.gpad; return; }
    const double dc = (double)__ldg(M.cell_dist + cell);
    lo = dc - M.ghd; hi = dc + M.ghd;
}

// Upper bound of the mesh SDF at a body-frame point without a search: the cell bracket's upper end, tightened by the exact distance
// to the cell's seed triangle (the triangle nearest to the cell centre — for most points of the cell THE nearest triangle). The
// signed distance never exceeds the distance to any one triangle.
__device__ __forceinline__ double mesh_upper(const DevMesh &M, d3 prel) {
    if (M.gdim[0] <= 0) return 1e300;
    const int cell = mesh_cell_index(M, prel);
    if (cell < 0) return 1e300;
    double hi = (double)__ldg(M.cell_dist + cell) + M.ghd;
    const int seed = (int)__ldg(M.cell_seed + cell);
    if (seed >= 0 && seed < M.ntris) {
        int f;
        const d3 e = prel - tri_closest_rec(prel, M.tris + TRI_STRIDE * (size_t)seed, f);
        hi = fmin(hi, sqrt(dot3(e, e)) * (1.0 + 1e-12));
    }
    return hi;
}

__device__ __forceinline__ d3 sv_body_point(const SvArgs &A, const TrajView &tr, d3 p, double t) {
    d3 x, v, a, j;
    traj_pvaj(tr, t, x, v, a, j);
    const rot3 R = quat_rot(flat_quat_only(A.cfg.fp, v, a));
    return rot_applyT(R, p - x);
}

// Exact mesh SDF for the lanes flagged in `need` (each with its own body-frame point): one warp-cooperative search per
// flagged lane, in lane order. A lane-per-query search costs ~10x more here because the interesting queries sit 1-2 m from
// the mesh, where a closest-triangle search prunes badly and 32 private traversals diverge.
__device__ __forceinline__ double mesh_sdf_each(const DevMesh &M, bool need, d3 prel, double reach, double dflt, int lane, WideStack *stk, d3 *gout = nullptr) {
    unsigned todo = __ballot_sync(0xffffffffu, need);
    double out = dflt;
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const d3 q = mk3(__shfl_sync(0xffffffffu, prel.x, src), __shfl_sync(0xffffffffu, prel.y, src), __shfl_sync(0xffffffffu, prel.z, src));
        d3 g = mk3(0, 0, 0);
        const double v = mesh_sdf_grad_warp_lat(M, q, reach, g, lane, stk);
        if (lane == src) { out = v; if (gout) *gout = g; }
    }
    return out;
}

// getSDFAtTimeStamp (swm:550-556), analytic shapes
__device__ __forceinline__ double sv_sdf_at(const SvArgs &A, const TrajView &tr, d3 p, double t) {
    return shape_sdf_analytic(A.shape, sv_body_point(A, tr, p, t));
}

__device__ __forceinline__ d3 shfl3(d3 v, int src) {
    return mk3(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src), __shfl_sync(0xffffffffu, v.z, src));
}

// Warp-cooperative getonlyGrad1 (analytic shapes) at a body-frame point known to every lane.
__device__ __forceinline__ d3 warp_grad(const DevShape &S, d3 tmp, int lane) {
    if (S.kind == ISDF_SHAPE_BALL || S.kind == ISDF_SHAPE_POINT) return unit3(tmp);
    d3 q = tmp;
    if (S.kind == ISDF_SHAPE_BOX) {
        if (lane == 1) q.x += 0.01; else if (lane == 2) q.y += 0.01; else if (lane == 3) q.z += 0.01;
        const double val = shape_sdf_analytic(S, q);
        const double f0 = __shfl_sync(0xffffffffu, val, 0);
        return mk3((__shfl_sync(0xffffffffu, val, 1) - f0) / 0.01, (__shfl_sync(0xffffffffu, val, 2) - f0) / 0.01,
                   (__shfl_sync(0xffffffffu, val, 3) - f0) / 0.01);
    }
    const double dx = 0.000005;
    if (lane < 6) {
        const int ax = lane >> 1;
        double c = (ax == 0 ? tmp.x : (ax == 1 ? tmp.y : tmp.z)) - dx;
        if (lane & 1) c = c + 2 * dx;
        if (ax == 0) q.x = c; else if (ax == 1) q.y = c; else q.z = c;
    }
    const double val = shape_sdf_analytic(S, q);
    const double gx = __shfl_sync(0xffffffffu, val, 1) - __shfl_sync(0xffffffffu, val, 0);
    const double gy = __shfl_sync(0xffffffffu, val, 3) - __shfl_sync(0xffffffffu, val, 2);
    const double gz = __shfl_sync(0xffffffffu, val, 5) - __shfl_sync(0xffffffffu, val, 4);
    return unit3(mk3(gx / (2 * dx), gy / (2 * dx), gz / (2 * dx)));
}

// gradientDescent (swm:1000-1062), one speculative warp pass per outer iteration.
// lanes 0..8: x - tau_d (taken when g > 0), lanes 9..17: x + tau_d (g < 0), lane 18: f(x), lanes 19..24: FD samples.
__device__ void sv_gradient_descent(const SvArgs &A, const TrajView &tr, d3 p, double t_min, double t_max, double x0,
                                    double &fx, double &x, unsigned &nevals, int lane) {
    const DevShape &S = A.shape;
    const double alpha = 0.02, tol = 1e-5;
    int iter = 0; bool stop = false;
    double prev_x = 10000000.0;
    x = x0;
    const bool central = S.kind != ISDF_SHAPE_BALL && S.kind != ISDF_SHAPE_POINT && S.kind != ISDF_SHAPE_BOX;
    while (iter < 300 && !stop && fabs(x - prev_x) > tol) {
        double t = x;
        if (lane < 18) {
            const int d = (lane % 9) + 1;
            double tau = alpha;
            for (int q = 1; q < d; q++) tau = 0.5 * tau;
            const double xc = (lane < 9) ? (x - tau * 1) : (x - tau * (-1));
            t = fmax(fmin(xc, t_max), t_min);
        }
        d3 xt, v, a, j;
        traj_pvaj(tr, t, xt, v, a, j);
        FlatState fs;
        flat_state(A.cfg.fp, v, a, j, fs);
        const rot3 R = quat_rot(flat_quat(fs));
        const d3 tmp = rot_applyT(R, p - xt);
        d3 q = tmp;
        if (central && lane >= 19 && lane < 25) {
            const double dx = 0.000005;
            const int ax = (lane - 19) >> 1;
            double c = (ax == 0 ? tmp.x : (ax == 1 ? tmp.y : tmp.z)) - dx;
            if ((lane - 19) & 1) c = c + 2 * dx;
            if (ax == 0) q.x = c; else if (ax == 1) q.y = c; else q.z = c;
        } else if (S.kind == ISDF_SHAPE_BOX && lane >= 19 && lane < 22) {
            if (lane == 19) q.x += 0.01; else if (lane == 20) q.y += 0.01; else q.z += 0.01;
        }
        const double val = shape_sdf_analytic(S, q);
        if (iter == 0) { fx = __shfl_sync(0xffffffffu, val, 18); nevals++; }
        // gradient of the SDF at (x, tmp@lane18)
        d3 g;
        if (S.kind == ISDF_SHAPE_BALL || S.kind == ISDF_SHAPE_POINT) g = shfl3(unit3(tmp), 18);
        else if (S.kind == ISDF_SHAPE_BOX) {
            const double f0 = __shfl_sync(0xffffffffu, val, 18);
            g = mk3((__shfl_sync(0xffffffffu, val, 19) - f0) / 0.01, (__shfl_sync(0xffffffffu, val, 20) - f0) / 0.01,
                    (__shfl_sync(0xffffffffu, val, 21) - f0) / 0.01);
        } else {
            const double dx = 0.000005;
            const double gx = __shfl_sync(0xffffffffu, val, 20) - __shfl_sync(0xffffffffu, val, 19);
            const double gy = __shfl_sync(0xffffffffu, val, 22) - __shfl_sync(0xffffffffu, val, 21);
            const double gz = __shfl_sync(0xffffffffu, val, 24) - __shfl_sync(0xffffffffu, val, 23);
            g = unit3(mk3(gx / (2 * dx), gy / (2 * dx), gz / (2 * dx)));
        }
        // d/dt of the SDF: grad . point_velocity, point_velocity = -(R^T v + omega x tmp)  (swm:655-661), on lane 18's pose
        const d3 omg = flat_omega(fs);
        const d3 rv = rot_applyT(R, v), wx = cross3(omg, tmp);
        const d3 pv = mk3(-(rv.x + wx.x), -(rv.y + wx.y), -(rv.z + wx.z));
        const double gd = __shfl_sync(0xffffffffu, dot3(g, pv), 18);
        const int sgn = (int)(gd > 0) - (int)(gd < 0);
        const unsigned ok = __ballot_sync(0xffffffffu, lane < 18 && (val - fx) < 0);
        const unsigned m = sgn > 0 ? (ok & 0x1ffu) : (sgn < 0 ? ((ok >> 9) & 0x1ffu) : 0u);
        prev_x = x;
        if (m) {
            const int d = __ffs(m);
            const int src = (sgn > 0 ? 0 : 9) + d - 1;
            x = __shfl_sync(0xffffffffu, t, src);
            fx = __shfl_sync(0xffffffffu, val, src);
            iter += d; nevals += d;
        } else {
            iter += 9; nevals += 9; stop = true;
        }
    }
}

// ---- chain-rule tail of one obstacle point (hpp:578-636): stores t*, sdf*, g_rel and the point's contribution to its piece ----
__device__ __forceinline__ void sv_point_tail(const SvArgs &A, const double *sC, const TrajView &tr, int pk, d3 p, bool found, double tstar,
                                              double sdf_value, d3 grel) {
    const DevCfg &cfg = A.cfg;
    int piece = -1;
    A.tstar[pk] = tstar; A.sdf[pk] = sdf_value;
    A.grel[3 * pk] = grel.x; A.grel[3 * pk + 1] = grel.y; A.grel[3 * pk + 2] = grel.z;
    double f, df;
    hinge(cfg.safety - sdf_value, 0.01, f, df);   // mu hard-coded 0.01 (hpp:851)
    if (found && f > 2.220446049250313e-16) {     // returns costp > DBL_EPSILON (hpp:865)
        double tl = tstar;
        const int i = traj_locate(tr, tl);
        PieceEval pe;
        piece_eval(sC + 6 * i, sC + 6 * A.N + 6 * i, sC + 12 * A.N + 6 * i, tl, pe);
        FlatState fs;
        flat_state(cfg.fp, pe.vel, pe.acc, pe.jer, fs);
        const quat4 q = flat_quat(fs);
        const rot3 R = quat_rot(q);
        const d3 wg = rot_apply(R, grel);
        const d3 dd = p - pe.pos;
        double jq[4];
        quat_pull(q, grel, dd, jq);
        const d3 gP = mk3(cfg.wp * (df * wg.x), cfg.wp * (df * wg.y), cfg.wp * (df * wg.z));
        const double gQ[4] = {cfg.wp * (-df * jq[0]), cfg.wp * (-df * jq[1]), cfg.wp * (-df * jq[2]), cfg.wp * (-df * jq[3])};
        const double pena = cfg.wp * f;
        d3 gV, gA, gJ;
        flat_adjoint(cfg.fp, fs, pe.vel, pe.acc, gQ, mk3(0, 0, 0), mk3(0, 0, 0), gV, gA, gJ);
        double *o = A.partial + (size_t)pk * PARTIAL_STRIDE;
#pragma unroll
        for (int k = 0; k < 6; k++) {
            o[k] = pe.b0[k] * gP.x + pe.b1[k] * gV.x + pe.b2[k] * gA.x + pe.b3[k] * gJ.x;
            o[6 + k] = pe.b0[k] * gP.y + pe.b1[k] * gV.y + pe.b2[k] * gA.y + pe.b3[k] * gJ.y;
            o[12 + k] = pe.b0[k] * gP.z + pe.b1[k] * gV.z + pe.b2[k] * gA.z + pe.b3[k] * gJ.z;
        }
        o[18] = (-dot3(gP, pe.vel) + -dot3(gV, pe.acc) + -dot3(gA, pe.jer) + -dot3(gJ, pe.sna));
        o[19] = pena;
        piece = i;
    }
    A.piece[pk] = piece;
}

// ---- k_sv_points_cta: one CTA (SVM_WARPS warps) per obstacle point (designed for mesh robots) ----------------------------------------
// The work per point is extremely uneven (half of the points never come within range; a few need >100 closest-triangle
// searches in sequence), and with 10^2-10^4 points the kernel is a single wave: its duration is the SLOWEST point, not the
// sum. So a point gets a whole CTA and the dependent chain is cut three ways:
//   * coarse / fine scans: SVM_THREADS samples per round; consecutive fine samples go to different warps, so the survivors of
//     the bracket pass (a contiguous run around the closest approach) are searched by all warps at once;
//   * sign descent: one outer iteration evaluates the step candidates x -/+ 0.02/2^d, d = 1..8, on the eight warps at once
//     (each a warp-cooperative search) and then replays the reference's sequential accept/reject logic on the results;
//   * the SDF value and gradient of an accepted candidate are carried into the next iteration (same point, same function),
//     which removes the re-evaluation at the new x — guarded by a bit-compare of the body-frame point.
// Decisions, values and the reference-equivalent evaluation count are those of the sequential algorithm.
constexpr int SVM_WARPS = 8;   // warps per obstacle point
constexpr int SVM_THREADS = SVM_WARPS * 32;

struct SvmShared {
    uint32_t flags[SV_FLAG_WORDS];
    WideStack stk[SVM_WARPS];
    double red_d[SVM_WARPS], red_t[SVM_WARPS];
    int red_i[SVM_WARPS];
    double cand_f[9], cand_x[9], cand_g[9][3], cand_q[9][3];
    double bc[4];
    double bestg[SVM_WARPS][32][6];      // fine scan: gradient and body-frame point of every lane's best sample (the descent starts there)
};

__device__ __forceinline__ bool same_bits(d3 a, d3 b) { return a.x == b.x && a.y == b.y && a.z == b.z; }

// gradientDescent (swm:1000-1062) for one point, executed by the whole CTA. Returns sdf(x), x and the unit gradient g at the
// body-frame point q of the final x.
// have0: (f0, g0) are the mesh SDF and its gradient at the body-frame point q0, already computed by the fine scan at its best sample — if
// that sample is the seed x0 (its body-frame point has the same bits), the descent's first search is that one and is not repeated.
__device__ __forceinline__ void svm_descent(const SvArgs &A, const TrajView &tr, d3 p, double t_min, double t_max, double x0, SvmShared &S,
                                            double &fx, double &x, d3 &g, d3 &gq, unsigned &nevals, int lane, int warp,
                                            bool have0, double f0, d3 g0, d3 q0) {
    const DevMesh &M = A.shape.mesh;
    WideStack *stk = &S.stk[warp];
    const double alpha = 0.02, tol = 1e-5;
    int iter = 0; bool stop = false, have = have0;
    double prev_x = 10000000.0;
    x = x0;
    g = have0 ? g0 : mk3(0, 0, 0); gq = have0 ? q0 : mk3(0, 0, 0);
    double fval = have0 ? f0 : 0.0;
    while (iter < 300 && !stop && fabs(x - prev_x) > tol) {
        d3 xt, v, a, j;
        traj_pvaj(tr, x, xt, v, a, j);
        FlatState fs;
        flat_state(A.cfg.fp, v, a, j, fs);
        const rot3 R = quat_rot(flat_quat(fs));
        const d3 tmp = rot_applyT(R, p - xt);
        if (!(have && same_bits(tmp, gq))) {          // CTA-uniform: every thread computed the same tmp
            if (warp == 0) {
                d3 g0 = mk3(0, 0, 0);
                const double f0 = mesh_sdf_grad_warp_lat(M, tmp, 1e300, g0, lane, stk);
                if (lane == 0) { S.bc[0] = f0; S.bc[1] = g0.x; S.bc[2] = g0.y; S.bc[3] = g0.z; }
            }
            __syncthreads();
            fval = S.bc[0]; g = mk3(S.bc[1], S.bc[2], S.bc[3]); gq = tmp; have = true;
            __syncthreads();
        }
        if (iter == 0) { fx = fval; if (warp == 0) nevals++; }
        const d3 omg = flat_omega(fs);
        const d3 rv = rot_applyT(R, v), wx = cross3(omg, tmp);
        const double gd = g.x * -(rv.x + wx.x) + g.y * -(rv.y + wx.y) + g.z * -(rv.z + wx.z);
        const int sgn = (int)(gd > 0) - (int)(gd < 0);
        prev_x = x;
        bool accepted = false;
        for (int b0 = 1; b0 < 10 && !accepted; b0 += SVM_WARPS) {
            const int mydiv = b0 + warp;
            if (mydiv < 10) {
                double tau = alpha;
                for (int q = 1; q < mydiv; q++) tau = 0.5 * tau;
                const double xc = fmax(fmin(x - tau * sgn, t_max), t_min);
                const d3 qc = sv_body_point(A, tr, p, xc);
                d3 g2 = mk3(0, 0, 0);
                const double fc = mesh_sdf_grad_warp_lat(M, qc, 1e300, g2, lane, stk);
                if (lane == 0) {
                    S.cand_f[mydiv - 1] = fc; S.cand_x[mydiv - 1] = xc;
                    S.cand_g[mydiv - 1][0] = g2.x; S.cand_g[mydiv - 1][1] = g2.y; S.cand_g[mydiv - 1][2] = g2.z;
                    S.cand_q[mydiv - 1][0] = qc.x; S.cand_q[mydiv - 1][1] = qc.y; S.cand_q[mydiv - 1][2] = qc.z;
                }
            }
            __syncthreads();
            const int dend = min(b0 + SVM_WARPS, 10);
            for (int div = b0; div < dend; div++) {      // the reference's sequential loop over the halvings
                iter = iter + 1;
                if (warp == 0) nevals++;
                const double fc = S.cand_f[div - 1];
                if ((fc - fx) < 0) {
                    x = S.cand_x[div - 1]; fx = fc; fval = fc;
                    g = mk3(S.cand_g[div - 1][0], S.cand_g[div - 1][1], S.cand_g[div - 1][2]);
                    gq = mk3(S.cand_q[div - 1][0], S.cand_q[div - 1][1], S.cand_q[div - 1][2]);
                    accepted = true;
                    break;
                }
                if (div == 9) stop = true;
            }
            __syncthreads();
        }
    }
}

// MESH = false: analytic shapes through the same CTA-per-point structure — the scans are 256 samples wide and exact (an analytic
// SDF is cheap, no bracket pass), the sign descent is the lane-speculative sv_gradient_descent on warp 0.
template <bool MESH>
__device__ __forceinline__ void sv_points_cta_body(const SvArgs &A, const int bx) {
    if (A.rank + A.world * bx >= A.P) return;   // batched launch: this problem has fewer points than the grid is wide (whole CTA leaves)
    const long long work_begin = clock64();
    extern __shared__ __align__(16) double smem[];
    double *sC = smem, *sT = smem + 18 * A.N;
    __shared__ SvmShared S;
#pragma nv_diag_suppress static_var_with_dynamic_init
    __shared__ cuda::barrier<cuda::thread_scope_block> bar;
    stage_traj_block(sC, sT, A.C, A.T, A.N, &bar);
    const TrajView tr = {sT, sC, A.N};
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pk = A.use_order ? A.order[bx] : A.rank + A.world * bx;     // grid.x >= number of points of this rank (batched launches: the largest problem's)
    const DevMesh &M = A.shape.mesh;
    WideStack *stk = &S.stk[warp];
    const d3 p = mk3(A.pts[3 * pk], A.pts[3 * pk + 1], A.pts[3 * pk + 2]);
    const DevCfg &cfg = A.cfg;
    const double dur = A.state[0];
    const int nc = A.meta[0];
    const double inf = 2 * cfg.safety + 0.1;   // safty_hor_inf (swm:383)

    double sdf_value = 1e1, tstar = A.tstar[pk];
    d3 grel = mk3(0, 0, 0);
    unsigned nevals = 0;      // per warp; lane 0 of every warp adds its share to the counter
    bool found = false;

    if (A.g_t) {
        sdf_value = A.g_s[pk]; tstar = A.g_t[pk]; grel = mk3(A.g_g[3 * pk], A.g_g[3 * pk + 1], A.g_g[3 * pk + 2]);
        found = true;
    } else {
        // ---- coarse scan (swm:392-421): in-range bitmap; the cell bracket settles all but a thin band around `inf` ---------
        // consecutive samples go to different warps (an obstacle point's undecided samples — the thin band around `inf` — are
        // consecutive in time and each costs a cooperative search: spread, they run on all warps at once)
        for (int w = tid; w < SV_FLAG_WORDS; w += SVM_THREADS) S.flags[w] = 0u;
        __syncthreads();
        for (int base = 0; base < nc; base += SVM_THREADS) {
            const int k = base + lane * SVM_WARPS + warp;
            bool in = false, undecided = false;
            d3 prel = mk3(0, 0, 0);
            if (k < nc) {
                const double *o = A.poses + 12 * (size_t)k;
                const d3 d = mk3(p.x - __ldg(o), p.y - __ldg(o + 1), p.z - __ldg(o + 2));
                prel = mk3(__ldg(o + 3) * d.x + __ldg(o + 6) * d.y + __ldg(o + 9) * d.z,
                           __ldg(o + 4) * d.x + __ldg(o + 7) * d.y + __ldg(o + 10) * d.z,
                           __ldg(o + 5) * d.x + __ldg(o + 8) * d.y + __ldg(o + 11) * d.z);
                if (MESH) {
                    double blo, bhi;
                    mesh_bracket(M, prel, blo, bhi);
                    if (bhi < inf) in = true;
                    else if (blo < inf) undecided = true;
                } else in = shape_sdf_analytic(A.shape, prel) < inf;
            }
            if (MESH) {
                const double v = mesh_sdf_each(M, undecided, prel, inf, inf, lane, stk);
                if (undecided) in = v < inf;
            }
            if (in) atomicOr(&S.flags[k >> 5], 1u << (k & 31));
        }
        __syncthreads();
        if (warp == 0) nevals += nc;
        const uint32_t *fl = S.flags;
        const int nwords = (nc + 31) >> 5;
        // last run entry (in-range sample whose predecessor is out of range): its SDF initialises range_mindis (quirk Q2)
        int last_entry = -1;
        for (int w = nwords - 1; w >= 0 && last_entry < 0; w--) {
            const uint32_t cur = fl[w];
            const uint32_t prevbit = (w > 0) ? (fl[w - 1] >> 31) : 0u;
            const uint32_t starts = cur & ~((cur << 1) | prevbit);
            if (starts) last_entry = w * 32 + (31 - __clz(starts));
        }
        if (last_entry >= 0) {
            double range_mindis;
            if (MESH) {
                if (warp == 0) {
                    d3 g_;
                    const double v = mesh_sdf_grad_warp_lat(M, sv_body_point(A, tr, p, A.times[last_entry]), inf, g_, lane, stk);
                    if (lane == 0) S.bc[0] = v;
                }
                __syncthreads();
                range_mindis = S.bc[0];
                __syncthreads();
            } else range_mindis = sv_sdf_at(A, tr, p, A.times[last_entry]);
            double range_time_seed = 0.0;
            double min_sdf_star = 1e1;
            d3 g_best = mk3(0, 0, 0), q_best = mk3(0, 0, 0);
            int pos = 0;
            while (pos < nc) {
                int kin = -1;
                for (int w = pos >> 5; w < nwords; w++) {
                    uint32_t cur = fl[w];
                    if (w == (pos >> 5)) cur &= ~((1u << (pos & 31)) - 1u);
                    if (cur) { kin = w * 32 + __ffs(cur) - 1; break; }
                }
                if (kin < 0) break;
                int kout = -1;
                for (int w = kin >> 5; w < nwords; w++) {
                    uint32_t cur = ~fl[w];
                    if (w == (kin >> 5)) cur &= ~((1u << (kin & 31)) - 1u);
                    if (w == nwords - 1 && (nc & 31)) cur &= (1u << (nc & 31)) - 1u;
                    if (cur) { kout = w * 32 + __ffs(cur) - 1; break; }
                }
                if (kout < 0) break;  // run still open at the end of the scan: dropped (quirk Q2)
                const double lb = fmax(0.0, A.times[kin] - 0.2);
                const double ub = fmin(dur, A.times[kout] + 0.2);
                // ---- fine scan of [lb, ub) at dt = 0.02 (swm:423-438): t advances by repeated addition -----------------
                // The reference keeps the FIRST sample attaining the minimum over the interval. A sample whose cell lower
                // bound exceeds the smallest cell upper bound of the interval cannot be that sample: pass 1 brackets every
                // sample from the cell grid (no search), pass 2 runs the exact search on the survivors only.
                const int first = lane * SVM_WARPS + warp;      // sample index of this thread in a round of SVM_THREADS
                double cut = 1e300;
                if (MESH) {
                    double t = lb;
                    for (int q = 0; q < first; q++) t += 0.02;
                    while (t < ub) {
                        cut = fmin(cut, mesh_upper(M, sv_body_point(A, tr, p, t)));
                        for (int q = 0; q < SVM_THREADS; q++) t += 0.02;
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) cut = fmin(cut, __shfl_xor_sync(0xffffffffu, cut, o));
                    if (lane == 0) S.red_d[warp] = cut;
                    __syncthreads();
                    cut = S.red_d[0];
                    for (int w = 1; w < SVM_WARPS; w++) cut = fmin(cut, S.red_d[w]);
                    __syncthreads();
                }
                bool seed_have = false; double seed_f = 0.0; d3 seed_g = mk3(0, 0, 0), seed_q = mk3(0, 0, 0);
                {
                    double t = lb;
                    for (int q = 0; q < first; q++) t += 0.02;
                    int mi = first;
                    double bd = 1e300, bt = 0.0; int bi = 0x7fffffff;
                    while (__any_sync(0xffffffffu, t < ub)) {
                        const bool valid = t < ub;
                        double dis = 1e300;
                        if (MESH) {
                            bool need = false;
                            d3 prel = mk3(0, 0, 0);
                            if (valid) {
                                prel = sv_body_point(A, tr, p, t);
                                double blo, bhi;
                                mesh_bracket(M, prel, blo, bhi);
                                need = blo <= cut;
                            }
                            d3 gl = mk3(0, 0, 0);
                            dis = mesh_sdf_each(M, need, prel, inf, 1e300, lane, stk, &gl);
                            if (dis < bd) { double *bg = S.bestg[warp][lane]; bg[0] = gl.x; bg[1] = gl.y; bg[2] = gl.z; bg[3] = prel.x; bg[4] = prel.y; bg[5] = prel.z; }
                        } else if (valid) dis = sv_sdf_at(A, tr, p, t);
                        nevals += __popc(__ballot_sync(0xffffffffu, valid));
                        if (dis < bd) { bd = dis; bi = mi; bt = t; }      // own samples come in increasing index order
                        for (int q = 0; q < SVM_THREADS; q++) t += 0.02;
                        mi += SVM_THREADS;
                    }
                    // first occurrence of the minimum: lexicographic (value, sample index) min over the CTA
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const double od = __shfl_xor_sync(0xffffffffu, bd, o);
                        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                        const double otm = __shfl_xor_sync(0xffffffffu, bt, o);
                        if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; bt = otm; }
                    }
                    if (lane == 0) { S.red_d[warp] = bd; S.red_i[warp] = bi; S.red_t[warp] = bt; }
                    __syncthreads();
                    bd = S.red_d[0]; bi = S.red_i[0]; bt = S.red_t[0];
                    for (int w = 1; w < SVM_WARPS; w++) {
                        const double od = S.red_d[w]; const int oi = S.red_i[w];
                        if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; bt = S.red_t[w]; }
                    }
                    if (MESH && bd < range_mindis && bd < inf && bi != 0x7fffffff) {   // the seed is this scan's best sample: its search result starts the descent
                        const double *bg = S.bestg[bi % SVM_WARPS][(bi % SVM_THREADS) / SVM_WARPS];
                        seed_have = true; seed_f = bd; seed_g = mk3(bg[0], bg[1], bg[2]); seed_q = mk3(bg[3], bg[4], bg[5]);
                    }
                    __syncthreads();
                    if (bd < range_mindis) { range_mindis = bd; range_time_seed = bt; }
                }
                // ---- descent inside the interval (swm:730-734) ---------------------------------------------------------
                const double tmin_ = fmax(0.0, lb), tmax_ = fmin(ub, dur);
                double sdf_star = 1e1, t_star = 0;
                d3 g_s = mk3(0, 0, 0), q_s = mk3(1e300, 1e300, 1e300);
                if (MESH) svm_descent(A, tr, p, tmin_, tmax_, range_time_seed, S, sdf_star, t_star, g_s, q_s, nevals, lane, warp, seed_have, seed_f, seed_g, seed_q);
                else {
                    if (warp == 0) {
                        sv_gradient_descent(A, tr, p, tmin_, tmax_, range_time_seed, sdf_star, t_star, nevals, lane);
                        if (lane == 0) { S.bc[0] = sdf_star; S.bc[1] = t_star; }
                    }
                    __syncthreads();
                    sdf_star = S.bc[0]; t_star = S.bc[1];
                    __syncthreads();
                }
                if (sdf_star < min_sdf_star) { min_sdf_star = sdf_star; tstar = t_star; found = true; g_best = g_s; q_best = q_s; }
                pos = kout;
            }
            if (found) {
                sdf_value = min_sdf_star;
                // getGradPrelAtTimeStamp (swm:566-572) at the winning t*: the descent already holds it unless the pose differs
                const d3 qf = sv_body_point(A, tr, p, tstar);
                if (MESH && same_bits(qf, q_best)) grel = g_best;
                else {
                    if (warp == 0) {
                        d3 g0 = mk3(0, 0, 0);
                        if (MESH) mesh_sdf_grad_warp_lat(M, qf, 1e300, g0, lane, stk);
                        else g0 = warp_grad(A.shape, qf, lane);
                        if (lane == 0) { S.bc[1] = g0.x; S.bc[2] = g0.y; S.bc[3] = g0.z; }
                    }
                    __syncthreads();
                    grel = mk3(S.bc[1], S.bc[2], S.bc[3]);
                }
            }
        }
    }
    if (lane == 0 && A.counter && nevals) atomicAdd(A.counter, (unsigned long long)nevals);
    if (tid == 0) sv_point_tail(A, sC, tr, pk, p, found, tstar, sdf_value, grel);
    if (tid == 0 && A.work) A.work[pk] = (unsigned)min((clock64() - work_begin) >> 4, 0xffffffffll);
}

// one CTA: this rank's points bucketed by the work they just reported (half-octave buckets), heaviest bucket first
__device__ __forceinline__ int sv_work_bucket(unsigned w) {
    if (w == 0) return 0;
    const int e = 31 - __clz(w);
    return min(63, 2 * e + (e > 0 ? (int)((w >> (e - 1)) & 1u) : 0));
}
__device__ __forceinline__ void sv_order_body(const SvArgs &A) {
    __shared__ unsigned hist[64], base[64];
    const int tid = threadIdx.x;
    if (tid < 64) hist[tid] = 0;
    __syncthreads();
    const int Mloc = (A.P - A.rank + A.world - 1) / A.world;
    for (int i = tid; i < Mloc; i += blockDim.x) atomicAdd(&hist[sv_work_bucket(A.work[A.rank + A.world * i])], 1u);
    __syncthreads();
    if (tid == 0) { unsigned run = 0; for (int b = 63; b >= 0; b--) { base[b] = run; run += hist[b]; } }
    __syncthreads();
    for (int i = tid; i < Mloc; i += blockDim.x) {
        const int pk = A.rank + A.world * i;
        A.order[atomicAdd(&base[sv_work_bucket(A.work[pk])], 1u)] = pk;
    }
}

// ---- reductions --------------------------------------------------------------------------------------------------
__device__ __forceinline__ void sv_reduce_body(const SvArgs &A, const int bx) {
    const int i = bx;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int Mloc = (A.P - A.rank + A.world - 1) / A.world;
    double acc[PARTIAL_STRIDE];
#pragma unroll
    for (int q = 0; q < PARTIAL_STRIDE; q++) acc[q] = 0.0;
    for (int m = threadIdx.x; m < Mloc; m += blockDim.x) {
        const int pk = A.rank + A.world * m;
        if (A.piece[pk] == i) {
            const double *o = A.partial + (size_t)pk * PARTIAL_STRIDE;
#pragma unroll
            for (int q = 0; q < PARTIAL_STRIDE; q++) acc[q] += o[q];
        }
    }
    __shared__ double red[8][PARTIAL_STRIDE];
#pragma unroll
    for (int q = 0; q < PARTIAL_STRIDE; q++) { const double s = warp_sum(acc[q]); if (lane == 0) red[warp][q] = s; }
    __syncthreads();
    if (threadIdx.x < PARTIAL_STRIDE) {
        const int q = threadIdx.x;
        double s = 0.0;
        for (int w = 0; w < 8; w++) s += red[w][q];
        if (q < 18) { const int ax = q / 6, k = q - 6 * ax; A.out[1 + (size_t)ax * 6 * A.N + 6 * i + k] = s; }
        else if (q == 18) A.piece_gdt[i] = s;
        else A.piece_cost[i] = s;
    }
}

__device__ __forceinline__ void sv_finish_body(const SvArgs &A, const int bx) {
    if (threadIdx.x != 0 || bx != 0) return;
    double c = 0.0;
    for (int i = 0; i < A.N; i++) c += A.piece_cost[i];
    A.out[0] = c;
    double run = 0.0;  // gradT(j) += gdT for all j < i (hpp:642-645)  <=>  gradT(j) = sum over pieces i > j
    for (int i = A.N - 1; i >= 0; i--) { A.out[1 + 18 * A.N + i] = run; run += A.piece_gdt[i]; }
    if (A.count_out) *A.count_out = __longlong_as_double(A.counter ? (long long)*(volatile unsigned long long *)A.counter : 0ll);
}

// ---- kernels: single problem (arguments in the constant bank) and batched (blockIdx.y = problem; the problem's argument view is built in
// shared memory from the batch description) — both run the SAME bodies, so a problem's swept-volume term is bit-identical whether it is
// evaluated alone or as one of B --------------------------------------------------------------------------------------------------------
struct SvBatch {
    SvArgs base;              // pointers = problem 0 / point 0; base.P unused
    int B;
    const int *pt_off;        // B + 1: problem b owns points [pt_off[b], pt_off[b+1])
    long long out_stride;     // doubles between two problems' out vectors (19N + 1)
};
__device__ __forceinline__ void sv_make_view(const SvBatch &Bt, int b, SvArgs &V) {
    const unsigned long long *src = reinterpret_cast<const unsigned long long *>(&Bt.base);
    unsigned long long *dst = reinterpret_cast<unsigned long long *>(&V);
    for (int k = threadIdx.x; k < (int)(sizeof(SvArgs) / 8); k += blockDim.x) dst[k] = src[k];
    __syncthreads();
    if (threadIdx.x == 0) {
        const int N = Bt.base.N, p0 = Bt.pt_off[b];
        V.P = Bt.pt_off[b + 1] - p0;
        V.T = Bt.base.T + (size_t)b * N; V.C = Bt.base.C + (size_t)b * 18 * N;
        V.pts = Bt.base.pts + (size_t)3 * p0; V.tstar = Bt.base.tstar + p0; V.sdf = Bt.base.sdf + p0; V.grel = Bt.base.grel + (size_t)3 * p0;
        V.times = Bt.base.times + (size_t)b * SV_MAX_COARSE; V.poses = Bt.base.poses + (size_t)b * 12 * SV_MAX_COARSE;
        V.meta = Bt.base.meta + (size_t)b * 4; V.state = Bt.base.state + (size_t)b * 4;
        V.partial = Bt.base.partial + (size_t)p0 * PARTIAL_STRIDE; V.piece = Bt.base.piece + p0;
        V.piece_gdt = Bt.base.piece_gdt + (size_t)b * N; V.piece_cost = Bt.base.piece_cost + (size_t)b * N;
        V.out = Bt.base.out + (size_t)b * Bt.out_stride;
    }
    __syncthreads();
}
static_assert(sizeof(SvArgs) % 8 == 0, "SvArgs is copied as 64-bit words");

__global__ void __launch_bounds__(256) k_sv_table(const __grid_constant__ SvArgs A) { sv_table_body(A, blockIdx.x); }
template <bool MESH>
__global__ void __launch_bounds__(SVM_THREADS) k_sv_points_cta(const __grid_constant__ SvArgs A) { sv_points_cta_body<MESH>(A, blockIdx.x); }
__global__ void __launch_bounds__(256) k_sv_reduce(const __grid_constant__ SvArgs A) { if ((int)blockIdx.x == A.N) sv_order_body(A); else sv_reduce_body(A, blockIdx.x); }
__global__ void k_sv_finish(const __grid_constant__ SvArgs A) { sv_finish_body(A, blockIdx.x); }

__global__ void __launch_bounds__(256) k_sv_table_b(const __grid_constant__ SvBatch Bt) { __shared__ SvArgs V; sv_make_view(Bt, blockIdx.y, V); sv_table_body(V, blockIdx.x); }
template <bool MESH>
__global__ void __launch_bounds__(SVM_THREADS) k_sv_points_cta_b(const __grid_constant__ SvBatch Bt) {
    __shared__ SvArgs V; sv_make_view(Bt, blockIdx.y, V); sv_points_cta_body<MESH>(V, blockIdx.x);
}
__global__ void __launch_bounds__(256) k_sv_reduce_b(const __grid_constant__ SvBatch Bt) { __shared__ SvArgs V; sv_make_view(Bt, blockIdx.y, V); sv_reduce_body(V, blockIdx.x); }
__global__ void k_sv_finish_b(const __grid_constant__ SvBatch Bt) { __shared__ SvArgs V; sv_make_view(Bt, blockIdx.y, V); sv_finish_body(V, blockIdx.x); }

// ---- host-side state ----------------------------------------------------------------------------------------------
struct SweptState {
    int P = 0;
    // traj_duration (updateTraj, swm:287-296) persists across evaluations: d_state[0] for the single-problem entry points, d_state_b[4 b]
    // for problem b of the batched callback — separate, so that neither path sees the other's trajectories
    DevBuf<double> d_pts, d_tstar, d_sdf, d_grel, d_times, d_poses, d_state, d_state_b, d_partial, d_piece_gdt, d_piece_cost;
    DevBuf<int> d_piece, d_meta;
    DevBuf<unsigned long long> d_counter;
    DevBuf<unsigned> d_work; DevBuf<int> d_order;
    bool order_ready = false; int order_rank = -1, order_world = -1;

    // the only place that replaces the point set: it gives up the current one (and any per-problem sets: set_points_batch sets B
    // after it) before it touches the buffers
    cudaError_t set_points(const double *pts, int n, cudaStream_t st) {
        cudaError_t e = cudaSuccess;
        P = 0; B = 0;
        if (n == 0) return e;
        if ((e = d_pts.upload(pts, (size_t)3 * n, st)) != cudaSuccess) return e;
        if ((e = d_tstar.ensure(n)) != cudaSuccess) return e;
        if ((e = d_sdf.ensure(n)) != cudaSuccess) return e;
        if ((e = d_grel.ensure((size_t)3 * n)) != cudaSuccess) return e;
        if ((e = d_partial.ensure((size_t)n * PARTIAL_STRIDE)) != cudaSuccess) return e;
        if ((e = d_piece.ensure(n)) != cudaSuccess) return e;
        if ((e = d_work.ensure(n)) != cudaSuccess) return e;
        if ((e = d_order.ensure(n)) != cudaSuccess) return e;
        order_ready = false;
        if ((e = cudaMemsetAsync(d_tstar.p, 0, sizeof(double) * n, st)) != cudaSuccess) return e;  // lastTstar := zeros (plan_manager.cpp:254)
        if ((e = cudaMemsetAsync(d_sdf.p, 0, sizeof(double) * n, st)) != cudaSuccess) return e;
        if ((e = cudaMemsetAsync(d_grel.p, 0, sizeof(double) * 3 * n, st)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
        P = n;
        return e;
    }
    cudaError_t ensure_common() {
        cudaError_t e;
        if ((e = d_times.ensure(SV_MAX_COARSE)) != cudaSuccess) return e;
        if ((e = d_poses.ensure((size_t)12 * SV_MAX_COARSE)) != cudaSuccess) return e;
        if ((e = d_meta.ensure(4)) != cudaSuccess) return e;
        if (d_state.n == 0) {
            if ((e = d_state.ensure(4)) != cudaSuccess) return e;
            if ((e = cudaMemset(d_state.p, 0, 4 * sizeof(double))) != cudaSuccess) return e;
        }
        if (d_counter.n == 0) {
            if ((e = d_counter.ensure(2)) != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    // count_out (host entry points only): where the count lands, behind the result vector
    cudaError_t launch(const DevCfg &cfg, const DevShape &shape, int N, const double *d_T, const double *d_C, double *d_out, double *count_out,
                       int rank, int world, cudaStream_t st, const double *g_t, const double *g_s, const double *g_g, int *launches) {
        cudaError_t e;
        if ((e = ensure_common()) != cudaSuccess) return e;
        if ((e = d_piece_gdt.ensure(N)) != cudaSuccess) return e;
        if ((e = d_piece_cost.ensure(N)) != cudaSuccess) return e;
        SvArgs A;
        A.cfg = cfg; A.shape = shape; A.N = N; A.T = d_T; A.C = d_C; A.P = P; A.pts = d_pts.p;
        A.tstar = d_tstar.p; A.sdf = d_sdf.p; A.grel = d_grel.p; A.times = d_times.p; A.poses = d_poses.p; A.meta = d_meta.p;
        A.state = d_state.p; A.partial = d_partial.p; A.piece = d_piece.p; A.piece_gdt = d_piece_gdt.p; A.piece_cost = d_piece_cost.p;
        A.out = d_out; A.counter = d_counter.p; A.count_out = count_out; A.rank = rank; A.world = world; A.g_t = g_t; A.g_s = g_s; A.g_g = g_g;
        // longest-first schedule (searching evaluations of a mesh robot only: the other kernels' points are cheap and uniform)
        const bool record = (g_t == nullptr) && shape.kind == ISDF_SHAPE_MESH;
        if (order_rank != rank || order_world != world) { order_ready = false; order_rank = rank; order_world = world; }
        A.work = record ? d_work.p : nullptr; A.order = d_order.p; A.use_order = (record && order_ready) ? 1 : 0;
        const size_t sm = sizeof(double) * 19 * (size_t)N;
        if (sm > 200 * 1024) return cudaErrorInvalidValue;
        if ((e = cudaMemsetAsync(d_counter.p, 0, sizeof(unsigned long long), st)) != cudaSuccess) return e;
        if (sm > 48 * 1024) {
            cudaFuncSetAttribute(k_sv_table, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            cudaFuncSetAttribute(k_sv_points_cta<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            cudaFuncSetAttribute(k_sv_points_cta<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        }
        k_sv_table<<<SV_TABLE_CTAS, SV_TABLE_THREADS, sm, st>>>(A);
        const int Mloc = (P - rank + world - 1) / world;
        if (Mloc > 0) {
            if (shape.kind == ISDF_SHAPE_MESH) k_sv_points_cta<true><<<(unsigned)Mloc, SVM_THREADS, sm, st>>>(A);
            else k_sv_points_cta<false><<<(unsigned)Mloc, SVM_THREADS, sm, st>>>(A);
        }
        k_sv_reduce<<<N + ((record && Mloc > 0) ? 1 : 0), 256, 0, st>>>(A);   // + one CTA that sorts the points for the next evaluation
        if (record && Mloc > 0) order_ready = true;
        k_sv_finish<<<1, 32, 0, st>>>(A);
        *launches = 3 + (Mloc > 0 ? 1 : 0);
        return cudaGetLastError();
    }
    // ---- batched: B problems, each with its own obstacle point set (concatenated; offsets), its own trajectory (T: B x N, C: B x 18N,
    // per-problem column-major blocks) and its own output vector (B x (19N+1)); one launch per stage, grid.y = problem -------------------
    int B = 0, maxP = 0;
    std::vector<int> h_off;
    DevBuf<int> d_off;
    cudaError_t set_points_batch(int nB, const int *off, const double *pts, cudaStream_t st) {
        cudaError_t e = set_points(pts, off[nB], st);
        if (e != cudaSuccess) return e;
        if ((e = d_off.upload(off, (size_t)nB + 1, st)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
        h_off.assign(off, off + nB + 1);
        maxP = 0;
        for (int b = 0; b < nB; b++) maxP = std::max(maxP, off[b + 1] - off[b]);
        B = nB;
        return cudaSuccess;
    }
    cudaError_t launch_batch(const DevCfg &cfg, const DevShape &shape, int N, const double *d_T, const double *d_Cpp, double *d_out, cudaStream_t st, int *launches) {
        cudaError_t e;
        if ((e = d_times.ensure((size_t)B * SV_MAX_COARSE)) != cudaSuccess) return e;
        if ((e = d_poses.ensure((size_t)12 * B * SV_MAX_COARSE)) != cudaSuccess) return e;
        if ((e = d_meta.ensure((size_t)4 * B)) != cudaSuccess) return e;
        if (d_state_b.n < (size_t)4 * B) {   // a problem's traj_duration starts at 0; growing B keeps the durations of the problems already there
            DevBuf<double> grown;
            if ((e = grown.ensure((size_t)4 * B)) != cudaSuccess) return e;
            if ((e = cudaMemsetAsync(grown.p, 0, sizeof(double) * 4 * B, st)) != cudaSuccess) return e;
            if (d_state_b.n && (e = cudaMemcpyAsync(grown.p, d_state_b.p, sizeof(double) * d_state_b.n, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return e;
            if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;   // the old buffer is freed below
            d_state_b = std::move(grown);
        }
        if (d_counter.n == 0) { if ((e = d_counter.ensure(2)) != cudaSuccess) return e; }
        if ((e = d_piece_gdt.ensure((size_t)B * N)) != cudaSuccess) return e;
        if ((e = d_piece_cost.ensure((size_t)B * N)) != cudaSuccess) return e;
        SvBatch Bt;
        SvArgs &A = Bt.base;
        A.cfg = cfg; A.shape = shape; A.N = N; A.T = d_T; A.C = d_Cpp; A.P = 0; A.pts = d_pts.p;
        A.tstar = d_tstar.p; A.sdf = d_sdf.p; A.grel = d_grel.p; A.times = d_times.p; A.poses = d_poses.p; A.meta = d_meta.p;
        A.state = d_state_b.p; A.partial = d_partial.p; A.piece = d_piece.p; A.piece_gdt = d_piece_gdt.p; A.piece_cost = d_piece_cost.p;
        A.out = d_out; A.counter = d_counter.p; A.count_out = nullptr; A.rank = 0; A.world = 1; A.g_t = nullptr; A.g_s = nullptr; A.g_g = nullptr;
        A.work = nullptr; A.order = nullptr; A.use_order = 0;
        Bt.B = B; Bt.pt_off = d_off.p; Bt.out_stride = 19ll * N + 1;
        const size_t sm = sizeof(double) * 19 * (size_t)N;
        if (sm > 200 * 1024) return cudaErrorInvalidValue;
        if ((e = cudaMemsetAsync(d_counter.p, 0, sizeof(unsigned long long), st)) != cudaSuccess) return e;
        if (sm > 48 * 1024) {
            cudaFuncSetAttribute(k_sv_table_b, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            cudaFuncSetAttribute(k_sv_points_cta_b<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
            cudaFuncSetAttribute(k_sv_points_cta_b<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        }
        k_sv_table_b<<<dim3(SV_TABLE_CTAS, B), SV_TABLE_THREADS, sm, st>>>(Bt);
        if (maxP > 0) {
            if (shape.kind == ISDF_SHAPE_MESH) k_sv_points_cta_b<true><<<dim3(maxP, B), SVM_THREADS, sm, st>>>(Bt);
            else k_sv_points_cta_b<false><<<dim3(maxP, B), SVM_THREADS, sm, st>>>(Bt);
        }
        k_sv_reduce_b<<<dim3(N, B), 256, 0, st>>>(Bt);
        k_sv_finish_b<<<dim3(1, B), 32, 0, st>>>(Bt);
        *launches = 3 + (maxP > 0 ? 1 : 0);
        return cudaGetLastError();
    }
};

}  // namespace isdf
