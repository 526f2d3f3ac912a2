// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_math.hpp header).
// Occupancy grid + AABB gather, trajectory evaluation, the discrete collision term (grad_cost_p wired into the
// time-integral loop), the swept-volume SDF query and the swept-volume penalty loop.
#pragma once
#include "oracle_math.hpp"
#include "oracle_shapes.hpp"
#ifdef _OPENMP
#include <omp.h>
#endif

namespace orc {

// ---------------------------------------------------------------------------------------------
// GridMap3D / PCSmapManager subset (grid:25-39, 135-194, 239-284; pcs:130-170). Occupancy is 1 byte per voxel
// here (the reference stores a double per voxel, GridMap3D.h:215); address = ix*Y*Z + iy*Z + iz (GridMap3D.h:194).
struct Grid {
    int X = 0, Y = 0, Z = 0;
    V3 bmin, bmax;
    double res = 1.0;
    const uint8_t *occ = nullptr;

    void create(const V3 &mn, const V3 &mx, double r) {  // createGridMap (grid:25-39)
        bmin = mn; bmax = mx; res = r;
        X = (int)std::ceil((mx.x - mn.x) / r); Y = (int)std::ceil((mx.y - mn.y) / r); Z = (int)std::ceil((mx.z - mn.z) / r);
    }
    bool in_map(const V3 &p) const {  // isInMap (grid:~60-101)
        return !(p.x < bmin.x || p.y < bmin.y || p.z < bmin.z || p.x > bmax.x || p.y > bmax.y || p.z > bmax.z);
    }
    void grid_index(const V3 &p, int id[3]) const {  // getGridIndex (grid:135-175), incl. its typo branches (quirk Q6)
        if (!in_map(p)) { id[0] = id[1] = id[2] = 0; return; }
        int ix = (int)std::floor((p.x - bmin.x) / res);
        int iy = (int)std::floor((p.y - bmin.y) / res);
        int iz = (int)std::floor((p.z - bmin.z) / res);
        if (ix < 0) ix = 0;
        if (ix >= X) ix = X - 1;
        if (iy < 0) ix = 0;  // sic
        if (iy >= Y) iy = Y - 1;
        if (iz < 0) ix = 0;  // sic
        if (iz >= Z) iz = Z - 1;
        id[0] = ix; id[1] = iy; id[2] = iz;
    }
    bool occupied(int ix, int iy, int iz) const {  // isIndexOccupied(int,int,int) (grid:239-284): out of range => occupied
        if (ix < 0 || ix >= X || iy < 0 || iy >= Y || iz < 0 || iz >= Z) return true;
        return occ[(size_t)ix * Y * Z + (size_t)iy * Z + iz] != 0;
    }
    V3 centre(int ix, int iy, int iz) const {  // getGridCubeCenter (grid:177-194)
        if (ix < 0 || ix >= X || iy < 0 || iy >= Y || iz < 0 || iz >= Z) return V3(0, 0, 0);
        return V3((ix + 0.5) * res, (iy + 0.5) * res, (iz + 0.5) * res) + bmin;
    }
    void proj_in_map(V3 &p) const {  // projInMap (pcs:130-137)
        for (int a = 0; a < 3; a++) { if (p[a] < bmin[a]) p[a] = bmin[a]; if (p[a] > bmax[a]) p[a] = bmax[a]; }
    }
    // index box of an AABB after projInMap (pcs:184-197)
    void index_box(const V3 &c, double h, int lo[3], int hi[3]) const {
        V3 c1 = c - V3(h, h, h), c2 = c + V3(h, h, h);
        proj_in_map(c1); proj_in_map(c2);
        grid_index(c1, lo); grid_index(c2, hi);
    }
    // The obstacle list of plan_manager.cpp:232-254: for every waypoint in order, getPointsInAABBOutOfLastOne (pcs:182-216)
    // inserts the occupied voxels of box(wp + offset) that are NOT in box(previous wp) into a map keyed by voxel id.
    // Output order here: first-inserting waypoint, then the reference's loop order (x, y, z ascending); the reference's own
    // order is the iteration order of an unordered_map (unspecified).
    void gather_obstacle_points(const std::vector<V3> &wps, double h, const V3 &offset, std::vector<V3> &out) const {
        std::vector<char> seen((size_t)X * Y * Z, 0);
        V3 last(999, 999, 999);                                     // tmp_pos initial value (plan_manager.cpp:228)
        for (const V3 &wp : wps) {
            int a0[3], a1[3], l0[3], l1[3];
            index_box(wp + offset, h, a0, a1);
            index_box(last, h, l0, l1);
            for (int i = a0[0]; i <= a1[0]; i++)
                for (int j = a0[1]; j <= a1[1]; j++)
                    for (int k = a0[2]; k <= a1[2]; k++) {
                        if (i > l1[0] || i < l0[0] || j > l1[1] || j < l0[1] || k > l1[2] || k < l0[2]) {
                            if (occupied(i, j, k)) {
                                char &sn = seen[((size_t)i * Y + j) * Z + k];
                                if (!sn) { sn = 1; out.push_back(centre(i, j, k)); }
                            }
                        }
                    }
            last = wp;
        }
    }
    // getPointsInAABB (pcs:148-170)
    void points_in_aabb(const V3 &c, double hx, double hy, double hz, std::vector<V3> &out) const {
        V3 c1 = c - V3(hx, hy, hz), c2 = c + V3(hx, hy, hz);
        proj_in_map(c1); proj_in_map(c2);
        int i1[3], i2[3];
        grid_index(c1, i1); grid_index(c2, i2);
        for (int i = i1[0]; i <= i2[0]; i++)
            for (int j = i1[1]; j <= i2[1]; j++)
                for (int k = i1[2]; k <= i2[2]; k++)
                    if (occupied(i, j, k)) out.push_back(centre(i, j, k));
    }
};

// ---------------------------------------------------------------------------------------------
struct Params {
    // flatness (config.hpp / flat:36-51)
    double mass = 0.61, grav = 9.8, dh = 0.10, dv = 0.10, cp = 0.01, veps = 1e-4;
    // penalties (hpp:678-692)
    double vmax = 10, omgmax = 10, thetamax = 100.0;
    double weight_v = 1000, weight_p = 4000, weight_omg = 1000, weight_theta = 1000;
    double smooth_fac = 1e-2, safety_hor = 0.866;
    int integral_res = 64;
    double bd = 13.0;  // kernel_size * occupancy_resolution (hpp:692)
    int threads = 1;   // threads_num (OpenMP build only)
    int with_dynamics = 1;  // include the vel / body-rate / tilt terms of addTimeIntPenaltyParallel (hpp:505-534)
    int with_collision = 1; // wire grad_cost_p into the sample loop the way hpp:619-626 does for the SV sibling
};

// MINCO coefficient block as the callback sees it: Eigen::MatrixX3d (6N x 3), column-major (hpp:434, 460).
struct Traj {
    int N = 0;
    const double *T = nullptr;
    const double *C = nullptr;  // C[col*6N + 6i + k] = t^k coefficient of piece i, axis col
    double c(int i, int k, int ax) const { return C[(size_t)ax * 6 * N + 6 * i + k]; }
    double total() const { double s = 0; for (int i = 0; i < N; i++) s += T[i]; return s; }  // traj:457-466
    // locatePieceIdx (traj:545-563): mutates t; strict > ; clamps past-the-end into the last piece (quirk Q12)
    int locate(double &t) const {
        int idx; double dur = 0;
        for (idx = 0; idx < N && t > (dur = T[idx]); idx++) t -= dur;
        if (idx == N) { idx--; t += T[idx]; }
        return idx;
    }
    // Piece::getPos_Vel_Acc_Jerk (traj:105-149): running powers of t over ascending coefficients
    void pvaj(double tabs, V3 &p, V3 &v, V3 &a, V3 &j) const {
        double t = tabs;
        const int i = locate(t);
        p = v = a = j = V3();
        double ptn = 1.0, vtn = 1.0, atn = 1.0, jtn = 1.0;
        int vn = 1, am = 1, an = 2, jl = 1, jm = 2, jn = 3;
        for (int k = 0; k <= 5; k++) {  // reference iterates its descending storage from the constant term up
            const V3 ck(c(i, k, 0), c(i, k, 1), c(i, k, 2));
            p += ptn * ck; ptn *= t;
            if (k >= 1) { v += (vn * vtn) * ck; vtn *= t; vn++; }
            if (k >= 2) { a += (am * an * atn) * ck; atn *= t; am++; an++; }
            if (k >= 3) { j += (jl * jm * jn * jtn) * ck; jtn *= t; jl++; jm++; jn++; }
        }
    }
};

struct EvalOut {
    double cost = 0;
    std::vector<double> gradC;  // 6N x 3 column-major
    std::vector<double> gradT;  // N
    long long n_pairs = 0;      // (sample, voxel) pairs that reached the SDF call
    long long n_sdf = 0;        // SDF evaluations counted for the SV path
};

// ---------------------------------------------------------------------------------------------
// grad_cost_p (hpp:766-824): one pose against the occupied voxels in its AABB.
inline bool grad_cost_p(const Params &P, const Grid &G, const Shape &S, const V3 &pos, const M3 &R, const double quat[4],
                        V3 &gradp, double grad_quat[4], double &costp, long long *npairs, bool fair = false) {
    costp = 0.0; gradp = V3(); for (int k = 0; k < 4; k++) grad_quat[k] = 0.0;
    std::vector<V3> ob;
    G.points_in_aabb(pos, P.bd / 2, P.bd / 2, P.bd / 2, ob);
    for (size_t i = 0; i < ob.size(); i++) {
        const V3 d = ob[i] - pos;
        const V3 prel = mulT(R, d);
        if (std::abs(prel.x) > P.bd / 2 || std::abs(prel.y) > P.bd / 2 || std::abs(prel.z) > P.bd / 2) continue;
        V3 grel;
        double sdf;
        if (npairs) (*npairs)++;
        if (fair) { if (!S.sdf_grad_reach(prel, P.safety_hor, sdf, grel)) continue; }   // exact culls of the "fair CPU" arm
        else sdf = S.sdf_grad(prel, grel);  // getSDFWithGradWhenRobotAtState (swm:537-541)
        double sdf_cost = 0, grad_out = 0.0;
        smoothedL1(P.safety_hor - sdf, P.smooth_fac, sdf_cost, grad_out);
        if (sdf_cost > 0) {
            costp += sdf_cost;
            gradp += grad_out * mul(R, grel);
            double sq[4];
            quat_jac_contract(quat, grel, d, sq);
            for (int k = 0; k < 4; k++) grad_quat[k] += -grad_out * sq[k];
        }
    }
    return costp > 0;
}

// One time sample of addTimeIntPenaltyParallel (hpp:454-552) with grad_cost_p re-inserted.
struct SampleContribution { double gdC[18]; double gdT; double cost; int piece; };

inline void eval_sample(const Params &P, const Grid *G, const Shape *S, const Flat &F, const Traj &tr, int count,
                        SampleContribution &out, long long *npairs, bool fair = false) {
    const int K = P.integral_res;
    const int j = count % (K + 1), i = count / (K + 1);
    const double integralFrac = 1.0 / K;
    const double step = tr.T[i] * integralFrac;
    const double s1 = j * step;
    double b0[6], b1[6], b2[6], b3[6], b4[6];
    beta_basis(s1, b0, b1, b2, b3, b4);
    V3 pos, vel, acc, jer, sna;
    for (int ax = 0; ax < 3; ax++)
        for (int k = 0; k < 6; k++) {
            const double ck = tr.c(i, k, ax);
            pos[ax] += ck * b0[k]; vel[ax] += ck * b1[k]; acc[ax] += ck * b2[k]; jer[ax] += ck * b3[k]; sna[ax] += ck * b4[k];
        }
    double quat[4]; V3 omg;
    F.forward(vel, acc, jer, quat, omg);
    const M3 R = quat_to_R(quat);

    double pena = 0.0;
    V3 gradVel, gradPos, gradOmg; double gradQuat[4] = {0, 0, 0, 0};
    if (P.with_dynamics) {
        const double cos_theta = 1.0 - 2.0 * (quat[1] * quat[1] + quat[2] * quat[2]);
        const double violaVel = dot(vel, vel) - P.vmax * P.vmax;
        const double violaOmg = dot(omg, omg) - P.omgmax * P.omgmax;
        const double violaTheta = std::acos(cos_theta) - P.thetamax;
        double f, df;
        if (smoothedL1(violaVel, P.smooth_fac, f, df)) { gradVel += (P.weight_v * df * 2.0) * vel; pena += P.weight_v * f; }
        if (smoothedL1(violaOmg, P.smooth_fac, f, df)) { gradOmg += (P.weight_omg * df * 2.0) * omg; pena += P.weight_omg * f; }
        if (smoothedL1(violaTheta, P.smooth_fac, f, df)) {
            const double sc = P.weight_theta * df / std::sqrt(1.0 - cos_theta * cos_theta) * 4.0;
            gradQuat[1] += sc * quat[1]; gradQuat[2] += sc * quat[2];
            pena += P.weight_theta * f;
        }
    }
    if (P.with_collision && G && S) {
        V3 gp; double gq[4], cp;
        if (grad_cost_p(P, *G, *S, pos, R, quat, gp, gq, cp, npairs, fair)) {  // wired as hpp:619-626
            gradPos += P.weight_p * gp;
            for (int k = 0; k < 4; k++) gradQuat[k] += P.weight_p * gq[k];
            pena += P.weight_p * cp;
        }
    }
    V3 gP, gV, gA, gJ;
    F.backward(vel, acc, jer, gradPos, gradVel, gradQuat, gradOmg, gP, gV, gA, gJ);
    const double node = (j == 0 || j == K) ? 0.5 : 1.0;
    const double alpha = j * integralFrac;
    for (int ax = 0; ax < 3; ax++)
        for (int k = 0; k < 6; k++)
            out.gdC[ax * 6 + k] = (b0[k] * gP[ax] + b1[k] * gV[ax] + b2[k] * gA[ax] + b3[k] * gJ[ax]) * node * step;
    out.gdT = (dot(gP, vel) + dot(gV, acc) + dot(gA, jer) + dot(gJ, sna)) * alpha * node * step + node * integralFrac * pena;
    out.cost = node * step * pena;
    out.piece = i;
}

// addTimeIntPenaltyParallel (hpp:432-554), accumulating into cost/gradC/gradT like the reference does.
// use_omp = false: serial, deterministic order (THE ORACLE).  use_omp = true: the reference's
// `parallel for schedule(dynamic)` + `critical` structure (the CPU baseline; nondeterministic order).
// rank/world: evaluate only samples with count % world == rank (partial sums; test harness for the multi-GPU sharding)
// fair = true (with use_omp): the "fair CPU" arm of BASELINE.md §2 — per-thread accumulators merged once instead of the critical section,
// and the exact culls of Shape::sdf_grad_reach; same cost and gradient up to summation order.
inline void eval_discrete(const Params &P, const Grid *G, const Shape *S, const Traj &tr, EvalOut &out, bool use_omp, int rank = 0, int world = 1,
                          bool fair = false) {
    Flat F; F.reset(P.mass, P.grav, P.dh, P.dv, P.cp, P.veps);
    const int N = tr.N, K = P.integral_res, total = N * (K + 1);
    out.gradC.assign((size_t)18 * N, 0.0); out.gradT.assign(N, 0.0); out.cost = 0; out.n_pairs = 0;
    auto accumulate = [&](const SampleContribution &c) {
        for (int ax = 0; ax < 3; ax++)
            for (int k = 0; k < 6; k++) out.gradC[(size_t)ax * 6 * N + 6 * c.piece + k] += c.gdC[ax * 6 + k];
        out.gradT[c.piece] += c.gdT;
        out.cost += c.cost;
    };
    if (!use_omp) {
        for (int count = 0; count < total; count++) {
            if (count % world != rank) continue;
            SampleContribution c; eval_sample(P, G, S, F, tr, count, c, &out.n_pairs); accumulate(c);
        }
        return;
    }
    if (fair) {
#ifdef _OPENMP
#pragma omp parallel num_threads(P.threads)
#endif
        {
            std::vector<double> lg((size_t)19 * N + 1, 0.0);   // thread-local [gradC | gradT | cost]
            long long lnp = 0;
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 4) nowait
#endif
            for (int count = 0; count < total; count++) {
                if (count % world != rank) continue;
                SampleContribution c;
                eval_sample(P, G, S, F, tr, count, c, &lnp, true);
                for (int ax = 0; ax < 3; ax++)
                    for (int k = 0; k < 6; k++) lg[(size_t)ax * 6 * N + 6 * c.piece + k] += c.gdC[ax * 6 + k];
                lg[(size_t)18 * N + c.piece] += c.gdT;
                lg[(size_t)19 * N] += c.cost;
            }
#ifdef _OPENMP
#pragma omp critical
#endif
            {
                for (size_t k = 0; k < (size_t)18 * N; k++) out.gradC[k] += lg[k];
                for (int k = 0; k < N; k++) out.gradT[k] += lg[(size_t)18 * N + k];
                out.cost += lg[(size_t)19 * N]; out.n_pairs += lnp;
            }
        }
        return;
    }
#ifdef _OPENMP
#pragma omp parallel for num_threads(P.threads) schedule(dynamic)
#endif
    for (int count = 0; count < total; count++) {
        if (count % world != rank) continue;
        SampleContribution c; long long np = 0;
        eval_sample(P, G, S, F, tr, count, c, &np);
#ifdef _OPENMP
#pragma omp critical
#endif
        { accumulate(c); out.n_pairs += np; }
    }
}

// ---------------------------------------------------------------------------------------------
// SweptVolumeManager subset (swm:287-296, 332-358, 367-445, 550-572, 593-662, 710-747, 1000-1062)
struct SweptVolume {
    const Params *P; const Shape *S; const Traj *tr; Flat F;
    double traj_duration = 0;
    long long n_sdf = 0;

    void update() { const double td = tr->total(); if (td < 3 * 1e2) traj_duration = td; }  // updateTraj (swm:287-296), quirk Q14

    void state(double t, V3 &x, M3 &R) const {  // getStateOnTrajStamp (swm:332-341)
        V3 v, a, j; tr->pvaj(t, x, v, a, j);
        double q[4]; F.forward(v, a, j, q);
        R = quat_to_R(q);
    }
    double sdf_at(const V3 &p, double t) {  // getSDFAtTimeStamp (swm:550-556) via posEva2Rel (swm:353-358)
        V3 x; M3 R; state(t, x, R); n_sdf++;
        return S->sdf(mulT(R, p - x));
    }
    V3 grad_prel_at(const V3 &p, double t) {  // getGradPrelAtTimeStamp (swm:566-572)
        V3 x; M3 R; state(t, x, R);
        return S->grad(mulT(R, p - x));
    }
    double sdf_dot_at(const V3 &p, double t) {  // getSDF_DOTAtTimeStampOptimized (swm:593-662)
        V3 x, v, a, j; tr->pvaj(t, x, v, a, j);
        double q[4]; V3 omg; F.forward(v, a, j, q, omg);
        const M3 R = quat_to_R(q);
        const V3 tmp = mulT(R, p - x);
        const V3 g = S->grad(tmp);
        // point_velocity = -(R^T v + w_hat * tmp)
        const V3 pv = -(mulT(R, v) + cross(omg, tmp));
        return dot(g, pv);
    }
    // choiceTInit with ranges (swm:367-445), quirk Q2 preserved
    void choice_t_init(const V3 &p, double dt, std::vector<double> &rl, std::vector<double> &rr, std::vector<double> &rts) {
        const double rough_dt = 0.2;
        double mindis = 1e9, range_mindis = 1e9, dis = 1e9, range_time_seed = 0.0, tou_lb = 0, tou_ub = 0;
        const double inf = 2 * P->safety_hor + 0.1;
        rl.clear(); rr.clear(); rts.clear();
        bool in_range = false;
        for (double t = 0; t < traj_duration; t += rough_dt) {
            dis = sdf_at(p, t);
            if (dis < mindis) mindis = dis;
            if (dis < inf) {
                if (!in_range) { in_range = true; range_mindis = dis; tou_lb = std::max(0.0, t - rough_dt); tou_ub = t; }
                else tou_ub = std::min(traj_duration, t + rough_dt);
            } else if (in_range) {
                in_range = false; tou_ub = std::min(traj_duration, t + rough_dt);
                rl.push_back(tou_lb); rr.push_back(tou_ub);
            }
        }
        const size_t n = rl.size();
        for (size_t i = 0; i < n; i++) {
            for (double t = rl[i]; t < rr[i]; t += dt) {
                dis = sdf_at(p, t);
                if (dis < range_mindis) { range_time_seed = t; range_mindis = dis; }
            }
            rts.push_back(range_time_seed);
        }
    }
    // test hook: choiceTInit's coarse loop as above, recorded instead of acted on. Sets bit k of bits (words of 32) when coarse sample k is
    // in range; returns the number of coarse samples (at most 32 * words: later samples are counted, not recorded). margin = the smallest
    // |dis - inf| over the samples (how far the closest coarse decision is from flipping). carried = closed runs after the first whose fine
    // scan leaves range_mindis unchanged, so that their descent starts from an earlier run's seed.
    int coarse(const V3 &p, uint32_t *bits, int words, double &margin, int &carried) {
        const double inf = 2 * P->safety_hor + 0.1;
        for (int w = 0; w < words; w++) bits[w] = 0u;
        margin = 1e300;
        int nc = 0;
        for (double t = 0; t < traj_duration; t += 0.2) {
            const double dis = sdf_at(p, t);
            margin = std::min(margin, std::abs(dis - inf));
            if (dis < inf && nc < 32 * words) bits[nc >> 5] |= 1u << (nc & 31);
            nc++;
        }
        std::vector<double> rl, rr, rts;
        choice_t_init(p, 0.02, rl, rr, rts);
        carried = 0;
        for (size_t i = 1; i < rts.size(); i++) carried += rts[i] == rts[i - 1];
        return nc;
    }
    // gradientDescent (swm:1000-1062): sign-descent with step halving, quirk Q5
    void gradient_descent(double t_min, double t_max, double x0, double &fx, double &x, const V3 &p) {
        const int max_iter = 300; const double alpha = 0.02, tol = 1e-5;
        double tau = alpha, g = 0.0, prev_x = 10000000.0;
        int iter = 0; bool stop = false;
        x = x0;
        while (iter < max_iter && !stop && std::abs(x - prev_x) > tol) {
            if (iter == 0) fx = sdf_at(p, x);
            g = sdf_dot_at(p, x);
            tau = alpha; prev_x = x;
            for (int div = 1; div < 10; div++) {
                iter = iter + 1;
                g = sdf_dot_at(p, x);
                double xc = x - tau * ((int)(g > 0) - (int)(g < 0));
                xc = std::max(std::min(xc, t_max), t_min);
                const double fc = sdf_at(p, xc);
                if ((fc - fx) < 0) { x = xc; fx = fc; break; }
                tau = 0.5 * tau;
                if (div == 9) stop = true;
            }
        }
    }
    // getSDFofSweptVolume<true>(p, time_seed_f, grad_prel, set_ts=false) (swm:710-747); quirks Q3, Q4
    double sdf_swept(const V3 &p, double &time_seed_f, V3 &grad_prel) {
        double t_star = 0, sdf_star = 1e1, min_sdf_star = 1e1;
        std::vector<double> rl, rr, rts;
        choice_t_init(p, 0.02, rl, rr, rts);
        for (size_t i = 0; i < rl.size(); i++) {
            const double tmin_ = std::max(0.0, rl[i]), tmax_ = std::min(rr[i], traj_duration);
            gradient_descent(tmin_, tmax_, rts[i], sdf_star, t_star, p);
            if (sdf_star < min_sdf_star) { min_sdf_star = sdf_star; time_seed_f = t_star; grad_prel = grad_prel_at(p, t_star); }
        }
        return min_sdf_star;
    }
};

// grad_cost_p_sw (hpp:827-866)
inline bool grad_cost_p_sw(const Params &P, const V3 &pos_eva, const V3 &pos_obj, const M3 &R, const double quat[4],
                           double sdf_value, const V3 &grel, V3 &gradp, double grad_quat[4], double &costp) {
    costp = 0; gradp = V3(); for (int k = 0; k < 4; k++) grad_quat[k] = 0;
    double sdf_cost = -1.0, dout = 0.0;
    smoothedL1(P.safety_hor - sdf_value, 0.01, sdf_cost, dout);
    if (sdf_cost > 0) {
        costp += sdf_cost;
        gradp += dout * mul(R, grel);
        const V3 d = pos_eva - pos_obj;
        double sq[4]; quat_jac_contract(quat, grel, d, sq);
        for (int k = 0; k < 4; k++) grad_quat[k] += -dout * sq[k];
    }
    return costp > 2.220446049250313e-16;  // DBL_EPSILON
}

// addSaftyPenaOnSweptVolumeParallel (hpp:557-649). tstar is lastTstar (in/out, hpp:576-578).
// If tstar_given != nullptr the t* search is skipped and the tail is evaluated at the given t*/sdf*/g_rel
// (parity tier T1, SURVEY §7).
struct SweptGiven { const double *tstar, *sdf, *grel; };
// prev_duration: the SweptVolumeManager's traj_duration before this evaluation (0 for a fresh manager), which a trajectory of 300 s or
// longer leaves in place (quirk Q14)
inline void eval_swept(const Params &P, const Shape &S, const Traj &tr, int npts, const double *pts, double *tstar,
                       EvalOut &out, bool use_omp, double *sdf_out = nullptr, double *grel_out = nullptr,
                       const SweptGiven *given = nullptr, double prev_duration = 0.0) {
    Flat F; F.reset(P.mass, P.grav, P.dh, P.dv, P.cp, P.veps);
    const int N = tr.N;
    out.gradC.assign((size_t)18 * N, 0.0); out.gradT.assign(N, 0.0); out.cost = 0; out.n_sdf = 0;
    auto body = [&](int k, double gdC[18], double &gdT, double &pena, int &piece, long long &nsdf) {
        SweptVolume sv; sv.P = &P; sv.S = &S; sv.tr = &tr; sv.F = F; sv.traj_duration = prev_duration; sv.update();
        const V3 pe(pts[3 * k], pts[3 * k + 1], pts[3 * k + 2]);
        V3 grel;  // uninitialised Vector3d in the reference (hpp:574); zero here — unused when no interval (quirk Q3)
        double sdf_value;
        if (given) {
            sdf_value = given->sdf[k]; tstar[k] = given->tstar[k];
            grel = V3(given->grel[3 * k], given->grel[3 * k + 1], given->grel[3 * k + 2]);
        } else {
            sdf_value = sv.sdf_swept(pe, tstar[k], grel);
        }
        nsdf = sv.n_sdf;
        if (sdf_out) sdf_out[k] = sdf_value;
        if (grel_out) { grel_out[3 * k] = grel.x; grel_out[3 * k + 1] = grel.y; grel_out[3 * k + 2] = grel.z; }
        double tl = tstar[k];
        const int i = tr.locate(tl);
        double b0[6], b1[6], b2[6], b3[6], b4[6];
        beta_basis(tl, b0, b1, b2, b3, b4);
        V3 pos, vel, acc, jer, sna;
        for (int ax = 0; ax < 3; ax++)
            for (int q = 0; q < 6; q++) {
                const double ck = tr.c(i, q, ax);
                pos[ax] += ck * b0[q]; vel[ax] += ck * b1[q]; acc[ax] += ck * b2[q]; jer[ax] += ck * b3[q]; sna[ax] += ck * b4[q];
            }
        double quat[4]; F.forward(vel, acc, jer, quat);
        const M3 R = quat_to_R(quat);
        V3 gradPos, gradVel, gradOmg; double gradQuat[4] = {0, 0, 0, 0};
        pena = 0.0;
        V3 gp; double gq[4], cp;
        if (grad_cost_p_sw(P, pe, pos, R, quat, sdf_value, grel, gp, gq, cp)) {
            gradPos += P.weight_p * gp;
            for (int q = 0; q < 4; q++) gradQuat[q] += P.weight_p * gq[q];
            pena += P.weight_p * cp;
        }
        V3 gP, gV, gA, gJ;
        F.backward(vel, acc, jer, gradPos, gradVel, gradQuat, gradOmg, gP, gV, gA, gJ);
        for (int ax = 0; ax < 3; ax++)
            for (int q = 0; q < 6; q++) gdC[ax * 6 + q] = b0[q] * gP[ax] + b1[q] * gV[ax] + b2[q] * gA[ax] + b3[q] * gJ[ax];
        gdT = (-dot(gP, vel) + -dot(gV, acc) + -dot(gA, jer) + -dot(gJ, sna));
        piece = i;
    };
    auto accumulate = [&](const double gdC[18], double gdT, double pena, int piece) {
        out.cost += pena;
        for (int ax = 0; ax < 3; ax++)
            for (int q = 0; q < 6; q++) out.gradC[(size_t)ax * 6 * N + 6 * piece + q] += gdC[ax * 6 + q];
        for (int j = 0; j < piece; j++) out.gradT[j] += gdT;  // hpp:642-645
    };
    if (!use_omp) {
        for (int k = 0; k < npts; k++) {
            double gdC[18], gdT, pena; int piece; long long ns;
            body(k, gdC, gdT, pena, piece, ns); accumulate(gdC, gdT, pena, piece); out.n_sdf += ns;
        }
        return;
    }
#ifdef _OPENMP
#pragma omp parallel for num_threads(P.threads) schedule(dynamic)
#endif
    for (int k = 0; k < npts; k++) {
        double gdC[18], gdT, pena; int piece; long long ns;
        body(k, gdC, gdT, pena, piece, ns);
#ifdef _OPENMP
#pragma omp critical
#endif
        { accumulate(gdC, gdT, pena, piece); out.n_sdf += ns; }
    }
}

}  // namespace orc
