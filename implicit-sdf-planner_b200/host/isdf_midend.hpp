// Host-side mid-end: OriTraj::costFunction (planner_algorithm/mid_end.hpp:262-304) with its pose term addPosePenalty (:201-260), and the
// getOriTraj driver (mid_end.cpp:3-94) on host/isdf_lbfgs.hpp. Same arithmetic as the device callback of isdf_midend_batch
// (csrc/isdf_midend.cuh + isdf_minco.cuh with seq_terms = 1): the pose term of every piece is computed into its own arrays (zero where there
// is none) and added to the energy partials entry by entry, the piece costs are added to the energy one at a time, every sum runs left to
// right — so host and device agree bit for bit. The definition, its quirk (the T entry carries the cost factor) and the IEEE form that
// replaces the reference's pow are documented in include/isdf.h.
#pragma once
#include "isdf_minco.hpp"
#include "isdf_cost_callback.hpp"
#include "isdf_lbfgs.hpp"
#include <cmath>
#include <vector>

namespace isdf_host {

struct MidEnd {
    int N = 0;                 // pieces
    int K = 64;                // integralRes (isdf_config.integral_intervs)
    double weight = 1000.0;    // weightPR
    double rho = 200.0;        // rho_mid_end
    int cancel_after = 8000;   // earlyExit: cancel once k > cancel_after; 0 = never
    MincoS3 minco;
    std::vector<double> Q, times, points, gradC, gradT, termC, termT, pc, gradPts, gradTimes;

    void setup(int pieces, const double *head3x3, const double *tail3x3, const double *waypoints) {
        N = pieces;
        minco.setConditions(head3x3, tail3x3, N);
        Q.assign(waypoints, waypoints + (size_t)3 * (N - 1));
        times.assign(N, 0.0); points.assign((size_t)3 * (N - 1), 0.0);
        gradC.assign((size_t)18 * N, 0.0); gradT.assign(N, 0.0); termC.assign((size_t)18 * N, 0.0); termT.assign(N, 0.0); pc.assign(N, 0.0);
        gradPts.assign((size_t)3 * (N - 1), 0.0); gradTimes.assign(N, 0.0);
    }

    // addPosePenalty into termC / termT / pc: piece i + 1 at s = T_{i+1} * (1 / K) against waypoint i
    void poseTerms(const double *coeffs) {
        std::fill(termC.begin(), termC.end(), 0.0); std::fill(termT.begin(), termT.end(), 0.0); std::fill(pc.begin(), pc.end(), 0.0);
        const double alpha = 1.0 / K;
        for (int seg = 1; seg < N; seg++) {
            const double s1 = alpha * times[seg], s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
            const double beta0[6] = {1.0, s1, s2, s3, s4, s5};
            const double beta1[6] = {0.0, 1.0, 2.0 * s1, 3.0 * s2, 4.0 * s3, 5.0 * s4};
            double d[3], v[3];
            for (int ax = 0; ax < 3; ax++) {
                const double *c = coeffs + (size_t)ax * 6 * N + 6 * seg;
                double p = 0.0, vv = 0.0;
                for (int k = 0; k < 6; k++) { p += c[k] * beta0[k]; vv += c[k] * beta1[k]; }
                d[ax] = p - Q[3 * (seg - 1) + ax];
                v[ax] = vv;
            }
            const double n = std::sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
            const double c3 = (n * n) * n;
            if (!(c3 > 0.0)) continue;                       // grad_cost_dir returns cost > 0 (mid_end.hpp:198)
            const double g2 = 3.0 * (n * n);
            double g[3];
            for (int ax = 0; ax < 3; ax++) g[ax] = g2 * (d[ax] / n);
            const double gv = alpha * ((g[0] * v[0] + g[1] * v[1]) + g[2] * v[2]);
            for (int ax = 0; ax < 3; ax++)
                for (int k = 0; k < 6; k++) termC[(size_t)ax * 6 * N + 6 * seg + k] = weight * (beta0[k] * g[ax]);
            termT[seg] = weight * (c3 * gv);                 // the reference's T entry, cost factor included (mid_end.hpp:256)
            pc[seg] = weight * c3;
        }
    }

    // lbfgs_eval_raw_t
    static double costFunction(void *ptr, const double *x, double *g, int n, double *p_cost) {
        MidEnd &o = *static_cast<MidEnd *>(ptr);
        const int dimTau = o.N, dimXi = 3 * (o.N - 1);
        if (p_cost) *p_cost = 0.0;
        if (n != dimTau + dimXi) return std::nan("");
        BackEnd::forwardT(x, o.times.data(), dimTau);
        for (int k = 0; k < dimXi; k++) o.points[k] = x[dimTau + k];
        o.minco.setParameters(o.points.data(), o.times.data());
        double cost = o.minco.getEnergy();
        o.minco.getEnergyPartialGradByCoeffs(o.gradC.data());
        o.minco.getEnergyPartialGradByTimes(o.gradT.data());
        o.poseTerms(o.minco.coeffs().data());
        for (size_t k = 0; k < o.gradC.size(); k++) o.gradC[k] = o.gradC[k] + o.termC[k];
        for (int i = 0; i < o.N; i++) o.gradT[i] = o.gradT[i] + o.termT[i];
        for (int i = 0; i < o.N; i++) cost += o.pc[i];
        o.minco.propagateGrad(o.gradC.data(), o.gradT.data(), o.gradPts.data(), o.gradTimes.data());
        double tsum = 0.0;
        for (int i = 0; i < dimTau; i++) tsum += o.times[i];
        cost += o.rho * tsum;
        for (int i = 0; i < dimTau; i++) o.gradTimes[i] += o.rho;
        BackEnd::backwardGradT(x, o.gradTimes.data(), g, dimTau);
        for (int k = 0; k < dimXi; k++) g[dimTau + k] = o.gradPts[k];
        return cost;
    }

    // earlyExit (mid_end.hpp:613-631) without its visualisation and sleep
    static int earlyExit(void *ptr, const double *, const double *, double, double, int k, int, int) {
        const MidEnd &o = *static_cast<const MidEnd *>(ptr);
        return o.cancel_after > 0 && k > o.cancel_after;
    }

    // getOriTraj (mid_end.cpp:3-94): x (4N-3) is set to [backwardT(init_time) | Q] and returns the solution; T (N) and coeffs (18N) are
    // forwardT + MINCO of it whatever the return code
    int getOriTraj(double init_time, const LbfgsParams &pr, double *x, double &f, double *T, double *coeffs, LbfgsStats *st = nullptr) {
        std::vector<double> t0(N, init_time);
        BackEnd::backwardT(t0.data(), x, N);
        for (int k = 0; k < 3 * (N - 1); k++) x[N + k] = Q[k];
        const int ret = lbfgs_optimize(4 * N - 3, x, f, &MidEnd::costFunction, nullptr, &MidEnd::earlyExit, this, pr, st);
        BackEnd::forwardT(x, times.data(), N);
        for (int k = 0; k < 3 * (N - 1); k++) points[k] = x[N + k];
        minco.setParameters(points.data(), times.data());
        if (T) for (int i = 0; i < N; i++) T[i] = times[i];
        if (coeffs) for (int k = 0; k < 18 * N; k++) coeffs[k] = minco.coeffs()[k];
        return ret;
    }
};

}  // namespace isdf_host
