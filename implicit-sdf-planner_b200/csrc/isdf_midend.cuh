// Mid-end pose term on the device: OriTraj::addPosePenalty (planner_algorithm/mid_end.hpp:201-260) for B problems at once, the one
// stage of OriTraj::costFunction (mid_end.hpp:262-304) that the back end's batched callback does not already have. The callback of
// isdf_midend_batch is k_minco_forward -> k_midend_pose -> k_minco_backward (seq_terms = 1), all three on the concatenated layout of
// isdf_minco.cuh.
//
// k_midend_pose: one thread per (problem, piece). Piece 0 has no term; piece i + 1 carries waypoint i's term, evaluated at
// s = T_{i+1} * (1 / K) of piece i + 1 (not at the junction where xi_i sits):
//   d = p(s) - Q_i, n = sqrt((d0 d0 + d1 d1) + d2 d2), c = (n n) n, g = (3 (n n)) (d / n),
//   gradC rows of piece i + 1 = w (beta0[k] g[ax]), gradT = w (c (alpha (g . v(s)))), piece cost = w c,
// and all three are zero unless c > 0 (grad_cost_dir's `return cost > 0`, mid_end.hpp:198). The T entry is the reference's, cost
// factor included; it is not the derivative of the cost (include/isdf.h). Every row of the output is written, so the buffer is the
// `disc_out` / `piece_cost` input of k_minco_backward with no clearing: zero where there is no term.
// The unit is compiled with -fmad=false and every sum runs left to right: host/isdf_midend.hpp does the same arithmetic, bit for bit.
// A ragged batch (poff != null, include/isdf.h) puts problem b's pieces at [poff[b], poff[b+1]) and its waypoints at rows
// [poff[b] - b, poff[b+1] - b - 1); a thread finds its problem by a binary search of the offsets.
#pragma once
#include "isdf_types.cuh"

namespace isdf {

struct MidendArgs {
    int B, N;                // problems, pieces per problem (ragged: unused)
    int P;                   // pieces of the batch (B N when uniform)
    const int *poff;         // may be null: B + 1 piece offsets of a ragged batch
    int K;                   // integralRes (isdf_config.integral_intervs)
    double weight;           // weightPR
    const double *T;         // P durations
    const double *C;         // 18P concatenated coefficient block (k_minco_forward's C)
    const double *wp;        // (P - B) x 3 waypoints Q
    double *out;             // 19P + 1: [unused | gradC 18P | gradT P], k_minco_backward's disc_out layout
    double *piece_cost;      // P
};

// the problem that owns row q of a ragged batch: the last b with off[b] <= q (off: B + 1 increasing offsets, off[0] = 0)
__device__ __forceinline__ int ragged_owner(const int *off, int B, long long q) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= q) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(128) k_midend_pose(const MidendArgs A) {
    const long long BN = A.P;
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= BN) return;
    const int b = A.poff ? ragged_owner(A.poff, A.B, q) : (int)(q / A.N);
    const int p0 = A.poff ? A.poff[b] : b * A.N, seg = (int)(q - p0);
    const size_t rows = (size_t)6 * BN;
    double beta0[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
    double gT = 0.0, cost = 0.0;
    bool on = false;
    if (seg > 0) {
        const double alpha = 1.0 / A.K;
        const double s1 = alpha * A.T[q], s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
        beta0[0] = 1.0; beta0[1] = s1; beta0[2] = s2; beta0[3] = s3; beta0[4] = s4; beta0[5] = s5;
        const double beta1[6] = {0.0, 1.0, 2.0 * s1, 3.0 * s2, 4.0 * s3, 5.0 * s4};
        const double *Q = A.wp + ((size_t)(p0 - b) + (seg - 1)) * 3;
        double d[3], v[3];
#pragma unroll
        for (int ax = 0; ax < 3; ax++) {
            const double *c = A.C + (size_t)ax * rows + (size_t)6 * q;
            double p = 0.0, vv = 0.0;
#pragma unroll
            for (int k = 0; k < 6; k++) { p += c[k] * beta0[k]; vv += c[k] * beta1[k]; }
            d[ax] = p - Q[ax];
            v[ax] = vv;
        }
        const double n = sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
        const double c3 = (n * n) * n;
        if (c3 > 0.0) {
            on = true;
            const double g2 = 3.0 * (n * n);
#pragma unroll
            for (int ax = 0; ax < 3; ax++) g[ax] = g2 * (d[ax] / n);
            const double gv = alpha * ((g[0] * v[0] + g[1] * v[1]) + g[2] * v[2]);
            gT = A.weight * (c3 * gv);
            cost = A.weight * c3;
        }
    }
#pragma unroll
    for (int ax = 0; ax < 3; ax++) {
        double *o = A.out + 1 + (size_t)ax * rows + (size_t)6 * q;
#pragma unroll
        for (int k = 0; k < 6; k++) o[k] = on ? A.weight * (beta0[k] * g[ax]) : 0.0;
    }
    A.out[1 + 18 * (size_t)BN + q] = gT;
    A.piece_cost[q] = cost;
}

// the starting point of getOriTraj (mid_end.cpp:21-36): tau = backwardT(init_time) for every piece, xi = the waypoints. X rows of x in all;
// ragged (poff, xoff: B + 1 piece and decision-vector offsets) or uniform (both null: N pieces each)
__global__ void __launch_bounds__(128) k_midend_init(int B, int N, const int *poff, const int *xoff, long long X, double tau0, const double *wp,
                                                     double *x) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= X) return;
    const int dim = 4 * N - 3;
    const int b = xoff ? ragged_owner(xoff, B, q) : (int)(q / dim);
    const int k = (int)(q - (xoff ? (long long)xoff[b] : (long long)b * dim));
    const int Nb = poff ? poff[b + 1] - poff[b] : N;
    const size_t w0 = poff ? (size_t)(poff[b] - b) : (size_t)b * (N - 1);   // the problem's first waypoint row
    x[q] = k < Nb ? tau0 : wp[3 * w0 + (k - Nb)];
}

}  // namespace isdf
