// Batched MINCO (s = 3, non-uniform time) on the device — the step on BOTH sides of the hot loop (SURVEY §8f row 1):
//   k_minco_forward : decision vector x_b = [tau (N) | xi (3(N-1))] -> T = forwardT(tau) (back_end_optimizer.hpp:214-241) ->
//                     banded system of MINCO_S3NU::setParameters (utils/minco.hpp:433-513), LU without pivoting
//                     (BandedSystem::factorizeLU, minco.hpp:99-135), solve (:137-166) -> coefficient block, jerk energy and
//                     its partial gradients (minco.hpp:530-582);
//   k_minco_backward: (dJ/dc, dJ/dT) -> solveAdj (minco.hpp:168-197) -> propogateGrad (minco.hpp:584-654) -> + rho ->
//                     backwardGradT / backwardGradP (hpp:283-330) -> gradient of the decision vector.
// One WARP per problem; the 6N x 6N band (13 diagonals) and the right-hand sides live in shared memory. The elimination is
// sequential in the pivot index — that is the algorithm — but every elementary update a(i,j) -= a(i,k) * a(k,j) of one pivot
// step is independent, so the lanes take one (i,j) pair each: the arithmetic (one multiply, one subtract per element, no
// FMA: the library is built with -fmad=false) and therefore every bit of the result equals the sequential host port
// (host/isdf_minco.hpp), which the CPU tests pin against the oracle's dense solve.
// The coefficient blocks of the B problems are written CONCATENATED (piece b*N + i of a 6BN x 3 column-major block), which is
// exactly what one launch of the discrete kernels consumes: the time-integral term couples nothing across pieces.
// A ragged batch (poff != null, include/isdf.h) gives problem b the pieces [poff[b], poff[b+1]) instead of [b N, b N + N): every per-piece
// array is indexed by the problem's first piece p0, x by 4 p0 - 3 b, and the per-problem arithmetic is the same, so a problem's bits do
// not depend on the batch around it.
#pragma once
#include "isdf_types.cuh"

namespace isdf {

struct MincoArgs {
    int B, N;                 // problems, pieces per problem (ragged: the most pieces of one problem)
    int P;                    // pieces of the batch (B N when uniform)
    const int *poff;          // may be null: B + 1 piece offsets of a ragged batch; null: problem b owns pieces [b N, b N + N)
    const double *x;          // B x (N + 3(N-1)) decision vectors (ragged: problem b's 4 N_b - 3 start at row 4 poff[b] - 3 b)
    const double *head, *tail;  // 3x3 column-major (columns p, v, a); bc_stride = 0: shared by the batch, 9: one per problem
    int bc_stride;
    double rho;
    double *T;                // P durations (concatenated)
    double *C;                // 18P coefficients: column-major over the 6P rows
    double *Cpp;              // may be null: 18P, the same coefficients as one column-major 6N x 3 block PER PROBLEM (swept-volume kernels)
    const double *sv_out;     // may be null: 19P + B, per problem [cost | gradC 18N | gradT N] of the batched swept-volume term
    double *lu;               // 78P: factored band of every problem (kept for the adjoint solve)
    double *energy;           // B
    double *gC_e, *gT_e;      // energy partials, same layouts as C / T
    const double *disc_out;   // [cost | gradC 18P | gradT P] of the concatenated time-integral evaluation (null: none)
    const double *piece_cost; // P per-piece cost terms of that evaluation
    double *cost;             // B
    double *grad;             // laid out as x
    int seq_terms;            // 1: the piece costs are added to the energy one at a time (the mid-end, isdf_midend.cuh); 0: summed first
    const double *T_in;       // may be null: P durations used as they are (isdf_trajectory_brake); null: T = forwardT(tau) of x
};

__device__ __forceinline__ double &band(double *a, int n, int i, int j) { return a[(size_t)(i - j + 6) * n + j]; }

// row of the monomial basis for derivative order `der` at time t (the reference's rows, no factorial normalisation)
__device__ __forceinline__ void minco_basis(double t, int der, double out[6]) {
#pragma unroll
    for (int k = 0; k < 6; k++) {
        if (k < der) { out[k] = 0.0; continue; }
        double c = 1.0;
        for (int q = 0; q < der; q++) c *= (k - q);
        double p = 1.0;
        for (int q = 0; q < k - der; q++) p *= t;
        out[k] = c * p;
    }
}
__device__ __forceinline__ void minco_put(double *a, int n, int row, int col0, const double r[6], double sgn) {
#pragma unroll
    for (int k = 0; k < 6; k++) if (r[k] != 0.0) band(a, n, row, col0 + k) = sgn * r[k];
}

__global__ void __launch_bounds__(32) k_minco_forward(const __grid_constant__ MincoArgs A) {
    extern __shared__ __align__(16) double sm[];
    const int b = blockIdx.x, lane = threadIdx.x;
    const int p0 = A.poff ? A.poff[b] : b * A.N, N = A.poff ? A.poff[b + 1] - p0 : A.N, n = 6 * N;   // first piece, pieces
    double *a = sm;                    // 13n
    double *rhs = sm + (size_t)13 * n; // 3n, column-major
    double *sT = rhs + (size_t)3 * n;  // N
    const double *x = A.x + (size_t)4 * p0 - 3 * b;
    const double *head = A.head + (size_t)b * A.bc_stride, *tail = A.tail + (size_t)b * A.bc_stride;
    for (int i = lane; i < N; i += 32) {
        double Ti;
        if (A.T_in) Ti = A.T_in[(size_t)p0 + i];
        else {
            const double t = x[i];
            Ti = t > 0.0 ? ((0.5 * t + 1.0) * t + 1.0) : 1.0 / ((0.5 * t - 1.0) * t + 1.0);
        }
        sT[i] = Ti;
        A.T[(size_t)p0 + i] = Ti;
    }
    for (int k = lane; k < 16 * n; k += 32) sm[k] = 0.0;
    __syncwarp();
    // rows: start conditions, per junction {jerk, snap continuity, waypoint, p/v/a continuity}, end conditions
    double r[6];
    if (lane < 3) {
        const int d = lane;
        minco_basis(0.0, d, r); minco_put(a, n, d, 0, r, 1.0);
        for (int ax = 0; ax < 3; ax++) rhs[(size_t)ax * n + d] = head[d * 3 + ax];
        minco_basis(sT[N - 1], d, r); minco_put(a, n, n - 3 + d, n - 6, r, 1.0);
        for (int ax = 0; ax < 3; ax++) rhs[(size_t)ax * n + n - 3 + d] = tail[d * 3 + ax];
    }
    for (int i = lane; i + 1 < N; i += 32) {
        const int c0 = 6 * i, c1 = 6 * (i + 1), r0 = 6 * i + 3;
        const double Ti = sT[i];
        minco_basis(Ti, 3, r); minco_put(a, n, r0, c0, r, 1.0); minco_basis(0.0, 3, r); minco_put(a, n, r0, c1, r, -1.0);
        minco_basis(Ti, 4, r); minco_put(a, n, r0 + 1, c0, r, 1.0); minco_basis(0.0, 4, r); minco_put(a, n, r0 + 1, c1, r, -1.0);
        minco_basis(Ti, 0, r); minco_put(a, n, r0 + 2, c0, r, 1.0);
        for (int ax = 0; ax < 3; ax++) rhs[(size_t)ax * n + r0 + 2] = x[N + 3 * i + ax];
        for (int d = 0; d < 3; d++) {
            minco_basis(Ti, d, r); minco_put(a, n, r0 + 3 + d, c0, r, 1.0);
            minco_basis(0.0, d, r); minco_put(a, n, r0 + 3 + d, c1, r, -1.0);
        }
    }
    __syncwarp();
    // ---- LU without pivoting (minco.hpp:99-135) -----------------------------------------------------------------------
    for (int k = 0; k + 1 < n; k++) {
        const int cnt = min(6, n - 1 - k);           // rows / columns k+1 .. k+cnt
        const double piv = band(a, n, k, k);
        if (lane < cnt) {
            double &m = band(a, n, k + 1 + lane, k);
            if (m != 0.0) m /= piv;
        }
        __syncwarp();
        for (int e = lane; e < cnt * cnt; e += 32) {
            const int i = k + 1 + e / cnt, j = k + 1 + e % cnt;
            const double m = band(a, n, i, k);
            if (m != 0.0) {
                const double u = band(a, n, k, j);
                if (u != 0.0) band(a, n, i, j) -= m * u;
            }
        }
        __syncwarp();
    }
    // ---- solve, three right-hand sides (minco.hpp:137-166) -------------------------------------------------------------
    for (int j = 0; j < n; j++) {
        const int cnt = min(6, n - 1 - j);
        if (lane < 3 * cnt) {
            const int i = j + 1 + lane / 3, c = lane % 3;
            const double m = band(a, n, i, j);
            if (m != 0.0) rhs[(size_t)c * n + i] -= m * rhs[(size_t)c * n + j];
        }
        __syncwarp();
    }
    for (int j = n - 1; j >= 0; j--) {
        if (lane < 3) rhs[(size_t)lane * n + j] /= band(a, n, j, j);
        __syncwarp();
        const int lo = max(0, j - 6), cnt = j - lo;
        if (lane < 3 * cnt) {
            const int i = lo + lane / 3, c = lane % 3;
            const double u = band(a, n, i, j);
            if (u != 0.0) rhs[(size_t)c * n + i] -= u * rhs[(size_t)c * n + j];
        }
        __syncwarp();
    }
    // ---- outputs ------------------------------------------------------------------------------------------------------
    const size_t rows = (size_t)6 * A.P;             // rows of the concatenated block
    for (int k = lane; k < 3 * n; k += 32) {
        const int ax = k / n, row = k - ax * n;
        A.C[(size_t)ax * rows + (size_t)6 * p0 + row] = rhs[k];
        if (A.Cpp) A.Cpp[(size_t)18 * p0 + k] = rhs[k];
    }
    for (int k = lane; k < 13 * n; k += 32) A.lu[(size_t)78 * p0 + k] = a[k];
    // energy partials (minco.hpp:550-582); the energy itself is summed in the reference's (piece, axis) order by lane 0
    double *term = a;                                  // band no longer needed in shared memory: reuse as 3N scratch
    __syncwarp();
    for (int i = lane; i < N; i += 32) {
        const double t1 = sT[i], t2 = t1 * t1, t3 = t2 * t1, t4 = t2 * t2, t5 = t4 * t1;
        double s = 0.0;
        for (int ax = 0; ax < 3; ax++) {
            const double c3 = rhs[(size_t)ax * n + 6 * i + 3], c4 = rhs[(size_t)ax * n + 6 * i + 4], c5 = rhs[(size_t)ax * n + 6 * i + 5];
            term[3 * i + ax] = 36.0 * c3 * c3 * t1 + 144.0 * c4 * c3 * t2 + 192.0 * c4 * c4 * t3 + 240.0 * c5 * c3 * t3 + 720.0 * c5 * c4 * t4 + 720.0 * c5 * c5 * t5;
            double *o = A.gC_e + (size_t)ax * rows + (size_t)6 * p0 + 6 * i;
            o[0] = 0.0; o[1] = 0.0; o[2] = 0.0;
            o[3] = 72.0 * c3 * t1 + 144.0 * c4 * t2 + 240.0 * c5 * t3;
            o[4] = 144.0 * c3 * t2 + 384.0 * c4 * t3 + 720.0 * c5 * t4;
            o[5] = 240.0 * c3 * t3 + 720.0 * c4 * t4 + 1440.0 * c5 * t5;
            s += 36.0 * c3 * c3 + 288.0 * c4 * c3 * t1 + 576.0 * c4 * c4 * t2 + 720.0 * c5 * c3 * t2 + 2880.0 * c5 * c4 * t3 + 3600.0 * c5 * c5 * t4;
        }
        A.gT_e[(size_t)p0 + i] = s;
    }
    __syncwarp();
    if (lane == 0) {
        double e = 0.0;
        for (int k = 0; k < 3 * N; k++) e += term[k];
        A.energy[b] = e;
    }
}

__global__ void __launch_bounds__(32) k_minco_backward(const __grid_constant__ MincoArgs A) {
    extern __shared__ __align__(16) double sm[];
    const int b = blockIdx.x, lane = threadIdx.x;
    const int p0 = A.poff ? A.poff[b] : b * A.N, N = A.poff ? A.poff[b + 1] - p0 : A.N, n = 6 * N;   // first piece, pieces
    double *a = sm;                     // 13n
    double *lam = sm + (size_t)13 * n;  // 3n
    double *gtm = lam + (size_t)3 * n;  // N: gradTimes
    const size_t rows = (size_t)6 * A.P, BN = (size_t)A.P;
    const double *sv = A.sv_out ? A.sv_out + (size_t)19 * p0 + b : nullptr;   // this problem's [cost | gradC 18N | gradT N]
    for (int k = lane; k < 13 * n; k += 32) a[k] = A.lu[(size_t)78 * p0 + k];
    for (int k = lane; k < 3 * n; k += 32) {
        const int ax = k / n, row = k - ax * n;
        const size_t g = (size_t)ax * rows + (size_t)6 * p0 + row;
        double v = A.gC_e[g];                                                   // accumulation order of costFunctionLmbm (hpp:386-405): energy partials,
        if (sv) v += sv[1 + k];                                                 // + swept-volume term,
        lam[k] = v + (A.disc_out ? A.disc_out[1 + g] : 0.0);                    // + time-integral term
    }
    __syncwarp();
    // ---- solveAdj (minco.hpp:168-197) -----------------------------------------------------------------------------------
    for (int j = 0; j < n; j++) {
        if (lane < 3) lam[(size_t)lane * n + j] /= band(a, n, j, j);
        __syncwarp();
        const int cnt = min(6, n - 1 - j);
        if (lane < 3 * cnt) {
            const int i = j + 1 + lane / 3, c = lane % 3;
            const double u = band(a, n, j, i);
            if (u != 0.0) lam[(size_t)c * n + i] -= u * lam[(size_t)c * n + j];
        }
        __syncwarp();
    }
    for (int j = n - 1; j >= 0; j--) {
        const int lo = max(0, j - 6), cnt = j - lo;
        if (lane < 3 * cnt) {
            const int i = lo + lane / 3, c = lane % 3;
            const double m = band(a, n, j, i);
            if (m != 0.0) lam[(size_t)c * n + i] -= m * lam[(size_t)c * n + j];
        }
        __syncwarp();
    }
    // ---- propogateGrad (minco.hpp:584-654) + rho + backwardGradT/P (hpp:283-330) -----------------------------------------
    double *g = A.grad + (size_t)4 * p0 - 3 * b;
    const double *x = A.x + (size_t)4 * p0 - 3 * b;
    for (int k = lane; k < 3 * (N - 1); k += 32) {
        const int i = k / 3, ax = k - 3 * i;
        g[N + k] = lam[(size_t)ax * n + 6 * i + 5];
    }
    for (int i = lane; i < N; i += 32) {
        const double Ti = A.T[(size_t)p0 + i];
        double s = 0.0;
        double r[6];
        for (int ax = 0; ax < 3; ax++) {
            double dval[6];
            const double *c = A.C + (size_t)ax * rows + (size_t)6 * p0 + 6 * i;
            for (int d = 1; d <= 5; d++) {
                minco_basis(Ti, d, r);
                double v = 0.0;
#pragma unroll
                for (int k = 0; k < 6; k++) v += r[k] * c[k];
                dval[d] = v;
            }
            const double *L = lam + (size_t)ax * n;
            if (i + 1 < N) {
                const int r0 = 6 * i + 3;
                s -= dval[4] * L[r0] + dval[5] * L[r0 + 1] + dval[1] * L[r0 + 2] + dval[1] * L[r0 + 3] + dval[2] * L[r0 + 4] + dval[3] * L[r0 + 5];
            } else {
                s -= dval[1] * L[n - 3] + dval[2] * L[n - 2] + dval[3] * L[n - 1];
            }
        }
        double gT = A.gT_e[(size_t)p0 + i];
        if (sv) gT += sv[1 + 18 * N + i];
        gT += (A.disc_out ? A.disc_out[1 + 18 * BN + (size_t)p0 + i] : 0.0);
        double gt = s + gT;
        gt += A.rho;
        gtm[i] = gt;
        const double tau = x[i];
        if (tau > 0) g[i] = gt * (tau + 1.0);
        else { const double den = (0.5 * tau - 1.0) * tau + 1.0; g[i] = gt * (1.0 - tau) / (den * den); }
    }
    if (lane == 0) {
        double cost = A.energy[b];
        if (sv) cost += sv[0];
        if (A.piece_cost && A.seq_terms) {
            for (int i = 0; i < N; i++) cost += A.piece_cost[(size_t)p0 + i];
        } else if (A.piece_cost) {
            double c = 0.0;
            for (int i = 0; i < N; i++) c += A.piece_cost[(size_t)p0 + i];
            cost += c;
        }
        double tsum = 0.0;
        for (int i = 0; i < N; i++) tsum += A.T[(size_t)p0 + i];
        cost += A.rho * tsum;
        A.cost[b] = cost;
    }
}

inline size_t minco_smem_bytes(int N) { return sizeof(double) * ((size_t)16 * 6 * N + N); }

}  // namespace isdf
