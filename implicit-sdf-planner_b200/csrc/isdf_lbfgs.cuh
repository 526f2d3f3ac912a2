// Device-resident lock-step L-BFGS: B independent instances of the reference's patched LBFGS-Lite fork (utils/include/utils/lbfgs.hpp:
// Lewis–Overton bracketing that returns on Armijo :290-430; cautious update + two-loop recursion :742-786; the fork's direction reset
// at the price of one more evaluation :788-811; stop tests :656-690) advanced together on the GPU. Every round = ONE batched callback
// (isdf_callback_batch_device: MINCO -> time-integral / collision term -> adjoint for all B problems) + ONE launch of k_lbfgs_feed,
// in which every instance consumes its (f, grad) and names the point it wants evaluated next. Iterates, histories and all bookkeeping
// stay in HBM; the host reads one integer per round (instances still running).
//
// k_lbfgs_feed is host/isdf_lbfgs.hpp's LbfgsInstance::feed transcribed statement for statement — one THREAD per instance, every dot
// product a left-to-right sum, compiled without FMA contraction (this header lives in the -fmad=false translation unit) — so an
// instance's iterates, iteration / evaluation counts and return code are bit-identical to the sequential host driver's
// (tests/test_gpu_lbfgs_device.py). The O(m n) arithmetic per round (n = 253, m = 16: ~10^4 flops per instance) is noise next to the
// callback (~0.3 ms of GPU time per instance), which is why one thread per instance is enough.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace isdf {

enum { LB_WANT_INIT = 0, LB_WANT_LS = 1, LB_WANT_RESET = 2, LB_DONE = 3 };
enum {   // lbfgs.hpp:148-197
    LB_CONVERGENCE = 0, LB_STOP = 1, LB_CANCELED = 2,
    LBERR_UNKNOWNERROR = -1024, LBERR_INVALID_N, LBERR_INVALID_MEMSIZE, LBERR_INVALID_GEPSILON, LBERR_INVALID_TESTPERIOD,
    LBERR_INVALID_DELTA, LBERR_INVALID_MINSTEP, LBERR_INVALID_MAXSTEP, LBERR_INVALID_FDECCOEFF, LBERR_INVALID_SCURVCOEFF,
    LBERR_INVALID_MACHINEPREC, LBERR_INVALID_MAXLINESEARCH, LBERR_INVALID_FUNCVAL, LBERR_MINIMUMSTEP, LBERR_MAXIMUMSTEP,
    LBERR_MAXIMUMLINESEARCH, LBERR_MAXIMUMITERATION, LBERR_WIDTHTOOSMALL, LBERR_INVALIDPARAMETERS, LBERR_INCREASEGRADIENT
};

struct LbfgsDevParams {
    int mem_size, past, max_iterations, max_linesearch;
    double g_epsilon, delta, min_step, max_step, f_dec_coeff, cautious_factor, machine_prec;
    int cancel_after;   // > 0: LB_CANCELED once k > cancel_after (the mid-end's progress callback earlyExit, mid_end.hpp:613-631); 0: never
};

constexpr int LB_NSCALAR = 8;   // fx, step, olddnorm, finit, dgtest, mu, nu, -
constexpr int LB_NINT = 12;     // phase, ret, k, end, bound, count, brackt, touched, iterations, evaluations, -, -

struct LbfgsArgs {
    int B, n;
    LbfgsDevParams pr;
    double *x;          // B x n: the point every instance wants evaluated next (in: starting points; out: solutions)
    const double *f;    // B: callback values at x
    const double *grad; // B x n
    double *xp, *g, *gp, *d;   // B x n each
    double *pf;         // B x max(1, past)
    double *alpha, *ys; // B x m each
    double *S, *Y;      // B x m x n each
    double *sc;         // B x LB_NSCALAR
    int *st;            // B x LB_NINT
    int *active;        // [0]: instances not DONE after this launch (zeroed by the host before each launch)
};

__device__ __forceinline__ double lb_dot(const double *a, const double *b, int n) { double s = 0; for (int i = 0; i < n; i++) s += a[i] * b[i]; return s; }
__device__ __forceinline__ double lb_norm_inf(const double *a, int n) { double m = 0; for (int i = 0; i < n; i++) m = fmax(m, fabs(a[i])); return m; }

__global__ void __launch_bounds__(64) k_lbfgs_feed(const LbfgsArgs A) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= A.B) return;
    const int n = A.n, m = A.pr.mem_size, past = A.pr.past;
    const LbfgsDevParams &pr = A.pr;
    int *st = A.st + (size_t)b * LB_NINT;
    int phase = st[0];
    if (phase == LB_DONE) return;
    double *sc = A.sc + (size_t)b * LB_NSCALAR;
    double *x = A.x + (size_t)b * n, *xp = A.xp + (size_t)b * n, *g = A.g + (size_t)b * n, *gp = A.gp + (size_t)b * n, *d = A.d + (size_t)b * n;
    double *pf = A.pf + (size_t)b * (past > 1 ? past : 1), *alpha = A.alpha + (size_t)b * m, *ys_hist = A.ys + (size_t)b * m;
    double *S = A.S + (size_t)b * m * n, *Y = A.Y + (size_t)b * m * n;
    const double *grad = A.grad + (size_t)b * n;
    const double f = A.f[b];
    double fx = sc[0], step = sc[1], olddnorm = sc[2], finit = sc[3], dgtest = sc[4], mu = sc[5], nu = sc[6];
    int ret = st[1], k = st[2], end = st[3], bound = st[4], count = st[5], brackt = st[6], touched = st[7], iterations = st[8], evaluations = st[9];

    // the continuation labels of LbfgsInstance: 0 nothing more, 1 begin_iteration, 2 after_line_search, 3 finish_direction
    int next = 0;
    auto finish = [&](int r) { ret = r; phase = LB_DONE; next = 0; };
    auto fail_line_search = [&](int r) { for (int i = 0; i < n; i++) { x[i] = xp[i]; g[i] = gp[i]; } finish(r); };

    if (phase == LB_WANT_INIT) {
        fx = f;
        for (int i = 0; i < n; i++) g[i] = grad[i];
        ++evaluations;
        pf[0] = fx;
        for (int i = 0; i < n; i++) d[i] = -g[i];
        if (lb_norm_inf(g, n) / fmax(1.0, lb_norm_inf(x, n)) < pr.g_epsilon) finish(LB_CONVERGENCE);
        else { step = 1.0 / sqrt(lb_dot(d, d, n)); k = 1; end = 0; bound = 0; next = 1; }
    } else if (phase == LB_WANT_LS) {
        fx = f;
        for (int i = 0; i < n; i++) g[i] = grad[i];
        ++count; ++evaluations;
        if (isinf(fx) || isnan(fx)) fail_line_search(LBERR_INVALID_FUNCVAL);
        else {
            bool armijo = false;
            if (fx > finit + step * dgtest) { nu = step; brackt = 1; }   // with_tole_ls / cast_x_range are off in this driver (as in the reference's configs)
            else armijo = true;
            if (armijo) next = 2;
            else if (pr.max_linesearch <= count) fail_line_search(LBERR_MAXIMUMLINESEARCH);
            else if (brackt && (nu - mu) < pr.machine_prec * nu) fail_line_search(LBERR_WIDTHTOOSMALL);
            else {
                if (brackt) step = 0.5 * (mu + nu); else step *= 2.0;
                if (step < pr.min_step) fail_line_search(LBERR_MINIMUMSTEP);
                else {
                    bool failed = false;
                    if (step > pr.max_step) { if (touched) { fail_line_search(LBERR_MAXIMUMSTEP); failed = true; } else { touched = 1; step = pr.max_step; } }
                    if (!failed) for (int i = 0; i < n; i++) x[i] = xp[i] + step * d[i];
                }
            }
        }
    } else {   // LB_WANT_RESET: the fork keeps fx and takes the fresh gradient (lbfgs.hpp:802-809)
        ++evaluations;
        for (int i = 0; i < n; i++) g[i] = grad[i];
        const double gn = sqrt(lb_dot(g, g, n));
        for (int q = 0; q < n; q++) d[q] = (gn > 0 ? -g[q] / gn : -g[q]) * olddnorm;
        next = 3;
    }

    if (next == 2) {   // after_line_search
        next = 0;
        iterations = k;
        bool stop = false;
        if (pr.cancel_after > 0 && k > pr.cancel_after) { finish(LB_CANCELED); stop = true; }   // where lbfgs.hpp:644-652 asks proc_progress
        if (!stop && lb_norm_inf(g, n) / fmax(1.0, lb_norm_inf(x, n)) < pr.g_epsilon) { finish(LB_CONVERGENCE); stop = true; }
        if (!stop && 0 < past) {
            if (past <= k) {
                const double rate = fabs(pf[k % past] - fx) / fmax(1.0, fabs(fx));
                if (rate < pr.delta) { finish(LB_STOP); stop = true; }
            }
            if (!stop) pf[k % past] = fx;
        }
        if (!stop && pr.max_iterations != 0 && pr.max_iterations <= k) { finish(LBERR_MAXIMUMITERATION); stop = true; }
        if (!stop) {
            ++k;
            double *s_end = S + (size_t)end * n, *y_end = Y + (size_t)end * n;
            for (int i = 0; i < n; i++) { s_end[i] = x[i] - xp[i]; y_end[i] = g[i] - gp[i]; }
            const double ys = lb_dot(y_end, s_end, n), yy = lb_dot(y_end, y_end, n);
            ys_hist[end] = ys;
            for (int i = 0; i < n; i++) d[i] = -g[i];
            const double cau = lb_dot(s_end, s_end, n) * sqrt(lb_dot(gp, gp, n)) * pr.cautious_factor;
            bool reset_direction = false;
            if (ys > cau) {
                ++bound; bound = m < bound ? m : bound;
                end = (end + 1) % m;
                int j = end;
                for (int i = 0; i < bound; ++i) {
                    j = (j + m - 1) % m;
                    alpha[j] = lb_dot(S + (size_t)j * n, d, n) / ys_hist[j];
                    const double *yj = Y + (size_t)j * n;
                    for (int q = 0; q < n; q++) d[q] += (-alpha[j]) * yj[q];
                }
                const double scal = ys / yy;
                for (int q = 0; q < n; q++) d[q] *= scal;
                for (int i = 0; i < bound; ++i) {
                    const double beta = lb_dot(Y + (size_t)j * n, d, n) / ys_hist[j];
                    const double *sj = S + (size_t)j * n;
                    for (int q = 0; q < n; q++) d[q] += (alpha[j] - beta) * sj[q];
                    j = (j + 1) % m;
                }
                if (sqrt(lb_dot(d, d, n)) >= 0.04 || lb_dot(d, g, n) >= 0) reset_direction = true;   // lbfgs.hpp:788
            } else {
                reset_direction = true;                                                            // lbfgs.hpp:797
                end = (end + 1) % m;
            }
            if (reset_direction) phase = LB_WANT_RESET;   // re-evaluate at the current x
            else next = 3;
        }
    }
    if (next == 3) {   // finish_direction
        next = 0;
        const double dn = sqrt(lb_dot(d, d, n));
        if (isinf(dn) || isnan(dn)) finish(LBERR_INVALID_FUNCVAL);
        else { olddnorm = dn; step = 1.0; next = 1; }
    }
    if (next == 1) {   // begin_iteration
        for (int i = 0; i < n; i++) { xp[i] = x[i]; gp[i] = g[i]; }
        if (!(step > 0.0)) fail_line_search(LBERR_INVALIDPARAMETERS);
        else {
            const double dginit = lb_dot(gp, d, n);
            if (0.0 < dginit) fail_line_search(LBERR_INCREASEGRADIENT);
            else {
                finit = fx; dgtest = pr.f_dec_coeff * dginit;
                count = 0; brackt = 0; touched = 0; mu = 0.0; nu = pr.max_step;
                for (int i = 0; i < n; i++) x[i] = xp[i] + step * d[i];
                phase = LB_WANT_LS;
            }
        }
    }
    sc[0] = fx; sc[1] = step; sc[2] = olddnorm; sc[3] = finit; sc[4] = dgtest; sc[5] = mu; sc[6] = nu;
    st[0] = phase; st[1] = ret; st[2] = k; st[3] = end; st[4] = bound; st[5] = count; st[6] = brackt; st[7] = touched; st[8] = iterations; st[9] = evaluations;
    if (phase != LB_DONE) atomicAdd(A.active, 1);
}

}  // namespace isdf
