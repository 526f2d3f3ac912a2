// Re-entrant L-BFGS driver with the semantics of the reference's patched LBFGS-Lite fork (utils/include/utils/lbfgs.hpp):
//   * Lewis–Overton bracketing line search that returns as soon as the ARMIJO condition holds — the fork comments the
//     weak-Wolfe branch out (lbfgs.hpp:352-388); optional tolerance term `with_tole_ls` and x(0) range casting (:133-142, :360-365);
//   * cautious update (Li & Fukushima) and two-loop recursion (lbfgs.hpp:742-786);
//   * the fork's direction patch: if ||d|| >= 0.04 or d.g >= 0 — or the cautious test fails — the direction is replaced by
//     steepest descent rescaled to the previous direction norm, at the price of one more callback evaluation (:788-811);
//   * first step 1/||d||, then 1 (:595, :821); stop tests: gradient (g_epsilon) and past/delta (:656-690); same return codes.
// Differences by design: plain pointers instead of Eigen (an Eigen overload is provided under ISDF_WITH_EIGEN), no globals
// (any number of instances can run concurrently — the reference's LMBM shim keeps its callback in file statics,
// lmbm.cpp:4-6), no console output. Callback evaluations are counted: they are the unit a faithful "iterations/s" needs.
#pragma once
#include <cmath>
#include <vector>
#include <algorithm>
#ifdef ISDF_WITH_EIGEN
#include <Eigen/Core>
#endif

namespace isdf_host {

struct LbfgsParams {   // lbfgs_parameter_t (lbfgs.hpp:40-142)
    int mem_size = 8;
    double g_epsilon = 1.0e-5;
    int past = 3;
    double delta = 1.0e-6;
    int max_iterations = 0;
    int max_linesearch = 64;
    double min_step = 1.0e-20;
    double max_step = 1.0e+20;
    double f_dec_coeff = 1.0e-4;
    double s_curv_coeff = 0.9;
    double cautious_factor = 1.0e-6;
    double machine_prec = 1.0e-16;
    bool with_tole_ls = false;
    bool cast_x_range = false;
    double x_min = 0.0, x_max = 0.0;
    int cancel_after = 0;   // lock-step driver only: LBFGS_CANCELED once k > cancel_after, where the sequential driver asks `progress`; 0 = never
};

enum {   // lbfgs.hpp:148-197
    LBFGS_CONVERGENCE = 0, LBFGS_STOP, LBFGS_CANCELED,
    LBFGSERR_UNKNOWNERROR = -1024, LBFGSERR_INVALID_N, LBFGSERR_INVALID_MEMSIZE, LBFGSERR_INVALID_GEPSILON, LBFGSERR_INVALID_TESTPERIOD,
    LBFGSERR_INVALID_DELTA, LBFGSERR_INVALID_MINSTEP, LBFGSERR_INVALID_MAXSTEP, LBFGSERR_INVALID_FDECCOEFF, LBFGSERR_INVALID_SCURVCOEFF,
    LBFGSERR_INVALID_MACHINEPREC, LBFGSERR_INVALID_MAXLINESEARCH, LBFGSERR_INVALID_FUNCVAL, LBFGSERR_MINIMUMSTEP, LBFGSERR_MAXIMUMSTEP,
    LBFGSERR_MAXIMUMLINESEARCH, LBFGSERR_MAXIMUMITERATION, LBFGSERR_WIDTHTOOSMALL, LBFGSERR_INVALIDPARAMETERS, LBFGSERR_INCREASEGRADIENT
};

// raw twins of lbfgs_evaluate_t / lbfgs_stepbound_t / lbfgs_progress_t (lbfgs.hpp:213-262)
typedef double (*lbfgs_eval_raw_t)(void *instance, const double *x, double *g, int n, double *p_cost);
typedef double (*lbfgs_stepbound_raw_t)(void *instance, const double *xp, const double *d, int n);
typedef int (*lbfgs_progress_raw_t)(void *instance, const double *x, const double *g, double fx, double step, int k, int ls, int n);

struct LbfgsStats { int iterations = 0; int evaluations = 0; };

namespace detail {
inline double dotn(const double *a, const double *b, int n) { double s = 0; for (int i = 0; i < n; i++) s += a[i] * b[i]; return s; }
inline double norm_inf(const double *a, int n) { double m = 0; for (int i = 0; i < n; i++) m = std::max(m, std::fabs(a[i])); return m; }

// line_search_lewisoverton (lbfgs.hpp:290-430)
inline int line_search(int n, double *x, double &f, double &fpos, double *g, double &stp, const double *s, const double *xp, const double *gp,
                       double stpmin, double stpmax, lbfgs_eval_raw_t eval, void *instance, const LbfgsParams &pr, LbfgsStats &st) {
    if (!(stp > 0.0)) return LBFGSERR_INVALIDPARAMETERS;
    const double dginit = dotn(gp, s, n);
    if (0.0 < dginit) return LBFGSERR_INCREASEGRADIENT;
    const double finit = f, dgtest = pr.f_dec_coeff * dginit;
    const int tol_sw = pr.with_tole_ls ? 1 : 0;
    int count = 0;
    bool brackt = false, touched = false;
    double mu = 0.0, nu = stpmax;
    for (;;) {
        for (int i = 0; i < n; i++) x[i] = xp[i] + stp * s[i];
        double f_cost = 0;
        f = eval(instance, x, g, n, &f_cost);
        (void)fpos;
        ++count; ++st.evaluations;
        const double stp_conv1 = (1.0 - stp) > 0.0 ? (0.05 * (1.0 - stp)) : 0.0;
        if (std::isinf(f) || std::isnan(f)) return LBFGSERR_INVALID_FUNCVAL;
        if (pr.cast_x_range && (x[0] > pr.x_max || x[0] < pr.x_min)) { nu = stp; brackt = true; }
        else if (f > finit + stp * dgtest + tol_sw * (stp_conv1 * finit)) { nu = stp; brackt = true; }
        else return count;   // Armijo holds: the fork returns here
        if (pr.max_linesearch <= count) return LBFGSERR_MAXIMUMLINESEARCH;
        if (brackt && (nu - mu) < pr.machine_prec * nu) return LBFGSERR_WIDTHTOOSMALL;
        if (brackt) stp = 0.5 * (mu + nu); else stp *= 2.0;
        if (stp < stpmin) return LBFGSERR_MINIMUMSTEP;
        if (stp > stpmax) { if (touched) return LBFGSERR_MAXIMUMSTEP; touched = true; stp = stpmax; }
    }
}
}  // namespace detail

// lbfgs_optimize (lbfgs.hpp:480-830)
inline int lbfgs_optimize(int n, double *x, double &f, lbfgs_eval_raw_t eval, lbfgs_stepbound_raw_t stepbound, lbfgs_progress_raw_t progress,
                          void *instance, const LbfgsParams &pr, LbfgsStats *stats_out = nullptr) {
    using namespace detail;
    const int m = pr.mem_size;
    if (n <= 0) return LBFGSERR_INVALID_N;
    if (m <= 0) return LBFGSERR_INVALID_MEMSIZE;
    if (pr.g_epsilon < 0.0) return LBFGSERR_INVALID_GEPSILON;
    if (pr.past < 0) return LBFGSERR_INVALID_TESTPERIOD;
    if (pr.delta < 0.0) return LBFGSERR_INVALID_DELTA;
    if (pr.min_step < 0.0) return LBFGSERR_INVALID_MINSTEP;
    if (pr.max_step < pr.min_step) return LBFGSERR_INVALID_MAXSTEP;
    if (!(pr.f_dec_coeff > 0.0 && pr.f_dec_coeff < 1.0)) return LBFGSERR_INVALID_FDECCOEFF;
    if (!(pr.s_curv_coeff < 1.0 && pr.s_curv_coeff > pr.f_dec_coeff)) return LBFGSERR_INVALID_SCURVCOEFF;
    if (!(pr.machine_prec > 0.0)) return LBFGSERR_INVALID_MACHINEPREC;
    if (pr.max_linesearch <= 0) return LBFGSERR_INVALID_MAXLINESEARCH;

    LbfgsStats st;
    std::vector<double> xp(n), g(n), grec(n), gp(n), d(n), pf(std::max(1, pr.past));
    std::vector<double> alpha(m, 0.0), ys_hist(m, 0.0), S((size_t)n * m, 0.0), Y((size_t)n * m, 0.0);
    double olddnorm = 1.0, p_cost = 0, p_cost_new = 0;
    double fx = eval(instance, x, g.data(), n, &p_cost);
    ++st.evaluations;
    pf[0] = fx;
    for (int i = 0; i < n; i++) d[i] = -g[i];
    int ret;
    if (norm_inf(g.data(), n) / std::max(1.0, norm_inf(x, n)) < pr.g_epsilon) {
        ret = LBFGS_CONVERGENCE;
    } else {
        double step = 1.0 / std::sqrt(dotn(d.data(), d.data(), n));
        int k = 1, end = 0, bound = 0;
        for (;;) {
            xp.assign(x, x + n);
            gp = g;
            double step_min = pr.min_step, step_max = pr.max_step;
            if (stepbound) {
                step_max = stepbound(instance, xp.data(), d.data(), n);
                step_max = step_max < pr.max_step ? step_max : pr.max_step;
                step = step < step_max ? step : 0.5 * step_max;
            }
            const int ls = line_search(n, x, fx, p_cost, g.data(), step, d.data(), xp.data(), gp.data(), step_min, step_max, eval, instance, pr, st);
            if (ls < 0) { std::copy(xp.begin(), xp.end(), x); g = gp; ret = ls; break; }
            st.iterations = k;
            if (progress && progress(instance, x, g.data(), fx, step, k, ls, n)) { ret = LBFGS_CANCELED; break; }
            if (norm_inf(g.data(), n) / std::max(1.0, norm_inf(x, n)) < pr.g_epsilon) { ret = LBFGS_CONVERGENCE; break; }
            if (0 < pr.past) {
                if (pr.past <= k) {
                    const double rate = std::fabs(pf[k % pr.past] - fx) / std::max(1.0, std::fabs(fx));
                    if (rate < pr.delta) { ret = LBFGS_STOP; break; }
                }
                pf[k % pr.past] = fx;
            }
            if (pr.max_iterations != 0 && pr.max_iterations <= k) { ret = LBFGSERR_MAXIMUMITERATION; break; }
            ++k;
            double *s_end = &S[(size_t)end * n], *y_end = &Y[(size_t)end * n];
            for (int i = 0; i < n; i++) { s_end[i] = x[i] - xp[i]; y_end[i] = g[i] - gp[i]; }
            const double ys = dotn(y_end, s_end, n), yy = dotn(y_end, y_end, n);
            ys_hist[end] = ys;
            for (int i = 0; i < n; i++) d[i] = -g[i];
            const double cau = dotn(s_end, s_end, n) * std::sqrt(dotn(gp.data(), gp.data(), n)) * pr.cautious_factor;
            bool reset_direction = false;
            if (ys > cau) {
                ++bound; bound = m < bound ? m : bound;
                end = (end + 1) % m;
                int j = end;
                for (int i = 0; i < bound; ++i) {
                    j = (j + m - 1) % m;
                    alpha[j] = dotn(&S[(size_t)j * n], d.data(), n) / ys_hist[j];
                    const double *yj = &Y[(size_t)j * n];
                    for (int q = 0; q < n; q++) d[q] += (-alpha[j]) * yj[q];
                }
                const double sc = ys / yy;
                for (int q = 0; q < n; q++) d[q] *= sc;
                for (int i = 0; i < bound; ++i) {
                    const double beta = dotn(&Y[(size_t)j * n], d.data(), n) / ys_hist[j];
                    const double *sj = &S[(size_t)j * n];
                    for (int q = 0; q < n; q++) d[q] += (alpha[j] - beta) * sj[q];
                    j = (j + 1) % m;
                }
                if (std::sqrt(dotn(d.data(), d.data(), n)) >= 0.04 || dotn(d.data(), g.data(), n) >= 0) reset_direction = true;   // lbfgs.hpp:788
            } else {
                reset_direction = true;                                                                                        // lbfgs.hpp:797
                end = (end + 1) % m;
            }
            if (reset_direction) {
                (void)eval(instance, x, grec.data(), n, &p_cost_new);
                ++st.evaluations;
                g = grec;
                const double gn = std::sqrt(dotn(grec.data(), grec.data(), n));
                for (int q = 0; q < n; q++) d[q] = (gn > 0 ? -grec[q] / gn : -grec[q]) * olddnorm;
            }
            const double dn = std::sqrt(dotn(d.data(), d.data(), n));
            if (std::isinf(dn) || std::isnan(dn)) { if (stats_out) *stats_out = st; return LBFGSERR_INVALID_FUNCVAL; }
            olddnorm = dn;
            step = 1.0;
        }
    }
    f = fx;
    if (stats_out) *stats_out = st;
    return ret;
}

// ---- lock-step batched driver ---------------------------------------------------------------------------------------------------
// B independent instances of the SAME algorithm as lbfgs_optimize above, advanced together: every round each unfinished instance
// names the point it needs evaluated next (a line-search trial or the direction-reset re-evaluation), ONE batched callback
// evaluates them all (isdf_callback_batch: MINCO + collision term + adjoint for all problems in three launches), and each instance
// consumes its result. An instance performs exactly the arithmetic of the sequential driver — it is the same code unrolled into a
// state machine — so its iterates, iteration and evaluation counts and return code are identical to running it alone
// (tests/test_host_adapters_cpu.py). No step bound / progress callback in this variant; its one progress rule is pr.cancel_after (the
// mid-end's earlyExit, mid_end.hpp:613-631), tested where the sequential driver calls `progress`.
typedef void (*lbfgs_eval_batch_t)(void *instance, int nb, const int *ids, const double *x /* nb x n */, double *f /* nb */, double *g /* nb x n */);

class LbfgsInstance {
public:
    enum Phase { WANT_INIT, WANT_LS, WANT_RESET, DONE };
    Phase phase = WANT_INIT;
    int ret = 0;
    LbfgsStats st;
    double fx = 0.0;

    void start(int n_, const double *x0, const LbfgsParams &pr_) {
        n = n_; pr = pr_; m = pr.mem_size;
        x.assign(x0, x0 + n); xp.assign(n, 0.0); g.assign(n, 0.0); gp.assign(n, 0.0); d.assign(n, 0.0);
        pf.assign(std::max(1, pr.past), 0.0);
        alpha.assign(m, 0.0); ys_hist.assign(m, 0.0); S.assign((size_t)n * m, 0.0); Y.assign((size_t)n * m, 0.0);
        phase = WANT_INIT; st = LbfgsStats(); olddnorm = 1.0;
    }
    const double *request() const { return x.data(); }      // the point to evaluate next (phase != DONE)
    const double *solution() const { return x.data(); }

    // consume f(request()), grad f(request())
    void feed(double f, const double *grad) {
        using namespace detail;
        if (phase == WANT_INIT) {
            fx = f; std::copy(grad, grad + n, g.begin()); ++st.evaluations;
            pf[0] = fx;
            for (int i = 0; i < n; i++) d[i] = -g[i];
            if (norm_inf(g.data(), n) / std::max(1.0, norm_inf(x.data(), n)) < pr.g_epsilon) { finish(LBFGS_CONVERGENCE); return; }
            step = 1.0 / std::sqrt(dotn(d.data(), d.data(), n));
            k = 1; end = 0; bound = 0;
            begin_iteration();
        } else if (phase == WANT_LS) {
            fx = f; std::copy(grad, grad + n, g.begin());
            ++count; ++st.evaluations;
            const double stp_conv1 = (1.0 - step) > 0.0 ? (0.05 * (1.0 - step)) : 0.0;
            const int tol_sw = pr.with_tole_ls ? 1 : 0;
            if (std::isinf(fx) || std::isnan(fx)) { fail_line_search(LBFGSERR_INVALID_FUNCVAL); return; }
            if (pr.cast_x_range && (x[0] > pr.x_max || x[0] < pr.x_min)) { nu = step; brackt = true; }
            else if (fx > finit + step * dgtest + tol_sw * (stp_conv1 * finit)) { nu = step; brackt = true; }
            else { after_line_search(count); return; }               // Armijo holds
            if (pr.max_linesearch <= count) { fail_line_search(LBFGSERR_MAXIMUMLINESEARCH); return; }
            if (brackt && (nu - mu) < pr.machine_prec * nu) { fail_line_search(LBFGSERR_WIDTHTOOSMALL); return; }
            if (brackt) step = 0.5 * (mu + nu); else step *= 2.0;
            if (step < pr.min_step) { fail_line_search(LBFGSERR_MINIMUMSTEP); return; }
            if (step > pr.max_step) { if (touched) { fail_line_search(LBFGSERR_MAXIMUMSTEP); return; } touched = true; step = pr.max_step; }
            for (int i = 0; i < n; i++) x[i] = xp[i] + step * d[i];
        } else if (phase == WANT_RESET) {
            ++st.evaluations;
            std::copy(grad, grad + n, g.begin());                      // the fork keeps fx and takes the fresh gradient (lbfgs.hpp:802-809)
            const double gn = std::sqrt(dotn(g.data(), g.data(), n));
            for (int q = 0; q < n; q++) d[q] = (gn > 0 ? -g[q] / gn : -g[q]) * olddnorm;
            finish_direction();
        }
    }

private:
    int n = 0, m = 0, k = 1, end = 0, bound = 0, count = 0;
    LbfgsParams pr;
    std::vector<double> x, xp, g, gp, d, pf, alpha, ys_hist, S, Y;
    double step = 0.0, olddnorm = 1.0, finit = 0.0, dgtest = 0.0, mu = 0.0, nu = 0.0;
    bool brackt = false, touched = false;

    void finish(int r) { ret = r; phase = DONE; }
    void fail_line_search(int r) { x = xp; g = gp; finish(r); }
    void begin_iteration() {
        using namespace detail;
        xp = x; gp = g;
        if (!(step > 0.0)) { fail_line_search(LBFGSERR_INVALIDPARAMETERS); return; }
        const double dginit = dotn(gp.data(), d.data(), n);
        if (0.0 < dginit) { fail_line_search(LBFGSERR_INCREASEGRADIENT); return; }
        finit = fx; dgtest = pr.f_dec_coeff * dginit;
        count = 0; brackt = false; touched = false; mu = 0.0; nu = pr.max_step;
        for (int i = 0; i < n; i++) x[i] = xp[i] + step * d[i];
        phase = WANT_LS;
    }
    void after_line_search(int ls) {
        using namespace detail;
        (void)ls;
        st.iterations = k;
        if (pr.cancel_after > 0 && k > pr.cancel_after) { finish(LBFGS_CANCELED); return; }
        if (norm_inf(g.data(), n) / std::max(1.0, norm_inf(x.data(), n)) < pr.g_epsilon) { finish(LBFGS_CONVERGENCE); return; }
        if (0 < pr.past) {
            if (pr.past <= k) {
                const double rate = std::fabs(pf[k % pr.past] - fx) / std::max(1.0, std::fabs(fx));
                if (rate < pr.delta) { finish(LBFGS_STOP); return; }
            }
            pf[k % pr.past] = fx;
        }
        if (pr.max_iterations != 0 && pr.max_iterations <= k) { finish(LBFGSERR_MAXIMUMITERATION); return; }
        ++k;
        double *s_end = &S[(size_t)end * n], *y_end = &Y[(size_t)end * n];
        for (int i = 0; i < n; i++) { s_end[i] = x[i] - xp[i]; y_end[i] = g[i] - gp[i]; }
        const double ys = dotn(y_end, s_end, n), yy = dotn(y_end, y_end, n);
        ys_hist[end] = ys;
        for (int i = 0; i < n; i++) d[i] = -g[i];
        const double cau = dotn(s_end, s_end, n) * std::sqrt(dotn(gp.data(), gp.data(), n)) * pr.cautious_factor;
        bool reset_direction = false;
        if (ys > cau) {
            ++bound; bound = m < bound ? m : bound;
            end = (end + 1) % m;
            int j = end;
            for (int i = 0; i < bound; ++i) {
                j = (j + m - 1) % m;
                alpha[j] = dotn(&S[(size_t)j * n], d.data(), n) / ys_hist[j];
                const double *yj = &Y[(size_t)j * n];
                for (int q = 0; q < n; q++) d[q] += (-alpha[j]) * yj[q];
            }
            const double sc = ys / yy;
            for (int q = 0; q < n; q++) d[q] *= sc;
            for (int i = 0; i < bound; ++i) {
                const double beta = dotn(&Y[(size_t)j * n], d.data(), n) / ys_hist[j];
                const double *sj = &S[(size_t)j * n];
                for (int q = 0; q < n; q++) d[q] += (alpha[j] - beta) * sj[q];
                j = (j + 1) % m;
            }
            if (std::sqrt(dotn(d.data(), d.data(), n)) >= 0.04 || dotn(d.data(), g.data(), n) >= 0) reset_direction = true;
        } else {
            reset_direction = true;
            end = (end + 1) % m;
        }
        if (reset_direction) { phase = WANT_RESET; return; }           // re-evaluate at the current x (request() == x)
        finish_direction();
    }
    void finish_direction() {
        using namespace detail;
        const double dn = std::sqrt(dotn(d.data(), d.data(), n));
        if (std::isinf(dn) || std::isnan(dn)) { finish(LBFGSERR_INVALID_FUNCVAL); return; }
        olddnorm = dn;
        step = 1.0;
        begin_iteration();
    }
};

// x: B x n (in: starting points, out: solutions), f: B, ret: B return codes, stats: B (may be null). Returns the number of rounds.
inline int lbfgs_optimize_batch(int B, int n, double *x, double *f, int *ret, lbfgs_eval_batch_t eval, void *instance, const LbfgsParams &pr,
                                LbfgsStats *stats = nullptr) {
    std::vector<LbfgsInstance> inst(B);
    for (int b = 0; b < B; b++) inst[b].start(n, x + (size_t)b * n, pr);
    std::vector<int> ids;
    std::vector<double> xb, fb, gb;
    int rounds = 0;
    for (;;) {
        ids.clear();
        for (int b = 0; b < B; b++) if (inst[b].phase != LbfgsInstance::DONE) ids.push_back(b);
        if (ids.empty()) break;
        const int nb = (int)ids.size();
        xb.resize((size_t)nb * n); fb.assign(nb, 0.0); gb.assign((size_t)nb * n, 0.0);
        for (int q = 0; q < nb; q++) std::copy(inst[ids[q]].request(), inst[ids[q]].request() + n, xb.begin() + (size_t)q * n);
        eval(instance, nb, ids.data(), xb.data(), fb.data(), gb.data());
        for (int q = 0; q < nb; q++) inst[ids[q]].feed(fb[q], gb.data() + (size_t)q * n);
        ++rounds;
    }
    for (int b = 0; b < B; b++) {
        std::copy(inst[b].solution(), inst[b].solution() + n, x + (size_t)b * n);
        f[b] = inst[b].fx; ret[b] = inst[b].ret;
        if (stats) stats[b] = inst[b].st;
    }
    return rounds;
}

#ifdef ISDF_WITH_EIGEN
// the reference's signature, for call sites such as mid_end.cpp:56-62
typedef double (*lbfgs_evaluate_t)(void *instance, const Eigen::VectorXd &x, Eigen::VectorXd &g, double &p_cost);
struct EigenThunk { lbfgs_evaluate_t fn; void *instance; };
inline double eigen_thunk_eval(void *th, const double *x, double *g, int n, double *p_cost) {
    EigenThunk *t = static_cast<EigenThunk *>(th);
    Eigen::VectorXd xv = Eigen::Map<const Eigen::VectorXd>(x, n), gv(n);
    double pc = 0;
    const double f = t->fn(t->instance, xv, gv, pc);
    Eigen::Map<Eigen::VectorXd>(g, n) = gv;
    if (p_cost) *p_cost = pc;
    return f;
}
inline int lbfgs_optimize(Eigen::VectorXd &x, double &f, lbfgs_evaluate_t eval, void *instance, const LbfgsParams &pr, LbfgsStats *st = nullptr) {
    EigenThunk th{eval, instance};
    return lbfgs_optimize((int)x.size(), x.data(), f, &eigen_thunk_eval, nullptr, nullptr, &th, pr, st);
}
#endif

}  // namespace isdf_host
