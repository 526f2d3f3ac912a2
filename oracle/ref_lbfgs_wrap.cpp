// ORACLE — TEST INFRASTRUCTURE ONLY.
// C wrapper around the reference's own L-BFGS (the patched LBFGS-Lite fork), compiled UNMODIFIED from where it lies:
//   /root/reference/src/utils/include/utils/lbfgs.hpp     lbfgs_optimize :480-830, line_search_lewisoverton :290-430
// against oracle/_shim_dyn/Eigen/Eigen (eager element-wise arithmetic, left-to-right reductions — see that header for what this does and
// does not pin). The built oracle/_ref/libref_lbfgs.so is kind "reference": it pins the product's host driver (host/isdf_lbfgs.hpp) —
// and through it the lock-step host and device drivers, which are tested bit-identical to that driver — on iterates, value, return code and
// evaluation count. The reference header prints progress to stdout on every iteration; the wrapper silences stdout for the duration.
#include <utils/lbfgs.hpp>
#include <cstdio>
#include <unistd.h>
#include <fcntl.h>

typedef double (*c_eval_t)(void *user, int n, const double *x, double *g);
struct Bridge { c_eval_t f; void *user; long evals; };
static double bridge_eval(void *inst, const Eigen::VectorXd &x, Eigen::VectorXd &g, double &p_cost) {
    Bridge *b = static_cast<Bridge *>(inst);
    b->evals++;
    p_cost = 0.0;
    return b->f(b->user, (int)x.size(), x.data(), g.data());
}

extern "C" int ref_lbfgs_optimize_ex(int n, double *x, double *f, c_eval_t eval, void *user, int mem_size, int past, double delta, double g_epsilon,
                                     int max_iterations, double min_step, int max_linesearch, double max_step, double f_dec_coeff, double cautious_factor,
                                     double machine_prec, long *evaluations) {
    lbfgs::lbfgs_parameter_t pr;
    pr.mem_size = mem_size; pr.past = past; pr.delta = delta; pr.g_epsilon = g_epsilon; pr.max_iterations = max_iterations; pr.min_step = min_step;
    pr.max_linesearch = max_linesearch; pr.max_step = max_step; pr.f_dec_coeff = f_dec_coeff; pr.cautious_factor = cautious_factor;
    pr.machine_prec = machine_prec;
    Eigen::VectorXd xv(n);
    for (int i = 0; i < n; i++) xv(i) = x[i];
    Bridge b{eval, user, 0};
    double fx = 0.0;
    fflush(stdout);
    const int saved = dup(1), nul = open("/dev/null", O_WRONLY);
    if (nul >= 0) dup2(nul, 1);
    const int ret = lbfgs::lbfgs_optimize(xv, fx, &bridge_eval, nullptr, nullptr, &b, pr);
    fflush(stdout);
    if (saved >= 0) { dup2(saved, 1); close(saved); }
    if (nul >= 0) close(nul);
    for (int i = 0; i < n; i++) x[i] = xv(i);
    *f = fx;
    if (evaluations) *evaluations = b.evals;
    return ret;
}

// the same with max_linesearch, max_step, f_dec_coeff, cautious_factor and machine_prec at lbfgs_parameter_t's defaults (the signature
// older callers were built against)
extern "C" int ref_lbfgs_optimize(int n, double *x, double *f, c_eval_t eval, void *user, int mem_size, int past, double delta, double g_epsilon,
                                  int max_iterations, double min_step, long *evaluations) {
    lbfgs::lbfgs_parameter_t d;
    return ref_lbfgs_optimize_ex(n, x, f, eval, user, mem_size, past, delta, g_epsilon, max_iterations, min_step, d.max_linesearch, d.max_step,
                                 d.f_dec_coeff, d.cautious_factor, d.machine_prec, evaluations);
}
