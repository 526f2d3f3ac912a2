"""A catalogue of L-BFGS runs, one per branch of the reference's patched LBFGS-Lite fork (utils/lbfgs.hpp: lbfgs_optimize :480-830,
line_search_lewisoverton :290-430) and of its three product drivers (host/isdf_lbfgs.hpp sequential and lock-step, csrc/isdf_lbfgs.cuh
k_lbfgs_feed). Each case is an objective, a full parameter set and a start; `reached(result)` shows from the return code or the trace that
the run took its branch. A direction reset re-evaluates the accepted point, so it shows in the trace as two consecutive identical points.

Every objective uses only IEEE-exact element-wise operations and math.fsum, so its bits do not depend on the machine, on numpy's SIMD
paths or on whether it is evaluated one instance at a time or for a whole batch.

Branches of the fork no objective can reach, so no case tries:
  * `step *= 2` (lbfgs.hpp:407): the line search only gets there after the Armijo test failed, which sets brackt; so it always bisects.
  * LBFGSERR_MAXIMUMSTEP (:420): a step above max_step is clamped once (touched); every later trial bisects towards mu = 0 below the
    clamped trial, so the step can never exceed max_step again.
  * LBFGSERR_INCREASEGRADIENT (:321): d is -g on the first iteration, -g / |g| * olddnorm after a reset (every product g_i * d_i <= 0), and
    a two-loop direction with d.g >= 0 is replaced by a reset (:788) — d.g is the same left-to-right sum as gp.d, since gp = g then.
    A NaN makes `0 < dginit` false.

One known divergence, recorded by the case "leading NaN gradient": the product's norm_inf starts at 0 and std::max / fmax skip a NaN, while
the Eigen stand-in's cwiseAbs().maxCoeff() starts at element 0 and so keeps a leading NaN. With g(x0) = [NaN, small...] and g_epsilon > 0
the product drivers report convergence at x0 (ret 0, one evaluation); the reference build goes on to step = 1 / |d| = NaN and returns
LBFGSERR_INVALIDPARAMETERS (-1006) from the line search, also at x0 after one evaluation. (The real Eigen's maxCoeff leaves NaN handling
unspecified.) That case is pinned to the product's host driver, and the reference build's answer is recorded beside it."""
import math
import numpy as np

CONVERGENCE, STOP, CANCELED = 0, 1, 2
ERR_INVALID_FUNCVAL, ERR_MINIMUMSTEP, ERR_MAXIMUMLINESEARCH, ERR_MAXIMUMITERATION = -1012, -1011, -1009, -1008
ERR_WIDTHTOOSMALL, ERR_INVALIDPARAMETERS = -1007, -1006

# isdf_lbfgs_default_params: the back end's settings
DEFAULTS = dict(mem_size=16, past=10, max_iterations=0, max_linesearch=64, g_epsilon=0.0, delta=1e-6, min_step=1e-32, max_step=1e20,
                f_dec_coeff=1e-4, cautious_factor=1e-6, machine_prec=1e-16)
HOST_KEYS = ("mem_size", "past", "delta", "g_epsilon", "max_iterations", "max_linesearch", "min_step", "max_step", "f_dec_coeff",
             "cautious_factor", "machine_prec")


def _rowsum(A):
    return np.array([math.fsum(r) for r in A.tolist()]) if A.shape[1] else np.zeros(A.shape[0])


# ---- objectives: X (B, n) -> (F (B,), G (B, n)) --------------------------------------------------------------------------------------
def quad(w, c):
    w, c = np.asarray(w, float), np.asarray(c, float)

    def fun(X):
        d = X - c
        return _rowsum(0.5 * w * d * d), w * d
    return fun


def quartic(w):
    w = np.asarray(w, float)

    def fun(X):
        x2 = X * X
        return _rowsum(w * x2 * x2), 4.0 * w * x2 * X
    return fun


def quad_quartic(w, c, v):
    q, w4, c = quad(w, c), np.asarray(v, float), np.asarray(c, float)

    def fun(X):
        F, G = q(X)
        d = X - c
        d2 = d * d
        return F + _rowsum(w4 * d2 * d2), G + 4.0 * w4 * d2 * d
    return fun


def rosen2(X):
    a, b = X[:, 0], X[:, 1]
    t, u = b - a * a, 1.0 - a
    F = 100.0 * t * t + u * u
    G = np.stack([-400.0 * a * t - 2.0 * u, 200.0 * t], axis=1)
    return F, G


def wall(fun, c, r, value=1e6):
    """fun inside the max-norm ball of radius r around c; a finite plateau `value` outside (the gradient stays fun's)"""
    c = np.asarray(c, float)

    def w(X):
        F, G = fun(X)
        out = np.abs(X - c).max(axis=1) > r
        return np.where(out, value, F), G
    return w


def beyond(fun, r, value):
    """fun where |x|_2 <= r; `value` (NaN or inf) beyond"""
    def w(X):
        F, G = fun(X)
        out = np.sqrt(_rowsum(X * X)) > r
        return np.where(out, value, F), G
    return w


def grad_poison(fun, where, value, i=0):
    """fun, but g[i] = value wherever where(X) holds"""
    def w(X):
        F, G = fun(X)
        G = G.copy()
        G[where(X), i] = value
        return F, G
    return w


def one(fun):
    """the single-instance form the host drivers call: x (n,) -> (f, g)"""
    def f1(x):
        F, G = fun(np.asarray(x, float)[None, :])
        return float(F[0]), G[0].copy()
    return f1


# ---- what a result shows ---------------------------------------------------------------------------------------------------------
def resets(trace):
    """direction resets: evaluations at the same point as the one before"""
    t = np.asarray(trace)
    return int(sum(np.array_equal(t[k], t[k - 1]) for k in range(1, len(t))))


def _grad0(case):
    return one(case["fun"])(case["x0"])[1]


class Case(dict):
    pass


def _case(name, fun, x0, reached, cancel_after=0, host_pinned=False, f_unwritten=False, **params):
    """host_pinned: the golden is the product's host driver (the reference build differs, see above); f_unwritten: the sequential drivers
    return without writing f (lbfgs.hpp:814-817), where the lock-step and device drivers report f(x)"""
    c = Case(name=name, fun=fun, x0=np.asarray(x0, float), params={**DEFAULTS, **params}, cancel_after=cancel_after, host_pinned=host_pinned,
             f_unwritten=f_unwritten)
    c["reached"] = lambda r, c=c: reached(r, c)
    return c


def cases():
    rng = np.random.default_rng(31)
    q4 = quad([1.0, 2.0, 3.0, 4.0], [0.5, -1.0, 2.0, 0.25])
    slow = quad_quartic([0.01, 0.2, 1.0, 3.0, 0.05], [1.0, -0.5, 0.25, 2.0, -1.5], [0.5, 0.1, 2.0, 0.01, 1.0])
    x_slow = np.array([2.5, 1.0, -1.0, 0.5, 0.5])
    unit = np.array([1.0, 0.0, 0.0, 0.0])          # |g(x0)| of quad(1, x0 - unit * s) is exactly s
    q1 = quad(np.ones(4), np.zeros(4))
    out = [
        _case("convergence at the start", q4, [0.5, -1.0, 2.0, 0.25], lambda r, c: r["ret"] == CONVERGENCE and r["evaluations"] == 1, g_epsilon=1e-5),
        _case("convergence after a line search", q4, np.zeros(4), lambda r, c: r["ret"] == CONVERGENCE and r["iterations"] >= 2, g_epsilon=1e-6, past=0,
              mem_size=8, max_iterations=200),
    ]
    for past in (1, 3, 10):
        out.append(_case(f"stop, past {past}", slow, x_slow, lambda r, c: r["ret"] == STOP and r["iterations"] > c["params"]["past"], past=past,
                         delta=1e-3 if past == 1 else 1e-4, mem_size=6, max_iterations=500))
    for it in (1, 7):
        out.append(_case(f"max iterations {it}", slow, x_slow, lambda r, c: r["ret"] == ERR_MAXIMUMITERATION and r["iterations"] == c["params"]["max_iterations"],
                         max_iterations=it, past=0, mem_size=8))
    # a plateau 0.01 around x0 that the first trials (steps 1/|g|, then halved: 1, 0.5, 0.25 along d) all land on
    q_far = quad(np.ones(4), [3.0, -2.0, 1.0, 4.0])
    out += [
        _case("max line search", wall(q_far, np.zeros(4), 0.01), np.zeros(4),
              lambda r, c: r["ret"] == ERR_MAXIMUMLINESEARCH and r["evaluations"] == 4 and np.array_equal(r["x"], c["x0"]), max_linesearch=3),
        # both tests true on the first failed trial: the line-search count is tested first
        _case("max line search before width", wall(q_far, np.zeros(4), 0.01), np.zeros(4),
              lambda r, c: r["ret"] == ERR_MAXIMUMLINESEARCH and r["evaluations"] == 2, max_linesearch=1, machine_prec=2.0),
        # machine_prec > 1: the first bracket (mu = 0, nu = step) is already "too narrow"; mu never leaves 0 in the fork
        _case("width too small", wall(q_far, np.zeros(4), 0.01), np.zeros(4),
              lambda r, c: r["ret"] == ERR_WIDTHTOOSMALL and r["evaluations"] == 2 and np.array_equal(r["x"], c["x0"]), machine_prec=2.0),
        # |g(x0)| = 2: the first step is 0.5, the bisected one 0.25 < min_step
        _case("minimum step", wall(q1, np.zeros(4), 0.01), -2.0 * unit,
              lambda r, c: r["ret"] == ERR_MINIMUMSTEP and r["evaluations"] == 2 and np.array_equal(r["x"], c["x0"]), min_step=0.3),
        _case("NaN value in the line search", beyond(q_far, 1.5, np.nan), np.array([1.0, -0.5, 0.2, 0.9]),
              lambda r, c: r["ret"] == ERR_INVALID_FUNCVAL and np.isnan(r["f"]) and np.array_equal(r["x"], c["x0"]), past=3, mem_size=8),
        _case("+inf value in the line search", beyond(q_far, 1.5, np.inf), np.array([1.0, -0.5, 0.2, 0.9]),
              lambda r, c: r["ret"] == ERR_INVALID_FUNCVAL and np.isinf(r["f"]) and np.array_equal(r["x"], c["x0"]), past=3, mem_size=8),
        # the first trial (x[0] 0 -> 0.75) is accepted with a finite value and an inf gradient: the next direction has norm NaN
        _case("inf gradient at an accepted point", grad_poison(q_far, lambda X: X[:, 0] > 0.5, np.inf), np.zeros(4),
              lambda r, c: r["ret"] == ERR_INVALID_FUNCVAL and r["iterations"] == 1 and not np.array_equal(r["x"], c["x0"]), f_unwritten=True),
        _case("NaN gradient at x0", grad_poison(q4, lambda X: np.ones(len(X), bool), np.nan, i=1), np.zeros(4),
              lambda r, c: r["ret"] == ERR_INVALIDPARAMETERS and r["evaluations"] == 1 and np.array_equal(r["x"], c["x0"]), g_epsilon=0.0),
    ]
    for ca in (1, 5):
        out.append(_case(f"cancel after {ca}", slow, x_slow, lambda r, c: r["ret"] == CANCELED and r["iterations"] == c["cancel_after"] + 1,
                         cancel_after=ca, past=0, mem_size=8))
    # |g(x0)| = 1.2: the first trial (step 1/1.2, distance 1) lands on the plateau (0.5 away), the bisected step 0.41 is clamped to 0.3
    out.append(_case("max_step clamp", wall(q1, -1.2 * unit, 0.5), -1.2 * unit,
                     lambda r, c: (np.array_equal(r["trace"][2], c["x0"] + 0.3 * -_grad0(c)) and not np.array_equal(r["trace"][1], r["trace"][2])
                                   and r["ret"] == ERR_MAXIMUMITERATION),
                     max_step=0.3, max_iterations=4, past=0))
    # ys > cau never holds: every iteration ends in a reset
    out.append(_case("cautious-update reset", slow, x_slow, lambda r, c: r["ret"] == ERR_MAXIMUMITERATION and resets(r["trace"]) == r["iterations"] - 1,
                     cautious_factor=1e6, max_iterations=8, past=0, mem_size=4))
    # strictly convex quadratic, cautious_factor 0: ys > 0 = cau and d.g < 0 always, so every reset is |d| >= 0.04
    out.append(_case("|d| >= 0.04 reset", quad([1.0, 5.0, 0.5, 2.0, 9.0], [3.0, -2.0, 1.0, 4.0, 0.5]), np.zeros(5),
                     lambda r, c: resets(r["trace"]) >= 2 and r["ret"] == ERR_MAXIMUMITERATION, cautious_factor=0.0, max_iterations=10, past=0, mem_size=5))
    # a quartic bowl at a small scale: two-loop steps stay below 0.04, so the history fills and its ring wraps
    ring_w = [1.0, 3.0, 0.3, 10.0, 0.7, 2.0, 5.0, 0.1]
    for m, it in ((1, 20), (3, 20), (64, 90)):
        out.append(_case(f"history ring, mem_size {m}", quartic(ring_w), rng.uniform(-0.02, 0.02, 8),
                         lambda r, c: (r["ret"] == ERR_MAXIMUMITERATION and r["iterations"] == c["params"]["max_iterations"]
                                       and r["iterations"] - 1 - resets(r["trace"]) > c["params"]["mem_size"]),
                         mem_size=m, max_iterations=it, past=0))
    out += [
        _case("n = 1", quad_quartic([2.0], [0.3], [1.0]), [2.0], lambda r, c: r["ret"] in (CONVERGENCE, STOP) and r["iterations"] >= 2,
              g_epsilon=1e-10, past=2, delta=1e-12, max_iterations=100),
        _case("n = 2", rosen2, [-1.2, 1.0], lambda r, c: r["ret"] in (CONVERGENCE, STOP) and r["iterations"] > 20, g_epsilon=1e-8, past=0,
              mem_size=8, max_iterations=2000),
        _case("n = 1157", quad_quartic(np.linspace(0.5, 4.0, 1157), ((np.arange(1157) * 37) % 101 - 50) / 25.0, np.linspace(0.0, 0.2, 1157)),
              np.zeros(1157), lambda r, c: r["ret"] == ERR_MAXIMUMITERATION and r["iterations"] == 12, max_iterations=12),
        _case("leading NaN gradient", grad_poison(quad(np.ones(4), np.full(4, 1e-9)), lambda X: np.ones(len(X), bool), np.nan, i=0), np.zeros(4),
              lambda r, c: r["ret"] == CONVERGENCE and r["evaluations"] == 1, g_epsilon=1e-5, host_pinned=True),
    ]
    return out


def host_kwargs(case):
    """keyword arguments of host_lib.lbfgs_minimize[_batch] and oracle_lib.RefLbfgs.minimize"""
    p = case["params"]
    return {k: p[k] for k in HOST_KEYS}


def sequential_kwargs(case):
    """the sequential drivers have no progress callback: a cancel after c iterations is pinned, as the mid-end pins it, by the
    max_iterations = c + 1 stop at the same iterate"""
    kw = host_kwargs(case)
    if case["cancel_after"]:
        kw["max_iterations"] = case["cancel_after"] + 1
    return kw


def sequential_ret(case, ret):
    """the return code the lock-step and device drivers give where the sequential run (sequential_kwargs) gave `ret`"""
    return CANCELED if case["cancel_after"] and ret == ERR_MAXIMUMITERATION else ret
