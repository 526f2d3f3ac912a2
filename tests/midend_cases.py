"""Shared pieces of the mid-end tests: A*-shaped paths and the waypoint rule, the product's host mid-end (host/isdf_midend.hpp through
libisdf_host.so), and the reference form of OriTraj::costFunction (mid_end.hpp:262-304: the reference-compiled MINCO of oracle/_ref/libref_minco.so
plus libm's pow, the std::pow of grad_cost_dir)."""
import ctypes as C
import math
import numpy as np

dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int)
LBFGS_STOP, LBFGS_CANCELED, LBFGSERR_MAXIMUMITERATION, LBFGSERR_INVALIDPARAMETERS, LBFGSERR_INVALID_FUNCVAL = 1, 2, -1008, -1006, -1012
# getOriTraj's L-BFGS settings (mid_end.cpp:48-54 with the shipped config): mem 16, past 10, delta 1e-6, g_epsilon 0, min_step 1e-32
LB = dict(mem_size=16, past=10, delta=1e-6, g_epsilon=0.0, max_iterations=100000, min_step=1e-32)


def waypoint_rule(path, res, parlength=3.0):
    """plan_manager.cpp:204-245 restated: the rows of path that become waypoints (N = len + 1); 1- and 2-node paths give none"""
    S = len(path)
    if S <= 2:
        return np.zeros((0, 3))
    gap = math.ceil(parlength / res)
    while gap >= S - 1:
        parlength /= 1.5
        gap = math.ceil(parlength / res)
    return np.array([path[i] for i in range(gap, S - 1, gap)]).reshape(-1, 3)


def astar_like_path(S, seed, res=1.0, origin=(0.0, 0.0, 0.0)):
    """S cube centres joined by 26-connected one-voxel steps, as isdf_frontend_path_batch returns them"""
    rng = np.random.default_rng(seed)
    steps = rng.integers(-1, 2, size=(max(S - 1, 0), 3))
    steps[np.all(steps == 0, axis=1)] = (1, 0, 0)
    vox = np.vstack([np.zeros((1, 3), dtype=np.int64), np.cumsum(steps, axis=0)])
    return (vox + 0.5) * res + np.asarray(origin, dtype=np.float64)


def problem(N, seed, res=1.0):
    """a plan of N pieces from an A*-shaped path (3 (N - 1) + 2 nodes at res 1: gap 3) -> head, tail (3x3, columns p, v, a), waypoints (N-1, 3)"""
    path = astar_like_path(3 * (N - 1) + 2, seed, res)
    Q = waypoint_rule(path, res)
    assert len(Q) == N - 1, (len(Q), N)
    head, tail = np.zeros((3, 3)), np.zeros((3, 3))
    head[:, 0], tail[:, 0] = path[0], path[-1]
    return head, tail, Q


def tau0(init_time=2.5):
    T = init_time
    return math.sqrt(2.0 * T - 1.0) - 1.0 if T > 1.0 else 1.0 - math.sqrt(2.0 / T - 1.0)


def start_point(N, Q, init_time=2.5):
    return np.concatenate([np.full(N, tau0(init_time)), np.asarray(Q, dtype=np.float64).reshape(-1)])


def forwardT(tau):
    return np.array([((0.5 * t + 1.0) * t + 1.0) if t > 0.0 else 1.0 / ((0.5 * t - 1.0) * t + 1.0) for t in tau])


def dT_dtau(tau):
    return np.array([(t + 1.0) if t > 0 else (1.0 - t) / (((0.5 * t - 1.0) * t + 1.0) ** 2) for t in tau])


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class HostMidEnd:
    """host/isdf_midend.hpp: MidEnd::costFunction, getOriTraj (sequential driver + earlyExit) and the lock-step driver with its cancel rule"""

    def __init__(self, head, tail, Q, K=64, weight=1000.0, rho=200.0, cancel_after=8000):
        import host_lib as H
        L = H.lib()
        L.isdf_host_midend_create.restype = C.c_void_p
        L.isdf_host_midend_create.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, dp, dp, dp]
        L.isdf_host_midend_destroy.argtypes = [C.c_void_p]
        L.isdf_host_midend_eval.restype = C.c_double
        L.isdf_host_midend_eval.argtypes = [C.c_void_p, C.c_int, dp, dp]
        L.isdf_host_midend_optimize.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double,
                                                dp, dp, dp, dp, ip, ip]
        L.isdf_host_midend_lockstep.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                                                C.c_double, dp, dp, ip, ip, ip]
        self.L = L
        Q = _f(Q).reshape(-1, 3)
        self.N = Q.shape[0] + 1
        self.head, self.tail, self.Q = _f(head), _f(tail), Q
        h, t = np.asfortranarray(self.head), np.asfortranarray(self.tail)
        q = _f(Q.reshape(-1)) if Q.size else np.zeros(1)
        self.h = L.isdf_host_midend_create(self.N, K, weight, rho, cancel_after, h.ctypes.data_as(dp), t.ctypes.data_as(dp), q.ctypes.data_as(dp))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.isdf_host_midend_destroy(self.h)
            self.h = None

    def cost(self, x):
        x = _f(x).copy()
        g = np.zeros_like(x)
        c = self.L.isdf_host_midend_eval(self.h, x.size, x.ctypes.data_as(dp), g.ctypes.data_as(dp))
        return c, g

    def optimize(self, init_time=2.5, **kw):
        p = dict(LB, **kw)
        n = 4 * self.N - 3
        x, T, Cc, f, it, ev = np.zeros(n), np.zeros(self.N), np.zeros(18 * self.N), C.c_double(0), C.c_int(0), C.c_int(0)
        r = self.L.isdf_host_midend_optimize(self.h, init_time, p["mem_size"], p["past"], p["delta"], p["g_epsilon"], p["max_iterations"], p["min_step"],
                                             x.ctypes.data_as(dp), C.byref(f), T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(it), C.byref(ev))
        return dict(ret=r, x=x, f=f.value, T=T, coeffs=Cc, iterations=it.value, evaluations=ev.value)

    @staticmethod
    def lockstep(mids, X0, cancel_after, **kw):
        p = dict(LB, **kw)
        B = len(mids)
        X = _f(X0).copy().reshape(-1)
        f, ret, it, ev = np.zeros(B), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        hs = (C.c_void_p * B)(*[m.h for m in mids])
        rounds = mids[0].L.isdf_host_midend_lockstep(B, hs, cancel_after, p["mem_size"], p["past"], p["delta"], p["g_epsilon"], p["max_iterations"],
                                                     p["min_step"], X.ctypes.data_as(dp), f.ctypes.data_as(dp), ret.ctypes.data_as(ip),
                                                     it.ctypes.data_as(ip), ev.ctypes.data_as(ip))
        return dict(rounds=rounds, x=X.reshape(B, -1), f=f, ret=ret, iterations=it, evaluations=ev)


def pose_terms(N, T, coeffs, Q, K, weight):
    """the pose term per piece from a coefficient block (6N x 3 column-major), the product's arithmetic: (cost w c_i, g . v at s, c_i)"""
    alpha = 1.0 / K
    out = []
    Cm = np.asarray(coeffs).reshape(3, 6 * N)
    for seg in range(1, N):
        s1 = alpha * T[seg]
        s2 = s1 * s1
        s3 = s2 * s1
        s4 = s2 * s2
        s5 = s4 * s1
        b0 = (1.0, s1, s2, s3, s4, s5)
        b1 = (0.0, 1.0, 2.0 * s1, 3.0 * s2, 4.0 * s3, 5.0 * s4)
        d, v = [], []
        for ax in range(3):
            c = Cm[ax, 6 * seg:6 * seg + 6]
            p = vv = 0.0
            for k in range(6):
                p += c[k] * b0[k]
                vv += c[k] * b1[k]
            d.append(p - Q[seg - 1][ax])
            v.append(vv)
        n = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        c3 = (n * n) * n
        if not c3 > 0.0:
            out.append((0.0, 0.0, 0.0))
            continue
        g = [(3.0 * (n * n)) * (d[k] / n) for k in range(3)]
        out.append((weight * c3, alpha * ((g[0] * v[0] + g[1] * v[1]) + g[2] * v[2]), c3))
    return out


def positions_at_s(N, T, coeffs, K):
    """p(T_{i+1} / K) of pieces 1 .. N-1 with the product's arithmetic: the waypoints that make every offset exactly zero"""
    alpha = 1.0 / K
    Cm = np.asarray(coeffs).reshape(3, 6 * N)
    out = []
    for seg in range(1, N):
        s1 = alpha * T[seg]
        s2 = s1 * s1
        b0 = (1.0, s1, s2, s2 * s1, s2 * s2, (s2 * s2) * s1)
        row = []
        for ax in range(3):
            p = 0.0
            for k in range(6):
                p += Cm[ax, 6 * seg + k] * b0[k]
            row.append(p)
        out.append(row)
    return np.array(out).reshape(-1, 3)


def ref_form_cost(rm, head, tail, Q, x, K=64, weight=1000.0, rho=200.0):
    """OriTraj::costFunction in the reference's form: the reference-compiled MINCO (rm = oracle_lib.RefMinco) and pow(|d|, 3),
    3 * pow(|d|, 2) * d.normalized() with libm's pow"""
    Q = np.asarray(Q, dtype=np.float64).reshape(-1, 3)
    N = Q.shape[0] + 1
    x = np.asarray(x, dtype=np.float64)
    tau, xi = x[:N], x[N:]
    T = forwardT(tau)
    inPs = xi.reshape(N - 1, 3).T
    co, cost, gC, gT = rm.forward(head, tail, inPs, T)
    gC, gT = gC.copy(), gT.copy()
    alpha = 1.0 / K
    Cm = co.reshape(3, 6 * N)
    for i in range(N - 1):
        seg = i + 1
        s1 = alpha * T[seg]
        b0 = np.array([1.0, s1, s1 ** 2, s1 ** 3, s1 ** 4, s1 ** 5])
        b1 = np.array([0.0, 1.0, 2 * s1, 3 * s1 ** 2, 4 * s1 ** 3, 5 * s1 ** 4])
        pos = np.array([float(np.dot(Cm[ax, 6 * seg:6 * seg + 6], b0)) for ax in range(3)])
        vel = np.array([float(np.dot(Cm[ax, 6 * seg:6 * seg + 6], b1)) for ax in range(3)])
        d = pos - Q[i]
        nrm = math.sqrt(float(np.dot(d, d)))
        cp = math.pow(nrm, 3)
        if not cp > 0:
            continue
        gp = 3 * math.pow(nrm, 2) * (d / nrm)
        for ax in range(3):
            gC[ax * 6 * N + 6 * seg:ax * 6 * N + 6 * seg + 6] += weight * (b0 * gp[ax])
        gT[seg] += weight * (cp * (alpha * float(np.dot(gp, vel))))
        cost += weight * cp
    gp_, gt_ = rm.backward(head, tail, inPs, T, gC, gT)
    cost += rho * float(np.sum(T))
    gt_ = gt_ + rho
    g = np.concatenate([gt_ * dT_dtau(tau), np.asarray(gp_).T.reshape(-1)])
    return cost, g


def ref_run_problem():
    """the plan of the whole-run comparison with the reference form (GPU test and golden fixture)"""
    return problem(8, 31)


def ref_form_optimize(rm, rl, head, tail, Q, init_time=2.5):
    """getOriTraj in the reference's form: the reference-compiled lbfgs.hpp (rl = oracle_lib.RefLbfgs) on ref_form_cost"""
    N = len(Q) + 1
    return rl.minimize(lambda x: ref_form_cost(rm, head, tail, Q, x), start_point(N, Q, init_time), **LB)


def trace_digest(trace):
    """SHA-256 of the evaluated points, in order, as float64 bytes: what the golden fixture keeps of an optimiser's trace"""
    import hashlib
    h = hashlib.sha256()
    for x in trace:
        h.update(np.ascontiguousarray(x, dtype=np.float64).tobytes())
    return h.hexdigest()
