"""TEST INFRASTRUCTURE: ctypes access to tests/sim_serial.cpp, the serial CPU restatement of the closed loop (isdf_simulate), built by
build() next to the library objects with the reference's flags and no contraction; and to oracle/_ref/libref_sim.so (oracle/sim.mk), the
reference's own Quadrotor, SO3Control, getControl and odeint behind oracle/ref_sim_wrap.cpp, whose answers tests/golden/sim_reference.npz
stores (tests/golden/make_sim_golden.py)."""
import ctypes as C
import os
import subprocess
import numpy as np
import isdf_b200 as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "sim_serial.cpp")
ORACLE_DIR = os.path.join(ROOT, "oracle")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_sim.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "sim_reference.npz")
LIB = os.path.join(ROOT, "implicit-sdf-planner_b200", "build", "libsim_serial.so")


def build(force=False):
    deps = [SRC, os.path.join(ROOT, "include", "isdf.h")]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([gxx, "-O3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", LIB, SRC])


_lib = None
dp = C.POINTER(C.c_double)


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        pp = C.POINTER(I.SimParams)
        L.sim_rollout.argtypes = [pp, C.c_int, dp, dp, dp, dp, C.c_int, C.c_int, C.c_int, dp, C.POINTER(I.SimSummary)]
        L.sim_rhs.argtypes = [pp, dp, dp, dp, dp, dp]
        L.sim_open_loop.argtypes = [pp, dp, dp, dp, C.c_int, C.POINTER(C.c_int64)]
        L.sim_open_loop.restype = C.c_int
        L.sim_get_control.argtypes = [pp, dp, dp, dp, dp]
        L.sim_set_input.argtypes = [pp, dp, dp]
        L.sim_set_input.restype = C.c_int
        L.sim_calculate_control.argtypes = [pp, dp, dp, dp, dp, dp, dp, dp, dp]
        _lib = L
    return _lib


def _d(a):
    return None if a is None else a.ctypes.data_as(dp)


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def ticks(p):
    m = int(p.sim_rate / p.cmd_rate)
    n_ticks = int(np.floor(p.t_end * p.cmd_rate)) + 1
    return n_ticks, m, (n_ticks - 1) // p.log_every + 1


def simulate(piece_off, T, coeffs, traj, init, dist, p, cap_log=None):
    """-> (log (R, cap_log, 21), list of summary dicts), rollout by rollout as isdf_simulate defines them"""
    off, T, Cc = np.asarray(piece_off), _f(T).reshape(-1), _f(coeffs).reshape(-1)
    init = _f(init).reshape(-1, I.SIM_INIT_DOUBLES)
    dist = None if dist is None else _f(dist).reshape(-1, 6)
    n_ticks, m, n_log = ticks(p)
    cap = n_log if cap_log is None else cap_log
    R = init.shape[0]
    log = np.empty((R, cap, I.SIM_DOUBLES))
    out = []
    for r in range(R):
        b = int(traj[r])
        p0, n = int(off[b]), int(off[b + 1] - off[b])
        s = I.SimSummary()
        Tb, Cb = np.ascontiguousarray(T[p0:p0 + n]), np.ascontiguousarray(Cc[18 * p0:18 * (p0 + n)])
        lr = np.ascontiguousarray(log[r])
        di = None if dist is None else np.ascontiguousarray(dist[r])
        lib().sim_rollout(C.byref(p), n, _d(Tb), _d(Cb), _d(np.ascontiguousarray(init[r])), _d(di), n_ticks, m, cap, _d(lr), C.byref(s))
        log[r] = lr
        out.append(s.as_dict())
    return log, out


def line_trajectories():
    """(piece_off, T, coeffs): two trajectories in the ragged layout, of two 1 s pieces and one, each piece a straight line at 1-2 m"""
    lines = (([0.0, 0.0, 1.5], [0.5, 0.2, 0.1]), ([0.5, 0.2, 1.6], [-0.3, 0.4, 0.0]), ([2.0, 1.0, 1.0], [0.2, -0.2, 0.3]))
    out = []
    for group in (lines[:2], lines[2:]):
        N = len(group)
        c = np.zeros(18 * N)   # 6N x 3 column-major, ascending powers
        for i, (p0, v) in enumerate(group):
            for d in range(3):
                c[6 * N * d + 6 * i], c[6 * N * d + 6 * i + 1] = p0[d], v[d]
        out.append(c)
    return np.array([0, 2, 3], dtype=np.int32), np.array([1.0, 1.0, 1.0]), np.concatenate(out)


def rhs(p, x, inp, dist=None):
    dx, acc = np.empty(22), np.empty(3)
    lib().sim_rhs(C.byref(p), _d(_f(x)), _d(_f(inp)), _d(None if dist is None else _f(dist)), _d(dx), _d(acc))
    return dx, acc


def open_loop(p, x, rpm, n, dist=None):
    """n steps at a fixed commanded rpm -> (x, counts dict, ok)"""
    x = _f(x).copy()
    cnt = (C.c_int64 * 5)()
    ok = lib().sim_open_loop(C.byref(p), _d(x), _d(_f(rpm)), _d(None if dist is None else _f(dist)), int(n), cnt)
    return x, dict(accepted=cnt[0], rejected=cnt[1], clamped=cnt[2], floor=cnt[3], rollbacks=cnt[4]), bool(ok)


def get_control(p, R, omega, force, quat, current_yaw=0.0):
    rpm = np.empty(4)
    cmd = _f(list(force) + list(quat) + [current_yaw])
    lib().sim_get_control(C.byref(p), _d(_f(R).reshape(9)), _d(_f(omega)), _d(cmd), _d(rpm))
    return rpm


def calculate_control(p, pos, vel, acc, dp_, dv, da):
    f, q = np.empty(3), np.empty(4)
    lib().sim_calculate_control(C.byref(p), _d(_f(pos)), _d(_f(vel)), _d(_f(acc)), _d(_f(dp_)), _d(_f(dv)), _d(_f(da)), _d(f), _d(q))
    return f, q


def set_input(p, rpm):
    out = np.empty(4)
    cl = lib().sim_set_input(C.byref(p), _d(_f(rpm)), _d(out))
    return out, bool(cl)


# ---- the reference-compiled simulator (oracle/_ref/libref_sim.so) ----
_ref = None


def ref_available():
    """builds the library where the reference tree exists (make's dependency check decides); elsewhere whatever library exists is kept"""
    subprocess.call(["make", "-C", ORACLE_DIR, "-f", "sim.mk"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return os.path.exists(REF_LIB)


def ref_lib():
    global _ref
    if _ref is None:
        L = C.CDLL(REF_LIB)
        pp = C.POINTER(I.SimParams)
        L.ref_sim_rhs.argtypes = [pp, dp, dp, dp, dp, dp]
        L.ref_sim_step.argtypes = [pp, dp, dp, dp, C.POINTER(C.c_int64)]
        L.ref_sim_step.restype = C.c_int
        L.ref_sim_set_input.argtypes = [pp, dp, dp]
        L.ref_sim_get_control.argtypes = [pp, dp, dp, dp, dp]
        L.ref_sim_calculate_control.argtypes = [pp, dp, dp, dp, dp, dp, dp, dp, dp]
        L.ref_sim_rollout.argtypes = [pp, C.c_int, dp, dp, dp, dp, C.c_int, C.c_int, C.c_int, dp, C.POINTER(I.SimSummary), C.POINTER(C.c_int)]
        _ref = L
    return _ref


def ref_rhs(p, x, rpm, dist=None):
    dx, acc = np.empty(22), np.empty(3)
    ref_lib().ref_sim_rhs(C.byref(p), _d(_f(x)), _d(_f(rpm)), _d(None if dist is None else _f(dist)), _d(dx), _d(acc))
    return dx, acc


def ref_step(p, x, rpm, dist=None):
    """one Quadrotor::step -> (x, dict(accepted, rejected, same, rollbacks, floor), status: 1 ok, 0 odeint gave up, -1 the 100000-try bound)"""
    x = _f(x).copy()
    cnt = (C.c_int64 * 5)()
    ok = ref_lib().ref_sim_step(C.byref(p), _d(x), _d(_f(rpm)), _d(None if dist is None else _f(dist)), cnt)
    return x, dict(accepted=cnt[0], rejected=cnt[1], same=cnt[2], rollbacks=cnt[3], floor=cnt[4]), int(ok)


def ref_set_input(p, rpm):
    out = np.empty(4)
    ref_lib().ref_sim_set_input(C.byref(p), _d(_f(rpm)), _d(out))
    return out


def ref_get_control(p, R, omega, force, quat, current_yaw=0.0):
    rpm = np.empty(4)
    ref_lib().ref_sim_get_control(C.byref(p), _d(_f(R).reshape(9)), _d(_f(omega)), _d(_f(list(force) + list(quat) + [current_yaw])), _d(rpm))
    return rpm


def ref_calculate_control(p, pos, vel, acc, dp_, dv, da):
    f, q = np.empty(3), np.empty(4)
    ref_lib().ref_sim_calculate_control(C.byref(p), _d(_f(pos)), _d(_f(vel)), _d(_f(acc)), _d(_f(dp_)), _d(_f(dv)), _d(_f(da)), _d(f), _d(q))
    return f, q


def ref_simulate(piece_off, T, coeffs, traj, init, dist, p, cap_log=None):
    """the reference driver's (log, summaries) in the layout of simulate(); asserts every step's counting run matched Quadrotor::step"""
    off, T, Cc = np.asarray(piece_off), _f(T).reshape(-1), _f(coeffs).reshape(-1)
    init = _f(init).reshape(-1, I.SIM_INIT_DOUBLES)
    dist = None if dist is None else _f(dist).reshape(-1, 6)
    n_ticks, m, n_log = ticks(p)
    cap = n_log if cap_log is None else cap_log
    log = np.empty((init.shape[0], cap, I.SIM_DOUBLES))
    out = []
    for r in range(init.shape[0]):
        b = int(traj[r])
        p0, n = int(off[b]), int(off[b + 1] - off[b])
        s, same = I.SimSummary(), C.c_int()
        lr = np.empty((cap, I.SIM_DOUBLES))
        di = None if dist is None else np.ascontiguousarray(dist[r])
        ref_lib().ref_sim_rollout(C.byref(p), n, _d(np.ascontiguousarray(T[p0:p0 + n])), _d(np.ascontiguousarray(Cc[18 * p0:18 * (p0 + n)])),
                                  _d(np.ascontiguousarray(init[r])), _d(di), n_ticks, m, cap, _d(lr), C.byref(s), C.byref(same))
        assert same.value == 1, "a counting run left a different state than Quadrotor::step"
        log[r] = lr
        out.append(s.as_dict())
    return log, out
