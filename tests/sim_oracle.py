"""TEST INFRASTRUCTURE: ctypes access to tests/sim_serial.cpp, the serial CPU restatement of the closed loop (isdf_simulate), built by
build() next to the library objects with the reference's flags and no contraction."""
import ctypes as C
import os
import subprocess
import numpy as np
import isdf_b200 as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "sim_serial.cpp")
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


def set_input(p, rpm):
    out = np.empty(4)
    cl = lib().sim_set_input(C.byref(p), _d(_f(rpm)), _d(out))
    return out, bool(cl)
