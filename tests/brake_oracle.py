"""Restatement of isdf_trajectory_brake's candidates (include/isdf.h) in FP64 in the header's operation order (Python floats round every
operation as the library's -fmad=false unit does): tau_max, tau_k, the equal durations, the waypoint times tau_k f_j, the head and tail
states and the waypoints by locatePieceIdx and getPos / getVel / getAcc, and the candidate's MINCO S3 solve by the host port (host_lib),
which is bit-identical to the device solve."""
import math
import numpy as np
import host_lib as H
import navigate_oracle as NO


def pva(T, Cc, t):
    """position, velocity and acceleration of one trajectory (T (N,), its 6N x 3 column-major block) at time t: locatePieceIdx, then the
    running powers of traj_pvaj / Piece::getPos_Vel_Acc_Jerk (integer factors multiplied first)"""
    T = [float(x) for x in T]
    i, tl = NO.locate(T, float(t))
    blk = NO._block(Cc, len(T))[i]
    out = []
    for ax in range(3):
        c = [float(x) for x in blk[ax]]
        p = v = a = 0.0
        ptn = vtn = atn = 1.0
        vn, am, an = 1, 1, 2
        for k in range(6):
            p += ptn * c[k]
            ptn *= tl
            if k >= 1:
                f = vn * vtn
                v += f * c[k]
                vtn *= tl
                vn += 1
            if k >= 2:
                f = (am * an) * atn
                a += f * c[k]
                atn *= tl
                am += 1
                an += 1
        out.append((p, v, a))
    return np.array([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out])


def tau_max(T, t_stop_max):
    """min(t_stop_max, D), D the left-to-right sum of T; None for NO_INPUT"""
    D = 0.0
    for x in T:
        D += float(x)
    ts = float(t_stop_max)
    tm = ts if ts < D else D
    if len(T) == 0 or math.isnan(ts) or not (tm > 0.0 and math.isfinite(tm)):
        return None
    return tm


def schedule(tm, k, K, M):
    """(tau_k, the M durations, the waypoint times tau_k f_j for j = 1 .. M-1)"""
    tau = tm * (float(k + 1) / float(K))
    dur = (tau + tau) / float(M)
    times = []
    for j in range(1, M):
        u = float(M - j) / float(M)
        f = 1.0 - u * u
        times.append(tau * f)
    return tau, np.full(M, dur), times


def candidate(T, Cc, t_stop_max, k, K, M):
    """candidate k of one trajectory -> dict(tau, T (M,), coeffs (18 M,) in its own 6M x 3 column-major block, head, tail, waypoints
    (3, M-1)), or None for NO_INPUT"""
    tm = tau_max(T, t_stop_max)
    if tm is None:
        return None
    tau, dur, times = schedule(tm, k, K, M)
    p0, v0, a0 = pva(T, Cc, 0.0)
    head = np.stack([p0, v0, a0], 1)
    tail = np.stack([pva(T, Cc, tau)[0], np.zeros(3), np.zeros(3)], 1)
    wps = np.stack([pva(T, Cc, s)[0] for s in times], 1) if times else np.zeros((3, 0))
    coeffs = H.minco_forward(head, tail, wps, dur)[0]
    return dict(tau=tau, T=dur, coeffs=coeffs, head=head, tail=tail, waypoints=wps, times=times)


def ragged_candidate(off, T, Cc, t_stop_max, b, k, K, M):
    """candidate k of trajectory b of a ragged batch"""
    a, e = int(off[b]), int(off[b + 1])
    return candidate(np.asarray(T)[a:e], np.asarray(Cc)[18 * a:18 * e], float(np.asarray(t_stop_max)[b]), k, K, M)
