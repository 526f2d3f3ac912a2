"""The failure contract shared by every entry point that has a host form and a `_device` form (include/isdf.h): both forms compute
equal values (the host evaluations add theirs to 0.0, so a -0.0 may come back as +0.0); a refused call returns the same code from both
forms, sets isdf_last_error and poisons every output the header names (host costs and f NaN, d_f NaN, every clearance and certificate summary); and a call moves the same statistics
(kernel_launches, and last_kernel_ms for the host forms that time their kernels). Every call runs on a fresh context, so that state
one call leaves behind (work-item schedules, warm starts) cannot tell the two forms apart."""
import ctypes as C
import math
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W

pytestmark = pytest.mark.gpu

K, N, N0 = 8, 4, 2            # pieces; N0 pieces per trajectory of the clearance check and the certificate
B, NB = 3, 3                  # problems and pieces per problem of the batched optimiser entry points
BMIN = [0.0, 0.0, 0.0]
OCC = W.random_map(24, 24, 24, p=0.01, seed=1, slabs=0)
T_, C_, WP_ = W.make_trajectory(N, [4, 4, 4], [20, 20, 20], seed=1)
T = np.ascontiguousarray(T_, dtype=np.float64)
CC = np.ascontiguousarray(C_, dtype=np.float64).reshape(-1)
PTS = W.gather_obstacle_points(OCC, BMIN, 1.0, WP_, 3.0)[:40]
DP, IP = C.POINTER(C.c_double), C.POINTER(C.c_int32)
# the pairs whose host form times its kernels into isdf_stats.last_kernel_ms
TIMED = {"eval_discrete", "eval_swept", "callback_batch", "frontend_feasibility"}


def problems():
    rng = np.random.default_rng(9)
    heads, tails, X = np.zeros((B, 3, 3)), np.zeros((B, 3, 3)), []
    for b in range(B):
        wp = W.random_walk_waypoints(NB, [4, 4, 4], [20, 20, 20], seed=200 + b)
        heads[b, :, 0], tails[b, :, 0] = wp[0], wp[-1]
        heads[b, :, 1] = rng.normal(size=3) * 0.3
        X.append(np.concatenate([rng.normal(size=NB) * 0.4 + 0.8, (wp[1:-1] + rng.normal(size=(NB - 1, 3)) * 0.2).reshape(-1)]))
    colmajor = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(-1)
    return colmajor(heads), colmajor(tails), np.ascontiguousarray(np.array(X)).reshape(-1)


HEAD, TAIL, X0 = problems()
DIM = 4 * NB - 3
WAYP = np.ascontiguousarray(X0.reshape(B, DIM)[:, NB:]).reshape(-1)


def dev(a):
    import torch
    return torch.tensor(np.ascontiguousarray(a), device="cuda")


def ptr(t, fault, first=False):
    """a device pointer; the first input of a call is NULL under the 'null' faults"""
    return None if (first and "null" in fault) else C.c_void_p(t.data_ptr())


def host_ptr(a, fault, first=False, kind=DP):
    return None if (first and "null" in fault) else a.ctypes.data_as(kind)


def stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def make_ev(fault, shape="Ball", points=False, kernels=False, esdf=False, scene=False):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs = K
    ev = I.Evaluator(cfg)
    if "nomap" not in fault:
        ev.set_map_u8(OCC, BMIN, 1.0)
    if "noshape" not in fault:
        ev.set_shape_named("Torus" if "shape" in fault else shape)
    if points and "nopoints" not in fault:
        ev.set_points(PTS)
    if kernels and "nokernels" not in fault:
        ev.frontend_build_kernels()
    if esdf and "noesdf" not in fault:
        ev.map_esdf()
    if scene and "noscene" not in fault:
        ev.set_sense_cloud((np.argwhere(OCC) + 0.5).astype(np.float32))
    if "shard" in fault:
        ev.set_shard(0, 2)
    return ev


# ---- the pairs: (host call, device call) -> (return code, outputs) ------------------------------------------------------------
def eval_host(name):
    def run(ev, h, fault):
        cost, gC, gT = C.c_double(0.0), np.zeros(18 * N), np.zeros(N)
        f = getattr(ev.lib, "isdf_" + name)
        r = f(h, 0 if "param" in fault else N, host_ptr(T, fault, True), host_ptr(CC, fault), C.byref(cost), gC.ctypes.data_as(DP), gT.ctypes.data_as(DP))
        return r, dict(out=np.concatenate([[cost.value], gC, gT]))
    return run


def eval_device(name):
    def run(ev, h, fault):
        dT, dC, dout = dev(T), dev(CC), dev(np.zeros(19 * N + 1))
        f = getattr(ev.lib, "isdf_" + name + "_device")
        r = f(h, 0 if "param" in fault else N, ptr(dT, fault, True), ptr(dC, fault), ptr(dout, fault), stream())
        return r, dict(out=dout.cpu().numpy())
    return run


def callback_host(ev, h, fault):
    cost, grad = np.zeros(B), np.zeros(B * DIM)
    r = ev.lib.isdf_callback_batch(h, B, 0 if "param" in fault else NB, host_ptr(HEAD, fault, True), host_ptr(TAIL, fault), 1, 20.0,
                                   host_ptr(X0, fault), cost.ctypes.data_as(DP), grad.ctypes.data_as(DP))
    return r, dict(cost=cost, grad=grad)


def callback_device(ev, h, fault):
    dh, dt, dx, dcost, dgrad = dev(HEAD), dev(TAIL), dev(X0), dev(np.zeros(B)), dev(np.zeros(B * DIM))
    r = ev.lib.isdf_callback_batch_device(h, B, 0 if "param" in fault else NB, ptr(dh, fault, True), ptr(dt, fault), 1, 20.0, ptr(dx, fault),
                                          ptr(dcost, fault), ptr(dgrad, fault), stream())
    return r, dict(cost=dcost.cpu().numpy(), grad=dgrad.cpu().numpy())


def lbfgs_params(ev, fault):
    return ev.lbfgs_params(max_iterations=4, mem_size=0 if "param" in fault else 8)


def ints():
    return [np.zeros(B, dtype=np.int32) for _ in range(3)]


def lbfgs_host(ev, h, fault):
    x, f, (ret, it, evs), rounds = X0.copy(), np.zeros(B), ints(), C.c_int32(0)
    r = ev.lib.isdf_lbfgs_batch(h, B, NB, host_ptr(HEAD, fault, True), host_ptr(TAIL, fault), 1, 20.0, C.byref(lbfgs_params(ev, fault)),
                                x.ctypes.data_as(DP), f.ctypes.data_as(DP), ret.ctypes.data_as(IP), it.ctypes.data_as(IP), evs.ctypes.data_as(IP),
                                C.byref(rounds))
    return r, dict(x=x, f=f, ret=ret, it=it, evs=evs, rounds=rounds.value)


def lbfgs_device(ev, h, fault):
    import torch
    dh, dt, dx, df = dev(HEAD), dev(TAIL), dev(X0), dev(np.zeros(B))
    di = torch.zeros(3 * B, dtype=torch.int32, device="cuda")
    rounds = C.c_int32(0)
    r = ev.lib.isdf_lbfgs_batch_device(h, B, NB, ptr(dh, fault, True), ptr(dt, fault), 1, 20.0, C.byref(lbfgs_params(ev, fault)), ptr(dx, fault),
                                       ptr(df, fault), ptr(di, fault), ptr(di[B:], fault), ptr(di[2 * B:], fault), C.byref(rounds), stream())
    i = di.cpu().numpy()
    return r, dict(x=dx.cpu().numpy(), f=df.cpu().numpy(), ret=i[:B], it=i[B:2 * B], evs=i[2 * B:], rounds=rounds.value)


def midend_params(ev, fault):
    p = ev.midend_params(max_iterations=12)
    if "param" in fault:
        p.reserved_ = 1
    return p


def midend_host(ev, h, fault):
    x, T_o, C_o, f, (ret, it, evs), rounds = np.zeros(B * DIM), np.zeros(B * NB), np.zeros(18 * B * NB), np.zeros(B), ints(), C.c_int32(0)
    r = ev.lib.isdf_midend_batch(h, B, NB, host_ptr(HEAD, fault, True), host_ptr(TAIL, fault), 1, C.byref(midend_params(ev, fault)),
                                 host_ptr(WAYP, fault), x.ctypes.data_as(DP), T_o.ctypes.data_as(DP), C_o.ctypes.data_as(DP), f.ctypes.data_as(DP),
                                 ret.ctypes.data_as(IP), it.ctypes.data_as(IP), evs.ctypes.data_as(IP), C.byref(rounds))
    return r, dict(x=x, T=T_o, coeffs=C_o, f=f, ret=ret, it=it, evs=evs, rounds=rounds.value)


def midend_device(ev, h, fault):
    import torch
    dh, dt, dw = dev(HEAD), dev(TAIL), dev(WAYP)
    dx, dT, dC, df = dev(np.zeros(B * DIM)), dev(np.zeros(B * NB)), dev(np.zeros(18 * B * NB)), dev(np.zeros(B))
    di = torch.zeros(3 * B, dtype=torch.int32, device="cuda")
    rounds = C.c_int32(0)
    r = ev.lib.isdf_midend_batch_device(h, B, NB, ptr(dh, fault, True), ptr(dt, fault), 1, C.byref(midend_params(ev, fault)), ptr(dw, fault),
                                        ptr(dx, fault), ptr(dT, fault), ptr(dC, fault), ptr(df, fault), ptr(di, fault), ptr(di[B:], fault),
                                        ptr(di[2 * B:], fault), C.byref(rounds), stream())
    i = di.cpu().numpy()
    return r, dict(x=dx.cpu().numpy(), T=dT.cpu().numpy(), coeffs=dC.cpu().numpy(), f=df.cpu().numpy(), ret=i[:B], it=i[B:2 * B],
                   evs=i[2 * B:], rounds=rounds.value)


def summaries(cls, raw):
    return [s.as_dict() for s in (cls * (N // N0)).from_buffer_copy(raw)]


def device_summary_buffer(cls, n=N // N0):
    import torch
    return torch.zeros(C.sizeof(cls) * n, dtype=torch.uint8, device="cuda")   # reads as "clear" until a failure poisons it


def clearance_params(ev, fault):
    return ev.clearance_params(0 if "param" in fault else K, 2.0, 0.5, N0)


def clearance_host(ev, h, fault):
    S = N * (K + 1)
    clear, vox, summ = np.zeros(S), np.zeros(S, dtype=np.int64), (I.ClearanceSummary * (N // N0))()
    r = ev.lib.isdf_trajectory_clearance(h, N, host_ptr(T, fault, True), host_ptr(CC, fault), C.byref(clearance_params(ev, fault)),
                                         clear.ctypes.data_as(DP), vox.ctypes.data_as(C.POINTER(C.c_int64)), summ)
    return r, dict(clear=clear, vox=vox, summary=[s.as_dict() for s in summ])


def clearance_device(ev, h, fault):
    S = N * (K + 1)
    dT, dC, dclear, dvox, dsum = dev(T), dev(CC), dev(np.zeros(S)), dev(np.zeros(S, dtype=np.int64)), device_summary_buffer(I.ClearanceSummary)
    r = ev.lib.isdf_trajectory_clearance_device(h, N, ptr(dT, fault, True), ptr(dC, fault), C.byref(clearance_params(ev, fault)), ptr(dclear, fault),
                                                ptr(dvox, fault), ptr(dsum, fault), stream())
    return r, dict(clear=dclear.cpu().numpy(), vox=dvox.cpu().numpy(), summary=summaries(I.ClearanceSummary, dsum.cpu().numpy().tobytes()))


SIZE = 2 ** 30   # max_samples_per_traj under the "size" faults: valid alone, but N (2 K + 1) + 3 B SIZE exceeds 31 bits


def certify_params(ev, fault):
    return ev.certify_params(K, 2.0, 0.5, N0, max_depth=65 if "param" in fault else None, max_samples=SIZE if "size" in fault else None)


def certify_host(ev, h, fault):
    summ = (I.CertifySummary * (N // N0))()
    r = ev.lib.isdf_trajectory_certify(h, N, host_ptr(T, fault, True), host_ptr(CC, fault), C.byref(certify_params(ev, fault)), summ)
    return r, dict(summary=[s.as_dict() for s in summ])


def certify_device(ev, h, fault):
    dT, dC, dsum = dev(T), dev(CC), device_summary_buffer(I.CertifySummary)
    r = ev.lib.isdf_trajectory_certify_device(h, N, ptr(dT, fault, True), ptr(dC, fault), C.byref(certify_params(ev, fault)), ptr(dsum, fault),
                                              stream())
    return r, dict(summary=summaries(I.CertifySummary, dsum.cpu().numpy().tobytes()))


def dynamics_params(ev, fault):
    return ev.dynamics_params(K, N0, max_depth=65 if "param" in fault else None, max_samples=SIZE if "size" in fault else None)


def dynamics_host(ev, h, fault):
    summ = (I.DynamicsSummary * (N // N0))()
    r = ev.lib.isdf_trajectory_dynamics(h, N, host_ptr(T, fault, True), host_ptr(CC, fault), C.byref(dynamics_params(ev, fault)), summ)
    return r, dict(summary=[s.as_dict() for s in summ])


def dynamics_device(ev, h, fault):
    dT, dC, dsum = dev(T), dev(CC), device_summary_buffer(I.DynamicsSummary)
    r = ev.lib.isdf_trajectory_dynamics_device(h, N, ptr(dT, fault, True), ptr(dC, fault), C.byref(dynamics_params(ev, fault)), ptr(dsum, fault),
                                               stream())
    return r, dict(summary=summaries(I.DynamicsSummary, dsum.cpu().numpy().tobytes()))


def nvox():
    return int(np.prod(OCC.shape))


def frontend_host(ev, h, fault):
    masks = np.zeros(4 * nvox(), dtype=np.uint32)
    return ev.lib.isdf_frontend_feasibility(h, host_ptr(masks, fault, True, C.POINTER(C.c_uint32))), dict(masks=masks)


def frontend_device(ev, h, fault):
    import torch
    d = torch.zeros(4 * nvox(), dtype=torch.int32, device="cuda")
    r = ev.lib.isdf_frontend_feasibility_device(h, ptr(d, fault, True), stream())
    return r, dict(masks=d.cpu().numpy().view(np.uint32))


# trajectory states: one trajectory, QS query times across it
OFF1 = np.array([0, N], dtype=np.int32)
QS = 64


def state_times(Q):
    return np.ascontiguousarray(np.linspace(0.0, float(T.sum()), Q)), np.zeros(Q, dtype=np.int32)


def states_host(ev, h, fault, Q=QS):
    times, traj = state_times(Q)
    out = np.zeros(Q * I.STATE_DOUBLES)
    r = ev.lib.isdf_trajectory_states(h, 0 if "param" in fault else 1, host_ptr(OFF1, fault, True, IP), T.ctypes.data_as(DP), CC.ctypes.data_as(DP),
                                      Q, traj.ctypes.data_as(IP), times.ctypes.data_as(DP), out.ctypes.data_as(DP))
    return r, dict(out=out)


def states_device(ev, h, fault):
    times, traj = state_times(QS)
    doff, dT, dC, dtraj, dtimes, dout = dev(OFF1), dev(T), dev(CC), dev(traj), dev(times), dev(np.zeros(QS * I.STATE_DOUBLES))
    r = ev.lib.isdf_trajectory_states_device(h, 0 if "param" in fault else 1, ptr(doff, fault, True), ptr(dT, fault), ptr(dC, fault), QS,
                                             ptr(dtraj, fault), ptr(dtimes, fault), ptr(dout, fault), stream())
    return r, dict(out=dout.cpu().numpy())


# posed body points: QP state records (every field drawn, so every input reaches the result), NBODY body points
QP, NBODY = 16, 7
STATES = np.random.default_rng(3).normal(size=QP * I.STATE_DOUBLES)
BODY = np.random.default_rng(4).normal(size=3 * NBODY)


def pose_points_host(ev, h, fault):
    out = np.zeros(QP * NBODY * 3)
    r = ev.lib.isdf_pose_points(h, QP, host_ptr(STATES, fault, True), -1 if "param" in fault else NBODY, BODY.ctypes.data_as(DP), out.ctypes.data_as(DP))
    return r, dict(out=out)


def pose_points_device(ev, h, fault):
    ds, db, dout = dev(STATES), dev(BODY), dev(np.zeros(QP * NBODY * 3))
    r = ev.lib.isdf_pose_points_device(h, QP, ptr(ds, fault, True), -1 if "param" in fault else NBODY, ptr(db, fault), ptr(dout, fault), stream())
    return r, dict(out=dout.cpu().numpy())


# closed loop: two rollouts of the trajectory, one under a side force
RS = 2
SIM_TRAJ = np.zeros(RS, dtype=np.int32)
SIM_DIST = np.zeros((RS, 6))
SIM_DIST[1, 1] = 0.5


def sim_setup(fault):
    p = I.sim_default_params(t_end=0.5, log_every=5)
    if "param" in fault:
        p.reserved_ = 1
    init = np.ascontiguousarray(I.sim_init_from_trajectories(OFF1, CC, SIM_TRAJ, p))
    return p, init, I.sim_log_records(p)


def sim_summaries(raw):
    return [s.as_dict() for s in (I.SimSummary * RS).from_buffer_copy(raw)]


def simulate_host(ev, h, fault):
    p, init, n_log = sim_setup(fault)
    log, summ = np.zeros(RS * n_log * I.SIM_DOUBLES), (I.SimSummary * RS)()
    r = ev.lib.isdf_simulate(h, 1, host_ptr(OFF1, fault, True, IP), T.ctypes.data_as(DP), CC.ctypes.data_as(DP), RS, SIM_TRAJ.ctypes.data_as(IP),
                             init.ctypes.data_as(DP), SIM_DIST.ctypes.data_as(DP), C.byref(p), n_log, log.ctypes.data_as(DP), summ)
    return r, dict(log=log, summary=[s.as_dict() for s in summ])


def simulate_device(ev, h, fault):
    import torch
    p, init, n_log = sim_setup(fault)
    doff, dT, dC, dtraj, dinit, ddist = dev(OFF1), dev(T), dev(CC), dev(SIM_TRAJ), dev(init), dev(SIM_DIST)
    dlog, dsum = dev(np.zeros(RS * n_log * I.SIM_DOUBLES)), torch.zeros(C.sizeof(I.SimSummary) * RS, dtype=torch.uint8, device="cuda")
    r = ev.lib.isdf_simulate_device(h, 1, ptr(doff, fault, True), ptr(dT, fault), ptr(dC, fault), RS, ptr(dtraj, fault), ptr(dinit, fault),
                                    ptr(ddist, fault), C.byref(p), n_log, ptr(dlog, fault), ptr(dsum, fault), stream())
    return r, dict(log=dlog.cpu().numpy(), summary=sim_summaries(dsum.cpu().numpy().tobytes()))


def poisoned_sim_summary(s):
    nans = ("max_err", "t_max_err", "rms_err", "final_err", "max_tilt", "max_omega", "t_diverged")
    counts = ("accepted", "rejected", "clamped_steps", "floor_contacts", "nan_rollbacks")
    return all(math.isnan(s[k]) for k in nans) and all(s[k] == -1 for k in counts) and s["diverged"] == 1


# ESDF queries, inside and outside the map
QE = 50
EPTS = np.random.default_rng(5).uniform(-2.0, 26.0, size=3 * QE)


def esdf_host(ev, h, fault):
    dist, grad = np.zeros(QE), np.zeros(3 * QE)
    r = ev.lib.isdf_esdf_query(h, 7 if "param" in fault else 2, host_ptr(EPTS, fault, True), QE, dist.ctypes.data_as(DP), grad.ctypes.data_as(DP))
    return r, dict(dist=dist, grad=grad)


def esdf_device(ev, h, fault):
    dp_, ddist, dgrad = dev(EPTS), dev(np.zeros(QE)), dev(np.zeros(3 * QE))
    r = ev.lib.isdf_esdf_query_device(h, 7 if "param" in fault else 2, ptr(dp_, fault, True), QE, ptr(ddist, fault), ptr(dgrad, fault), stream())
    return r, dict(dist=ddist.cpu().numpy(), grad=dgrad.cpu().numpy())


# poses as (x, y, z, w, qx, qy, qz) records, in groups of QG
QC, QG = 12, 6


def pose_records():
    rng = np.random.default_rng(6)
    q = rng.normal(size=(QC, 4))
    return np.ascontiguousarray(np.concatenate([rng.uniform(2.0, 22.0, size=(QC, 3)), q / np.linalg.norm(q, axis=1, keepdims=True)], axis=1))


POSES = pose_records()


def pose_clearance_params(ev, fault):
    p = ev.pose_clearance_params(2.0, 0.5, QG)
    if "param" in fault:
        p.reserved_ = 1
    return p


def pose_clearance_host(ev, h, fault):
    clear, vox, summ = np.zeros(QC), np.zeros(QC, dtype=np.int64), (I.ClearanceSummary * (QC // QG))()
    base = POSES.ctypes.data
    r = ev.lib.isdf_pose_clearance(h, QC, None if "null" in fault else C.cast(base, DP), C.cast(base + 24, DP), 7,
                                   C.byref(pose_clearance_params(ev, fault)), clear.ctypes.data_as(DP), vox.ctypes.data_as(C.POINTER(C.c_int64)), summ)
    return r, dict(clear=clear, vox=vox, summary=[s.as_dict() for s in summ])


def pose_clearance_device(ev, h, fault):
    dpose, dclear, dvox = dev(POSES), dev(np.zeros(QC)), dev(np.zeros(QC, dtype=np.int64))
    dsum = device_summary_buffer(I.ClearanceSummary, QC // QG)
    r = ev.lib.isdf_pose_clearance_device(h, QC, ptr(dpose, fault, True), C.c_void_p(dpose.data_ptr() + 24), 7, C.byref(pose_clearance_params(ev, fault)),
                                          ptr(dclear, fault), ptr(dvox, fault), ptr(dsum, fault), stream())
    return r, dict(clear=dclear.cpu().numpy(), vox=dvox.cpu().numpy(), summary=summaries(I.ClearanceSummary, dsum.cpu().numpy().tobytes()))


# the certified swept volume of the trajectory on a 1-unit grid around it
def swept_setup(ev, fault):
    p = ev.swept_params(K, max_depth=65 if "param" in fault else None)
    return p, I.swept_grid_for(T, CC, 1.0, p.band, 1.0)


def swept_grid_host(ev, h, fault):
    p, g = swept_setup(ev, fault)
    n = g.X * g.Y * g.Z
    val, low, ts, dec = np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n, dtype=np.uint8)
    r = ev.lib.isdf_swept_volume_grid(h, N, host_ptr(T, fault, True), CC.ctypes.data_as(DP), C.byref(p), C.byref(g), val.ctypes.data_as(DP),
                                      low.ctypes.data_as(DP), ts.ctypes.data_as(DP), dec.ctypes.data_as(C.POINTER(C.c_uint8)), None)
    return r, dict(value=val, lower=low, tstar=ts, decided=dec)


def swept_grid_device(ev, h, fault):
    p, g = swept_setup(ev, fault)
    n = g.X * g.Y * g.Z
    dT, dC, dval, dlow, dts, ddec = dev(T), dev(CC), dev(np.zeros(n)), dev(np.zeros(n)), dev(np.zeros(n)), dev(np.zeros(n, dtype=np.uint8))
    r = ev.lib.isdf_swept_volume_grid_device(h, N, ptr(dT, fault, True), ptr(dC, fault), C.byref(p), C.byref(g), ptr(dval, fault), ptr(dlow, fault),
                                             ptr(dts, fault), ptr(ddec, fault), None, stream())
    return r, dict(value=dval.cpu().numpy(), lower=dlow.cpu().numpy(), tstar=dts.cpu().numpy(), decided=ddec.cpu().numpy())


# depth images of the map's occupied voxel centres at the poses above
def sense_host(ev, h, fault):
    p = I.sense_params(width=64, height=48)
    depth = np.zeros(QC * p.height * p.width, dtype=np.int32)
    base = POSES.ctypes.data
    r = ev.lib.isdf_sense_depth(h, 0 if "param" in fault else QC, None if "null" in fault else C.c_void_p(base), C.c_void_p(base + 24), 7,
                                C.byref(p), depth.ctypes.data_as(C.c_void_p))
    return r, dict(depth=depth)


def sense_device(ev, h, fault):
    import torch
    p = I.sense_params(width=64, height=48)
    dpose, ddepth = dev(POSES), torch.zeros(QC * p.height * p.width, dtype=torch.int32, device="cuda")
    r = ev.lib.isdf_sense_depth_device(h, 0 if "param" in fault else QC, ptr(dpose, fault, True), C.c_void_p(dpose.data_ptr() + 24), 7, C.byref(p),
                                       ptr(ddepth, fault), stream())
    return r, dict(depth=ddepth.cpu().numpy())


# front-end paths and planning: BP (start, goal) pairs between traversable voxels of OCC, found once on a context of their own. The
# offset arrays start as SENTINEL, so that a test sees which calls write them.
BP, SENTINEL = 6, -7
CAP = 4096    # path nodes and planned pieces; 1 under the "cap" faults
_ENDS = []


def path_ends():
    if not _ENDS:
        import frontpath_oracle as FO
        ev = make_ev("", kernels=True)
        trav = np.argwhere(FO.traversable(OCC, ev.frontend_feasibility(*OCC.shape)))
        ev.close()
        v = trav[np.random.default_rng(8).choice(len(trav), 2 * BP, replace=False)] + 0.5
        _ENDS.extend([np.ascontiguousarray(v[:BP]), np.ascontiguousarray(v[BP:])])
    return _ENDS


def sentinels():
    return np.full(BP + 1, SENTINEL, dtype=np.int32)


def path_setup(fault, pairs):
    starts, goals = path_ends()
    prm = I.FrontPathParams()
    prm.reserved_[0] = 1 if "param" in fault else 0
    return (starts if pairs else np.ascontiguousarray(starts[0])), goals, prm, 1 if "cap" in fault else CAP


def path_host(pairs):
    def run(ev, h, fault):
        starts, goals, prm, cap = path_setup(fault, pairs)
        xyz, rp, off, cost, found = np.zeros(3 * cap), np.zeros(2 * cap), sentinels(), np.zeros(BP), np.zeros(BP, dtype=np.uint8)
        outs = (xyz.ctypes.data_as(DP), rp.ctypes.data_as(DP), off.ctypes.data_as(IP), cost.ctypes.data_as(DP), found.ctypes.data_as(C.POINTER(C.c_uint8)))
        if pairs:   # two fields at a time: three chunks
            r = ev.lib.isdf_frontend_path_pairs(h, BP, host_ptr(starts, fault, True), goals.ctypes.data_as(DP), C.byref(prm), 2, cap, *outs)
        else:
            r = ev.lib.isdf_frontend_path_batch(h, host_ptr(starts, fault, True), BP, goals.ctypes.data_as(DP), C.byref(prm), cap, *outs)
        return r, dict(xyz=xyz, rp=rp, offsets=off, cost=cost, found=found)
    return run


def path_device(pairs):
    def run(ev, h, fault):
        starts, goals, prm, cap = path_setup(fault, pairs)
        dxyz, drp, doff, dcost, dfound = dev(np.zeros(3 * cap)), dev(np.zeros(2 * cap)), dev(sentinels()), dev(np.zeros(BP)), dev(np.zeros(BP, dtype=np.uint8))
        dg = dev(goals)
        outs = (ptr(dxyz, fault), ptr(drp, fault), ptr(doff, fault), ptr(dcost, fault), ptr(dfound, fault), stream())
        if pairs:
            ds = dev(starts)
            r = ev.lib.isdf_frontend_path_pairs_device(h, BP, ptr(ds, fault, True), ptr(dg, fault), C.byref(prm), 2, cap, *outs)
        else:
            r = ev.lib.isdf_frontend_path_batch_device(h, host_ptr(starts, fault, True), BP, ptr(dg, fault), C.byref(prm), cap, *outs)
        return r, dict(xyz=dxyz.cpu().numpy(), rp=drp.cpu().numpy(), offsets=doff.cpu().numpy(), cost=dcost.cpu().numpy(), found=dfound.cpu().numpy())
    return run


# planning: plan_pairs with both certificates and every output; plan_batch with no certificate and only the required outputs (path_off,
# path_xyz, certify and dynamics NULL)
def plan_setup(ev, fault, pairs):
    starts, goals = path_ends()
    p = ev.plan_params(backend_max_iterations=60, flags=(I.PLAN_CERTIFY | I.PLAN_DYNAMICS) if pairs else 0)
    if "param" in fault:
        p.flags = 4   # unknown
    return (starts if pairs else np.ascontiguousarray(starts[0])), goals, p, 1 if "cap" in fault else CAP


def plan_results(raw):
    return [s.as_dict() for s in (I.PlanResult * BP).from_buffer_copy(raw)]


def plan_host(pairs):
    def run(ev, h, fault):
        starts, goals, p, cap = plan_setup(ev, fault, pairs)
        po, T_o, C_o, res = sentinels(), np.zeros(cap), np.zeros(18 * cap), (I.PlanResult * BP)()
        tail = (cap, po.ctypes.data_as(IP), T_o.ctypes.data_as(DP), C_o.ctypes.data_as(DP), res)
        out = dict(piece_off=po, T=T_o, coeffs=C_o)
        if pairs:
            pf, xyz, cs, ds = sentinels(), np.zeros(3 * CAP), (I.CertifySummary * BP)(), (I.DynamicsSummary * BP)()
            r = ev.lib.isdf_plan_pairs(h, BP, host_ptr(starts, fault, True), goals.ctypes.data_as(DP), C.byref(p), 0, CAP, pf.ctypes.data_as(IP),
                                       xyz.ctypes.data_as(DP), *tail, cs, ds)
            out.update(path_off=pf, path_xyz=xyz, certify=np.frombuffer(bytes(cs), np.uint8), dynamics=np.frombuffer(bytes(ds), np.uint8))
        else:
            r = ev.lib.isdf_plan_batch(h, host_ptr(starts, fault, True), BP, goals.ctypes.data_as(DP), C.byref(p), 0, None, None, *tail, None, None)
        return r, dict(out, results=plan_results(bytes(res)))
    return run


def plan_device(pairs):
    def run(ev, h, fault):
        import torch
        starts, goals, p, cap = plan_setup(ev, fault, pairs)
        dpo, dT, dC, dg = dev(sentinels()), dev(np.zeros(cap)), dev(np.zeros(18 * cap)), dev(goals)
        dres = torch.zeros(C.sizeof(I.PlanResult) * BP, dtype=torch.uint8, device="cuda")
        tail = (cap, ptr(dpo, fault), ptr(dT, fault), ptr(dC, fault), ptr(dres, fault))
        out = {}
        if pairs:
            dst, dpf, dxyz = dev(starts), dev(sentinels()), dev(np.zeros(3 * CAP))
            dcs, dds = device_summary_buffer(I.CertifySummary, BP), device_summary_buffer(I.DynamicsSummary, BP)
            r = ev.lib.isdf_plan_pairs_device(h, BP, ptr(dst, fault, True), ptr(dg, fault), C.byref(p), 0, CAP, ptr(dpf, fault), ptr(dxyz, fault),
                                              *tail, ptr(dcs, fault), ptr(dds, fault), stream())
            out = dict(path_off=dpf.cpu().numpy(), path_xyz=dxyz.cpu().numpy(), certify=dcs.cpu().numpy(), dynamics=dds.cpu().numpy())
        else:
            r = ev.lib.isdf_plan_batch_device(h, host_ptr(starts, fault, True), BP, ptr(dg, fault), C.byref(p), 0, None, None, *tail, None, None,
                                              stream())
        return r, dict(out, piece_off=dpo.cpu().numpy(), T=dT.cpu().numpy(), coeffs=dC.cpu().numpy(),
                       results=plan_results(dres.cpu().numpy().tobytes()))
    return run


def poisoned_plan_result(s):
    return s["stage"] == I.PLAN_FAILED and all(math.isnan(s[k]) for k in ("path_cost", "midend_f", "backend_f", "duration"))


PATH_FAULTS = {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "nokernels": -2, "shard": -4, "nokernels+null": -1}
PLAN_FAULTS = {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "nokernels": -2, "shard": -4}


# name -> (host, device, make_ev keywords, {fault: code}). "nomap+null" / "shard+null" pin the order of the checks: the state is
# checked before the pointers; "size+nomap" / "size+shard" pin where each certificate checks its 31-bit size: after the state checks
# for the clearance certificate, before the shard check for the dynamic-limit certificate.
PAIRS = {
    "eval_discrete": (eval_host("eval_discrete"), eval_device("eval_discrete"), {},
                      {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "nomap+null": -2}),
    "eval_swept": (eval_host("eval_swept"), eval_device("eval_swept"), dict(points=True),
                   {"ctx": -1, "null": -1, "param": -1, "noshape": -2, "nopoints": -2}),
    "callback_batch": (callback_host, callback_device, {},
                       {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "shard": -2, "nomap+null": -2}),
    "lbfgs_batch": (lbfgs_host, lbfgs_device, {},
                    {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "shard": -2, "nomap+null": -2}),
    "midend_batch": (midend_host, midend_device, {}, {"ctx": -1, "null": -1, "param": -1, "shard": -2, "shard+null": -2}),
    "trajectory_clearance": (clearance_host, clearance_device, {},
                             {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "shard": -4, "nomap+null": -2}),
    "trajectory_certify": (certify_host, certify_device, {},
                           {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "shape": -4, "shard": -4, "nomap+null": -2,
                            "size": -1, "size+nomap": -2, "size+shard": -4}),
    "trajectory_dynamics": (dynamics_host, dynamics_device, {}, {"ctx": -1, "null": -1, "param": -1, "shard": -4, "size": -1, "size+shard": -1}),
    "frontend_feasibility": (frontend_host, frontend_device, dict(kernels=True),
                             {"ctx": -1, "null": -1, "nomap": -2, "nokernels": -2, "nokernels+null": -2}),
    "trajectory_states": (states_host, states_device, {}, {"ctx": -1, "null": -1, "param": -1}),
    "pose_points": (pose_points_host, pose_points_device, {}, {"ctx": -1, "null": -1, "param": -1}),
    "simulate": (simulate_host, simulate_device, {}, {"ctx": -1, "null": -1, "param": -1}),
    "esdf_query": (esdf_host, esdf_device, dict(esdf=True), {"ctx": -1, "null": -1, "param": -1, "noesdf": -2}),
    "pose_clearance": (pose_clearance_host, pose_clearance_device, {},
                       {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "shard": -4}),
    "swept_volume_grid": (swept_grid_host, swept_grid_device, {}, {"ctx": -1, "null": -1, "param": -1, "noshape": -2, "shard": -4}),
    "sense_depth": (sense_host, sense_device, dict(scene=True), {"ctx": -1, "null": -1, "param": -1, "noscene": -2}),
    # the path calls check their pointers before the state ("nokernels+null")
    "frontend_path_batch": (path_host(False), path_device(False), dict(kernels=True), PATH_FAULTS),
    "frontend_path_pairs": (path_host(True), path_device(True), dict(kernels=True), PATH_FAULTS),
    "plan_batch": (plan_host(False), plan_device(False), dict(kernels=True), PLAN_FAULTS),
    "plan_pairs": (plan_host(True), plan_device(True), dict(kernels=True), PLAN_FAULTS),
}
# the pairs whose device form poisons its outputs with a kernel (counted in kernel_launches) when it has a context
POISON_KERNEL = {"simulate"}


def call(pair, form, fault):
    """one call on a fresh context: (code, isdf_last_error, outputs, kernel_launches delta, whether last_kernel_ms changed)"""
    host, device, kw, _ = PAIRS[pair]
    ev = make_ev(fault, **kw)
    import torch
    torch.cuda.synchronize()
    s0 = ev.stats()
    ev.lib.isdf_default_config(None)                        # a known message, so that a refusal must write its own
    stale = ev.lib.isdf_last_error()
    r, outs = (host if form == "host" else device)(ev, None if fault == "ctx" else ev.h, fault)
    torch.cuda.synchronize()
    err = ev.lib.isdf_last_error()
    s1 = ev.stats()
    ev.close()
    return r, (err if err != stale else b""), outs, s1.kernel_launches - s0.kernel_launches, s1.last_kernel_ms != s0.last_kernel_ms


def same(a, b):
    if isinstance(a, list):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    a, b = np.asarray(a), np.asarray(b)   # the host evaluations add their result to 0.0, which turns -0.0 into +0.0
    return a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


@pytest.mark.parametrize("pair", list(PAIRS))
def test_host_and_device_forms_agree(pair):
    rh, eh, oh, nh, msh = call(pair, "host", "")
    rd, ed, od, nd, msd = call(pair, "device", "")
    assert rh == 0 and rd == 0, (eh, ed)
    assert same(oh, od), pair
    assert nh == nd and nh > 0
    assert msh == (pair in TIMED) and not msd


def poisoned_summary(s):
    if "upper" in s:   # isdf_dynamics_summary
        bounds = ("upper", "attained", "t_attained", "thrust_lower", "thrust_attained_min", "t_thrust_attained_min")
        return (s["verdict"] == 0 and all(np.all(np.isnan(s[k])) for k in bounds) and s["violated"] == s["undecided"] == 0 and
                s["samples"] == s["undecided_intervals"] == s["depth"] == -1)
    if "verdict" in s:
        return (s["verdict"] == 0 and all(math.isnan(s[k]) for k in ("lower_bound", "min_clearance", "t_min", "first_hit")) and
                s["voxel_min"] == -1 and s["samples"] == s["undecided_intervals"] == s["depth"] == -1)
    return (s["collision_free"] == 0 and all(math.isnan(s[k]) for k in ("min_clearance", "t_min", "first_hit")) and
            s["voxel_min"] == s["piece_min"] == s["sample_min"] == s["colliding_samples"] == -1)


@pytest.mark.parametrize("pair,fault", [(p, f) for p, v in PAIRS.items() for f in v[3]])
def test_refusals_agree_and_poison(pair, fault):
    code = PAIRS[pair][3][fault]
    for form in ("host", "device"):
        r, err, outs, launches, ms = call(pair, form, fault)
        assert r == code and err, (form, r, err)
        assert launches == (pair in POISON_KERNEL and form == "device" and fault != "ctx") and not ms, form
        # poisoned outputs (include/isdf.h); a device form cannot write to a device pointer without a context
        if form == "host" or fault != "ctx":
            if pair == "eval_discrete" or pair == "eval_swept":
                assert form == "device" or math.isnan(outs["out"][0])
            elif pair == "callback_batch":
                assert form == "device" or np.all(np.isnan(outs["cost"]))
            elif pair in ("lbfgs_batch", "midend_batch"):
                assert np.all(np.isnan(outs["f"])), form
            elif pair in ("trajectory_clearance", "trajectory_certify", "trajectory_dynamics", "pose_clearance"):
                assert all(poisoned_summary(s) for s in outs["summary"]), (form, outs["summary"])
            elif pair == "simulate":
                assert all(poisoned_sim_summary(s) for s in outs["summary"]), (form, outs["summary"])
            elif pair == "swept_volume_grid":
                assert all(np.all(np.isnan(outs[k])) for k in ("value", "lower", "tstar")) and not outs["decided"].any(), form
            elif pair in ("plan_batch", "plan_pairs"):
                assert all(poisoned_plan_result(s) for s in outs["results"]), (form, outs["results"])


# The path and planning calls write their offsets once the sizes are known, also when a cap is too small: then both forms report the same
# sizes (and the planning results are poisoned). A call refused before the run leaves them as they were.
OFFSETS = {"frontend_path_batch": ["offsets"], "frontend_path_pairs": ["offsets"], "plan_batch": ["piece_off"], "plan_pairs": ["path_off", "piece_off"]}


@pytest.mark.parametrize("pair,fault", [(p, f) for p in OFFSETS for f in ["cap"] + list(PAIRS[p][3])])
def test_offsets_of_refused_path_and_plan_calls(pair, fault):
    (rh, _, oh, nh, _), (rd, _, od, nd, _) = call(pair, "host", fault), call(pair, "device", fault)
    assert rh == rd == PAIRS[pair][3].get(fault, -1)
    for k in OFFSETS[pair]:
        assert np.array_equal(oh[k], od[k]), (k, oh[k], od[k])
        assert (oh[k] == SENTINEL).all() == (fault != "cap"), (k, oh[k])
    if fault == "cap":
        assert nh == nd > 0
        if pair.startswith("plan"):
            assert same(oh["results"], od["results"]) and all(poisoned_plan_result(s) for s in oh["results"])


def swept_sdf_host(ev):
    p = ev.swept_params(K)
    val, low, ts, dec = np.zeros(QE), np.zeros(QE), np.zeros(QE), np.zeros(QE, dtype=np.uint8)
    r = ev.lib.isdf_swept_volume_sdf(ev.h, N, T.ctypes.data_as(DP), CC.ctypes.data_as(DP), C.byref(p), QE, EPTS.ctypes.data_as(DP),
                                     val.ctypes.data_as(DP), low.ctypes.data_as(DP), ts.ctypes.data_as(DP), dec.ctypes.data_as(C.POINTER(C.c_uint8)))
    return r, dict(value=val, lower=low, tstar=ts, decided=dec)


# host forms of different families in a row, their staged sizes growing and then shrinking: every host form stages through the
# context's one pinned and one device block
SHARED = [("states, large Q", lambda ev: states_host(ev, ev.h, "", Q=200_000)), ("clearance", lambda ev: clearance_host(ev, ev.h, "")),
          ("certify", lambda ev: certify_host(ev, ev.h, "")), ("callback", lambda ev: callback_host(ev, ev.h, "")),
          ("lbfgs", lambda ev: lbfgs_host(ev, ev.h, "")), ("swept volume sdf", swept_sdf_host), ("pose clearance", lambda ev: pose_clearance_host(ev, ev.h, "")),
          ("states, small Q", lambda ev: states_host(ev, ev.h, "", Q=5))]


def test_host_forms_in_a_row_equal_fresh_contexts():
    ev = make_ev("")
    shared = [call(ev) for _, call in SHARED]
    ev.close()
    for (name, call), (r, outs) in zip(SHARED, shared):
        fresh = make_ev("")
        rf, outs_f = call(fresh)
        fresh.close()
        assert r == 0 and rf == 0, name
        assert same(outs, outs_f), name
