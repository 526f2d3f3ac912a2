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


def make_ev(fault, shape="Ball", points=False, kernels=False):
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
    if "shard" in fault:
        ev.set_shard(0, 2)
    return ev


# ---- the eight pairs: (host call, device call) -> (return code, outputs) ------------------------------------------------------------
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


def device_summary_buffer(cls):
    import torch
    return torch.zeros(C.sizeof(cls) * (N // N0), dtype=torch.uint8, device="cuda")   # reads as "clear" until a failure poisons it


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


def certify_params(ev, fault):
    return ev.certify_params(K, 2.0, 0.5, N0, max_depth=65 if "param" in fault else None)


def certify_host(ev, h, fault):
    summ = (I.CertifySummary * (N // N0))()
    r = ev.lib.isdf_trajectory_certify(h, N, host_ptr(T, fault, True), host_ptr(CC, fault), C.byref(certify_params(ev, fault)), summ)
    return r, dict(summary=[s.as_dict() for s in summ])


def certify_device(ev, h, fault):
    dT, dC, dsum = dev(T), dev(CC), device_summary_buffer(I.CertifySummary)
    r = ev.lib.isdf_trajectory_certify_device(h, N, ptr(dT, fault, True), ptr(dC, fault), C.byref(certify_params(ev, fault)), ptr(dsum, fault),
                                              stream())
    return r, dict(summary=summaries(I.CertifySummary, dsum.cpu().numpy().tobytes()))


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


# name -> (host, device, make_ev keywords, {fault: code}). "nomap+null" / "shard+null" pin the order of the checks: the state is
# checked before the pointers.
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
                           {"ctx": -1, "null": -1, "param": -1, "nomap": -2, "noshape": -2, "shape": -4, "shard": -4, "nomap+null": -2}),
    "frontend_feasibility": (frontend_host, frontend_device, dict(kernels=True),
                             {"ctx": -1, "null": -1, "nomap": -2, "nokernels": -2, "nokernels+null": -2}),
}


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
        assert launches == 0 and not ms, form
        # poisoned outputs (include/isdf.h); a device form cannot write to a device pointer without a context
        if form == "host" or fault != "ctx":
            if pair == "eval_discrete" or pair == "eval_swept":
                assert form == "device" or math.isnan(outs["out"][0])
            elif pair == "callback_batch":
                assert form == "device" or np.all(np.isnan(outs["cost"]))
            elif pair in ("lbfgs_batch", "midend_batch"):
                assert np.all(np.isnan(outs["f"])), form
            elif pair in ("trajectory_clearance", "trajectory_certify"):
                assert all(poisoned_summary(s) for s in outs["summary"]), (form, outs["summary"])
