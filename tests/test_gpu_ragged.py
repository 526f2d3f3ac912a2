"""Ragged batches (include/isdf.h): problems of different piece counts in one call. Uniform offsets give the uniform calls' outputs bit for
bit; every problem of a mixed batch equals the same problem alone (and the sequential host drivers); instances that stop at different
rounds keep their own exits; the device forms equal the host forms; the refusals leave the context as it was; the planning call runs one
mid-end and one back end for plans of many N."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import midend_cases as M
import workloads as W
from common import small_case, BMIN, MESHES

pytestmark = pytest.mark.gpu

MIXED = [17, 1, 290, 3, 64, 2, 17, 3, 1, 64]   # N = 1, 2, 3, 17, 64 and 290, repeats, unsorted


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _ev(robot="Ball", K=16):
    cfg, occ, _, _, _ = small_case(N=6, K=K, seed=3)
    cfg.vmax, cfg.omgmax = 1.2, 0.5
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    else:
        ev.set_shape_named(robot)
    return ev, occ


def _problem(N, seed):
    """(head, tail, x) of one back-end problem of N pieces: a random walk through the map, perturbed"""
    rng = np.random.default_rng(seed)
    wp = W.random_walk_waypoints(N, [0, 0, 0], [50, 50, 34], seed=seed)
    h, t = np.zeros((3, 3)), np.zeros((3, 3))
    h[:, 0], t[:, 0] = wp[0], wp[-1]
    h[:, 1] = rng.normal(size=3) * 0.3
    tau = rng.normal(size=N) * 0.4 + 0.8
    return h, t, np.concatenate([tau, (wp[1:-1] + rng.normal(size=(N - 1, 3)) * 0.2).reshape(-1)])


def _problems(Ns, seed=300):
    ps = [_problem(N, seed + 7 * b) for b, N in enumerate(Ns)]
    return np.array([p[0] for p in ps]), np.array([p[1] for p in ps]), [p[2] for p in ps]


def _points(ev, x, N, occ):
    """the problem's obstacle list around its waypoints (a few occupied voxels for N = 1)"""
    if N > 1:
        pts = ev.gather_obstacle_points(x[N:].reshape(N - 1, 3), 3.0, [0.0, 0.0, 0.0])[0]
        if len(pts):
            return pts[:400]
    return (np.argwhere(occ)[:30] + 0.5).astype(np.float64)


# ---- uniform offsets == the uniform calls ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robot,swept", [("Ball", False), ("Ball", True), ("mesh", True)])
def test_uniform_offsets_equal_the_uniform_callback(robot, swept):
    ev, occ = _ev(robot)
    B, N0 = 5, 6
    heads, tails, xs = _problems([N0] * B)
    if swept:
        ev.set_points_batch([_points(ev, xs[b], N0, occ) for b in range(B)])
    for it in range(2):                                     # two evaluations: the persisted durations carry over identically
        X = np.array(xs) + 0.05 * it
        c0, g0 = ev.callback_batch(heads, tails, 20.0, X)
        T0, C0, e0 = ev.batch_trajectories(B, N0)
        c1, g1 = ev.callback_batch_ragged(heads, tails, 20.0, list(X))
        T1, C1, e1 = ev.batch_trajectories_ragged([N0] * B)
        assert _same(c0, c1) and _same(g0, np.array(g1)), it
        assert _same(T0, np.concatenate(T1)) and _same(C0, I.Ragged([N0] * B).pack_coeffs(C1)) and _same(e0, e1), it
    ev.close()


def test_uniform_offsets_equal_the_uniform_lbfgs_and_midend():
    ev, _ = _ev()
    B, N0 = 6, 5
    heads, tails, xs = _problems([N0] * B, seed=500)
    prm = ev.lbfgs_params(max_iterations=12, mem_size=8, past=3, delta=1e-7)
    u = ev.lbfgs_batch(heads, tails, 20.0, np.array(xs), prm)
    r = ev.lbfgs_batch_ragged(heads, tails, 20.0, xs, prm)
    assert _same(u["x"], np.array(r["x"])) and all(_same(u[k], r[k]) for k in ("f", "ret", "iterations", "evaluations", "rounds"))
    mh, mt, Q = [], [], []
    for b in range(B):
        h, t, q = M.problem(N0, 60 + b)
        mh.append(h); mt.append(t); Q.append(q.reshape(N0 - 1, 3))
    mh, mt, Q = np.array(mh), np.array(mt), np.array(Q)
    u = ev.midend_batch(mh, mt, Q)
    r = ev.midend_batch_ragged(mh, mt, list(Q))
    assert _same(u["x"], np.array(r["x"])) and _same(u["T"], np.array(r["T"])) and _same(u["coeffs"], I.Ragged([N0] * B).pack_coeffs(r["coeffs"]))
    assert all(_same(u[k], r[k]) for k in ("f", "ret", "iterations", "evaluations", "rounds"))
    X = np.array([M.start_point(N0, Q[b]) for b in range(B)]) + 0.1
    c0, g0 = ev.midend_callback_batch(mh, mt, Q, X)
    c1, g1 = ev.midend_callback_batch_ragged(mh, mt, list(Q), list(X))
    assert _same(c0, c1) and _same(g0, np.array(g1))
    ev.close()


# ---- mixed N == each problem alone -------------------------------------------------------------------------------------------------
def test_mixed_callback_with_swept_term_equals_each_problem_alone():
    Ns = MIXED
    ev, occ = _ev()
    heads, tails, xs = _problems(Ns)
    sets = [_points(ev, xs[b], N, occ) for b, N in enumerate(Ns)]
    long_b = 0                                              # N = 17: under 300 s at the first evaluation, over it at the second
    X1 = [x.copy() for x in xs]
    X1[long_b][:Ns[long_b]] = 3.0                           # T = 8.5 s per piece: 144.5 s
    X2 = [x + 0.01 for x in X1]
    X2[long_b][:Ns[long_b]] = 5.3                           # about 20.3 s per piece: 345 s, the search keeps the first duration
    ev.set_points_batch(sets)
    got = []
    for X in (X1, X2):
        c, g = ev.callback_batch_ragged(heads, tails, 20.0, X)
        T, Cc, e = ev.batch_trajectories_ragged(Ns)
        got.append((c, g, T, Cc, e))
    assert sum(T.size for T in got[1][2]) == sum(Ns) and sum(got[1][2][long_b]) > 300.0 > sum(got[0][2][long_b])
    ev.close()
    for b, N in enumerate(Ns):
        alone, _ = _ev()
        alone.set_points_batch([sets[b]])
        for k, X in enumerate((X1, X2)):
            c, g = alone.callback_batch(heads[b], tails[b], 20.0, X[b][None, :])
            T, Cc, e = alone.batch_trajectories(1, N)
            gc, gg, gT, gC, ge = got[k]
            assert c[0] == gc[b] and _same(g[0], gg[b]), (b, N, k)
            assert _same(T, gT[b]) and _same(Cc, gC[b]) and e[0] == ge[b], (b, N, k)
        alone.close()


def test_mixed_lbfgs_equals_each_problem_alone_and_the_host_driver():
    import host_lib as H
    Ns = MIXED
    ev, _ = _ev()
    heads, tails, xs = _problems(Ns, seed=700)
    max_it = 8
    prm = ev.lbfgs_params(max_iterations=max_it, mem_size=8, past=3, delta=1e-7)
    r = ev.lbfgs_batch_ragged(heads, tails, 20.0, xs, prm)
    assert r["rounds"] >= r["evaluations"].max() and r["iterations"].max() >= 3
    for b, N in enumerate(Ns):
        u = ev.lbfgs_batch(heads[b], tails[b], 20.0, xs[b][None, :], prm)
        assert _same(u["x"][0], r["x"][b]) and u["f"][0] == r["f"][b], (b, N)
        assert (u["ret"][0], u["iterations"][0], u["evaluations"][0]) == (r["ret"][b], r["iterations"][b], r["evaluations"][b]), (b, N)

        def fun(x, b=b):
            c, g = ev.callback_batch(heads[b], tails[b], 20.0, x[None, :])
            return float(c[0]), g[0]
        h = H.lbfgs_minimize(fun, xs[b], mem_size=8, past=3, delta=1e-7, g_epsilon=0.0, max_iterations=max_it)
        assert (h["ret"], h["iterations"], h["evaluations"]) == (r["ret"][b], r["iterations"][b], r["evaluations"][b]), (b, N)
        assert _same(h["x"], r["x"][b]) and h["f"] == r["f"][b], (b, N)
    ev.close()


def _midend_problems(Ns, seed=900):
    heads, tails, Q = [], [], []
    for b, N in enumerate(Ns):
        h, t, q = M.problem(N, seed + b)
        heads.append(h); tails.append(t); Q.append(q.reshape(N - 1, 3))
    return np.array(heads), np.array(tails), Q


def test_mixed_midend_equals_each_problem_alone_and_the_host_driver():
    Ns = MIXED
    ev, _ = _ev(K=64)
    heads, tails, Q = _midend_problems(Ns)
    p = ev.midend_params(cancel_after=40)
    r = ev.midend_batch_ragged(heads, tails, Q, p)
    for b, N in enumerate(Ns):
        u = ev.midend_batch(heads[b:b + 1], tails[b:b + 1], Q[b][None], p)
        assert _same(u["x"][0], r["x"][b]) and _same(u["T"][0], r["T"][b]) and _same(u["coeffs"], r["coeffs"][b]) and _same(u["f"][0], r["f"][b]), (b, N)
        assert (u["ret"][0], u["iterations"][0], u["evaluations"][0]) == (r["ret"][b], r["iterations"][b], r["evaluations"][b]), (b, N)
        h = M.HostMidEnd(heads[b], tails[b], Q[b], K=64, cancel_after=40).optimize()
        assert (h["ret"], h["iterations"], h["evaluations"]) == (r["ret"][b], r["iterations"][b], r["evaluations"][b]), (b, N)
        assert _same(h["x"], r["x"][b]) and _same(h["T"], r["T"][b]) and _same(h["coeffs"], r["coeffs"][b]), (b, N)
        if h["ret"] == M.LBFGSERR_INVALID_FUNCVAL and np.isnan(h["f"]) and not np.isnan(r["f"][b]):
            assert r["f"][b] == M.HostMidEnd(heads[b], tails[b], Q[b], K=64).cost(r["x"][b])[0], (b, N)   # the direction-norm exit: f at x
        else:
            assert _same(h["f"], r["f"][b]), (b, N)
    X = [M.start_point(N, Q[b]) + 0.05 for b, N in enumerate(Ns)]
    c, g = ev.midend_callback_batch_ragged(heads, tails, Q, X, p)
    for b, N in enumerate(Ns):
        hc, hg = M.HostMidEnd(heads[b], tails[b], Q[b], K=64, cancel_after=40).cost(X[b])
        assert c[b] == hc and _same(g[b], hg), (b, N)
    ev.close()


# ---- instances that stop at different rounds ----------------------------------------------------------------------------------------
def test_capped_and_cancelled_instances_keep_their_own_exits():
    ev, _ = _ev(K=64)
    Ns = [2, 40, 1, 9, 3, 40]
    heads, tails, xs = _problems(Ns, seed=1100)
    full = ev.lbfgs_batch_ragged(heads, tails, 20.0, xs, ev.lbfgs_params(max_iterations=30, mem_size=8, past=3, delta=1e-7))
    cap = int(np.sort(full["evaluations"])[len(Ns) // 2])     # some instances finish before the cap, the others are capped
    prm = ev.lbfgs_params(max_iterations=30, mem_size=8, past=3, delta=1e-7, max_rounds=cap)
    r = ev.lbfgs_batch_ragged(heads, tails, 20.0, xs, prm)
    assert r["rounds"] == cap and (r["ret"] == -1008).any() and (full["evaluations"] < cap).any()
    for b in range(len(Ns)):
        u = ev.lbfgs_batch(heads[b], tails[b], 20.0, xs[b][None, :], prm)
        assert _same(u["x"][0], r["x"][b]) and u["f"][0] == r["f"][b] and u["ret"][0] == r["ret"][b], b
        assert u["iterations"][0] == r["iterations"][b] and u["evaluations"][0] == r["evaluations"][b], b
        if full["evaluations"][b] < cap:
            assert r["ret"][b] == full["ret"][b] and _same(r["x"][b], full["x"][b]), b
    mh, mt, Q = _midend_problems(Ns, seed=1200)
    p = ev.midend_params(cancel_after=3, max_rounds=9)
    m = ev.midend_batch_ragged(mh, mt, Q, p)
    assert (m["ret"] == M.LBFGS_CANCELED).any() and (m["ret"] == -1008).any(), m["ret"]
    for b in range(len(Ns)):
        u = ev.midend_batch(mh[b:b + 1], mt[b:b + 1], Q[b][None], p)
        assert _same(u["x"][0], m["x"][b]) and _same(u["f"][0], m["f"][b]) and u["ret"][0] == m["ret"][b], b
        assert _same(u["T"][0], m["T"][b]) and _same(u["coeffs"], m["coeffs"][b]), b
    ev.close()


# ---- device forms ----------------------------------------------------------------------------------------------------------------------
def test_device_forms_equal_the_host_forms():
    import torch
    Ns = [5, 1, 12, 3]
    ev, occ = _ev()
    heads, tails, xs = _problems(Ns, seed=1300)
    L = I.Ragged(Ns)
    dv = lambda a: torch.tensor(np.ascontiguousarray(a).reshape(-1), dtype=torch.float64, device="cuda")
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(-1)
    d_h, d_t = dv(cm(heads)), dv(cm(tails))
    B, X = L.B, 4 * L.P - 3 * L.B
    s = torch.cuda.Stream()
    # callback
    c, g = ev.callback_batch_ragged(heads, tails, 20.0, xs)
    d_x, d_c, d_g = dv(L.pack_x(xs)), torch.zeros(B, dtype=torch.float64, device="cuda"), torch.zeros(X, dtype=torch.float64, device="cuda")
    with torch.cuda.stream(s):
        ev.callback_batch_ragged_device(L.piece_off, d_h.data_ptr(), d_t.data_ptr(), 1, 20.0, d_x.data_ptr(), d_c.data_ptr(), d_g.data_ptr(), s.cuda_stream)
    s.synchronize()
    assert _same(d_c.cpu().numpy(), c) and _same(d_g.cpu().numpy(), L.pack_x(g))
    # L-BFGS
    prm = ev.lbfgs_params(max_iterations=10, mem_size=8, past=3, delta=1e-7)
    r = ev.lbfgs_batch_ragged(heads, tails, 20.0, xs, prm)
    d_x, d_f, d_i = dv(L.pack_x(xs)), torch.zeros(B, dtype=torch.float64, device="cuda"), torch.zeros(3 * B, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        rounds = ev.lbfgs_batch_ragged_device(L.piece_off, d_h.data_ptr(), d_t.data_ptr(), 1, 20.0, d_x.data_ptr(), d_f.data_ptr(), d_i.data_ptr(),
                                              d_i.data_ptr() + 4 * B, d_i.data_ptr() + 8 * B, prm, s.cuda_stream)
    s.synchronize()
    i = d_i.cpu().numpy()
    assert rounds == r["rounds"] and _same(d_x.cpu().numpy(), L.pack_x(r["x"])) and _same(d_f.cpu().numpy(), r["f"])
    assert _same(i[:B], r["ret"]) and _same(i[B:2 * B], r["iterations"]) and _same(i[2 * B:], r["evaluations"])
    # mid-end
    mh, mt, Q = _midend_problems(Ns, seed=1400)
    p = ev.midend_params(cancel_after=30)
    m = ev.midend_batch_ragged(mh, mt, Q, p)
    d_h, d_t, d_q = dv(cm(mh)), dv(cm(mt)), dv(L.pack_waypoints(Q))
    d_x, d_T, d_C, d_f = (torch.zeros(n, dtype=torch.float64, device="cuda") for n in (X, L.P, 18 * L.P, B))
    d_i = torch.zeros(3 * B, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        rounds = ev.midend_batch_ragged_device(L.piece_off, d_h.data_ptr(), d_t.data_ptr(), 1, d_q.data_ptr(), d_x.data_ptr(), d_T.data_ptr(),
                                               d_C.data_ptr(), d_f.data_ptr(), d_i.data_ptr(), d_i.data_ptr() + 4 * B, d_i.data_ptr() + 8 * B, p,
                                               s.cuda_stream)
    s.synchronize()
    i = d_i.cpu().numpy()
    assert rounds == m["rounds"] and _same(d_x.cpu().numpy(), L.pack_x(m["x"])) and _same(d_f.cpu().numpy(), m["f"])
    assert _same(d_T.cpu().numpy(), L.pack_T(m["T"])) and _same(d_C.cpu().numpy(), L.pack_coeffs(m["coeffs"]))
    assert _same(i[:B], m["ret"]) and _same(i[B:2 * B], m["iterations"]) and _same(i[2 * B:], m["evaluations"])
    ev.close()


# ---- errors ---------------------------------------------------------------------------------------------------------------------------
def _raw_callback(ev, off, xs, heads, tails):
    off = np.ascontiguousarray(off, dtype=np.int32)
    B = off.size - 1
    x = np.ascontiguousarray(np.concatenate([np.asarray(v).reshape(-1) for v in xs]) if len(xs) else np.zeros(1))
    cost, grad = np.zeros(max(B, 1)), np.zeros(max(x.size, 1))
    h, t = I._colmajor(heads), I._colmajor(tails)
    r = ev.lib.isdf_callback_batch_ragged(ev.h, B, off.ctypes.data_as(C.POINTER(C.c_int32)), I._dp(h), I._dp(t), 1, 20.0, I._dp(x), I._dp(cost),
                                          I._dp(grad))
    return r, cost


def test_errors_leave_the_context_as_it_was():
    Ns = [3, 1, 5]
    ev, occ = _ev()
    heads, tails, xs = _problems(Ns, seed=1500)
    ev.set_points_batch([_points(ev, xs[b], N, occ) for b, N in enumerate(Ns)])
    ref = ev.callback_batch_ragged(heads, tails, 20.0, xs)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)

    def still_same():
        c, g = ev.callback_batch_ragged(heads, tails, 20.0, xs)
        assert _same(c, ref[0]) and all(_same(a, b) for a, b in zip(g, ref[1]))

    for off, code in (([1, 4, 5, 10], -1), ([0, 3, 3, 9], -1), ([0, 3, 2, 9], -1)):
        r, cost = _raw_callback(ev, off, xs, heads, tails)
        assert r == code and np.isnan(cost).all(), off
        still_same()
    big = [0, 3, 4, 4 + 291]                                # N_b = 291
    xb = xs[:2] + [np.zeros(4 * 291 - 3)]
    r, cost = _raw_callback(ev, big, xb, heads, tails)
    assert r == -4 and np.isnan(cost).all()
    still_same()
    f = np.ones(3)
    prm = ev.lbfgs_params()
    off = np.array([0, 3, 4, 9], dtype=np.int32)
    assert ev.lib.isdf_lbfgs_batch_ragged(ev.h, 3, None, I._dp(I._colmajor(heads)), I._dp(I._colmajor(tails)), 1, 20.0, C.byref(prm),
                                          I._dp(np.zeros(27)), I._dp(f), None, None, None, None) == -1 and np.isnan(f).all()
    f = np.ones(3)
    mp = ev.midend_params()
    assert ev.lib.isdf_midend_batch_ragged(ev.h, 3, off.ctypes.data_as(ip), I._dp(I._colmajor(heads)), I._dp(I._colmajor(tails)), 1, C.byref(mp), None,
                                           I._dp(np.zeros(27)), None, None, I._dp(f), None, None, None, None) == -1 and np.isnan(f).all()   # waypoints NULL, P > B
    still_same()
    # a registered point-set B that differs from the call's: no swept term (the uniform calls' rule), the time-integral term alone
    c2, g2 = ev.callback_batch_ragged(heads[:2], tails[:2], 20.0, xs[:2])
    ev.set_points_batch([])
    c2n, g2n = ev.callback_batch_ragged(heads[:2], tails[:2], 20.0, xs[:2])
    assert _same(c2, c2n) and all(_same(a, b) for a, b in zip(g2, g2n))
    ev.set_points_batch([_points(ev, xs[b], N, occ) for b, N in enumerate(Ns)])
    # sharded context
    ev.set_shard(0, 2)
    r, cost = _raw_callback(ev, [0, 3, 4, 9], xs, heads, tails)
    assert r == -2 and np.isnan(cost).all()
    ev.set_shard(0, 1)
    # a winding-sign mesh refuses the swept term
    V, F = MESHES["rcone"]()
    ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0], I.MESH_SIGN_WINDING)
    r, cost = _raw_callback(ev, [0, 3, 4, 9], xs, heads, tails)
    assert r == -4 and np.isnan(cost).all()
    ev.set_shape_named("Ball")
    still_same_after_reset = ev.callback_batch_ragged(heads, tails, 20.0, xs)
    assert np.isfinite(still_same_after_reset[0]).all()
    ev.close()


# ---- the planning call ----------------------------------------------------------------------------------------------------------------
def test_plan_runs_one_midend_and_one_back_end_over_many_N():
    import test_gpu_plan as TP
    occ, start, goals = TP._scene(24, seed=11)
    ev = TP._ev("Ball", occ)
    p = TP._params(ev, backend_max_iterations=40)
    got, info = ev.plan_batch(start, goals, p)
    fresh = TP._ev("Ball", occ)
    ref = TP._compose(fresh, start, goals, p)
    fresh.close()
    ev.close()
    Ns = {r["pieces"] for r in got if r["stage"] in (I.OPTIMISED, I.MIDEND_FAILED)}
    assert len(Ns) >= 8 and info["groups"] == len(Ns), (Ns, info)
    assert max(r["duration"] for r in ref) < 300.0
    for b in range(len(goals)):
        TP._check_plan(got[b], ref[b], b)
    be = [r["backend_evaluations"] for r in got if r["stage"] == I.OPTIMISED]
    assert be and info["backend_rounds"] == max(be), (info, be)
    print("N", sorted(Ns), "info", info)
