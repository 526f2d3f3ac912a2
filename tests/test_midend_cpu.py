"""The mid-end on the CPU: waypoint selection (isdf_path_waypoints) against plan_manager.cpp:204-245 restated, the product's host cost
(host/isdf_midend.hpp, which the device callback equals bit for bit) against the reference form of OriTraj::costFunction and against finite
differences — its T-gradient quirk included — and the host drivers against the reference-compiled lbfgs.hpp."""
import os
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import midend_cases as M

REF = os.path.exists(O.REF_MINCO) and os.path.exists(O.REF_LBFGS)
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "midend_reference.npz")


def _paths(sizes, seed):
    return [M.astar_like_path(S, seed + k, res=0.37) for k, S in enumerate(sizes)]


@pytest.mark.parametrize("res", [0.1, 0.25, 0.3, 0.4, 1.0, 3.0, 4.0])
def test_path_waypoints_equal_plan_manager_rule(res):
    """every path size 1..200 in one call: the waypoints and N of every plan equal the restated loop, including non-integer quotients
    and several /1.5 reductions; 1- and 2-node paths give N = 1 (the reference never terminates there)"""
    paths = [M.astar_like_path(S, 1000 + S, res=res) for S in range(1, 201)]
    wps, pieces = I.path_waypoints(paths, res)
    for S, p, w, n in zip(range(1, 201), paths, wps, pieces):
        ref = M.waypoint_rule(p, res)
        assert n == len(ref) + 1 and np.array_equal(w, ref), (S, res)
        if S <= 2:
            assert n == 1
    # 3.0 / 0.4 = 7.5 and 3.0 / 0.25 = 12: ceil rounds the first up, leaves the second
    assert I.path_waypoints([M.astar_like_path(40, 1)], 0.4)[1][0] == len(range(8, 39, 8)) + 1
    assert I.path_waypoints([M.astar_like_path(40, 1)], 0.25)[1][0] == len(range(12, 39, 12)) + 1


def test_path_waypoints_reductions_and_offsets():
    import ctypes as C
    lib = I.load_library()
    # parlength / res = 3 -> gap 3 needs S - 1 > 3; S = 4 divides once (2 / 1 -> gap 2), S = 3 twice (gap 2, then gap 1)
    for S, gap in ((3, 1), (4, 2), (5, 3)):
        w, n = I.path_waypoints([M.astar_like_path(S, 7)], 1.0)
        assert n[0] == len(range(gap, S - 1, gap)) + 1
    # offsets: several plans back to back
    paths = _paths([5, 1, 17, 2, 64], 3)
    wps, pieces = I.path_waypoints(paths, 0.37)
    xyz = np.concatenate(paths)
    off = np.cumsum([0] + [len(p) for p in paths]).astype(np.int32)
    total = int(sum(len(w) for w in wps))
    ipp, dp = C.POINTER(C.c_int32), C.POINTER(C.c_double)
    out, wo, pc = np.zeros((total, 3)), np.zeros(6, dtype=np.int32), np.zeros(5, dtype=np.int32)
    assert lib.isdf_path_waypoints(5, off.ctypes.data_as(ipp), xyz.ctypes.data_as(dp), 0.37, 3.0, total, out.ctypes.data_as(dp), wo.ctypes.data_as(ipp),
                                   pc.ctypes.data_as(ipp)) == 0
    assert np.array_equal(out, np.concatenate(wps)) and np.array_equal(pc, pieces) and wo[-1] == total
    # cap one short: refused, the offsets still report what is needed
    wo[:] = 0
    assert lib.isdf_path_waypoints(5, off.ctypes.data_as(ipp), xyz.ctypes.data_as(dp), 0.37, 3.0, total - 1, out.ctypes.data_as(dp),
                                   wo.ctypes.data_as(ipp), pc.ctypes.data_as(ipp)) == -1
    assert wo[-1] == total
    # bad arguments
    bad_off = off.copy(); bad_off[2] = bad_off[1]                                   # an empty path
    for args in ((5, bad_off, 0.37, 3.0), (5, off, 0.0, 3.0), (5, off, float("nan"), 3.0), (5, off, 0.37, -1.0), (0, off, 0.37, 3.0)):
        B, o, res, pl = args
        assert lib.isdf_path_waypoints(B, o.ctypes.data_as(ipp), xyz.ctypes.data_as(dp), res, pl, total, out.ctypes.data_as(dp), wo.ctypes.data_as(ipp),
                                       pc.ctypes.data_as(ipp)) == -1, args
    assert lib.isdf_path_waypoints(1, None, None, 1.0, 3.0, 0, None, None, None) == -1


def _cost_cases():
    out = []
    for N in (1, 2, 3, 17, 64):
        for seed in (0, 1):
            head, tail, Q = M.problem(N, 500 + 7 * N + seed)
            rng = np.random.default_rng(N * 10 + seed)
            x = M.start_point(N, Q)
            x[:N] += rng.normal(size=N) * 0.3
            x[N:] += rng.normal(size=3 * (N - 1)) * 0.4
            if N > 1:
                head[:, 1] = rng.normal(size=3) * 0.5
            out.append((N, head, tail, Q, x))
    return out


def test_host_cost_against_reference_form():
    """the product's host cost (IEEE form) against the reference form (reference-compiled MINCO + libm pow): cost and gradient within 1e-10
    relative; the maxima observed are recorded in DESIGN §3.10"""
    zl = None if REF else np.load(GOLD)
    rm = O.RefMinco() if REF else None
    worst_c = worst_g = 0.0
    for k, (N, head, tail, Q, x) in enumerate(_cost_cases()):
        c, g = M.HostMidEnd(head, tail, Q).cost(x)
        if rm is not None:
            rc, rg = M.ref_form_cost(rm, head, tail, Q, x)
        else:
            rc, rg = float(zl[f"cost{k}_c"]), zl[f"cost{k}_g"]
        ec = abs(c - rc) / abs(rc)
        eg = float(np.max(np.abs(g - rg))) / float(np.max(np.abs(rg)))
        worst_c, worst_g = max(worst_c, ec), max(worst_g, eg)
        assert np.isfinite(c) and ec <= 1e-10 and eg <= 1e-10, (N, ec, eg)
    print(f"host vs reference form: cost rel {worst_c:.2e}, grad rel (max-norm) {worst_g:.2e}")


def test_fd_xi_and_tau_quirk():
    """central differences: the xi gradient is the derivative of the cost; the tau gradient differs from it by exactly the quirk term
    w (c_i - 1) alpha (g . v) dT/dtau of piece i + 1 (the reference multiplies the T entry by the cost)"""
    for N in (3, 8):
        head, tail, Q = M.problem(N, 77 + N)
        rng = np.random.default_rng(N)
        x = M.start_point(N, Q)
        x[:N] += rng.normal(size=N) * 0.2
        x[N:] += rng.normal(size=3 * (N - 1)) * 0.3
        me = M.HostMidEnd(head, tail, Q)
        c, g = me.cost(x)
        fd = np.zeros_like(x)
        for j in range(x.size):
            h = 1e-6 * max(1.0, abs(x[j]))
            xp, xm = x.copy(), x.copy()
            xp[j] += h; xm[j] -= h
            fd[j] = (me.cost(xp)[0] - me.cost(xm)[0]) / (2 * h)
        scale = np.max(np.abs(fd))
        assert np.max(np.abs(g[N:] - fd[N:])) <= 1e-5 * scale, N
        import host_lib as H
        T = M.forwardT(x[:N])
        co, _, _, _ = H.minco_forward(head, tail, x[N:].reshape(N - 1, 3).T, T)
        terms = M.pose_terms(N, T, co, Q, 64, 1000.0)
        quirk = np.zeros(N)
        for seg, (wc, gv, c3) in enumerate(terms, start=1):
            quirk[seg] = 1000.0 * (c3 - 1.0) * gv
        predicted = quirk * M.dT_dtau(x[:N])
        assert np.max(np.abs(predicted)) > 1e-3 * scale                                  # the quirk is visible ...
        assert np.max(np.abs((g[:N] - fd[:N]) - predicted)) <= 1e-5 * max(scale, np.max(np.abs(predicted))), N   # ... and exactly it


def test_zero_offset_adds_nothing():
    """waypoints set to the positions the trajectory evaluates to at s: d = 0 exactly, so the pose term contributes nothing — cost and
    gradient equal those of weight 0"""
    import host_lib as H
    N = 6
    head, tail, Q = M.problem(N, 3)
    x = M.start_point(N, Q)
    x[:N] += np.linspace(-0.3, 0.4, N)
    T = M.forwardT(x[:N])
    co, _, _, _ = H.minco_forward(head, tail, x[N:].reshape(N - 1, 3).T, T)
    Qz = M.positions_at_s(N, T, co, 64)
    assert all(t == (0.0, 0.0, 0.0) for t in M.pose_terms(N, T, co, Qz, 64, 1000.0))
    c, g = M.HostMidEnd(head, tail, Qz).cost(x)
    c0, g0 = M.HostMidEnd(head, tail, Qz, weight=0.0).cost(x)
    assert c == c0 and np.array_equal(g, g0)


def _lbfgs_cases():
    cases = [("stop", 3, 11, {}), ("stop", 8, 12, {}), ("stop", 17, 13, {}), ("cancel", 8, 14, {"cancel_after": 5})]
    return cases


def _ref_run(k, me, x0, kw):
    if REF:
        return O.RefLbfgs().minimize(me.cost, x0, **kw)
    zl = np.load(GOLD)
    return {"ret": int(zl[f"lb{k}_ret"]), "evaluations": int(zl[f"lb{k}_evals"]), "trace_sha256": str(zl[f"lb{k}_trace_sha256"]), "x": zl[f"lb{k}_x"],
            "f": float(zl[f"lb{k}_f"])}


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def test_lbfgs_drivers_against_reference_compiled_lbfgs():
    """the reference's own lbfgs.hpp (oracle/_ref/libref_lbfgs.so) run on the product's host cost visits the same points, in order, as the
    product's sequential driver, and getOriTraj (the same driver with earlyExit) returns the same solution, value, code and counts. The reference
    build has no progress callback, so a cancelled run (k > cancel_after, cancel_after < past: the delta test cannot fire first) is pinned
    against its max_iterations = cancel_after + 1 stop, which breaks at the same k after the same evaluations; only the code differs
    (LBFGS_CANCELED here, LBFGSERR_MAXIMUMITERATION there). A NaN waypoint ends both at the first line search with the same code."""
    import host_lib as H
    stops = 0
    for k, (kind, N, seed, extra) in enumerate(_lbfgs_cases() + [("nan", 4, 15, {})]):
        head, tail, Q = M.problem(N, seed)
        if kind == "nan":
            Q = Q.copy(); Q[1, 2] = np.nan
        cancel = extra.get("cancel_after", 8000)
        me = M.HostMidEnd(head, tail, Q, cancel_after=cancel)
        x0 = M.start_point(N, Q)
        kw = dict(M.LB)
        if kind == "cancel":
            kw["max_iterations"] = cancel + 1
        a = _ref_run(k, me, x0, kw)
        b = me.optimize()
        if kind == "cancel":
            assert b["ret"] == M.LBFGS_CANCELED and a["ret"] == M.LBFGSERR_MAXIMUMITERATION and b["iterations"] == cancel + 1
        else:
            assert a["ret"] == b["ret"], (kind, N, a["ret"], b["ret"])
        stops += b["ret"] == M.LBFGS_STOP
        assert a["evaluations"] == b["evaluations"], (kind, N)
        assert _same(a["x"], b["x"]) and _same(a["f"], b["f"]), (kind, N)
        if kind != "cancel":   # every evaluated point: the product's sequential driver without a progress callback
            c = H.lbfgs_minimize(lambda x: me.cost(x), x0, **{q: v for q, v in kw.items() if q != "min_step"})
            if "trace" in a:
                assert len(c["trace"]) == len(a["trace"]) and all(_same(p, q) for p, q in zip(a["trace"], c["trace"])), (kind, N)
            else:
                assert M.trace_digest(c["trace"]) == a["trace_sha256"], (kind, N)
        if kind == "nan":
            assert b["ret"] == M.LBFGSERR_INVALIDPARAMETERS and np.isnan(b["f"])
    assert stops >= 3


def test_lockstep_host_driver_cancel_rule_equals_sequential():
    """the lock-step batched host driver with pr.cancel_after gives every instance the sequential getOriTraj result: a batch mixing plans
    that stop and one cancelled after 7 iterations"""
    mids, X0, seq = [], [], []
    for k, seed in enumerate((21, 22, 23)):
        head, tail, Q = M.problem(5, seed)
        me = M.HostMidEnd(head, tail, Q, cancel_after=7 if k == 1 else 8000)
        mids.append(me); X0.append(M.start_point(5, Q)); seq.append(me.optimize())
    # the lock-step driver takes one cancel_after for the batch: run the cancelled instance in its own batch
    a = M.HostMidEnd.lockstep([mids[0], mids[2]], [X0[0], X0[2]], 8000)
    b = M.HostMidEnd.lockstep([mids[1]], [X0[1]], 7)
    for q, (res, i) in enumerate(((a, 0), (a, 1), (b, 0))):
        s = seq[(0, 2, 1)[q]]
        assert res["ret"][i] == s["ret"] and res["iterations"][i] == s["iterations"] and res["evaluations"][i] == s["evaluations"]
        assert np.array_equal(res["x"][i], s["x"]) and res["f"][i] == s["f"]
    assert b["ret"][0] == M.LBFGS_CANCELED and b["iterations"][0] == 8


def test_midend_params_defaults_and_layout():
    import ctypes as C
    lib = I.load_library()
    p = I.MidendParams()
    assert lib.isdf_midend_default_params(C.byref(p)) == 0 and lib.isdf_midend_default_params(None) == -1
    assert (p.weight_pr, p.rho, p.init_time, p.cancel_after, p.reserved_) == (1000.0, 200.0, 2.5, 8000, 0)
    assert (p.lbfgs.mem_size, p.lbfgs.past, p.lbfgs.max_iterations, p.lbfgs.g_epsilon, p.lbfgs.delta, p.lbfgs.min_step) == (16, 10, 100000, 0.0, 1e-6, 1e-32)
    assert C.sizeof(I.MidendParams) == 112
    # argument checks run before any device call
    x, g, cost = np.zeros(5), np.zeros(5), np.zeros(1)
    dp = C.POINTER(C.c_double)
    assert lib.isdf_midend_callback_batch(None, 1, 2, None, None, 0, C.byref(p), None, x.ctypes.data_as(dp), cost.ctypes.data_as(dp),
                                          g.ctypes.data_as(dp)) == -1 and np.isnan(cost[0])
