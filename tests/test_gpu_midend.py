"""The mid-end on the device: isdf_midend_callback_batch and isdf_midend_batch(_device) bit-identical to the host restatement
(host/isdf_midend.hpp) problem by problem, back-end state untouched by mid-end calls, argument errors, the whole generateTraj chain on a map,
and one run against the reference form."""
import os
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import midend_cases as M
from common import small_case, BMIN, MESHES

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "midend_reference.npz")


def _ctx(K=64):
    cfg = I.default_config_values()
    cfg.integral_intervs = K
    return I.Evaluator(cfg)


def _batch(B, N, seed, jitter=0.0):
    heads, tails, Qs = [], [], []
    for b in range(B):
        h, t, Q = M.problem(N, seed + b)
        if jitter:
            h[:, 1] = np.random.default_rng(seed + b).normal(size=3) * jitter
        heads.append(h); tails.append(t); Qs.append(Q.reshape(N - 1, 3))
    return np.array(heads), np.array(tails), np.array(Qs).reshape(B, N - 1, 3)


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("per_problem_bc", [0, 1])
@pytest.mark.parametrize("N0", [1, 2, 3, 8, 33, 64, 290])
def test_callback_equals_host_cost(N0, per_problem_bc):
    ev = _ctx(K=16)
    B = 5
    heads, tails, Q = _batch(B, N0, 40 + N0, jitter=0.3)
    if not per_problem_bc:
        heads[:], tails[:] = heads[0], tails[0]
    rng = np.random.default_rng(N0)
    X = np.array([M.start_point(N0, Q[b]) for b in range(B)])
    X[:, :N0] += rng.normal(size=(B, N0)) * 0.3
    X[:, N0:] += rng.normal(size=(B, 3 * (N0 - 1))) * 0.4
    if N0 > 2:   # problem 1: the zero-offset case — every waypoint where its piece evaluates, so d = 0 exactly
        import host_lib as H
        T = M.forwardT(X[1, :N0])
        co, _, _, _ = H.minco_forward(heads[1], tails[1], X[1, N0:].reshape(N0 - 1, 3).T, T)
        Q[1] = M.positions_at_s(N0, T, co, 16)
    c, g = ev.midend_callback_batch(heads if per_problem_bc else heads[0], tails if per_problem_bc else tails[0], Q, X)
    for b in range(B):
        hc, hg = M.HostMidEnd(heads[b], tails[b], Q[b], K=16).cost(X[b])
        assert c[b] == hc and np.array_equal(g[b], hg), (N0, b)
    if N0 > 2:
        c0, g0 = ev.midend_callback_batch(heads, tails, Q, X, ev.midend_params(weight_pr=0.0))
        assert c[1] == c0[1] and np.array_equal(g[1], g0[1])
    ev.close()


def test_callback_refuses_291_pieces():
    ev = _ctx()
    heads, tails, Q = _batch(1, 291, 3)
    with pytest.raises(I.IsdfError) as e:
        ev.midend_callback_batch(heads[0], tails[0], Q, M.start_point(291, Q[0])[None, :])
    assert e.value.code == -4
    ev.close()


def _host_runs(heads, tails, Q, cancel=8000, K=64):
    out = []
    for b in range(len(heads)):
        me = M.HostMidEnd(heads[b], tails[b], Q[b], K=K, cancel_after=cancel)
        out.append(dict(me.optimize(), cost=me.cost))
    return out


def _check_against_host(dev, host, N0):
    T = dev["T"].reshape(-1, N0)
    Cc = dev["coeffs"].reshape(3, -1, 6 * N0)
    for b, h in enumerate(host):
        assert dev["ret"][b] == h["ret"] and dev["iterations"][b] == h["iterations"] and dev["evaluations"][b] == h["evaluations"], b
        assert _same(dev["x"][b], h["x"]), b
        if h["ret"] == M.LBFGSERR_INVALID_FUNCVAL and np.isnan(h["f"]) and not np.isnan(dev["f"][b]):
            assert dev["f"][b] == h["cost"](dev["x"][b])[0], b     # the direction-norm exit: f is the cost at x (include/isdf.h)
        else:
            assert _same(dev["f"][b], h["f"]), b
        assert _same(T[b], h["T"]) and _same(Cc[:, b, :].reshape(-1), h["coeffs"]), b


@pytest.mark.parametrize("B,N0", [(1, 8), (37, 5), (1024, 3)])
def test_midend_batch_equals_sequential_host_driver(B, N0):
    ev = _ctx()
    heads, tails, Q = _batch(B, N0, 1000)
    if B >= 37:
        Q[3, 1, 0] = np.nan                                    # a NaN instance stops alone; the others are unchanged
    dev = ev.midend_batch(heads, tails, Q)
    _check_against_host(dev, _host_runs(heads, tails, Q), N0)
    if B >= 37:
        assert np.isnan(dev["f"][3]) and dev["ret"][3] < 0 and np.all(np.isfinite(np.delete(dev["f"], 3)))
        alone = ev.midend_batch(heads[5:6], tails[5:6], Q[5:6])            # one problem alone == inside the batch
        assert _same(alone["x"][0], dev["x"][5]) and alone["ret"][0] == dev["ret"][5] and alone["evaluations"][0] == dev["evaluations"][5]
    assert dev["rounds"] >= dev["evaluations"].max()
    print(f"B={B} N0={N0}: rounds {dev['rounds']}, iterations mean {dev['iterations'].mean():.1f} max {dev['iterations'].max()}, "
          f"ret {dict(zip(*np.unique(dev['ret'], return_counts=True)))}")
    ev.close()


def test_midend_cancel_and_device_entry_point():
    import torch
    ev = _ctx()
    B, N0 = 6, 6
    heads, tails, Q = _batch(B, N0, 77)
    p = ev.midend_params(cancel_after=4)
    dev = ev.midend_batch(heads, tails, Q, p)
    _check_against_host(dev, _host_runs(heads, tails, Q, cancel=4), N0)
    assert np.all(dev["ret"] == M.LBFGS_CANCELED) and np.all(dev["iterations"] == 5)
    # the device entry point on a side stream: the same bits
    dv = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2)).reshape(-1)
    d_h, d_t, d_q = dv(cm(heads)), dv(cm(tails)), dv(Q.reshape(-1))
    d_x, d_T, d_C, d_f = (torch.zeros(n, dtype=torch.float64, device="cuda") for n in (B * (4 * N0 - 3), B * N0, 18 * B * N0, B))
    d_i = torch.zeros(3 * B, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        rounds = ev.midend_batch_device(B, N0, d_h.data_ptr(), d_t.data_ptr(), 1, d_q.data_ptr(), d_x.data_ptr(), d_T.data_ptr(), d_C.data_ptr(),
                                        d_f.data_ptr(), d_i.data_ptr(), d_i.data_ptr() + 4 * B, d_i.data_ptr() + 8 * B, p, s.cuda_stream)
    s.synchronize()
    i = d_i.cpu().numpy()
    assert rounds == dev["rounds"] and np.array_equal(d_x.cpu().numpy().reshape(B, -1), dev["x"]) and np.array_equal(d_f.cpu().numpy(), dev["f"])
    assert np.array_equal(d_T.cpu().numpy(), dev["T"].reshape(-1)) and np.array_equal(d_C.cpu().numpy(), dev["coeffs"])
    assert np.array_equal(i[:B], dev["ret"]) and np.array_equal(i[B:2 * B], dev["iterations"]) and np.array_equal(i[2 * B:], dev["evaluations"])
    ev.close()


def test_midend_leaves_back_end_state_alone():
    """a back-end callback / lbfgs sequence with swept point sets gives the same bits with and without mid-end calls in between, and
    isdf_get_batch_trajectories and every stats field but kernel_launches are unchanged by them"""
    cfg, occ, _, _, _ = small_case(N=6, K=16, seed=3)
    import test_gpu_lbfgs_device as L
    heads, tails, X = L.problems(4, 5)
    hM, tM, QM = _batch(3, 7, 900)

    def run(with_mid):
        ev = I.Evaluator(cfg)
        ev.set_map_u8(occ, BMIN, 1.0)
        ev.set_shape_named("Ball")
        ev.set_points_batch([np.asarray(occ.nonzero(), float).T[:40] + 0.5 + k for k in range(4)])
        out = [ev.callback_batch(heads, tails, 20.0, X)]
        if with_mid:
            traj, st = ev.batch_trajectories(4, 5), ev.stats()
            ev.midend_batch(hM, tM, QM)
            ev.midend_callback_batch(hM, tM, QM, np.array([M.start_point(7, QM[b]) for b in range(3)]))
            traj2, st2 = ev.batch_trajectories(4, 5), ev.stats()
            assert all(np.array_equal(a, b) for a, b in zip(traj, traj2))
            assert st2.kernel_launches > st.kernel_launches
            for f, _ in I.Stats._fields_:
                if f != "kernel_launches":
                    assert getattr(st, f) == getattr(st2, f), f
        out.append(ev.lbfgs_batch(heads, tails, 20.0, X, ev.lbfgs_params(max_iterations=6, mem_size=8, past=3)))
        out.append(ev.callback_batch(heads, tails, 20.0, out[-1]["x"]))
        out.append(ev.batch_trajectories(4, 5))
        ev.close()
        return out
    a, b = run(False), run(True)
    assert np.array_equal(a[0][0], b[0][0]) and np.array_equal(a[0][1], b[0][1])
    for k in ("x", "f", "ret", "iterations", "evaluations", "rounds"):
        assert _same(a[1][k], b[1][k]), k
    assert np.array_equal(a[2][0], b[2][0]) and np.array_equal(a[2][1], b[2][1])
    assert all(np.array_equal(p, q) for p, q in zip(a[3], b[3]))


def test_midend_argument_errors():
    import ctypes as C
    ev = _ctx()
    lib, dp = ev.lib, C.POINTER(C.c_double)
    heads, tails, Q = _batch(2, 4, 5)
    X = np.array([M.start_point(4, Q[b]) for b in range(2)])
    reserved = ev.midend_params()
    reserved.reserved_ = 1
    bad = [reserved, ev.midend_params(init_time=0.0), ev.midend_params(weight_pr=float("nan")), ev.midend_params(cancel_after=-1),
           ev.midend_params(mem_size=0)]
    for p in bad:
        with pytest.raises(I.IsdfError) as e:
            ev.midend_callback_batch(heads, tails, Q, X, p)
        assert e.value.code == -1
        with pytest.raises(I.IsdfError):
            ev.midend_batch(heads, tails, Q, p)
    cost, g, f = np.zeros(2), np.zeros(X.size), np.zeros(2)
    h, t = np.zeros(18), np.zeros(18)
    p = ev.midend_params()
    assert lib.isdf_midend_callback_batch(ev.h, 0, 4, h.ctypes.data_as(dp), t.ctypes.data_as(dp), 1, C.byref(p), None, None, cost.ctypes.data_as(dp), None) == -1
    assert lib.isdf_midend_callback_batch(ev.h, 2, 4, h.ctypes.data_as(dp), t.ctypes.data_as(dp), 1, C.byref(p), None, X.ctypes.data_as(dp),
                                          cost.ctypes.data_as(dp), g.ctypes.data_as(dp)) == -1 and np.all(np.isnan(cost))
    assert lib.isdf_midend_batch(ev.h, 2, 4, h.ctypes.data_as(dp), t.ctypes.data_as(dp), 1, C.byref(p), None, X.ctypes.data_as(dp), None, None,
                                 f.ctypes.data_as(dp), None, None, None, None) == -1 and np.all(np.isnan(f))
    assert lib.isdf_midend_batch(ev.h, 2, 4, h.ctypes.data_as(dp), t.ctypes.data_as(dp), 1, None, Q.ctypes.data_as(dp), X.ctypes.data_as(dp), None,
                                 None, f.ctypes.data_as(dp), None, None, None, None) == -1
    lib.isdf_set_shard(ev.h, 0, 2)
    f[:] = 0
    assert lib.isdf_midend_batch(ev.h, 2, 4, h.ctypes.data_as(dp), t.ctypes.data_as(dp), 1, C.byref(p), Q.ctypes.data_as(dp), X.ctypes.data_as(dp),
                                 None, None, f.ctypes.data_as(dp), None, None, None, None) == -2 and np.all(np.isnan(f))
    ev.close()


@pytest.mark.parametrize("robot", ["Ball", "mesh"])
def test_generate_traj_chain_end_to_end(robot):
    """frontend_path_batch (one start, 8 goals) -> waypoints -> mid-end per N group -> gather_obstacle_points (half = bd/3) ->
    set_points_batch -> lbfgs_batch from the mid-end x; every stage equals its standalone call and every cost is finite"""
    import workloads as W
    cfg = I.default_config_values()
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    cfg.integral_intervs, cfg.kernel_size = 16, 5
    occ = W.three_slit_map(48, 48, 48, noise=0.01, seed=4)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0.1, 0.0, -0.1, 120.0, 10.0, 0.0])
    else:
        ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    free = np.argwhere(occ == 0)
    rng = np.random.default_rng(5)
    start = free[np.argmin(np.abs(free - [4, 4, 24]).sum(1))] + 0.5
    goals = free[rng.choice(len(free), 8, replace=False)] + 0.5
    fp = ev.frontend_path_batch(start, goals)
    found = np.flatnonzero(fp["found"])
    assert found.size >= 1, fp["found"]
    fp = {k: ([v[b] for b in found] if isinstance(v, list) else v) for k, v in fp.items()}
    groups = ev.midend_from_paths(fp)
    half = cfg.kernel_size * cfg.occupancy_resolution / 3.0
    report = []
    for g in groups:
        alone = ev.midend_batch(g["head"], g["tail"], g["waypoints"])
        for k in ("x", "f", "ret", "iterations", "evaluations", "T", "coeffs"):
            assert _same(alone[k], g[k]), k
        assert np.all(np.isfinite(g["f"]))
        pts = [ev.gather_obstacle_points(g["waypoints"][q], half)[0] if g["N"] > 1 else np.zeros((0, 3)) for q in range(len(g["idx"]))]
        ok = [q for q in range(len(g["idx"])) if g["ret"][q] >= 0]          # plan_manager.cpp:277: the back end runs only on success
        if not ok:
            continue
        sel = lambda a: np.asarray(a)[ok]
        ev.set_points_batch([pts[q] if len(pts[q]) else np.asarray(g["waypoints"][q][:1]) for q in ok])
        c0, _ = ev.callback_batch(sel(g["head"]), sel(g["tail"]), 20.0, sel(g["x"]))
        be = ev.lbfgs_batch(sel(g["head"]), sel(g["tail"]), 20.0, sel(g["x"]), ev.lbfgs_params(max_iterations=20))
        assert np.all(np.isfinite(c0)) and np.all(np.isfinite(be["f"]))
        T, Cc, _ = ev.batch_trajectories(len(ok), g["N"])
        _, _, summ = ev.trajectory_clearance(T, Cc, 4, 2.0, cfg.safety_hor, N0=g["N"])
        report.append((g["N"], len(ok), [round(s["min_clearance"], 3) for s in summ]))
        ev.set_points_batch([])
    print("generateTraj chain (N, plans, min clearance):", report)
    ev.close()


def test_midend_against_reference_form():
    """one whole getOriTraj against the reference form (reference-compiled MINCO, lbfgs.hpp and pow): same sign of the return code, final cost
    within 1e-4 relative; the iterations and the largest waypoint difference are reported"""
    head, tail, Q = M.ref_run_problem()
    N = len(Q) + 1
    if os.path.exists(O.REF_MINCO) and os.path.exists(O.REF_LBFGS):
        r = M.ref_form_optimize(O.RefMinco(), O.RefLbfgs(), head, tail, Q)
    else:
        z = np.load(GOLD)
        r = dict(ret=int(z["run_ret"]), f=float(z["run_f"]), x=z["run_x"], evaluations=int(z["run_evals"]))
    ev = _ctx()
    dev = ev.midend_batch(head[None], tail[None], Q[None])
    assert (dev["ret"][0] >= 0) == (r["ret"] >= 0)
    assert abs(dev["f"][0] - r["f"]) <= 1e-4 * abs(r["f"])
    print(f"mid-end vs reference form: ret {dev['ret'][0]} / {r['ret']}, iterations {dev['iterations'][0]}, evaluations {dev['evaluations'][0]} / "
          f"{r['evaluations']}, f rel {abs(dev['f'][0] - r['f']) / abs(r['f']):.2e}, max waypoint diff {np.abs(dev['x'][0][N:] - r['x'][N:]).max():.3e}")
    ev.close()
