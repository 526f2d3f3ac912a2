"""The planning step (isdf_plan_batch): every output bit-identical to the composition of the public calls on a fresh context, each goal
alone equal to the batch (also past 300 s, where the durations rule matters), one test per stage, the error paths and the state the call
leaves behind."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
from common import MESHES

pytestmark = pytest.mark.gpu


def _cfg(ks=11):
    cfg = I.default_config_values()
    cfg.integral_intervs, cfg.kernel_size = 16, ks
    return cfg


def _ev(robot, occ, cfg=None, kernels=True):
    ev = I.Evaluator(cfg or _cfg())
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0.1, 0.0, -0.1, 120.0, 10.0, 0.0])
    else:
        ev.set_shape_named(robot)
    if kernels:
        ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    return ev


def _scene(n_goals, seed=5):
    occ = W.three_slit_map(48, 48, 48, noise=0.01, seed=4)
    free = np.argwhere(occ == 0)
    rng = np.random.default_rng(seed)
    start = free[np.argmin(np.abs(free - [4, 4, 24]).sum(1))] + 0.5
    goals = free[rng.choice(len(free), n_goals, replace=False)] + 0.5
    return occ, start, goals


def _params(ev, **kw):
    kw.setdefault("backend_max_iterations", 60)
    return ev.plan_params(**kw)


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _summ_same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return all(_same(a[k], b[k]) for k in a)


def _compose(ev, start, goals, p):
    """the public calls of include/isdf.h's definition, one stage at a time"""
    B = len(goals)
    fp = ev.frontend_path_batch(start, goals)
    wps, pieces = I.path_waypoints(fp["paths"], ev.map_info()["res"], p.parlength)
    out = [dict(stage=I.NO_PATH if not fp["found"][b] else I.TOO_LONG, path=fp["paths"][b], pieces=int(pieces[b]) if fp["found"][b] else 0,
                obstacle_points=0, midend_ret=0, backend_ret=0, backend_iterations=0, backend_evaluations=0, path_cost=fp["costs"][b],
                midend_f=np.nan, backend_f=np.nan, duration=0.0, T=np.zeros(0), coeffs=np.zeros(0), certify=None, dynamics=None)
           for b in range(B)]
    Ns = sorted({int(pieces[b]) for b in range(B) if fp["found"][b] and pieces[b] <= 290})
    for N in Ns:
        idx = [b for b in range(B) if fp["found"][b] and pieces[b] == N]
        Bg = len(idx)
        head, tail = np.zeros((Bg, 3, 3)), np.zeros((Bg, 3, 3))
        for q, b in enumerate(idx):
            head[q, :, 0], tail[q, :, 0] = fp["paths"][b][0], fp["paths"][b][-1]
        wp = np.array([wps[b] for b in idx]).reshape(Bg, N - 1, 3)
        m = ev.midend_batch(head, tail, wp, p.midend)
        ok = [q for q in range(Bg) if m["ret"][q] >= 0]
        Tg, Cg = m["T"].reshape(Bg, N).copy(), m["coeffs"].reshape(3, Bg, 6 * N).copy()
        for q, b in enumerate(idx):
            out[b].update(stage=I.MIDEND_FAILED, midend_f=m["f"][q], midend_ret=m["ret"][q])
        if ok:
            lists = [ev.gather_obstacle_points(wp[q], p.half_extent, p.offset)[0] if N > 1 else np.zeros((0, 3)) for q in ok]
            ev.set_points_batch(lists if sum(len(x) for x in lists) else [])
            be = ev.lbfgs_batch(head[ok], tail[ok], p.rho, m["x"][ok], p.backend)
            ev.callback_batch(head[ok], tail[ok], p.rho, be["x"])
            T, Cc, _ = ev.batch_trajectories(len(ok), N)
            for k, q in enumerate(ok):
                Tg[q], Cg[:, q, :] = T.reshape(-1, N)[k], Cc.reshape(3, -1, 6 * N)[:, k, :]
                out[idx[q]].update(stage=I.OPTIMISED, obstacle_points=len(lists[k]), backend_f=be["f"][k], backend_ret=be["ret"][k],
                                   backend_iterations=be["iterations"][k], backend_evaluations=be["evaluations"][k])
        cs = ds = [None] * Bg
        if p.flags & I.PLAN_CERTIFY:
            c = p.certify
            cs = ev.trajectory_certify(Tg.reshape(-1), Cg.reshape(-1), c.clearance.samples_per_piece, c.clearance.reach, c.clearance.margin, N0=N,
                                       max_depth=c.max_depth, max_samples=c.max_samples_per_traj)
        if p.flags & I.PLAN_DYNAMICS:
            pd = I.DynamicsParams.from_buffer_copy(p.dynamics)
            pd.pieces_per_traj = N
            ds = ev.trajectory_dynamics(Tg.reshape(-1), Cg.reshape(-1), pd)
        for q, b in enumerate(idx):
            td = 0.0
            for t in Tg[q]:
                td += t
            out[b].update(T=Tg[q], coeffs=Cg[:, q, :].reshape(-1), duration=td, certify=cs[q], dynamics=ds[q])
    return out


def _check_plan(got, ref, b):
    for k in ("stage", "pieces", "obstacle_points", "midend_ret", "backend_ret", "backend_iterations", "backend_evaluations", "path_cost",
              "midend_f", "backend_f", "duration", "path", "T", "coeffs"):
        assert _same(got[k], ref[k]), (b, k, got[k], ref[k])
    assert got["path_nodes"] == len(ref["path"])
    for k in ("certify", "dynamics"):
        if ref[k] is None and got[k] is not None:         # no trajectory: the certificate's failed-call summary
            assert ref["T"].size == 0 and got[k]["verdict"] == 0 and got[k]["samples"] == -1, (b, k)
        else:
            assert _summ_same(got[k], ref[k]), (b, k)


@pytest.mark.parametrize("robot", ["Ball", "mesh"])
def test_plan_equals_the_public_call_composition(robot):
    occ, start, goals = _scene(12)
    ev = _ev(robot, occ)
    p = _params(ev)
    got, info = ev.plan_batch(start, goals, p)
    again, _ = ev.plan_batch(start, goals, p)                     # run to run
    ev.close()
    fresh = _ev(robot, occ)
    ref = _compose(fresh, start, goals, p)
    fresh.close()
    assert max(r["duration"] for r in ref) < 300.0
    assert sum(r["stage"] == I.OPTIMISED for r in got) >= 2 and info["groups"] >= 1 and info["backend_rounds"] > 0
    assert sum(r["obstacle_points"] for r in got) > 0
    for b in range(len(goals)):
        _check_plan(got[b], ref[b], b)
        _check_plan(again[b], got[b], b)
    assert all(v >= 0 for k, v in info.items() if k.endswith("_ms"))
    print(robot, "stages", [r["stage"] for r in got], "N", [r["pieces"] for r in got], "info", info)


def test_each_goal_alone_equals_the_batch_past_300_s():
    occ, start, goals = _scene(8, seed=9)
    ev = _ev("Ball", occ)
    # long pieces, a mid-end stopped early by its cancel rule (a success, so the back end runs) and a small time weight
    p = _params(ev, midend_init_time=200.0, midend_rho=1e-3, midend_cancel_after=3, rho=1e-3, backend_max_iterations=30)
    got, _ = ev.plan_batch(start, goals, p)
    assert max(r["duration"] for r in got if r["stage"] == I.OPTIMISED) >= 300.0, [(r["stage"], r["duration"]) for r in got]
    perm = np.random.default_rng(1).permutation(len(goals))
    shuffled, _ = ev.plan_batch(start, goals[perm], p)
    for k, b in enumerate(perm):
        _check_plan(shuffled[k], got[b], b)
    for b in range(len(goals)):
        alone, _ = ev.plan_batch(start, goals[b:b + 1], p)
        _check_plan(alone[0], got[b], b)
    ev.close()


def test_no_path():
    occ, start, goals = _scene(2)
    occ = occ.copy()
    occ[30:35, 30:35, 30:35] = 1
    occ[31:34, 31:34, 31:34] = 0                                 # a free pocket no path reaches
    ev = _ev("Ball", occ)
    got, _ = ev.plan_batch(start, np.array([[32.5, 32.5, 32.5], goals[0]]), _params(ev))
    assert got[0]["stage"] == I.NO_PATH and got[0]["pieces"] == 0 and got[0]["T"].size == 0 and got[0]["path_nodes"] == 1
    assert np.isinf(got[0]["path_cost"]) and got[0]["certify"]["verdict"] == 0 and np.isnan(got[0]["certify"]["lower_bound"])
    assert got[1]["stage"] in (I.OPTIMISED, I.MIDEND_FAILED)
    ev.close()


def test_goal_equal_to_start():
    occ, start, _ = _scene(1)
    ev = _ev("Ball", occ)
    got, _ = ev.plan_batch(start, start[None], _params(ev))
    g = got[0]
    assert g["path_nodes"] == 1 and g["pieces"] == 1 and g["obstacle_points"] == 0 and g["T"].size == 1 and g["coeffs"].size == 18
    assert g["stage"] in (I.OPTIMISED, I.MIDEND_FAILED)
    ev.close()


def test_too_long():
    occ = np.zeros((300, 3, 3), dtype=np.uint8)                  # a corridor: the shortest path is the straight line of 299 voxels
    ev = _ev("Ball", occ, _cfg(ks=5))
    got, info = ev.plan_batch([0.5, 1.5, 1.5], [[298.5, 1.5, 1.5], [20.5, 1.5, 1.5]], _params(ev, parlength=1.0))
    assert got[0]["stage"] == I.TOO_LONG and got[0]["pieces"] > 290 and got[0]["T"].size == 0
    assert got[1]["stage"] in (I.OPTIMISED, I.MIDEND_FAILED) and got[1]["pieces"] == 20 and info["groups"] == 1
    ev.close()


def test_midend_failed_returns_the_midend_trajectory():
    occ, start, goals = _scene(4)
    ev = _ev("Ball", occ)
    p = _params(ev, midend_max_rounds=1)
    got, info = ev.plan_batch(start, goals, p)
    fresh = _ev("Ball", occ)
    ref = _compose(fresh, start, goals, p)
    fresh.close()
    assert info["backend_rounds"] == 0
    for b, g in enumerate(got):
        if g["stage"] == I.NO_PATH:
            continue
        assert g["stage"] == I.MIDEND_FAILED and g["midend_ret"] == -1008 and np.isnan(g["backend_f"]) and g["T"].size == g["pieces"]
        _check_plan(g, ref[b], b)
    ev.close()


def _raw_plan(ev, p, start, goals, cap_nodes=10000, cap_pieces=10000):
    B = len(goals)
    ip = C.POINTER(C.c_int32)
    st, gl = np.ascontiguousarray(start, dtype=np.float64), np.ascontiguousarray(goals, dtype=np.float64)
    pf, po = np.zeros(B + 1, dtype=np.int32), np.zeros(B + 1, dtype=np.int32)
    xyz, T, Cc = np.zeros((max(cap_nodes, 1), 3)), np.zeros(max(cap_pieces, 1)), np.zeros(18 * max(cap_pieces, 1))
    res, cs, ds = (I.PlanResult * B)(), (I.CertifySummary * B)(), (I.DynamicsSummary * B)()
    dp = C.POINTER(C.c_double)
    r = ev.lib.isdf_plan_batch(ev.h, st.ctypes.data_as(dp), B, gl.ctypes.data_as(dp), C.byref(p), cap_nodes, pf.ctypes.data_as(ip),
                               xyz.ctypes.data_as(dp), cap_pieces, po.ctypes.data_as(ip), T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), res, cs, ds)
    return r, pf, po, res, cs, ds


def test_error_paths():
    occ, start, goals = _scene(3)
    ev = _ev("Ball", occ, kernels=False)                        # no front-end kernels
    p = _params(ev)
    r, _, _, res, cs, ds = _raw_plan(ev, p, start, goals)
    assert r == -2 and all(x.stage == -1 and np.isnan(x.midend_f) and np.isnan(x.backend_f) for x in res)
    assert all(s.verdict == 0 and np.isnan(s.lower_bound) for s in cs) and all(s.samples == -1 for s in ds)
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    for field, value, code in (("reserved_", 1, -1), ("flags", 4, -1)):
        q = _params(ev)
        setattr(q, field, value)
        assert _raw_plan(ev, q, start, goals)[0] == code, field
    q = _params(ev)
    q.certify.clearance.pieces_per_traj = 3
    assert _raw_plan(ev, q, start, goals)[0] == -1
    q = _params(ev)
    q.dynamics.pieces_per_traj = 3
    assert _raw_plan(ev, q, start, goals)[0] == -1
    q = _params(ev, midend_init_time=0.0)
    assert _raw_plan(ev, q, start, goals)[0] == -1
    full, _ = ev.plan_batch(start, goals, p)                    # caps too small: the sizes needed are reported
    nodes, pieces = sum(g["path_nodes"] for g in full), sum(g["T"].size for g in full)
    r, pf, po, res, _, _ = _raw_plan(ev, p, start, goals, cap_nodes=nodes - 1)
    assert r == -1 and pf[-1] == nodes and po[-1] == pieces and all(x.stage == -1 for x in res)
    r, pf, po, _, _, _ = _raw_plan(ev, p, start, goals, cap_pieces=pieces - 1)
    assert r == -1 and po[-1] == pieces
    ev.set_shard(0, 2)
    assert _raw_plan(ev, p, start, goals)[0] == -4
    ev.set_shard(0, 1)
    ev.set_shape_named("Torus")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    k0 = ev.stats().kernel_launches
    assert _raw_plan(ev, _params(ev), start, goals)[0] == -4    # the certificate refuses the Torus before any work
    assert ev.stats().kernel_launches == k0
    no_cert = _params(ev, flags=I.PLAN_DYNAMICS)
    got, _ = ev.plan_batch(start, goals, no_cert)
    assert all(g["certify"] is None for g in got)
    ev.close()


def test_state_left_behind():
    occ, start, goals = _scene(4)
    ev = _ev("Ball", occ)
    ev.set_points(np.argwhere(occ)[:50] + 0.5)
    got, _ = ev.plan_batch(start, goals, _params(ev))
    assert any(g["stage"] == I.OPTIMISED for g in got)
    dp = C.POINTER(C.c_double)
    T, Cc = np.ones(2), np.zeros(36)
    assert ev.lib.isdf_eval_swept(ev.h, 2, T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(C.c_double(0.0)), np.zeros(36).ctypes.data_as(dp),
                                  np.zeros(2).ctypes.data_as(dp)) == -2
    import test_gpu_lbfgs_device as L
    heads, tails, X = L.problems(3, 5)
    after = ev.callback_batch(heads, tails, 20.0, X)
    ev.set_points_batch([])
    off = ev.callback_batch(heads, tails, 20.0, X)
    assert np.array_equal(after[0], off[0]) and np.array_equal(after[1], off[1])
    ev.close()
