"""Dynamic-limit certificate (isdf_trajectory_dynamics) on the GPU: soundness against dense reference values, violations between the back
end's samples that its penalty misses, the other verdicts, agreement with the serial restatement (tests/dynlimits_oracle.py), the thrust
against the reference-compiled FlatnessMap::forward, bit identity (run to run, both entry points, alone vs batch, after the device L-BFGS),
refusals and state isolation."""
import ctypes as C
import math
import os
import sys
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
import dynlimits_oracle as DO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "flat_forward_reference.npz")


def cubic_peak():
    """max over [0, 0.5] of t (t - 0.5) (t - 1), at t = 0.5 - sqrt(1/12)"""
    t = 0.5 - math.sqrt(1.0 / 12.0)
    return t, t * (t - 0.5) * (t - 1.0)


def speed_bump(V0, A):
    """one piece, T = 1: v_x = V0 + A t (t - 0.5) (t - 1), at rest in y and z; x = V0 t + A (t^4/4 - t^3/2 + t^2/4)"""
    c = np.zeros((3, 6))
    c[0, 1], c[0, 2], c[0, 3], c[0, 4] = V0, 0.25 * A, -0.5 * A, 0.25 * A
    c[2, 0] = 5.0
    return np.array([1.0]), c.reshape(-1)


def jerk_bump(B, T):
    """one piece of duration T: j_y = B t (t - T), zero at both ends and B T^2 / 4 in the middle; |a| stays below B T^3 / 6"""
    c = np.zeros((3, 6))
    c[1, 4], c[1, 5] = -B * T / 24.0, B / 60.0
    c[2, 0] = 5.0
    return np.array([T]), c.reshape(-1)


def dense_extrema(cfg, T, Cc, n=2001):
    """per quantity max (and thrust min) over n times per piece, from the reference values"""
    mx, tmin = np.full(5, -np.inf), np.inf
    for i in range(len(T)):
        vals, _ = DO.dense(cfg, T, Cc, i, np.linspace(0.0, T[i], n))
        mx = np.fmax(mx, np.nanmax(vals, axis=0))
        tmin = min(tmin, np.nanmin(vals[:, 4]))
    return mx, tmin


def random_trajs(count, seed):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        n = int(rng.choice([1, 2, 5, 16, 64]))
        T, Cc, _ = W.make_trajectory(n, [0, 0, 0], [30, 30, 20], seed=int(rng.integers(1 << 30)), piece_time=float(rng.uniform(0.4, 2.5)), jitter=0.3)
        out.append((T, Cc))
    return out


def aggressive_trajs():
    g = 9.8
    out = []
    c = np.zeros((3, 6)); c[0, 2] = 0.5 * g * math.tan(math.radians(80.0)); c[0, 3] = 40.0; c[1, 3] = -30.0; c[2, 1] = 1.0
    out.append((np.array([0.25]), c.reshape(-1)))
    rng = np.random.default_rng(3)
    for k in range(3):
        c = rng.normal(0, 1, (3, 6)) * np.array([5, 4, 3, 2, 1.5, 1.0])
        out.append((np.array([0.6 + 0.2 * k]), c.reshape(-1)))
    return out


def batch_of(trajs):
    N0 = max(len(T) for T, _ in trajs)
    Ts, Cs = [], []
    for T, Cc in trajs:
        n = len(T)
        c = np.asarray(Cc).reshape(3, 6 * n)
        if n < N0:   # pad with hover pieces at the last position
            pad = np.zeros((3, 6 * (N0 - n)))
            Tp = np.full(N0 - n, 0.5)
            T = np.concatenate([T, Tp]); c = np.concatenate([c, pad], axis=1)
        Ts.append(T); Cs.append(c)
    return np.concatenate(Ts), np.concatenate(Cs, axis=1).reshape(-1), N0


def cfg_of(drag=True, veps=1e-4, K=64):
    cfg = I.default_config_values()
    if not drag:
        cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
    cfg.speed_eps = veps
    cfg.integral_intervs = K
    return cfg


@pytest.mark.parametrize("drag,veps", [(True, 1e-4), (False, 1e-4), (True, 0.0)])
def test_bounds_enclose_dense_extrema(drag, veps):
    cfg = cfg_of(drag, veps)
    ev = I.Evaluator(cfg, device=0)
    for T, Cc in random_trajs(6, seed=5 + int(drag)) + aggressive_trajs():
        s = ev.trajectory_dynamics(T, Cc, K=8, max_depth=20, max_samples=4000)[0]
        mx, tmin = dense_extrema(cfg, T, Cc)
        toff = np.concatenate([[0.0], np.cumsum(T)[:-1]])
        for q in range(5):
            # attained: the reference value at the attained time itself (it need not lie on the dense grid)
            i = int(np.searchsorted(toff, s["t_attained"][q], side="right") - 1)
            at, _ = DO.dense(cfg, T, Cc, i, np.array([s["t_attained"][q] - toff[i]]))
            if q == 3:
                assert s["upper"][3] >= mx[3] - 1e-7 and s["attained"][3] <= at[0, 3] + 1e-7
                continue
            tol = 1e-9 * max(1.0, mx[q])
            assert s["upper"][q] >= mx[q] - tol, (q, s["upper"][q], mx[q])
            assert s["attained"][q] <= at[0, q] + tol, (q, s["attained"][q], at[0, q])
        assert s["thrust_lower"] <= tmin + 1e-9 * max(1.0, abs(tmin)) and s["thrust_lower"] <= s["thrust_attained_min"]
        i = int(np.searchsorted(toff, s["t_thrust_attained_min"], side="right") - 1)
        at, _ = DO.dense(cfg, T, Cc, i, np.array([s["t_thrust_attained_min"] - toff[i]]))
        assert s["thrust_attained_min"] >= at[0, 4] - 1e-9 * max(1.0, abs(at[0, 4]))
        assert np.all(s["attained"] <= s["upper"])
    ev.close()


def test_speed_violation_between_samples():
    cfg = cfg_of(K=2)
    cfg.flags = I.WITH_DYNAMICS
    tpk, bump = cubic_peak()
    T, Cc = speed_bump(9.5, 30.0)                 # |v| = 9.5 at the three samples, 9.5 + 30 * 0.0481 = 10.94 at t = 0.211
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(np.zeros((16, 16, 16), np.uint8), [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    cost, _, _ = ev.eval_discrete(T, Cc)
    assert cost == 0.0
    s = ev.trajectory_dynamics(T, Cc)[0]
    assert s["verdict"] == I.VIOLATING and s["violated"] & 1
    assert 0.0 < s["t_attained"][0] < 0.5 and abs(s["t_attained"][0] - tpk) < 0.02
    assert s["attained"][0] > cfg.vmax and s["upper"][0] >= 9.5 + 30.0 * bump
    ev.close()


def test_body_rate_violation_between_samples():
    cfg = cfg_of(K=1)
    cfg.flags = I.WITH_DYNAMICS
    Tp = 0.04
    T, Cc = jerk_bump(-600.0 / Tp ** 2, Tp)       # j_y = 0 at both samples, 150 m/s^3 in the middle, |a| <= 4 m/s^2
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(np.zeros((16, 16, 16), np.uint8), [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    cost, _, _ = ev.eval_discrete(T, Cc)
    assert cost == 0.0
    s = ev.trajectory_dynamics(T, Cc)[0]
    mx, _ = dense_extrema(cfg, T, Cc)
    assert mx[2] > cfg.omgmax
    assert s["verdict"] == I.VIOLATING and s["violated"] & 4 and not s["violated"] & 1
    assert 0.25 * Tp < s["t_attained"][2] < 0.75 * Tp and s["attained"][2] > cfg.omgmax
    ev.close()


def test_other_verdicts():
    cfg = cfg_of()
    ev = I.Evaluator(cfg, device=0)
    c = np.zeros((3, 6)); c[:, 0] = [1, 2, 3]; c[0, 2] = 0.1
    s = ev.trajectory_dynamics(np.array([2.0]), c.reshape(-1))[0]
    assert s["verdict"] == I.FEASIBLE and s["undecided"] == 0 and s["violated"] == 0
    # within tol of the limit between samples: the coarse round cannot decide it at max_depth 0
    _, bump = cubic_peak()
    T, Cc = speed_bump(9.5, (cfg.vmax - 2e-4 - 9.5) / bump)
    s0 = ev.trajectory_dynamics(T, Cc, K=2, max_depth=0)[0]
    assert s0["verdict"] == 0 and s0["undecided"] & 1 and s0["undecided_intervals"] > 0 and s0["samples"] == 3
    s1 = ev.trajectory_dynamics(T, Cc, K=2)[0]
    assert s1["verdict"] == I.FEASIBLE and s1["upper"][0] <= cfg.vmax
    # a non-finite coefficient
    bad = Cc.copy(); bad[3] = np.inf
    s = ev.trajectory_dynamics(T, bad, K=2)[0]
    assert s["verdict"] == I.VIOLATING and math.isnan(s["upper"][0])
    # near free fall: zu vanishes at t = 0, so the body rate cannot be bounded there
    c = np.zeros((3, 6)); c[2, 0] = 10.0; c[2, 2] = -0.5 * cfg.grav_acc
    s = ev.trajectory_dynamics(np.array([0.5]), c.reshape(-1), K=4)[0]
    assert s["verdict"] == 0 and s["undecided"] & 4 and s["upper"][2] == math.inf
    ev.close()


def test_device_agrees_with_restatement():
    cfg = cfg_of()
    ev = I.Evaluator(cfg, device=0)
    cases = random_trajs(4, seed=11) + aggressive_trajs()
    for kw in (dict(K=8), dict(K=4, max_depth=3, max_samples=20), dict(K=8, amax=40.0, thrust_min=2.0, thrust_max=9.0, omgmax=3.0)):
        for T, Cc in cases:
            p = ev.dynamics_params(**kw)
            d = ev.trajectory_dynamics(T, Cc, params=p)[0]
            o = DO.certify(cfg, T, Cc, p)[0][0]
            for q in range(5):
                assert d["upper"][q] >= o["upper"][q] * (1 - 1e-12) - 1e-12, (kw, q)
                if np.isfinite(o["upper"][q]):
                    assert abs(d["upper"][q] - o["upper"][q]) <= 1e-9 * max(1.0, abs(o["upper"][q])), (kw, q)
                assert abs(d["attained"][q] - o["attained"][q]) <= 1e-9 * max(1.0, abs(o["attained"][q]))
            for f in ("verdict", "violated", "undecided", "samples", "undecided_intervals", "depth"):
                assert d[f] == o[f], (kw, f, d[f], o[f])
    ev.close()


def test_thrust_at_samples_equals_reference_forward():
    g = np.load(GOLDEN)
    for tag, drag in (("drag", True), ("nodrag", False)):
        cfg = cfg_of(drag)
        ev = I.Evaluator(cfg, device=0)
        v, a, thr = g[f"{tag}_v"], g[f"{tag}_a"], g[f"{tag}_thr"]
        n = len(thr)
        # one piece per input with v(t) = v + a t over a duration so short that both samples evaluate (v, a)
        c = np.zeros((n, 3, 6)); c[:, :, 1] = v; c[:, :, 2] = 0.5 * a
        Cc = c.transpose(1, 0, 2).reshape(-1)
        summ = ev.trajectory_dynamics(np.full(n, 1e-300), Cc, K=1, N0=1, max_depth=0, tol_thrust=math.inf)
        hi = np.array([s["attained"][4] for s in summ])
        lo = np.array([s["thrust_attained_min"] for s in summ])
        scale = np.maximum(np.abs(thr), 1.0)
        assert np.max(np.abs(hi - thr) / scale) <= 1e-12 and np.max(np.abs(lo - thr) / scale) <= 1e-12
        ev.close()


def raw_summaries(d_sum, B):
    raw = d_sum.cpu().numpy().tobytes()
    return [bytes(raw[168 * b:168 * (b + 1)]) for b in range(B)]


def test_bit_identity_entry_points_batch_and_runs():
    import torch
    cfg = cfg_of()
    ev = I.Evaluator(cfg, device=0)
    trajs = random_trajs(5, seed=21) + aggressive_trajs()
    T, Cc, N0 = batch_of(trajs)
    B = len(T) // N0
    for kw in (dict(K=8), dict(K=8, max_samples=7), dict(K=4, max_depth=2, tol_v=math.inf)):
        p = ev.dynamics_params(N0=N0, **kw)
        host = (I.DynamicsSummary * B)()
        ev._check(ev.lib.isdf_trajectory_dynamics(ev.h, len(T), I._dp(T), I._dp(Cc), C.byref(p), host))
        hb = [bytes(host)[168 * b:168 * (b + 1)] for b in range(B)]
        dT, dC = torch.from_numpy(T).cuda(), torch.from_numpy(Cc).cuda()
        d_sum = torch.zeros(21 * B, dtype=torch.float64, device="cuda")
        for _ in range(2):
            ev.trajectory_dynamics_device(len(T), dT.data_ptr(), dC.data_ptr(), p, d_sum.data_ptr(), torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            assert raw_summaries(d_sum, B) == hb
        for b in range(B):   # alone
            p1 = ev.dynamics_params(N0=N0, **kw)
            one = (I.DynamicsSummary * 1)()
            Tb, Cb = T[b * N0:(b + 1) * N0], np.asarray(Cc).reshape(3, -1)[:, 6 * N0 * b:6 * N0 * (b + 1)].reshape(-1).copy()
            ev._check(ev.lib.isdf_trajectory_dynamics(ev.h, N0, I._dp(Tb), I._dp(Cb), C.byref(p1), one))
            assert bytes(one) == hb[b], (kw, b)
    ev.close()


def test_bit_identity_after_device_lbfgs_1024_restarts():
    import torch
    sys.path.insert(0, ROOT)
    sys.dont_write_bytecode = True
    import bench as BN
    w, cfg, occ, T, Cc, V, F = BN.make_workload(True)
    ev = I.Evaluator(cfg, device=0)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_mesh(V, F, w["poly_params"], I.MESH_SIGN_EXACT)
    Bt, N0 = 1024, 64
    xs, heads, tails = BN.batch_problems(Bt, N0, w["map_dim"])
    hh, tt = heads.reshape(Bt, 3, 3).transpose(0, 2, 1), tails.reshape(Bt, 3, 3).transpose(0, 2, 1)
    ev.lbfgs_batch(hh, tt, 20.0, xs, ev.lbfgs_params(max_iterations=8))
    Tb, Cb, _ = ev.batch_trajectories(Bt, N0)
    dT, dC = torch.from_numpy(Tb).cuda(), torch.from_numpy(Cb).cuda()
    st = torch.cuda.current_stream().cuda_stream
    for kw in (dict(), dict(max_samples=16, max_depth=4)):
        p = ev.dynamics_params(N0=N0, **kw)
        d_sum = torch.zeros(21 * Bt, dtype=torch.float64, device="cuda")
        ev.trajectory_dynamics_device(Bt * N0, dT.data_ptr(), dC.data_ptr(), p, d_sum.data_ptr(), st)
        torch.cuda.synchronize()
        r0 = raw_summaries(d_sum, Bt)
        ev.trajectory_dynamics_device(Bt * N0, dT.data_ptr(), dC.data_ptr(), p, d_sum.data_ptr(), st)
        torch.cuda.synchronize()
        assert raw_summaries(d_sum, Bt) == r0
        for b in (0, 1, 517, Bt - 1):
            one = (I.DynamicsSummary * 1)()
            p1 = ev.dynamics_params(N0=N0, **kw)
            Tp, Cp = Tb[b * N0:(b + 1) * N0].copy(), Cb.reshape(3, -1)[:, 6 * N0 * b:6 * N0 * (b + 1)].reshape(-1).copy()
            ev._check(ev.lib.isdf_trajectory_dynamics(ev.h, N0, I._dp(Tp), I._dp(Cp), C.byref(p1), one))
            assert bytes(one) == r0[b], (kw, b)
    ev.close()


def test_refusals_poison_and_isolation():
    cfg = cfg_of(K=8)
    cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    ev = I.Evaluator(cfg, device=0)
    T, Cc, wp = W.make_trajectory(4, [2, 2, 2], [28, 28, 28], seed=4, jitter=0.3)

    def refused(code, N=None, **kw):
        p = ev.dynamics_params()
        for k, v in kw.items():
            if k == "reserved":
                p.reserved_[1] = v
            else:
                setattr(p, k, v)
        s = (I.DynamicsSummary * 4)()
        for x in s:
            x.verdict = 7
        r = ev.lib.isdf_trajectory_dynamics(ev.h, len(T) if N is None else N, I._dp(T), I._dp(Cc), C.byref(p), s)
        assert r == code, (kw, r)
        assert s[0].verdict == 0 and math.isnan(s[0].upper[0]) and math.isnan(s[0].thrust_lower) and s[0].samples == -1

    for kw in (dict(samples_per_piece=0), dict(pieces_per_traj=3), dict(pieces_per_traj=-1), dict(max_depth=65), dict(max_depth=-1),
               dict(max_samples_per_traj=-1), dict(tol_v=-1.0), dict(tol_thrust=math.nan), dict(vmax=math.nan), dict(thrust_min=5.0, thrust_max=4.0),
               dict(reserved=1), dict(max_samples_per_traj=1 << 30)):
        refused(-1, **kw)
    refused(-1, N=0)
    p = ev.dynamics_params()
    assert ev.lib.isdf_trajectory_dynamics_device(ev.h, len(T), None, None, C.byref(p), None, None) == -1
    ev.set_shard(0, 2)
    refused(-4)
    ev.set_shard(0, 1)
    # the context still works, and a dynamics call changes no other state
    occ = W.random_map(32, 32, 32, p=0.02, seed=3)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    c0, g0, t0 = ev.eval_discrete(T, Cc)
    pts = W.gather_obstacle_points(occ, [0, 0, 0], 1.0, wp, 3.0)[:50]
    ev.set_points(pts)
    sv0 = ev.eval_swept(T, Cc)
    st0 = ev.stats()
    s = ev.trajectory_dynamics(T, Cc)[0]
    st1 = ev.stats()
    assert s["verdict"] in (-1, 0, 1) and st1.kernel_launches > st0.kernel_launches
    for f in ("evals_discrete", "evals_swept", "last_pairs", "last_sdf_evals", "last_kernel_ms"):
        assert getattr(st1, f) == getattr(st0, f), f
    c1, g1, t1 = ev.eval_discrete(T, Cc)
    sv1 = ev.eval_swept(T, Cc)
    assert c1 == c0 and np.array_equal(g1, g0) and np.array_equal(t1, t0)
    assert sv1[0] == sv0[0] and np.array_equal(sv1[1], sv0[1])
    s2 = ev.trajectory_dynamics(T, Cc)[0]
    assert all(np.array_equal(np.asarray(s2[k]), np.asarray(v)) for k, v in s.items())
    ev.close()


def test_batch_trajectories_unchanged_by_a_dynamics_call():
    w_cfg = cfg_of(K=16)
    w_cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
    ev = I.Evaluator(w_cfg, device=0)
    occ = W.random_map(32, 32, 32, p=0.02, seed=3)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named("Ball")
    sys.path.insert(0, ROOT)
    sys.dont_write_bytecode = True
    import bench as BN
    Bt, N0 = 4, 6
    xs, heads, tails = BN.batch_problems(Bt, N0, 32)
    hh, tt = heads.reshape(Bt, 3, 3).transpose(0, 2, 1), tails.reshape(Bt, 3, 3).transpose(0, 2, 1)
    ev.lbfgs_batch(hh, tt, 20.0, xs, ev.lbfgs_params(max_iterations=3))
    Tb0, Cb0, x0 = ev.batch_trajectories(Bt, N0)
    ev.trajectory_dynamics(Tb0, Cb0, N0=N0)
    Tb1, Cb1, x1 = ev.batch_trajectories(Bt, N0)
    assert np.array_equal(Tb0, Tb1) and np.array_equal(Cb0, Cb1) and np.array_equal(np.asarray(x0), np.asarray(x1))
    ev.close()
