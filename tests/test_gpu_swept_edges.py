"""Edges of the swept-volume search on the device (k_sv_table + k_sv_points_cta): the interval fixtures of tests/sv_intervals.py, odd and
very long trajectories, the persisted trajectory duration of updateTraj (quirk Q14) on the single-problem and batched paths, batched =
single bit for bit, and the device entry point.

The strict contract (analytic shapes without libm calls, and mesh robots): the same hit set and reference-equivalent SDF evaluation count
as the oracle, t* within 1e-12, SV-SDF within 1e-10, g_rel within 1e-8 (a 5e-6 central difference), cost and gradient within 1e-9."""
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import sv_intervals as S
from common import small_case, rel_l2, BMIN, MESHES

pytestmark = pytest.mark.gpu


def check_strict(ev, got, ref, what, counted=True):
    """got = eval_swept's (cost, gradC, gradT); ref = oracle_lib.eval_swept's dict on the same points"""
    ts, sd, gr = ev.swept_results()
    hit = ref["sdf"] < 9.99
    assert np.array_equal(sd < 9.99, hit), f"{what}: hit sets differ at points {np.flatnonzero((sd < 9.99) != hit)[:10]}"
    dt, ds, dg = (float(np.abs(a - b).max()) if a.size else 0.0 for a, b in ((ts, ref["tstar"]), (sd, ref["sdf"]), (gr, ref["grel"])))
    c, gC, gT = got
    dc = abs(c - ref["cost"]) / max(abs(ref["cost"]), 1e-300) if ref["cost"] != 0 else abs(c)
    rg = rel_l2(np.concatenate([gC, gT]), np.concatenate([ref["gradC"], ref["gradT"]]))
    evals = ev.stats().last_sdf_evals
    print(f"{what}: points {len(ts)} hits {hit.sum()} max|dt*| {dt:.1e} max|dsdf| {ds:.1e} max|dg_rel| {dg:.1e} cost rel {dc:.1e} grad rel-L2 {rg:.1e} "
          f"evals {evals} vs {ref['nsdf']}")
    assert dt <= 1e-12 and ds <= 1e-10 and dg <= 1e-8, what
    assert dc <= 1e-9 and rg <= 1e-9, what
    if counted:
        assert evals == ref["nsdf"], what


def near_points(T, Cc, n, seed, spread=3.0, t_max=None):
    """n points scattered around the trajectory at random times (first t_max seconds)"""
    rng = np.random.default_rng(seed)
    t = rng.uniform(0, T.sum() if t_max is None else t_max, n)
    pos, _, _, _ = O.traj_eval(T, Cc, t)
    return pos[:, :3] + rng.uniform(-spread, spread, (n, 3))


def minco_traj(N, T, seed, step=1.0):
    wp = W.random_walk_waypoints(N, [0, 0, 0], [50, 50, 34], seed=seed, step=step)
    head, tail = np.zeros((3, 3)), np.zeros((3, 3))
    head[:, 0], tail[:, 0] = wp[0], wp[-1]
    T = np.full(N, float(T)) if np.isscalar(T) else np.asarray(T, float)
    Cc, _, _, _ = O.minco_forward(head, tail, wp[1:-1].T, T)
    return T, Cc


# ---- interval fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robot,nc", [(robot, nc) for robot in S.ROBOTS for nc in (64, 97)])
def test_interval_fixtures_match_the_oracle_exactly(robot, nc):
    f = S.fixture(robot, nc)
    ref = O.eval_swept(O.config_from(f["cfg"]), S.oracle_robot(robot), f["T"], f["C"], f["pts"])
    ev = I.Evaluator(f["cfg"])
    S.set_robot(ev, robot)
    ev.set_points(f["pts"])
    got = ev.eval_swept(f["T"], f["C"])
    check_strict(ev, got, ref, f"{robot} nc={nc} (N={f['T'].size})")
    ts, sd, _ = ev.swept_results()
    for c in ("G", "H", "B_alone"):        # no closed run: SV-SDF 10, t* untouched (0 after set_points)
        k = f["cats"][c]
        assert np.all(sd[k] == 10.0) and np.all(ts[k] == 0.0), c
    ev.close()


# ---- trajectory length and layout ---------------------------------------------------------------------------------------------------------
def test_odd_piece_count_single_problem():
    """odd N: the trajectory block is staged by the cooperative loop, not the bulk copy"""
    cfg, occ, T, Cc, wp = small_case(N=5, K=16, seed=9, noise=0.05)
    pts = W.gather_obstacle_points(occ, BMIN, 1.0, wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0)[:300]
    for name in ("Torus", "CSG"):
        ref = O.eval_swept(O.config_from(cfg), O.Shape.named(name), T, Cc, pts)
        ev = I.Evaluator(cfg)
        ev.set_shape_named(name)
        ev.set_points(pts)
        check_strict(ev, ev.eval_swept(T, Cc), ref, f"{name} N=5")
        ev.close()


@pytest.mark.parametrize("N", [331, 1347])
def test_longest_trajectories(N):
    """just under 300 s: ~1500 coarse samples (all six table CTAs, bitmap words up to 46); 19 N doubles of dynamic shared memory above
    48 KB (opt-in). N = 1347 is the largest the shared-memory block holds; N = 1348 is refused and the context keeps working."""
    cfg = small_case()[0]
    T, Cc = minco_traj(N, 299.0 / N, seed=N)
    pts = near_points(T, Cc, 120, seed=N, spread=2.5)
    ref = O.eval_swept(O.config_from(cfg), O.Shape.named("Torus"), T, Cc, pts, use_omp=True)
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Torus")
    ev.set_points(pts)
    got = ev.eval_swept(T, Cc)
    check_strict(ev, got, ref, f"Torus N={N} ({T.sum():.1f} s)")
    assert (ref["sdf"] < 9.99).sum() >= 20
    if N == 1347:
        with pytest.raises(I.IsdfError) as e:
            ev.eval_swept(np.full(N + 1, 0.2), np.zeros(18 * (N + 1)))
        assert e.value.code == -1                       # ISDF_ERR_INVALID
        again = ev.eval_swept(T, Cc)
        assert again[0] == got[0] and np.array_equal(again[1], got[1]) and np.array_equal(again[2], got[2])
    ev.close()


# ---- persisted trajectory duration (updateTraj, swm:287-296; quirk Q14) ---------------------------------------------------------------------
def test_fresh_context_ignores_a_trajectory_of_300_s_or_more():
    cfg = small_case()[0]
    T, Cc = minco_traj(4, 80.0, seed=21, step=3.0)           # 320 s
    pts = near_points(T, Cc, 80, seed=1, spread=1.0)
    ref = O.eval_swept(O.config_from(cfg), O.Shape.named("Torus"), T, Cc, pts)
    assert ref["cost"] == 0.0 and ref["nsdf"] == 0 and ref["duration"] == 0.0
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Torus")
    ev.set_points(pts)
    c, gC, gT = ev.eval_swept(T, Cc)
    ts, sd, _ = ev.swept_results()
    assert c == 0.0 and not gC.any() and not gT.any() and np.all(sd == 10.0) and np.all(ts == 0.0)
    assert ev.stats().last_sdf_evals == 0
    ev.close()


def test_long_trajectory_scans_the_previous_duration():
    """200 s, then 310 s: the second evaluation scans the first 200 s of the new trajectory, as the oracle replays it"""
    cfg = small_case()[0]
    T1, C1 = minco_traj(4, 50.0, seed=22, step=3.0)
    T2, C2 = minco_traj(4, 77.5, seed=23, step=3.0)
    pts = np.concatenate([near_points(T1, C1, 60, seed=2, spread=1.5), near_points(T2, C2, 60, seed=3, spread=1.5, t_max=200.0)])
    osh, ocfg = O.Shape.named("Torus"), O.config_from(cfg)
    r1 = O.eval_swept(ocfg, osh, T1, C1, pts)
    r2 = O.eval_swept(ocfg, osh, T2, C2, pts, prev_duration=r1["duration"])
    assert r1["duration"] == T1.sum() and r2["duration"] == r1["duration"] and (r2["sdf"] < 9.99).sum() >= 10
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Torus")
    ev.set_points(pts)
    check_strict(ev, ev.eval_swept(T1, C1), r1, "200 s")
    ev.set_points(pts)                                   # t* back to 0, as the oracle starts
    check_strict(ev, ev.eval_swept(T2, C2), r2, "310 s after 200 s")
    ev.close()


def tau_for(T):
    """forwardT^-1 (back_end_optimizer.hpp:214-241) for durations above 1 s: T = (tau / 2 + 1) tau + 1"""
    return -1.0 + np.sqrt(1.0 + 2.0 * (np.asarray(T, float) - 1.0))


class Batch:
    """B problems of N0 pieces with fixed waypoints; per call each problem's piece duration is chosen"""

    def __init__(self, ev, cfg, B, N0=4, seed=40):
        self.ev, self.cfg, self.B, self.N0 = ev, cfg, B, N0
        self.heads, self.tails, self.xi, self.psets = [], [], [], []
        for b in range(B):
            wp = W.random_walk_waypoints(N0, [0, 0, 0], [50, 50, 34], seed=seed + b, step=3.0)
            h, t = np.zeros((3, 3)), np.zeros((3, 3))
            h[:, 0], t[:, 0] = wp[0], wp[-1]
            self.heads.append(h); self.tails.append(t); self.xi.append(wp[1:-1].reshape(-1))
            rng = np.random.default_rng(seed + b)
            self.psets.append(np.concatenate([w + rng.uniform(-1.5, 1.5, (12, 3)) for w in wp]))

    def run(self, piece_T, nb=None):
        """callback over the first nb problems with piece durations piece_T[b]; returns the swept term rows and (T_b, C_b) per problem"""
        nb = self.B if nb is None else nb
        X = np.array([np.concatenate([np.full(self.N0, tau_for(piece_T[b])), self.xi[b]]) for b in range(nb)])
        self.ev.callback_batch(np.array(self.heads[:nb]), np.array(self.tails[:nb]), 20.0, X)
        T, Cc, _ = self.ev.batch_trajectories(nb, self.N0)
        Cm = Cc.reshape(3, 6 * nb * self.N0)
        trajs = [(T[b * self.N0:(b + 1) * self.N0], Cm[:, 6 * self.N0 * b:6 * self.N0 * (b + 1)].reshape(-1)) for b in range(nb)]
        return self.ev.dbg_batch_swept_out(nb, self.N0), trajs

    def check(self, rows, trajs, prev, what):
        """problem b's swept term against the oracle started from the persisted duration prev[b]; returns the durations after"""
        osh, ocfg, out = O.Shape.named("Torus"), O.config_from(self.cfg), []
        for b, (T, Cc) in enumerate(trajs):
            ref = O.eval_swept(ocfg, osh, T, Cc, self.psets[b], prev_duration=prev[b])
            N0 = self.N0
            c, gC, gT = rows[b][0], rows[b][1:1 + 18 * N0], rows[b][1 + 18 * N0:]
            if ref["cost"] == 0.0:
                assert c == 0.0 and not gC.any() and not gT.any(), f"{what}: problem {b} (prev {prev[b]:.1f} s) cost {c:.3e}, expected 0"
            else:
                assert abs(c - ref["cost"]) <= 1e-9 * abs(ref["cost"]), f"{what}: problem {b} cost {c} vs {ref['cost']} (prev {prev[b]:.1f} s)"
                assert rel_l2(np.concatenate([gC, gT]), np.concatenate([ref["gradC"], ref["gradT"]])) <= 1e-9, f"{what}: problem {b}"
            out.append(ref["duration"])
        return out


def test_single_and_batched_paths_keep_separate_durations():
    """the single-problem entry points and every batched problem keep their own persisted duration, in either order and across a growing B"""
    cfg, occ, *_ = small_case(N=4, K=16, seed=3, flags=I.WITH_DYNAMICS)
    osh, ocfg = O.Shape.named("Torus"), O.config_from(cfg)
    T200, C200 = minco_traj(4, 50.0, seed=31, step=3.0)
    T310, C310 = minco_traj(4, 77.5, seed=31, step=3.0)
    psingle = near_points(T200, C200, 80, seed=4, spread=1.5)
    SHORT, LONG = 30.0, 80.0                              # piece durations: 120 s and 320 s trajectories

    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("Torus")
    bt = Batch(ev, cfg, 3)
    # single first: its duration becomes 200 s
    ev.set_points(psingle)
    r = O.eval_swept(ocfg, osh, T200, C200, psingle)
    check_strict(ev, ev.eval_swept(T200, C200), r, "single 200 s")
    # batch of one, 320 s: problem 0 has no previous duration of its own -> scans nothing
    ev.set_points_batch(bt.psets[:1])
    rows, trajs = bt.run([LONG], nb=1)
    assert not rows.any(), "batched problem 0 scanned the single path's duration"
    dur = bt.check(rows, trajs, [0.0], "B=1 long after single")
    # batch of one, 120 s, then B grows to 3 with problems 0 and 1 long: problem 0 keeps 120 s, problem 1 (new) has none
    rows, trajs = bt.run([SHORT], nb=1)
    dur = bt.check(rows, trajs, dur, "B=1 short")
    assert abs(dur[0] - 4 * SHORT) < 1e-6
    ev.set_points_batch(bt.psets)
    rows, trajs = bt.run([LONG, LONG, SHORT])
    assert rows[0].any() and not rows[1].any()
    dur = bt.check(rows, trajs, dur + [0.0, 0.0], "B=3 after growing")
    # the single path still has its own 200 s
    ev.set_points(psingle)
    r = O.eval_swept(ocfg, osh, T310, C310, psingle, prev_duration=T200.sum())
    assert r["cost"] > 0
    check_strict(ev, ev.eval_swept(T310, C310), r, "single 310 s after the batches")
    # and the batched problems still have theirs
    ev.set_points_batch(bt.psets)
    rows, trajs = bt.run([LONG, LONG, LONG])
    bt.check(rows, trajs, dur, "B=3 all long")
    ev.close()

    # the other order: batched durations first, then a fresh single path
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    ev.set_shape_named("Torus")
    bt = Batch(ev, cfg, 2)
    ev.set_points_batch(bt.psets)
    rows, trajs = bt.run([SHORT, SHORT])
    dur = bt.check(rows, trajs, [0.0, 0.0], "B=2 short")
    ev.set_points(psingle)
    c, gC, gT = ev.eval_swept(T310, C310)
    assert c == 0.0 and not gC.any() and not gT.any() and ev.stats().last_sdf_evals == 0, "the single path scanned a batched problem's duration"
    ev.set_points_batch(bt.psets)
    rows, trajs = bt.run([LONG, LONG])
    bt.check(rows, trajs, dur, "B=2 long after the single path")
    ev.close()


# ---- batched = single, bit for bit ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robot", ["Torus", "mesh"])
def test_batched_swept_term_equals_single_problem_bit_for_bit(robot):
    cfg, occ, *_ = small_case(N=5, K=16, seed=3, flags=I.WITH_DYNAMICS)
    B, N0 = 6, 5
    rng = np.random.default_rng(8)
    heads, tails, X, psets = [], [], [], []
    for b in range(B):
        wp = W.random_walk_waypoints(N0, [0, 0, 0], [50, 50, 34], seed=500 + b)
        h, t = np.zeros((3, 3)), np.zeros((3, 3))
        h[:, 0], t[:, 0] = wp[0], wp[-1]
        heads.append(h); tails.append(t)
        X.append(np.concatenate([rng.normal(size=N0) * 0.3 + 0.9, wp[1:-1].reshape(-1)]))
        pts = np.concatenate([w + rng.uniform(-2.5, 2.5, (10 + 6 * b, 3)) for w in wp])
        psets.append(pts[:0] if b == 2 else pts[:1] if b == 4 else pts)      # one empty problem, one 1-point problem
    X = np.array(X)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, [0, 0, 0, 120, 0, 0])
    else:
        ev.set_shape_named(robot)
    ev.set_points_batch(psets)
    ev.callback_batch(np.array(heads), np.array(tails), 20.0, X)
    T, Cc, _ = ev.batch_trajectories(B, N0)
    Cm = Cc.reshape(3, 6 * B * N0)
    single = {}
    for b in range(B):
        if len(psets[b]) == 0:
            continue
        ev.set_points(psets[b])
        c, gC, gT = ev.eval_swept(T[b * N0:(b + 1) * N0], Cm[:, 6 * N0 * b:6 * N0 * (b + 1)].reshape(-1))
        single[b] = (np.concatenate([[c], gC, gT]), *ev.swept_results())
    ev.set_points_batch(psets)                           # set_points gave the batched sets up: register them again (t* from 0 on both sides)
    ev.callback_batch(np.array(heads), np.array(tails), 20.0, X)
    rows = ev.dbg_batch_swept_out(B, N0)
    ts, sd, gr = ev.swept_results()
    off = np.concatenate([[0], np.cumsum([len(p) for p in psets])])
    hits = 0
    for b in range(B):
        if b not in single:
            assert not rows[b].any()
            continue
        out, t1, s1, g1 = single[b]
        sl = slice(off[b], off[b + 1])
        assert np.array_equal(ts[sl], t1) and np.array_equal(sd[sl], s1) and np.array_equal(gr[sl], g1), f"problem {b}: per-point results differ"
        assert np.array_equal(rows[b], out), f"problem {b}: swept term differs, max |diff| {np.abs(rows[b] - out).max():.3e}"
        hits += int((s1 < 9.99).sum())
    print(f"{robot}: {sum(len(p) for p in psets)} points, {hits} hits, bit-identical in all {len(single)} problems with points")
    assert hits >= 10 and any(rows[b][0] > 0 for b in single)
    ev.close()


# ---- device entry point --------------------------------------------------------------------------------------------------------------------
def test_device_entry_point_matches_host_entry_point():
    import torch
    cfg, occ, T, Cc, wp = small_case(N=4, K=16, seed=5, noise=0.05)
    pts = W.gather_obstacle_points(occ, BMIN, 1.0, wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0)[:300]
    ev = I.Evaluator(cfg)
    ev.set_shape_named("SmoothIntersection")
    ev.set_points(pts)
    c, gC, gT = ev.eval_swept(T, Cc)
    host = np.concatenate([[c], gC, gT])
    ts0, sd0, gr0 = ev.swept_results()
    assert c > 0
    N = T.size
    dev = dict(dtype=torch.float64, device="cuda")
    cases = {}
    dT, dC = torch.tensor(T, **dev), torch.tensor(np.asarray(Cc).reshape(-1), **dev)
    cases["aligned, current stream"] = (dT, dC, torch.cuda.current_stream())
    bT, bC = torch.zeros(N + 1, **dev), torch.zeros(18 * N + 1, **dev)     # views 8 bytes into their allocations: not 16-byte aligned
    bT[1:] = dT; bC[1:] = dC
    assert bT[1:].data_ptr() % 16 == 8 and bC[1:].data_ptr() % 16 == 8
    cases["8-byte offset, side stream"] = (bT[1:], bC[1:], torch.cuda.Stream())
    for what, (tT, tC, st) in cases.items():
        out = torch.full((19 * N + 1,), float("nan"), **dev)     # overwritten, not accumulated into
        torch.cuda.synchronize()
        ev.eval_swept_device(N, tT.data_ptr(), tC.data_ptr(), out.data_ptr(), st.cuda_stream)
        st.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got, host), f"{what}: max |diff| {np.nanmax(np.abs(got - host)):.3e}"
        ts, sd, gr = ev.swept_results()
        assert np.array_equal(ts, ts0) and np.array_equal(sd, sd0) and np.array_equal(gr, gr0), what
    ev.close()
