"""GPU: every consumer of the vehicle model and the penalty weights at vehicles other than the default one (tests/vehicles.py).

At the default vehicle horiz_drag == vert_drag and the three dynamic weights are equal, so a kernel parameter block that swaps them, reads the
mass for dh / mass, or hard-codes gravity or speed_eps computes the default's numbers. Here each consumer is held to the contract its own test
states, at three vehicles on which those mistakes all show, and each test first shows that its reference moves by at least 100 times the
test's tolerance under every such mistake the consumer can see (vehicles.sensitivity prints the margins and the mistakes it skips, with the
reason: a consumer that does not read the parameter). References at wrong vehicles are the oracle's and the restatements', which
tests/test_vehicles_cpu.py pins to the reference-compiled flatness map at the right ones."""
import math
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import states_oracle as SO
import certify_oracle as CE
import clearance_oracle as CO
import dynlimits_oracle as DO
import vehicles as VH
from common import small_case, rel_l2, BMIN, MESHES
from test_reference_pins import relerr

pytestmark = pytest.mark.gpu
ULP = 2.0 ** -52
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]      # the bench robot's poly_params
BOX_HALF = [0.9, 0.5, 0.3]


# ---- isdf_dbg_flatness: the flatness map and adjoint as compiled into the epilogue -------------------------------------------------------
@pytest.mark.parametrize("tag", VH.TAGS)
def test_device_flatness_equals_reference_at_vehicle(tag):
    """quat 1e-14, omega 1e-12, adjoint 1e-11 against the reference-compiled flatness.hpp at the vehicle (the committed outputs; the CPU tests
    hold them to the live library where it exists). The map reads neither dv nor the weights, nor the mass when dh = 0, nor speed_eps when
    cp = 0."""
    z = VH.golden(tag)
    cfg = VH.config(tag)
    ev = I.Evaluator(cfg)
    q, o, gV, gA, gJ = ev.dbg_flatness(z["v"], z["a"], z["j"], z["qg"], z["og"], z["vg"])
    ev.close()
    assert np.all(np.isfinite(q))
    errs = relerr(q, z["quat"]) / 1e-14, relerr(o, z["omg"]) / 1e-12, relerr(np.concatenate([gV, gA, gJ], axis=1), z["back"][:, 3:]) / 1e-11
    print(f"[{tag}] quat / omega / adjoint error in units of the tolerance: {errs[0]:.2e} {errs[1]:.2e} {errs[2]:.2e}")
    assert max(errs) <= 1.0, errs

    def moved(_, c):
        qw, ow = O.flat_forward_batch(O.config_from(c), z["v"], z["a"], z["j"])
        bw = O.flat_backward_batch(O.config_from(c), z["v"], z["a"], z["j"], z["pg"], z["vg"], z["qg"], z["og"])
        return max(relerr(qw, z["quat"]) / 1e-14, relerr(ow, z["omg"]) / 1e-12, relerr(bw[:, 3:], z["back"][:, 3:]) / 1e-11)
    VH.sensitivity(cfg, VH.FLAT, moved, 1.0, f"dbg_flatness [{tag}]")


# ---- isdf_trajectory_states and isdf_pose_points -------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", VH.TAGS)
def test_states_and_pose_points_equal_reference_at_vehicle(tag):
    """every record bit-identical to the reference-compiled process() state at the vehicle (N = 1, 2, 7, 64, 290), and the robot posed at
    those states bit-identical to the NumPy transform. The records read no weight."""
    z = VH.golden(tag)
    cfg = VH.config(tag)
    ev = I.Evaluator(cfg)
    body = np.load(__file__.replace("test_gpu_vehicles.py", "golden/ref_meshes.npz"))["drone_V"]
    moved = {name: 0.0 for name, _ in VH.wrong(cfg)}
    for c, rec_ref in zip(z["cases"], z["rec"]):
        rg = (np.array([0, c["N"]], dtype=np.int32), c["T"], c["coeffs"])
        rec = ev.trajectory_states(rg, np.zeros(c["times"].size, dtype=np.int32), c["times"])
        assert SO.same_bits(rec, rec_ref), f"N={c['N']}: {np.argwhere(rec.view(np.uint64) != rec_ref.view(np.uint64))[:5]}"
        fin = np.isfinite(rec).all(axis=1)
        assert SO.same_bits(ev.pose_points(rec[fin], body), SO.pose_points(rec[fin], body))
        for name, wc in VH.wrong(cfg):
            q, o, thr = SO.flat_forward_yaw0(VH.par(wc), rec_ref[fin, 3:6], rec_ref[fin, 6:9], rec_ref[fin, 9:12])
            moved[name] = max(moved[name], relerr(np.concatenate([q, o, thr[:, None]], axis=1), rec_ref[fin, 12:20]))
    ev.close()
    VH.sensitivity(cfg, VH.THRUST, lambda name, _: moved[name], ULP, f"trajectory_states [{tag}]")


# ---- isdf_eval_discrete: penalties, pose and adjoint in the epilogue --------------------------------------------------------------------
def hinge_config(cfg, T, Cc):
    """vmax, omgmax, thetamax and smoothing_eps such that every hinge of the epilogue has samples in its smoothing band (0 < x < mu) and in
    its linear part (x > mu): mu is half the smallest spread above the medians, and each limit sits 0.25 mu below the first sample from the
    median up that keeps the limit positive"""
    K = cfg.integral_intervs
    toff = np.concatenate([[0.0], np.cumsum(T)[:-1]])
    t = np.concatenate([toff[i] + np.arange(K + 1) * (T[i] / K) for i in range(len(T))])
    ev = O.traj_eval(T, Cc, t)[0]
    q, o = O.flat_forward_batch(O.config_from(cfg), ev[:, 3:6], ev[:, 6:9], ev[:, 9:12])
    y = [(ev[:, 3:6] ** 2).sum(1), (o ** 2).sum(1), np.arccos(1.0 - 2.0 * (q[:, 1] ** 2 + q[:, 2] ** 2))]
    mu = 0.5 * min(x.max() - np.median(x) for x in y)
    lim = [np.sort(x)[np.flatnonzero((np.arange(x.size) >= x.size // 2) & (np.sort(x) > 0.25 * mu))[0]] - 0.25 * mu for x in y]
    cfg.vmax, cfg.omgmax, cfg.thetamax, cfg.smoothing_eps = math.sqrt(lim[0]), math.sqrt(lim[1]), lim[2], mu
    for x, lo in zip(y, (cfg.vmax ** 2, cfg.omgmax ** 2, cfg.thetamax)):
        assert np.any((x - lo > 0) & (x - lo < mu)) and np.any(x - lo > mu), "fixture: a hinge without samples in both branches"
    return cfg


@pytest.mark.parametrize("robot", ["TwistBox", "mesh"])
@pytest.mark.parametrize("tag", VH.TAGS)
def test_discrete_equals_oracle_at_vehicle(tag, robot):
    """WITH_DYNAMICS | WITH_COLLISION, every hinge in both branches: cost and gradient within 1e-6 of the oracle (check_eval of
    test_gpu_parity.py), the same pair count. The back end's cost reads no thrust, so neither dv nor the mass beyond dh / mass: those wrong
    vehicles are skipped."""
    cfg, occ, T, Cc, _ = small_case(N=4, K=16, seed=3)
    cfg = hinge_config(VH.config(tag, cfg), T, Cc)
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, BMIN, 1.0)
    if robot == "mesh":
        V, F = MESHES["rcone"]()
        ev.set_shape_mesh(V, F, PP)
        osh = O.Shape.mesh(V, F, PP)
    else:
        ev.set_shape_named(robot)
        osh = O.Shape.named(robot)
    c, gC, gT = ev.eval_discrete(T, Cc)
    pairs = ev.stats().last_pairs
    ev.close()
    oc, ogC, ogT, opairs = O.eval_discrete(O.config_from(cfg), occ, BMIN, 1.0, osh, T, Cc)
    assert opairs > 0 and pairs == opairs
    assert abs(c - oc) <= 1e-6 * abs(oc) and rel_l2(np.concatenate([gC, gT]), np.concatenate([ogC, ogT])) <= 1e-6

    def moved(_, wc):
        wcost, wgC, wgT, _ = O.eval_discrete(O.config_from(wc), occ, BMIN, 1.0, osh, T, Cc)
        return max(abs(wcost - oc) / abs(oc), rel_l2(np.concatenate([wgC, wgT]), np.concatenate([ogC, ogT])))
    VH.sensitivity(cfg, VH.FLAT + VH.WEIGHTS, moved, 1e-6, f"eval_discrete {robot} [{tag}]")


# ---- isdf_eval_swept ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", VH.TAGS)
def test_swept_equals_oracle_at_vehicle(tag):
    """the strict swept contract of test_gpu_swept_edges.py (hit set, t* 1e-12, SV-SDF 1e-10, g_rel 1e-8, evaluation count, cost and gradient
    1e-9) with the mesh robot, whose pose the vehicle sets. The swept term reads the pose and weight_p; no thrust and no dynamic weight."""
    from test_gpu_swept_edges import check_strict
    cfg, occ, T, Cc, wp = small_case(N=4, K=16, seed=3, flags=I.WITH_DYNAMICS)
    cfg = VH.config(tag, cfg)
    V, F = MESHES["rcone"]()
    osh = O.Shape.mesh(V, F, PP)
    pts = W.gather_obstacle_points(occ, BMIN, 1.0, wp, cfg.kernel_size * cfg.occupancy_resolution / 3.0)[:200]
    ev = I.Evaluator(cfg)
    ev.set_shape_mesh(V, F, PP)
    ev.set_points(pts)
    got = ev.eval_swept(T, Cc)
    ref = O.eval_swept(O.config_from(cfg), osh, T, Cc, pts)
    assert ref["cost"] > 0
    check_strict(ev, got, ref, f"swept [{tag}]")
    ev.close()

    def moved(_, wc):
        w = O.eval_swept(O.config_from(wc), osh, T, Cc, pts)
        return max(abs(w["cost"] - ref["cost"]) / ref["cost"], rel_l2(np.concatenate([w["gradC"], w["gradT"]]), np.concatenate([ref["gradC"], ref["gradT"]])))
    VH.sensitivity(cfg, VH.FLAT + ("wp",), moved, 1e-9, f"eval_swept [{tag}]")


# ---- isdf_trajectory_clearance -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", VH.TAGS)
def test_clearance_equals_oracle_at_vehicle(tag):
    """per-sample clearance within 1e-12 of clearance_oracle and the same witnesses (as test_gpu_clearance.py) for a box robot, whose
    clearance depends on its attitude. The check reads the pose only."""
    from test_gpu_clearance import Robot, compare, traj_in, maps
    occ, bmin, res = maps()["random_1.0"]
    cfg = VH.config(tag)
    cfg.flags, cfg.integral_intervs = I.WITH_COLLISION, 8
    robot = Robot("Box")
    T, Cc = traj_in(bmin, np.array(occ.shape) * res, seed=0)
    reach = 2.5
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, bmin, res)
    robot.set_on(ev)
    clear, vox, _ = ev.trajectory_clearance(T, Cc, 8, reach, reach)
    ev.close()
    ref = CO.clearance(O.config_from(cfg), occ, bmin, res, robot.osdf, T, Cc, 8, reach, reach, keep_candidates=True)
    compare(clear, vox, ref, reach, 1e-12)
    assert (vox >= 0).sum() >= 3

    def moved(_, wc):
        w = CO.clearance(O.config_from(wc), occ, bmin, res, robot.osdf, T, Cc, 8, reach, reach)
        return float(np.abs(w["clear"] - ref["clear"]).max())
    VH.sensitivity(cfg, VH.FLAT, moved, 1e-12, f"trajectory_clearance [{tag}]")


# ---- isdf_trajectory_certify: the motion bound --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", VH.TAGS)
def test_certify_bound_at_vehicle(tag):
    """the device motion bound D within rounding of certify_oracle.bound and at least the dense displacement of the box's corners (as
    test_bound_sound_and_tight); the certificate's lower bound on the clearance at most the dense clearance minimum. The bound reads the
    rotation enclosure, i.e. the flatness map's attitude."""
    cfg = VH.config(tag)
    cfg.flags, cfg.integral_intervs = I.WITH_COLLISION, 8
    ev = I.Evaluator(cfg)
    ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
    reach = 2.0
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + reach
    T, Cc, _ = W.make_trajectory(4, [0, 0, 0], [30, 30, 30], seed=6, jitter=0.4)
    rng = np.random.default_rng(0)
    piece, ta, tb = [], [], []
    for i in range(4):
        for h in (T[i] / 16, T[i] / 64, 1e-6):
            a = rng.uniform(0, T[i] - h)
            for x, y in ((a, a + h), (T[i] - h, T[i]), (0.0, h)):
                piece.append(i); ta.append(x); tb.append(y)
    D, r = ev.dbg_certify_bound(T, Cc, reach, piece, ta, tb)
    body = CE.box_corners(BOX_HALF)
    o = np.zeros_like(D)
    for k in range(len(piece)):
        c = CE.piece_coeffs(Cc, 4, piece[k])
        for e, te in enumerate((ta[k], tb[k])):
            o[k, e] = CE.bound(cfg, r, H, c, ta[k], tb[k], te)
            assert D[k, e] >= o[k, e] * (1 - 1e-12), (k, e, D[k, e], o[k, e])
            assert D[k, e] <= o[k, e] * (1 + 1e-9) + CE.eps_pad(cfg, r, H, c, te), (k, e, D[k, e], o[k, e])
            assert D[k, e] >= CE.displacement(cfg, T, Cc, piece[k], ta[k], tb[k], te, body, n=401), (k, e)
    # the certificate end to end on a map: its lower bound never exceeds the dense minimum
    occ = W.random_map(32, 32, 32, p=0.02, seed=3)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    s = ev.trajectory_certify(T, Cc, 4, reach, 0.5)[0]
    dense = ev.trajectory_clearance(T, Cc, 2 ** 12, reach, 0.0)[2][0]["min_clearance"]
    assert s["lower_bound"] <= dense + 1e-12, (s, dense)
    ev.close()

    def moved(_, wc):
        w = np.array([[CE.bound(wc, r, H, CE.piece_coeffs(Cc, 4, piece[k]), ta[k], tb[k], te) for te in (ta[k], tb[k])] for k in range(len(piece))])
        return float(np.max(np.abs(w - o) / o))
    VH.sensitivity(cfg, VH.FLAT, moved, 1e-9, f"certify bound [{tag}]")


# ---- isdf_trajectory_dynamics ------------------------------------------------------------------------------------------------------------
def dense_values(cfg, T, Cc, i, t):
    """dynlimits_oracle.dense with the flatness map of the reference-compiled library where it exists, else the oracle's (pinned to it at
    these vehicles by test_vehicles_cpu.py)"""
    c = DO.piece_coeffs(Cc, len(T))[i]
    v, a, j = DO.vaj_exact(c, t)
    vd, ad, jd = (np.asarray(x, float) for x in (v, a, j))
    q, o = O.RefFlat(O.config_from(cfg)).forward(vd, ad, jd) if O.ref_flat_available() else O.flat_forward_batch(O.config_from(cfg), vd, ad, jd)
    cz = 1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2)
    return np.stack([np.asarray(np.sqrt((v * v).sum(1)), float), np.asarray(np.sqrt((a * a).sum(1)), float), np.linalg.norm(o, axis=1),
                     np.arccos(np.clip(cz, -1, 1)), DO.thrust_exact(cfg, v, a)], axis=1)


@pytest.mark.parametrize("tag", VH.TAGS)
def test_dynamics_at_vehicle(tag):
    """the proven bounds enclose the dense extrema (as test_bounds_enclose_dense_extrema) and the thrust at the samples equals the reference
    FlatnessMap::forward's (the process() records of the vehicle golden) to 1e-12 (as test_thrust_at_samples_equals_reference_forward). The
    thrust reads the mass and dv raw; no weight."""
    from test_gpu_dynlimits import random_trajs, aggressive_trajs
    cfg = VH.config(tag)
    ev = I.Evaluator(cfg, device=0)
    for T, Cc in random_trajs(3, seed=5) + aggressive_trajs():
        s = ev.trajectory_dynamics(T, Cc, K=8, max_depth=20, max_samples=4000)[0]
        mx, tmin = np.full(5, -np.inf), np.inf
        for i in range(len(T)):
            vals = dense_values(cfg, T, Cc, i, np.linspace(0.0, T[i], 2001))
            mx, tmin = np.fmax(mx, np.nanmax(vals, axis=0)), min(tmin, np.nanmin(vals[:, 4]))
        for q in range(5):
            tol = 1e-7 if q == 3 else 1e-9 * max(1.0, mx[q])
            assert s["upper"][q] >= mx[q] - tol, (q, s["upper"][q], mx[q])
        assert s["thrust_lower"] <= tmin + 1e-9 * max(1.0, abs(tmin))
        assert np.all(s["attained"] <= s["upper"])
    # the thrust at samples: one piece per reference record with v(t) = v + a t over a duration so short that both samples evaluate (v, a)
    rec = np.concatenate(VH.golden(tag)["rec"])
    rec = rec[np.isfinite(rec).all(axis=1)][::7]
    v, a, thr = rec[:, 3:6], rec[:, 6:9], rec[:, 19]
    n = len(thr)
    c = np.zeros((n, 3, 6)); c[:, :, 1] = v; c[:, :, 2] = 0.5 * a
    summ = ev.trajectory_dynamics(np.full(n, 1e-300), c.transpose(1, 0, 2).reshape(-1), K=1, N0=1, max_depth=0, tol_thrust=math.inf)
    ev.close()
    scale = np.maximum(np.abs(thr), 1.0)
    hi = np.array([x["attained"][4] for x in summ])
    lo = np.array([x["thrust_attained_min"] for x in summ])
    assert np.max(np.abs(hi - thr) / scale) <= 1e-12 and np.max(np.abs(lo - thr) / scale) <= 1e-12
    VH.sensitivity(cfg, VH.THRUST, lambda _, wc: float(np.max(np.abs(DO.thrust_exact(wc, v, a) - thr) / scale)), 1e-12, f"dynamics thrust [{tag}]")


# ---- isdf_swept_volume_sdf ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", VH.TAGS)
def test_swept_volume_equals_restatement_at_vehicle(tag):
    """the certified swept-volume SDF of an offset, rotated box decision for decision against sweptvol_oracle's refinement (compare of
    test_gpu_swept_volume_oracle.py: value 1e-12, t*, decided). It reads the pose and the rotation enclosure."""
    from test_gpu_swept_volume_oracle import Robot, trajectory, points_for, refine_all, compare
    robot = Robot("BoxRT")
    T, Cc = trajectory("traj")
    cfg = VH.config(tag)
    cfg.integral_intervs = 8
    ev = I.Evaluator(cfg)
    robot.set_on(ev)
    prm = ev.swept_params(K=8, tol=1e-3)
    P = points_for(robot, T, Cc, prm.band, seed=3)
    ref = refine_all(cfg, robot, T, Cc, prm, P)
    v, lo, ts, dec = ev.swept_volume_sdf(T, Cc, P, prm)
    ev.close()
    compare(ref, v, lo, ts, dec, f"swept volume [{tag}]")
    rv = np.array([x["value"] for x in ref])

    def moved(_, wc):
        return float(np.abs(np.array([x["value"] for x in refine_all(wc, robot, T, Cc, prm, P)]) - rv).max())
    VH.sensitivity(cfg, VH.FLAT, moved, 1e-12, f"swept_volume_sdf [{tag}]")


# ---- isdf_plan_batch ------------------------------------------------------------------------------------------------------------------
def test_plan_equals_the_public_call_composition_heavy():
    """isdf_plan_batch at the heavy vehicle bit-identical to the composition of the public calls on a fresh context at the same config (as
    test_plan_equals_the_public_call_composition); every wrong vehicle the planner reads changes the planned trajectories by far more than an
    ulp. The plan's certificates run at their defaults; the planner reads the thrust only through the dynamic-limit certificate."""
    from test_gpu_plan import _ev, _scene, _params, _compose, _check_plan, _cfg
    occ, start, goals = _scene(6)
    cfg = VH.config("heavy", _cfg())

    def plan(c):
        ev = _ev("mesh", occ, cfg=c)
        got, _ = ev.plan_batch(start, goals, _params(ev))
        ev.close()
        return got
    got = plan(cfg)
    fresh = _ev("mesh", occ, cfg=cfg)
    ref = _compose(fresh, start, goals, _params(fresh))
    fresh.close()
    assert sum(r["stage"] == I.OPTIMISED for r in got) >= 2
    for b in range(len(goals)):
        _check_plan(got[b], ref[b], b)
    opt = [b for b in range(len(goals)) if got[b]["stage"] == I.OPTIMISED]

    def moved(_, wc):
        w = plan(wc)
        return max(float(np.max(np.abs(w[b]["coeffs"] - got[b]["coeffs"]))) / float(np.max(np.abs(got[b]["coeffs"])))
                   if w[b]["coeffs"].shape == got[b]["coeffs"].shape else 1.0 for b in opt)
    VH.sensitivity(cfg, VH.FLAT + VH.WEIGHTS, moved, ULP, "plan_batch [heavy]")
