"""Planning through what has been seen (DESIGN §3.23): the front end's surcharge on unknown voxels (isdf_frontpath_params.unknown_weight),
the known-prefix gather (isdf_gather_obstacle_points_batch_known) and ISDF_PLAN_KNOWN_PREFIX, against tests/known_plan_oracle.py.
  weight 0     every front-end output and every isdf_plan_states output equals the call with NULL / default params, bit for bit;
  weight > 0   on seeded maps with known grids from isdf_map_mark_known boxes and from isdf_map_observe, the fields of the single, batch,
               pairs and multi-source calls equal the weighted serial Dijkstra bit for bit, paths follow the weighted parent rule, costs are
               g(t), and pairs agree across max_fields 0 / 1 and permutations;
  gather       known_rows lists equal the numpy restatement; with nothing known the plan flag changes nothing; the plan's obstacle_points
               are the restatement's counts from each path's k*;
  refusals     negative, NaN and infinite weights and non-zero reserved_ are refused by the front end and the planning step;
  navigate     the wall scenario of test_gpu_navigate_unknown.py under unknown="occupied" with plan_params(unknown_weight=1,
               flags=PLAN_CERTIFY | PLAN_KNOWN_PREFIX): every flown position lies in a known voxel, the true clearance stays >= 0 and two
               runs give identical logs. Recorded on an H100 80GB HBM3 at 700 W (DESIGN §3.23), next to the same rigs without the params
               (test_gpu_navigate_unknown.py):
                 front + back, 60 rounds: 24 commits in rounds 0-24, then held to the end (TIMEOUT); furthest x 23.5 (without: a commit
                   every round, never past x 34.4); minimum true clearance 0.866 m;
                 four cameras fx = fy = 200, 120 rounds: 30 commits in rounds 0-31, then held to the end (TIMEOUT); furthest x 16.7, past
                   the wall (without: ARRIVED after 46 rounds, 33 commits); minimum true clearance 0.866 m.
               The held vehicle stands at the edge of its known prefix: the last known row's box holds the unknown voxels it must pass to
               reach the crossing, so every stop it is offered ends before them. Nothing here asserts progress."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import frontpath_oracle as FO
import known_plan_oracle as KO
from test_gpu_plan import _ev as _plan_ev, _scene, _params, _same, _summ_same
from test_gpu_navigate import _wall_cloud, _ev as _nav_ev, _min_true_clearance
from test_gpu_observe import _records, _wall_poses
from test_gpu_navigate_unknown import START, GOAL, rig, seed_box, _summary, _positions, _same_logs

pytestmark = pytest.mark.gpu


def _fields(ev, starts, shape, w):
    import torch
    S = len(starts)
    d_g = torch.empty(S * int(np.prod(shape)), dtype=torch.float64, device="cuda")
    if S == 1:
        ev.frontend_path_field_device(starts[0], d_g.data_ptr(), unknown_weight=w)
    else:
        ev.frontend_path_fields_device(starts, d_g.data_ptr(), unknown_weight=w)
    torch.cuda.synchronize()
    return d_g.cpu().numpy().reshape((S,) + tuple(shape))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _marked_scene(seed=3):
    """the planning tests' three-slit map with seeded known boxes (isdf_map_mark_known)"""
    occ, start, goals = _scene(8, seed=seed)
    ev = _plan_ev("Ball", occ)
    rng = np.random.default_rng(seed)
    lo = rng.uniform(0, 40, (6, 3))
    ev.map_mark_known(np.concatenate([lo, lo + rng.uniform(4, 20, (6, 3))], 1))
    lo = start - 6.0
    ev.map_mark_known(np.concatenate([lo, start + 6.0]).reshape(1, 6))   # the start's surroundings
    return ev, occ, start, goals


def _observed_scene():
    """the wall scene at 1 m: the scene fused into the map, then 24 seeded poses observed"""
    scene = _wall_cloud()
    ev = _nav_ev(scene)
    ev.map_fuse_cloud(scene)
    ev.map_observe(_records(*_wall_poses(24, 5)), params=I.sense_params(sensing_horizon=12.0))
    occ = ev.get_map_u8()
    rng = np.random.default_rng(9)
    free = np.argwhere(occ == 0)
    pts = free[rng.choice(len(free), 9, replace=False)] + 0.5
    return ev, occ, pts[0], pts[1:]


SCENES = {"mark_known": _marked_scene, "observe": _observed_scene}


@pytest.mark.parametrize("scene", list(SCENES))
def test_weight_zero_equals_null_params(scene):
    ev, occ, start, goals = SCENES[scene]()
    a = ev.frontend_path_batch(start, goals)
    b = ev.frontend_path_batch(start, goals, unknown_weight=0.0)
    assert all(_same(a[k], b[k]) for k in ("xyz", "rp", "offsets", "costs", "found"))
    assert np.array_equal(_bits(_fields(ev, [start], occ.shape, None)), _bits(_fields(ev, [start], occ.shape, 0.0)))
    starts = np.concatenate([[start], goals[:3]])
    assert np.array_equal(_bits(_fields(ev, starts, occ.shape, None)), _bits(_fields(ev, starts, occ.shape, 0.0)))
    heads = np.zeros((len(goals), 9))
    heads[:, :3] = start
    p0 = _params(ev, flags=I.PLAN_CERTIFY)
    pz = _params(ev, flags=I.PLAN_CERTIFY, unknown_weight=0.0)
    ra, _ = ev.plan_states(heads, goals, p0)
    rb, _ = ev.plan_states(heads, goals, pz)
    keys = ("stage", "path_nodes", "pieces", "obstacle_points", "midend_ret", "backend_ret", "backend_iterations", "path_cost", "midend_f",
            "backend_f", "duration", "path", "T", "coeffs")
    assert all(_same(x[k], y[k]) for x, y in zip(ra, rb) for k in keys) and all(_summ_same(x["certify"], y["certify"]) for x, y in zip(ra, rb))
    ev.close()


@pytest.mark.parametrize("scene", list(SCENES))
@pytest.mark.parametrize("w", [0.5, 3.0])
def test_weighted_fields_and_paths_equal_the_serial_dijkstra(scene, w):
    ev, occ, start, goals = SCENES[scene]()
    info = ev.map_info()
    bmin, res = np.asarray(info["bmin"]), info["res"]
    known = ev.get_map_known_u8().astype(bool)
    assert known.any() and not known.all()
    trav = FO.traversable(occ, ev.frontend_feasibility(*occ.shape))
    vox = lambda p: tuple(np.floor((np.asarray(p) - bmin) / res).astype(int))   # noqa: E731
    src = vox(start)
    ref = KO.dijkstra(trav, known, src, w)
    assert not np.array_equal(_bits(ref), _bits(FO.dijkstra(trav, src))), "the surcharge changes nothing on this scene"
    assert np.array_equal(_bits(_fields(ev, [start], occ.shape, w)[0]), _bits(ref))
    starts = np.concatenate([[start], goals[:3], [start]])   # a repeated start shares no state with its twin
    got = _fields(ev, starts, occ.shape, w)
    for s, p in enumerate(starts):
        assert np.array_equal(_bits(got[s]), _bits(KO.dijkstra(trav, known, vox(p), w))), s
    res_b = ev.frontend_path_batch(start, goals, unknown_weight=w)
    for b, g in enumerate(goals):
        t = vox(g)
        assert res_b["found"][b] == np.isfinite(ref[t])
        assert _same(res_b["costs"][b], ref[t] if np.isfinite(ref[t]) else np.inf)
        nodes = np.floor((res_b["paths"][b] - bmin) / res).astype(int)
        assert np.array_equal(nodes, KO.path(ref, known, src, t, w) if np.isfinite(ref[t]) else np.array([src]))
        one = ev.frontend_path(start, g, unknown_weight=w)
        assert _same(one[0], res_b["paths"][b]) and _same(one[1], res_b["roll_pitch"][b]) and _same(one[2], res_b["costs"][b])
    # pairs: each pair alone, across max_fields and a permutation
    pst = np.concatenate([np.repeat([start], 3, 0), goals[:4]])   # three pairs share a start voxel
    pgl = np.concatenate([goals[:3], goals[4:8][::-1]])
    full = ev.frontend_path_pairs(pst, pgl, unknown_weight=w)
    for mf in (0, 1):
        again = ev.frontend_path_pairs(pst, pgl, max_fields=mf, unknown_weight=w)
        assert all(_same(full[k], again[k]) for k in ("xyz", "rp", "offsets", "costs", "found"))
    perm = np.random.default_rng(1).permutation(len(pst))
    pp = ev.frontend_path_pairs(pst[perm], pgl[perm], max_fields=1, unknown_weight=w)
    for k, b in enumerate(perm):
        assert _same(pp["paths"][k], full["paths"][b]) and _same(pp["costs"][k], full["costs"][b])
    for b in range(len(pst)):
        one = ev.frontend_path(pst[b], pgl[b], unknown_weight=w)
        assert _same(one[0], full["paths"][b]) and _same(one[2], full["costs"][b])
    ev.close()


def test_known_rows_gather_equals_the_restatement():
    occ, _, _ = _scene(1)
    ev = _plan_ev("Ball", occ, kernels=False)
    info = ev.map_info()
    bmin, bmax, res = np.asarray(info["bmin"]), np.asarray(info["bmax"]), info["res"]
    rng = np.random.default_rng(4)
    walk = lambda n, s: np.cumsum(rng.normal(size=(n, 3)) * 1.5, axis=0) + s   # noqa: E731
    plans = [np.zeros((0, 3)), walk(1, [10.0, 20.0, 15.0]), walk(40, [24.0, 24.0, 17.0]), walk(12, [5.0, 40.0, 30.0]),
             np.array([[-3.0, 2.0, 1.0], [47.0, 50.0, 40.0]]), walk(25, [30.0, 10.0, 9.0])]
    h, off = 13.0 / 3.0, np.array([0.25, -0.5, 0.0])
    # nothing known: every known row lists every voxel of its boxes
    rows = np.array([0, 1, 7, 12, 1, 30], dtype=np.int32)
    got = ev.gather_obstacle_points_batch(plans, h, off, known_rows=rows)
    for b, wp in enumerate(plans):
        assert _same(got[b], KO.gather(occ, None, bmin, bmax, res, wp, h, off, rows[b]).reshape(-1, 3)), b
    plain = ev.gather_obstacle_points_batch(plans, h, off)
    zero = ev.gather_obstacle_points_batch(plans, h, off, known_rows=np.zeros(len(plans), np.int32))
    assert all(_same(a, b) for a, b in zip(plain, zero))
    # seeded known boxes and observed-free voxels of any row count
    lo = rng.uniform(0, 40, (8, 3))
    ev.map_mark_known(np.concatenate([lo, lo + rng.uniform(3, 15, (8, 3))], 1))
    known = ev.get_map_known_u8().astype(bool)
    for trial in range(3):
        rows = rng.integers(0, 45, len(plans)).astype(np.int32)
        got = ev.gather_obstacle_points_batch(plans, h, off, known_rows=rows, set_as_points=trial == 0)
        for b, wp in enumerate(plans):
            assert _same(got[b], KO.gather(occ, known, bmin, bmax, res, wp, h, off, rows[b]).reshape(-1, 3)), (trial, b)
    bad = np.zeros(len(plans), np.int32)
    bad[2] = -1
    with pytest.raises(I.IsdfError):
        ev.gather_obstacle_points_batch(plans, h, off, known_rows=bad)
    ev.close()


def _plan_expected_points(ev, plan, occ, known, p):
    """the restatement's obstacle count of an OPTIMISED plan under ISDF_PLAN_KNOWN_PREFIX"""
    info = ev.map_info()
    bmin, bmax, res = np.asarray(info["bmin"]), np.asarray(info["bmax"]), info["res"]
    nodes = np.floor((plan["path"] - bmin) / res).astype(int)
    S, N = len(nodes), plan["pieces"]
    g = KO.waypoint_gap(S, res, p.parlength)
    wps = plan["path"][[(j + 1) * g for j in range(N - 1)]] if N > 1 else np.zeros((0, 3))
    rows = KO.known_rows(nodes, known, g, N)
    return len(KO.gather(occ, known, bmin, bmax, res, wps, p.half_extent, np.asarray(p.offset[:]), rows)), rows


def test_plan_known_prefix_gathers_the_restatement_and_nothing_known_changes_nothing():
    occ, start, goals = _scene(6, seed=11)
    ev = _plan_ev("Ball", occ)
    heads = np.zeros((len(goals), 9))
    heads[:, :3] = start
    keys = ("stage", "path_nodes", "pieces", "obstacle_points", "midend_ret", "backend_ret", "backend_iterations", "path_cost", "midend_f",
            "backend_f", "duration", "path", "T", "coeffs")
    # nothing known: k* = 0, the flag gathers what no flag gathers
    a, _ = ev.plan_states(heads, goals, _params(ev, flags=I.PLAN_CERTIFY))
    b, _ = ev.plan_states(heads, goals, _params(ev, flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_PREFIX))
    assert all(_same(x[k], y[k]) for x, y in zip(a, b) for k in keys) and all(_summ_same(x["certify"], y["certify"]) for x, y in zip(a, b))
    # known space around the start and along a band: the flag's counts are the restatement's
    ev.map_mark_known(np.array([[0, 0, 0, 30, 30, 48], [start[0] - 8, start[1] - 8, 0, start[0] + 8, start[1] + 8, 48]], dtype=np.float64))
    known = ev.get_map_known_u8().astype(bool)
    for w in (0.0, 2.0):
        p = _params(ev, flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_PREFIX, unknown_weight=w)
        got, _ = ev.plan_states(heads, goals, p)
        some_rows = False
        for r in got:
            if r["stage"] != I.OPTIMISED:
                continue
            n, rows = _plan_expected_points(ev, r, occ, known, p)
            assert r["obstacle_points"] == n
            some_rows |= rows > 0
        assert some_rows, "no plan has a known row: the test checks nothing"
        again, _ = ev.plan_states(heads, goals, p)
        assert all(_same(x[k], y[k]) for x, y in zip(got, again) for k in keys)
    ev.close()


def test_refusals():
    import torch
    ev, occ, start, goals = _marked_scene()
    d_g = torch.empty(occ.size, dtype=torch.float64, device="cuda")
    st = (C.c_double * 3)(*start)
    for w, res in ((-1.0, None), (np.nan, None), (np.inf, None), (-0.0, 0), (0.0, 0), (1e300, 0)):
        prm = I.FrontPathParams(unknown_weight=w)
        rc = ev.lib.isdf_frontend_path_field_device(ev.h, st, C.byref(prm), d_g.data_ptr(), None)
        assert (rc == -1) if res is None else (rc == 0), w
        p = _params(ev, flags=I.PLAN_CERTIFY)
        p.frontpath.unknown_weight = w
        if res is None:
            with pytest.raises(I.IsdfError):
                ev.plan_pairs(np.array([start]), goals[:1], p)
    for k in range(2):
        prm = I.FrontPathParams()
        prm.reserved_[k] = 1
        assert ev.lib.isdf_frontend_path_field_device(ev.h, st, C.byref(prm), d_g.data_ptr(), None) == -1
        p = _params(ev, flags=I.PLAN_CERTIFY)
        p.frontpath.reserved_[k] = 1
        with pytest.raises(I.IsdfError):
            ev.plan_pairs(np.array([start]), goals[:1], p)
    p = _params(ev, flags=I.PLAN_CERTIFY | 4)   # 4 is not a flag
    with pytest.raises(I.IsdfError):
        ev.plan_pairs(np.array([start]), goals[:1], p)
    ev.close()


def _run(cams, rounds, w=1.0, **cam):
    scene = _wall_cloud()
    ev = _nav_ev(scene)
    out = ev.navigate(START, GOAL, rounds=rounds, horizon=0.5, sense_every=25, tol=1.0,
                      plan_params=ev.plan_params(flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_PREFIX, unknown_weight=w, backend_max_iterations=200),
                      sense_params=rig(cams, **cam), fallback="brake", unknown="occupied", known_boxes=seed_box(START[0]))
    known = ev.get_map_known_u8().astype(bool)
    ev.close()
    return out, scene, known


def _check_run(out, scene, known):
    clear = _min_true_clearance(out, scene)
    pos = _positions(out)
    a = out["actions"][:, 0]
    print(_summary(out), "rounds", len(out["times"]), "min true clearance", clear, "furthest x", pos[:, 0].min(), "arrived",
          out["status"][0] == I.NAV_ARRIVED, "actions", a)
    assert clear >= 0.0
    idx = np.floor(pos).astype(int)   # the frame is [0, 40] x [0, 24] x [0, 8] at 1 m
    assert known[idx[:, 0], idx[:, 1], idx[:, 2]].all(), "a flown position left the known region"
    assert (out["verdicts"][a == I.NAV_COMMITTED, 0] == I.CERTIFIED).all()


def test_prefer_known_front_and_back_rig():
    out, scene, known = _run(2, 60)
    _check_run(out, scene, known)
    again, _, _ = _run(2, 60)
    assert _same_logs(out, again)


def test_prefer_known_four_wide_cameras():
    out, scene, known = _run(4, 120, fx=200.0, fy=200.0)
    _check_run(out, scene, known)
    again, _, _ = _run(4, 120, fx=200.0, fy=200.0)
    assert _same_logs(out, again)
