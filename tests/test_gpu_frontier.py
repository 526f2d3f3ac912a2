"""Frontiers of known space, frontier goals and known-only planning (DESIGN §3.24), against tests/frontier_oracle.py.
  frontiers   on seeded maps with known grids from isdf_map_mark_known boxes and from isdf_map_observe of the wall poses: T_b, F, the labels
              and the cluster table equal the restatement bit for bit (T_b's masks from isdf_frontend_feasibility on a second context whose
              map is the blocked grid), through both forms;
  goals       every pair's record equals the restatement (its g is the serial Dijkstra's over T_b), host and device forms agree, under
              pair permutations, for max_fields 0 and 1, and run to run; nothing known: no frontier and NONE unless start voxel == goal
              voxel; everything known: no frontier and GOAL wherever the goal is reachable;
  known-only  plans under ISDF_PLAN_KNOWN_ONLY follow the parent rule over T_b, keep every node but the start in T_b, gather every row from
              the blocked grid, and equal the same call with ISDF_PLAN_KNOWN_PREFIX added;
  refusals    bad goal_weight, min_cluster_voxels < 1, a non-zero reserved_, an unknown flag (4 still is one);
  navigate    the wall scenario under unknown="occupied" with explore=True and PLAN_CERTIFY | PLAN_KNOWN_PREFIX: every flown position lies
              in a known voxel, the true clearance stays >= 0, and two runs give identical logs. Whether the vehicle arrives is printed,
              not asserted. Recorded on an H100 80GB HBM3 at 700 W (DESIGN §3.24):
                front + back, 60 rounds: 23 rounds flown, furthest x 23.5, then held 37 rounds (TIMEOUT), 39 frontier plans;
                four cameras fx = fy = 200, 120 rounds: 14 rounds flown, furthest x 23.5, then held 106 rounds (TIMEOUT), 107 frontier plans;
                minimum true clearance 0.866 m in both. The vehicle reaches a frontier and is held there: at rest its cameras see
                nothing new, and with goal_weight 1 the frontier voxel it stands on keeps the least score."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import frontier_oracle as FR
import known_plan_oracle as KO
from test_gpu_plan import _ev as _plan_ev, _params, _same
from test_gpu_navigate import _wall_cloud, _ev as _nav_ev, _min_true_clearance
from test_gpu_plan_known import _marked_scene, _observed_scene
from test_gpu_navigate_unknown import START, GOAL, rig, seed_box, _summary, _positions, _same_logs

pytestmark = pytest.mark.gpu


def _scene(name):
    """-> ev, occ, start, goals, twin(u8 grid) -> a context like ev's with that map"""
    if name == "mark_known":
        ev, occ, start, goals = _marked_scene()
        return ev, occ, start, goals, lambda u8: _plan_ev("Ball", u8)
    ev, occ, start, goals = _observed_scene()
    info = ev.map_info()

    def twin(u8):
        t = _nav_ev(_wall_cloud())
        t.set_map_u8(u8, info["bmin"], info["res"])
        return t
    return ev, occ, start, goals, twin


def _oracle(ev, occ, twin):
    info = ev.map_info()
    known = ev.get_map_known_u8().astype(bool)
    To = FR.traversable(occ, ev.frontend_feasibility(*occ.shape))
    blk = FR.blocked(occ, known)
    t = twin(blk.astype(np.uint8))
    Tb = FR.traversable(blk, t.frontend_feasibility(*occ.shape))
    t.close()
    F = FR.frontier(To, Tb)
    lab, table = FR.clusters(F, np.asarray(info["bmin"]), info["res"])
    return dict(known=known, To=To, Tb=Tb, F=F, lab=lab, table=table, bmin=np.asarray(info["bmin"]), res=info["res"])


def _check_frontiers(fr, o):
    F = o["F"]
    assert fr["info"]["traversable_blocked"] == int(o["Tb"].sum())
    assert fr["info"]["frontier_voxels"] == int(F.sum()) and fr["info"]["clusters"] == len(o["table"])
    flat = np.arange(F.size, dtype=np.int64).reshape(F.shape)
    assert np.array_equal(fr["voxels"], flat[F]) and np.array_equal(fr["cluster_of"], o["lab"][F])
    for rec, c in zip(fr["clusters"], o["table"]):
        assert rec["id"] == c["id"] and rec["size"] == c["size"]
        assert np.array_equal(rec["bmin"], c["bmin"]) and np.array_equal(rec["bmax"], c["bmax"])
        assert np.array_equal(rec["centroid"].view(np.uint64), c["centroid"].view(np.uint64))


SCENES = ["mark_known", "observe"]


@pytest.mark.parametrize("scene", SCENES)
def test_frontiers_equal_the_restatement(scene):
    import torch
    ev, occ, start, goals, twin = _scene(scene)
    o = _oracle(ev, occ, twin)
    assert o["F"].any() and len(o["table"]) > 1 and not np.array_equal(o["Tb"], o["To"])
    fr = ev.map_frontiers()
    assert np.array_equal(ev.dbg_frontpath_traversable(), o["Tb"])   # the last traversability built: T_b
    _check_frontiers(fr, o)
    n, nc = fr["info"]["frontier_voxels"], fr["info"]["clusters"]
    dv, dc = torch.empty(n, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.int64, device="cuda")
    dt = torch.empty((nc, 64), dtype=torch.uint8, device="cuda")
    with pytest.raises(I.IsdfError):   # a cap too small
        ev.map_frontiers_device(n - 1, dv.data_ptr(), dc.data_ptr(), nc, dt.data_ptr())
    info = ev.map_frontiers_device(n, dv.data_ptr(), dc.data_ptr(), nc, dt.data_ptr())
    assert info["frontier_voxels"] == n
    assert np.array_equal(dv.cpu().numpy(), fr["voxels"]) and np.array_equal(dc.cpu().numpy(), fr["cluster_of"])
    assert np.array_equal(dt.cpu().numpy().reshape(-1).view(I.FRONTIER_CLUSTER_DTYPE), fr["clusters"])
    ev.close()


def _expected(o, starts, goals, **kw):
    dims = o["F"].shape
    out = []
    for s, gl in zip(starts, goals):
        g = FR.field(o["Tb"], FR.voxel(s, o["bmin"], o["res"], dims))
        out.append(FR.select(g, o["F"], o["lab"], o["table"], gl, FR.voxel(gl, o["bmin"], o["res"], dims), o["bmin"], o["res"], **kw))
    return out


def _records_equal(got, exp):
    for r, e in zip(got, exp):
        assert r["kind"] == e["kind"] and r["voxel"] == e["voxel"] and r["cluster"] == e["cluster"], (r, e)
        for k in ("g", "score"):
            assert np.float64(r[k]).view(np.uint64) == np.float64(e[k]).view(np.uint64), (k, r, e)
        assert np.array_equal(np.asarray(r["point"]).view(np.uint64), np.asarray(e["point"]).view(np.uint64))


def _pairs(o, goals):
    """four pairs from one start in T_b (seeded), three from the goals, and a start that is its own goal"""
    tb = np.argwhere(o["Tb"])
    start = o["bmin"] + (tb[np.random.default_rng(6).integers(len(tb))] + 0.5) * o["res"]
    far = np.array([[0.5, 0.5, 0.5]]) if goals.max() > 30 else np.array([[2.5, 12.5, 4.5]])
    starts = np.concatenate([np.repeat([start], 4, 0), goals[:3], [start]])
    gls = np.concatenate([goals[3:6], far, goals[5:8], [start]])
    return starts, gls


@pytest.mark.parametrize("scene", SCENES)
def test_frontier_goals_equal_the_restatement(scene):
    import torch
    ev, occ, start, goals, twin = _scene(scene)
    o = _oracle(ev, occ, twin)
    starts, gls = _pairs(o, goals)
    for kw in (dict(), dict(goal_weight=2.5, min_cluster_voxels=20)):
        p = ev.frontier_params(**kw)
        got, info = ev.frontier_goals(starts, gls, p)
        exp = _expected(o, starts, gls, **kw)
        print(kw, [int(r["kind"]) for r in got])
        _records_equal(got, exp)
        assert info["frontier_voxels"] == int(o["F"].sum())
        if not kw:
            assert any(r["kind"] == I.FRONTIER_FRONTIER for r in got) and any(r["kind"] == I.FRONTIER_GOAL for r in got)
        for mf in (0, 1):
            again, _ = ev.frontier_goals(starts, gls, p, max_fields=mf)
            assert np.array_equal(again.view(np.uint8), got.view(np.uint8))
        perm = np.random.default_rng(2).permutation(len(starts))
        pp, _ = ev.frontier_goals(starts[perm], gls[perm], p, max_fields=1)
        assert np.array_equal(pp.view(np.uint8), got[perm].view(np.uint8))
        dr, _ = ev.frontier_goals_device(torch.as_tensor(starts, device="cuda"), torch.as_tensor(gls, device="cuda"), p)
        assert np.array_equal(I.decode_frontier_goals(dr).view(np.uint8), got.view(np.uint8))
    ev.close()


def test_nothing_known_and_everything_known():
    occ, start, goals = __import__("test_gpu_plan")._scene(6, seed=3)
    ev = _plan_ev("Ball", occ)
    starts, gls = np.repeat([start], len(goals) + 1, 0), np.concatenate([goals, [start]])
    fr = ev.map_frontiers()
    assert fr["info"]["traversable_blocked"] == 0 and len(fr["voxels"]) == 0 and len(fr["clusters"]) == 0
    got, _ = ev.frontier_goals(starts, gls)
    assert list(got["kind"]) == [I.FRONTIER_NONE] * len(goals) + [I.FRONTIER_GOAL]
    ev.map_mark_known(np.array([[-1.0, -1.0, -1.0, 60.0, 60.0, 60.0]]))
    fr = ev.map_frontiers()
    assert fr["info"]["traversable_blocked"] > 0 and len(fr["voxels"]) == 0
    got, _ = ev.frontier_goals(starts, gls)
    found = ev.frontend_path_batch(start, gls)["found"]
    assert np.array_equal(got["kind"] == I.FRONTIER_GOAL, found) and ((got["kind"] == I.FRONTIER_GOAL) | (got["kind"] == I.FRONTIER_NONE)).all()
    ev.close()


@pytest.mark.parametrize("scene", SCENES)
def test_known_only_plans_follow_t_b(scene):
    ev, occ, start, goals, twin = _scene(scene)
    o = _oracle(ev, occ, twin)
    info = ev.map_info()
    bmin, bmax, res = np.asarray(info["bmin"]), np.asarray(info["bmax"]), info["res"]
    start = _pairs(o, goals)[0][0]   # in T_b
    rec, _ = ev.frontier_goals(np.repeat([start], len(goals), 0), goals)
    targets = np.asarray(rec["point"])
    heads = np.zeros((len(goals), 9))
    heads[:, :3] = start
    p = _params(ev, flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_ONLY)
    got, _ = ev.plan_states(heads, targets, p)
    both, _ = ev.plan_states(heads, targets, _params(ev, flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_ONLY | I.PLAN_KNOWN_PREFIX))
    weighted, _ = ev.plan_states(heads, targets, _params(ev, flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_ONLY, unknown_weight=2.0))
    keys = ("stage", "path_nodes", "pieces", "obstacle_points", "midend_ret", "backend_ret", "path_cost", "midend_f", "backend_f", "path", "T",
            "coeffs")
    assert all(_same(x[k], y[k]) for x, y in zip(got, both) for k in keys)
    assert all(_same(x[k], y[k]) for x, y in zip(got, weighted) for k in keys)
    src = FR.voxel(start, bmin, res, occ.shape)
    g = FR.field(o["Tb"], src)
    optimised = 0
    for r, t in zip(got, targets):
        tv = FR.voxel(t, bmin, res, occ.shape)
        nodes = np.floor((r["path"] - bmin) / res).astype(int)
        assert _same(r["path_cost"], g[tv])
        assert np.array_equal(nodes, KO.path(g, None, src, tv, 0.0) if np.isfinite(g[tv]) else np.array([src]))
        assert o["Tb"][tuple(nodes[1:].T)].all()
        if r["stage"] != I.OPTIMISED:
            continue
        optimised += 1
        S, N = len(nodes), r["pieces"]
        gap = KO.waypoint_gap(S, res, p.parlength)
        wps = r["path"][[(j + 1) * gap for j in range(N - 1)]] if N > 1 else np.zeros((0, 3))
        assert r["obstacle_points"] == len(KO.gather(occ, o["known"], bmin, bmax, res, wps, p.half_extent, np.asarray(p.offset[:]), N - 1))
    assert optimised > 0
    ev.close()


def test_refusals():
    ev, occ, start, goals, _ = _scene("mark_known")
    lib = ev.lib
    st, gl = np.ascontiguousarray([start]), np.ascontiguousarray(goals[:1])
    out = np.zeros(1, dtype=I.FRONTIER_GOAL_DTYPE)
    call = lambda p: lib.isdf_frontier_goals(ev.h, 1, I._dp(st.reshape(-1)), I._dp(gl.reshape(-1)), C.byref(p), 0, out.ctypes.data, None)  # noqa: E731
    assert call(ev.frontier_params()) == 0
    for kw in (dict(goal_weight=0.0), dict(goal_weight=-1.0), dict(goal_weight=np.nan), dict(goal_weight=np.inf), dict(min_cluster_voxels=0),
               dict(min_cluster_voxels=-3), dict(reserved_=1)):
        assert call(ev.frontier_params(**kw)) == -1, kw
    assert lib.isdf_frontier_goals(ev.h, 1, I._dp(st.reshape(-1)), I._dp(gl.reshape(-1)), None, -1, out.ctypes.data, None) == -1
    for flags in (I.PLAN_CERTIFY | 4, I.PLAN_CERTIFY | 32):
        with pytest.raises(I.IsdfError):
            ev.plan_pairs(st, gl, _params(ev, flags=flags))
    ev.plan_pairs(st, gl, _params(ev, flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_ONLY))
    ev.close()


def _run(cams, rounds, **cam):
    scene = _wall_cloud()
    ev = _nav_ev(scene)
    out = ev.navigate(START, GOAL, rounds=rounds, horizon=0.5, sense_every=25, tol=1.0,
                      plan_params=ev.plan_params(flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_PREFIX, unknown_weight=1.0, backend_max_iterations=200),
                      sense_params=rig(cams, **cam), fallback="brake", unknown="occupied", known_boxes=seed_box(START[0]), explore=True)
    known = ev.get_map_known_u8().astype(bool)
    ev.close()
    return out, scene, known


def _check_run(out, scene, known):
    clear = _min_true_clearance(out, scene)
    pos = _positions(out)
    a = out["actions"][:, 0]
    print(_summary(out), "rounds", len(out["times"]), "min true clearance", clear, "furthest x", pos[:, 0].min(), "arrived",
          out["status"][0] == I.NAV_ARRIVED, "frontier plans", out["frontier_plans"], "kinds", out["subgoal_kinds"][:, 0], "actions", a)
    assert clear >= 0.0
    idx = np.floor(pos).astype(int)   # the frame is [0, 40] x [0, 24] x [0, 8] at 1 m
    assert known[idx[:, 0], idx[:, 1], idx[:, 2]].all(), "a flown position left the known region"
    assert out["subgoal_kinds"].shape == out["actions"].shape and out["frontier_plans"][0] == int((out["subgoal_kinds"] == I.FRONTIER_FRONTIER).sum())


def test_explore_needs_unknown_occupied():
    ev = _nav_ev(_wall_cloud())
    with pytest.raises(ValueError):
        ev.navigate(START, GOAL, rounds=1, horizon=0.5, explore=True)
    ev.close()


def test_explore_front_and_back_rig():
    out, scene, known = _run(2, 60)
    _check_run(out, scene, known)
    again, _, _ = _run(2, 60)
    assert _same_logs(out, again)


def test_explore_four_wide_cameras():
    out, scene, known = _run(4, 120, fx=200.0, fy=200.0)
    _check_run(out, scene, known)
    again, _, _ = _run(4, 120, fx=200.0, fy=200.0)
    assert _same_logs(out, again)
