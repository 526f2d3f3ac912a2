"""Evaluator.navigate: vehicles fly to their goals through a world they only see through the reference's depth camera, fusing what they
sense into one map and replanning from their moving states. Scenarios (recorded in DESIGN §3.20):
  wall   a 40 x 24 x 8 m frame at 1 m (Ball robot, vmax 3 m/s), the box [18, 21] x [6, 18] x [0, 8] (a wall 3 m thick), start
         (2.5, 12.5, 4.5), goal (36.5, 12.5, 4.5), camera horizon 15 m, rounds of 0.5 s: the wall is out of range at the start, so the
         first plan flies straight through it and a later check must catch it;
  fleet  the same world, 4 vehicles at y = 3.5, 9.5, 14.5, 20.5 flying +x.
Every flown pose is held against the whole world (pose_clearance_device in a context holding the true map)."""
import numpy as np
import pytest
import isdf_b200 as I
from test_gpu_plan import _cfg

pytestmark = pytest.mark.gpu

DIMS, BMIN, RES = (40, 24, 8), np.zeros(3), 1.0


def _wall_cloud(step=0.25):
    """the surface of the box [18, 21] x [6, 18] x [0, 8] as float32 points"""
    xs, ys, zs = np.arange(18, 21 + 1e-9, step), np.arange(6, 18 + 1e-9, step), np.arange(0, 8 + 1e-9, step)
    faces = []
    for x in (18.0, 21.0):
        Y, Z = np.meshgrid(ys, zs, indexing="ij"); faces.append(np.stack([np.full(Y.size, x), Y.ravel(), Z.ravel()], 1))
    for y in (6.0, 18.0):
        X, Z = np.meshgrid(xs, zs, indexing="ij"); faces.append(np.stack([X.ravel(), np.full(X.size, y), Z.ravel()], 1))
    X, Y = np.meshgrid(xs, ys, indexing="ij"); faces.append(np.stack([X.ravel(), Y.ravel(), np.full(X.size, 8.0)], 1))
    return np.concatenate(faces).astype(np.float32)


def _nav_cfg():
    cfg = _cfg()
    cfg.vmax = 3.0
    return cfg


def _ev(scene):
    ev = I.Evaluator(_nav_cfg())
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    ev.set_map_u8(np.zeros(DIMS, np.uint8), BMIN, RES)
    ev.set_sense_cloud(scene)
    return ev


def _truth(scene):
    ev = I.Evaluator(_cfg())
    ev.set_shape_named("Ball")
    ev.set_map_u8(np.zeros(DIMS, np.uint8), BMIN, RES)
    ev.map_fuse_cloud(scene)   # the whole world in the same frame
    return ev


def _run(starts, goals, rounds=60):
    scene = _wall_cloud()
    ev = _ev(scene)
    out = ev.navigate(starts, goals, rounds=rounds, horizon=0.5, sense_every=25, tol=1.0,
                      plan_params=ev.plan_params(flags=I.PLAN_CERTIFY, backend_max_iterations=200),
                      sense_params=I.sense_params(sensing_horizon=15.0))
    ev.close()
    return out, scene


def _min_true_clearance(out, scene):
    import torch
    tr = _truth(scene)
    m = np.inf
    for _, lg in out["logs"]:
        rec = lg.reshape(-1, I.SIM_DOUBLES).contiguous()
        Q = rec.shape[0]
        p = tr.pose_clearance_params()
        clear = torch.empty(Q, dtype=torch.float64, device="cuda")
        vox = torch.empty(Q, dtype=torch.int64, device="cuda")
        summ = torch.empty((1, 48), dtype=torch.uint8, device="cuda")
        base = rec.data_ptr()
        tr.pose_clearance_device(Q, base + 8, base + 56, I.SIM_DOUBLES, p, clear.data_ptr(), vox.data_ptr(), summ.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
        m = min(m, float(clear.min()))
    tr.close()
    return m


def test_hidden_wall_triggers_a_replan_and_the_vehicle_arrives():
    starts, goals = np.array([[2.5, 12.5, 4.5]]), np.array([[36.5, 12.5, 4.5]])
    out, scene = _run(starts, goals)
    print({k: out[k] for k in ("status", "rounds_flown", "replans", "failed_replans", "uncertified_rounds")}, out["actions"].T,
          out["replan_stages"].T, out["replan_verdicts"].T)
    assert out["actions"][0, 0] == I.NAV_REPLANNED
    assert (out["actions"][1:, 0] == I.NAV_REPLANNED).any(), "the check never caught the wall"
    assert out["status"][0] == I.NAV_ARRIVED
    assert _min_true_clearance(out, scene) >= 0.0
    # two runs give identical logs
    again, _ = _run(starts, goals)
    assert len(again["logs"]) == len(out["logs"])
    for (ia, la), (ib, lb) in zip(out["logs"], again["logs"]):
        assert np.array_equal(ia, ib) and torch_equal(la, lb)


def torch_equal(a, b):
    import torch
    return bool(torch.equal(a.isnan(), b.isnan())) and bool(torch.equal(torch.nan_to_num(a), torch.nan_to_num(b)))


def test_a_fleet_arrives_and_never_touches_the_world():
    ys = [3.5, 9.5, 14.5, 20.5]
    starts = np.array([[2.5, y, 4.5] for y in ys])
    goals = np.array([[36.5, y, 4.5] for y in ys])
    out, scene = _run(starts, goals)
    print({k: out[k] for k in ("status", "rounds_flown", "replans", "failed_replans", "uncertified_rounds")}, out["actions"].T,
          out["replan_stages"].T, out["replan_verdicts"].T)
    assert (out["status"] == I.NAV_ARRIVED).all(), out["status"]
    assert _min_true_clearance(out, scene) >= 0.0
    assert len(out["times"]) == out["actions"].shape[0] and all(v >= 0 for t in out["times"] for v in t.values())
