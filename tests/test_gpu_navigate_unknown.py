"""Evaluator.navigate(unknown="occupied"): certificates against occupied-or-unseen space, and vehicles that commit only to stops inside what
their cameras have seen. Scenario (recorded in DESIGN §3.22): the wall test's frame, robot and scene (tests/test_gpu_navigate.py), start
(36.5, 12.5, 4.5), goal (2.5, 12.5, 4.5): the vehicle flies -x, away from the reference camera, which looks along body x (world +x, yaw 0).
Under "occupied" the space first known is the 5 x 5 x 5-voxel block around the start.
  free, front camera      the vehicle never sees what lies ahead and flies into the wall: a flown pose has negative true clearance;
  occupied, front camera  it never leaves the known region, and every flown pose is clear;
  occupied, front + back  it commits round after round and every flown pose is clear, but it does not get past the first metres: the
                          route bends toward the wall's corner, and the voxels diagonally ahead of it lie in the gap between the
                          cameras' 79.2 deg fields of view until the vehicle is within its margin of them (a four-camera rig of the
                          reference camera leaves 10.8 deg gaps at the diagonals and does the same);
  occupied, four wide     four cameras with fx = fy = 200 (116 x 100 deg fields, overlapping): it arrives, taking NAV_COMMITTED rounds,
                          and every flown pose is clear;
and two runs give identical logs, and unknown="free" passed explicitly equals omitting it."""
import numpy as np
import pytest
import isdf_b200 as I
from test_gpu_navigate import _wall_cloud, _ev, _min_true_clearance, torch_equal

pytestmark = pytest.mark.gpu

START, GOAL = np.array([[36.5, 12.5, 4.5]]), np.array([[2.5, 12.5, 4.5]])
CAM02BODY = np.array([[0, 0, 1, 0], [-1, 0, 0, 0], [0, -1, 0, 0], [0, 0, 0, 1]], dtype=np.float64)


def rig(k, **kw):
    """k cameras at yaw 0, 180 (k = 2) or 0, 90, 180, 270 degrees (k = 4): cam_to_body = Rz(yaw) cam02body, exact in FP64; kw replaces
    other camera fields (e.g. fx, fy)"""
    yaws = {1: [0], 2: [0, 2], 4: [0, 1, 2, 3]}[k]
    cams = []
    for q in yaws:
        c, s = [(1, 0), (0, 1), (-1, 0), (0, -1)][q]
        Rz = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=np.float64)
        cams.append(I.sense_params(sensing_horizon=15.0, cam_to_body=(Rz @ CAM02BODY).reshape(-1), **kw))
    return cams


def seed_box(p, half=2.5):
    """the 5 x 5 x 5-voxel block around a voxel-centre position, as a closed box"""
    return np.concatenate([np.asarray(p) - half, np.asarray(p) + half]).reshape(1, 6)


def _run(unknown=None, cams=1, rounds=120, **cam):
    scene = _wall_cloud()
    ev = _ev(scene)
    kw = {} if unknown is None else dict(unknown=unknown)
    if unknown == "occupied":
        kw["known_boxes"] = seed_box(START[0])
    out = ev.navigate(START, GOAL, rounds=rounds, horizon=0.5, sense_every=25, tol=1.0,
                      plan_params=ev.plan_params(flags=I.PLAN_CERTIFY, backend_max_iterations=200),
                      sense_params=rig(cams, **cam) if cams > 1 else I.sense_params(sensing_horizon=15.0), fallback="brake", **kw)
    known = ev.get_map_known_u8().astype(bool)
    assert ev.unknown_policy() == I.UNKNOWN_FREE   # restored on return
    ev.close()
    return out, scene, known


def _summary(out):
    keys = ("status", "rounds_flown", "replans", "failed_replans", "uncertified_rounds", "brakes", "held_rounds", "commits")
    return {k: out[k] for k in keys if k in out}


def _positions(out):
    return np.concatenate([lg[:, :, 1:4].reshape(-1, 3).cpu().numpy() for _, lg in out["logs"]])


def _same_logs(a, b):
    return np.array_equal(a["actions"], b["actions"]) and len(a["logs"]) == len(b["logs"]) and all(
        np.array_equal(ia, ib) and torch_equal(la, lb) for (ia, la), (ib, lb) in zip(a["logs"], b["logs"]))


def test_free_flies_into_the_unseen_wall():
    out, scene, known = _run()
    clear = _min_true_clearance(out, scene)
    print(_summary(out), out["actions"][:, 0], "min true clearance", clear)
    assert clear < 0.0   # what unknown="occupied" exists for
    assert not known.any() and "commits" not in out and all("observe" not in t for t in out["times"])
    explicit, _, _ = _run("free")
    assert _same_logs(out, explicit) and np.array_equal(out["status"], explicit["status"])


def test_occupied_front_camera_stays_in_the_known_region():
    out, scene, known = _run("occupied")
    clear = _min_true_clearance(out, scene)
    print(_summary(out), out["actions"][:, 0], "min true clearance", clear)
    assert clear >= 0.0
    pos = _positions(out)
    idx = np.floor(pos).astype(int)   # the frame is [0, 40] x [0, 24] x [0, 8] at 1 m
    assert known[idx[:, 0], idx[:, 1], idx[:, 2]].all(), "a flown position left the known region"
    assert out["status"][0] != I.NAV_ARRIVED
    assert all("observe" in t for t in out["times"])


def test_occupied_front_and_back_commits_and_stays_clear():
    out, scene, known = _run("occupied", cams=2, rounds=60)
    clear = _min_true_clearance(out, scene)
    a = out["actions"][:, 0]
    print(_summary(out), a, "min true clearance", clear, "last position", _positions(out)[-1])
    assert clear >= 0.0
    assert (a == I.NAV_COMMITTED).any() and out["commits"][0] == int((a == I.NAV_COMMITTED).sum())
    assert (out["verdicts"][a == I.NAV_COMMITTED, 0] == I.CERTIFIED).all()
    pos = _positions(out)
    idx = np.floor(pos).astype(int)
    assert known[idx[:, 0], idx[:, 1], idx[:, 2]].all()


def test_occupied_wide_rig_arrives_with_commits():
    out, scene, known = _run("occupied", cams=4, fx=200.0, fy=200.0)
    clear = _min_true_clearance(out, scene)
    a = out["actions"][:, 0]
    print(_summary(out), a, "min true clearance", clear)
    assert clear >= 0.0
    assert out["status"][0] == I.NAV_ARRIVED
    assert (a == I.NAV_COMMITTED).any() and out["commits"][0] == int((a == I.NAV_COMMITTED).sum())
    assert (out["verdicts"][a == I.NAV_COMMITTED, 0] == I.CERTIFIED).all()
    again, _, _ = _run("occupied", cams=4, fx=200.0, fy=200.0)
    assert _same_logs(out, again)
