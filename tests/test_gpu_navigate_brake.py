"""Evaluator.navigate(fallback="brake"): a vehicle whose replan fails brakes to a certified stop instead of flying on, and is then held.
Scenario (recorded in DESIGN §3.21): the wall test's frame, robot and camera (tests/test_gpu_navigate.py), start (2.5, 12.5, 4.5), goal
(31.5, 12.5, 4.5) inside the closed box shell [30, 33] x [11, 14] x [3, 6]. The shell is out of camera range at the start, so the first
plan flies to the goal; once a face next to the goal is fused the goal voxel is not traversable for the Ball robot and every replan is
NO_PATH. With "brake" the vehicle stops short of the shell and waits there (TIMEOUT); with "keep" (the control) it flies its colliding
trajectory into the shell."""
import numpy as np
import pytest
import isdf_b200 as I
from test_gpu_navigate import _ev, _min_true_clearance, torch_equal

pytestmark = pytest.mark.gpu

START, GOAL = np.array([[2.5, 12.5, 4.5]]), np.array([[31.5, 12.5, 4.5]])


def _shell_cloud(lo=(30.0, 11.0, 3.0), hi=(33.0, 14.0, 6.0), step=0.25):
    """the surface of the box [lo, hi] as float32 points"""
    ax = [np.arange(l, h + 1e-9, step) for l, h in zip(lo, hi)]
    faces = []
    for d in range(3):
        u, v = [ax[e] for e in range(3) if e != d]
        U, V = np.meshgrid(u, v, indexing="ij")
        for c in (lo[d], hi[d]):
            cols = [None, None, None]
            cols[d] = np.full(U.size, c)
            rest = [e for e in range(3) if e != d]
            cols[rest[0]], cols[rest[1]] = U.ravel(), V.ravel()
            faces.append(np.stack(cols, 1))
    return np.concatenate(faces).astype(np.float32)


def _run(fallback, rounds=40):
    scene = _shell_cloud()
    ev = _ev(scene)
    out = ev.navigate(START, GOAL, rounds=rounds, horizon=0.5, sense_every=25, tol=1.0,
                      plan_params=ev.plan_params(flags=I.PLAN_CERTIFY, backend_max_iterations=200),
                      sense_params=I.sense_params(sensing_horizon=15.0), fallback=fallback)
    ev.close()
    return out, scene


def _summary(out):
    keys = ("status", "rounds_flown", "replans", "failed_replans", "uncertified_rounds", "brakes", "held_rounds")
    return {k: out[k] for k in keys if k in out}


def test_brake_stops_short_of_an_enclosed_goal_and_holds():
    out, scene = _run("brake")
    a = out["actions"][:, 0]
    clear = _min_true_clearance(out, scene)
    print(_summary(out), a, out["replan_stages"][:, 0], "min true clearance", clear)
    assert a[0] == I.NAV_REPLANNED
    braked = np.nonzero(a == I.NAV_BRAKED)[0]
    assert braked.size >= 1, "no stop was taken"
    assert (a[braked[0] + 1:] == I.NAV_HELD).any(), "the vehicle was never held after its stop"
    assert out["brakes"][0] == braked.size and out["held_rounds"][0] == int((a == I.NAV_HELD).sum())
    # every failed replan after the shell was seen is NO_PATH
    fails = out["replan_stages"][a != I.NAV_REPLANNED, 0]
    assert (fails[fails != I.NAV_NO_TRAJECTORY] == I.NO_PATH).all()
    assert out["status"][0] == I.NAV_TIMEOUT
    # a BRAKED round flies a certified stop, and held rounds fly nothing
    assert (out["verdicts"][a == I.NAV_BRAKED, 0] == I.CERTIFIED).all()
    assert (out["verdicts"][a == I.NAV_HELD, 0] == I.NAV_NO_TRAJECTORY).all()
    assert clear >= 0.0
    assert all("brake" in t for t in out["times"])
    # two runs give identical logs
    again, _ = _run("brake")
    assert np.array_equal(again["actions"], out["actions"]) and len(again["logs"]) == len(out["logs"])
    for (ia, la), (ib, lb) in zip(out["logs"], again["logs"]):
        assert np.array_equal(ia, ib) and torch_equal(la, lb)


def test_keep_flies_into_the_shell():
    out, scene = _run("keep")
    clear = _min_true_clearance(out, scene)
    print(_summary(out), out["actions"][:, 0], "min true clearance", clear)
    assert "brakes" not in out and "held_rounds" not in out and all("brake" not in t for t in out["times"])
    assert out["uncertified_rounds"][0] > 0
    assert not (out["actions"] == I.NAV_BRAKED).any() and not (out["actions"] == I.NAV_HELD).any()
