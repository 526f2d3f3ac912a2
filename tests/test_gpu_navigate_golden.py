"""Evaluator.navigate computes exactly what it computed when tests/golden/navigate_reference.npz was recorded (by
tests/golden/make_navigate_golden.py): one run per branch of its round loop,
  fleet     the fleet scenario of tests/test_gpu_navigate.py (fallback "keep");
  brake     the enclosed goal of tests/test_gpu_navigate_brake.py (fallback "brake": stops and held rounds);
  unknown   unknown="occupied" with the four wide cameras of tests/test_gpu_navigate_unknown.py (commits);
  explore   explore=True with the front and back rig of tests/test_gpu_frontier.py (frontier plans);
  boxes     bench_navigate.py's box world with 16 vehicles, "brake" + "occupied" + 4 cameras + prefer-known 1 + explore, 40 rounds: the
            only run where plans, commits, stops, held vehicles and frontier plans are spliced across many vehicles in one round.
Compared: the result's key set, every count, the per-round tables, each logged round's vehicles and a SHA-256 of its log's bytes, and
the stage names of every round's times. Persistent grids are sized by the SM count, so a device with another SM count is skipped."""
import hashlib
import os
import sys

import numpy as np
import pytest
import isdf_b200 as I

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "navigate_reference.npz")
TABLES = ("status", "rounds_flown", "replans", "failed_replans", "uncertified_rounds", "brakes", "held_rounds", "commits", "frontier_plans",
          "actions", "verdicts", "replan_stages", "replan_verdicts", "subgoal_kinds")


def _fleet():
    from test_gpu_navigate import _run
    ys = [3.5, 9.5, 14.5, 20.5]
    return _run(np.array([[2.5, y, 4.5] for y in ys]), np.array([[36.5, y, 4.5] for y in ys]))[0]


def _brake():
    from test_gpu_navigate_brake import _run
    return _run("brake")[0]


def _unknown():
    from test_gpu_navigate_unknown import _run
    return _run("occupied", cams=4, fx=200.0, fy=200.0)[0]


def _explore():
    from test_gpu_frontier import _run
    return _run(2, 60)[0]


def _boxes(B=16):
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench_navigate as BN
    cfg = I.default_config_values()
    cfg.integral_intervs, cfg.kernel_size, cfg.vmax = 16, 11, 3.0
    sv = torch.cuda.current_stream().cuda_stream
    truth = I.Evaluator(cfg)
    truth.set_shape_named("Ball")
    scene = BN.world(truth)
    truth.set_map_u8(np.zeros(BN.DIMS, np.uint8), BN.BMIN, BN.RES)
    truth.map_fuse_cloud_device(scene, stream=sv)
    starts, goals = BN.pairs(truth.get_map_u8(), B, 7 + B)
    truth.close()
    ev = I.Evaluator(cfg)
    ev.set_shape_named("Ball")
    ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
    ev.set_map_u8(np.zeros(BN.DIMS, np.uint8), BN.BMIN, BN.RES)
    ev.set_sense_cloud_device(scene, stream=sv)
    out = ev.navigate(starts, goals, rounds=40, horizon=0.5, sense_every=25, tol=1.0,
                      plan_params=ev.plan_params(flags=I.PLAN_CERTIFY | I.PLAN_KNOWN_PREFIX, unknown_weight=1.0, backend_max_iterations=200),
                      sense_params=BN.rig(4), fallback="brake", unknown="occupied", known_boxes=np.concatenate([starts - 2.5, starts + 2.5], 1),
                      explore=True)
    ev.close()
    return out


SCENARIOS = dict(fleet=_fleet, brake=_brake, unknown=_unknown, explore=_explore, boxes=_boxes)


def record(out):
    """the non-timing outputs of one navigate result, as small numpy arrays"""
    rec = {k: np.asarray(out[k]) for k in TABLES if k in out}
    rec["keys"] = np.array(sorted(out))
    rec["log_vehicles"] = np.concatenate([np.asarray(vi, dtype=np.int64) for vi, _ in out["logs"]] or [np.zeros(0, np.int64)])
    rec["log_sizes"] = np.array([len(vi) for vi, _ in out["logs"]], dtype=np.int64)
    rec["log_sha256"] = np.array([np.frombuffer(hashlib.sha256(lg.contiguous().cpu().numpy().tobytes()).digest(), np.uint8)
                                  for _, lg in out["logs"]], dtype=np.uint8).reshape(-1, 32)
    rec["times_stages"] = np.array([list(t) for t in out["times"]])
    return rec


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_navigate_reproduces_the_recording(name):
    import torch
    ref = np.load(FIXTURE)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != int(ref["sm_count"]):
        pytest.skip(f"recorded on {ref['device']} with {int(ref['sm_count'])} SMs; this device has {sms}")
    got = record(SCENARIOS[name]())
    want = {k.split(".", 1)[1]: ref[k] for k in ref.files if k.startswith(name + ".")}
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].shape == want[k].shape and np.array_equal(got[k], want[k]), k
