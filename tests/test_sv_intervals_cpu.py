"""The swept-volume interval fixtures (tests/sv_intervals.py) checked against the oracle alone: the trajectories take nc = 0 and 1 (mod 32)
coarse samples, every category holds at least three points, every coarse decision is at least DELTA from flipping, and the points the
search must leave alone (never in range, in range throughout, only an open run) keep SV-SDF 10 and their previous t*. No GPU needed."""
import numpy as np
import pytest
import oracle_lib as O
import sv_intervals as S

CASES = [(robot, nc) for robot in S.ROBOTS for nc in (64, 97)]


@pytest.mark.parametrize("robot,nc", CASES)
def test_every_category_is_populated(robot, nc):
    f = S.fixture(robot, nc)
    assert f["nc"] == nc and f["nc"] % 32 == nc % 32 and nc % 32 in (0, 1)
    assert f["margin"].min() >= S.DELTA
    counts = {c: len(v) for c, v in f["cats"].items()}
    print(robot, nc, "points", len(f["pts"]), counts, f"min coarse margin {f['margin'].min():.2e}")
    assert all(n >= 3 for n in counts.values()), counts


@pytest.mark.parametrize("robot,nc", CASES)
def test_oracle_leaves_points_without_a_closed_run_alone(robot, nc):
    f = S.fixture(robot, nc)
    ocfg = O.config_from(f["cfg"])
    t0 = np.full(len(f["pts"]), -1.0)
    ref = O.eval_swept(ocfg, S.oracle_robot(robot), f["T"], f["C"], f["pts"], tstar=t0)
    none = np.concatenate([f["cats"]["G"], f["cats"]["H"], f["cats"]["B_alone"]])
    assert np.all(ref["sdf"][none] == 10.0) and np.all(ref["tstar"][none] == -1.0)
    closed = np.setdiff1d(np.arange(len(f["pts"])), none)
    assert np.all(ref["sdf"][closed] < 10.0) and np.all(ref["tstar"][closed] >= 0.0)
    # the coarse hook counts the samples the evaluation's own loop takes: nc coarse SDF evaluations per point at least
    assert ref["nsdf"] >= nc * len(f["pts"])
