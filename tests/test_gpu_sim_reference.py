"""isdf_simulate on the GPU against the reference's own simulator (tests/golden/sim_reference.npz, from oracle/_ref/libref_sim.so), and a
branch matrix of the closed loop's definition (include/isdf.h "closed loop") against the serial restatement tests/sim_serial.cpp.
Counts are exact. Logs and summaries agree to an absolute 1e-10, against the reference and against the serial restatement alike: what
separates the device from both is its libm (sin, cos, atan2, asin, acos, pow may differ from glibc's in the last ulp), carried through
the closed loop; the largest difference measured on an H100 was 1.8e-11, in the rpm entries (~1e4, whose ulp is 1.8e-12)."""
import numpy as np
import pytest
import isdf_b200 as I
import sim_oracle as S

pytestmark = pytest.mark.gpu

SUMMARY_FIELDS = [n for n, _ in I.SimSummary._fields_]
COUNTS = ("accepted", "rejected", "clamped_steps", "floor_contacts", "nan_rollbacks", "diverged")
TOL = 1e-10


def params_from(b):
    return I.SimParams.from_buffer_copy(np.asarray(b, dtype=np.uint8).tobytes())


@pytest.fixture(scope="module")
def ev():
    e = I.Evaluator(device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def golden():
    z = np.load(S.GOLDEN)
    return {k: z[k] for k in z.files}


def agree(log, summ, rlog, rsumm, tol=TOL):
    assert np.array_equal(np.isnan(log), np.isnan(rlog))
    fin = np.isfinite(rlog)
    err = np.abs(log[fin] - rlog[fin]).max(initial=0.0)
    assert err <= tol, err
    for a, b in zip(summ, rsumm):
        for c in COUNTS:
            assert a[c] == b[c], (c, a[c], b[c])
        for c in ("max_err", "rms_err", "final_err", "max_tilt", "max_omega", "t_max_err", "t_diverged"):
            assert (np.isnan(a[c]) and np.isnan(b[c])) or abs(a[c] - b[c]) <= tol, (c, a[c], b[c])
    return err


@pytest.mark.parametrize("name", ["default", "vehicle", "ratio1", "ratio20", "floor", "gust", "hold", "rollback"])
def test_device_matches_reference(ev, golden, name):
    k = f"roll/{name}/"
    p = params_from(golden[k + "params"])
    tr = (golden["traj/off"], golden["traj/T"], golden["traj/C"])
    log, summ = ev.simulate(tr, golden[k + "traj"], golden[k + "init"], golden[k + "dist"], p)
    rsumm = [dict(zip(SUMMARY_FIELDS, row)) for row in golden[k + "summary"]]
    print(name, "max |device - reference|:", agree(log, summ, golden[k + "log"], rsumm))


# ---- branch matrix against the serial restatement ----
trajectories = S.line_trajectories


def rollouts(off, Cc, R, p, seed=0, rpm=None):
    rng = np.random.default_rng(seed)
    traj = (np.arange(R) % (off.size - 1)).astype(np.int32)
    init = I.sim_init_from_trajectories(off, Cc, traj, p, rpm=rpm)
    init[:, 0:3] += rng.normal(scale=0.05, size=(R, 3))
    dist = np.zeros((R, 6))
    dist[:, 0:3] = rng.normal(scale=0.1, size=(R, 3))
    dist[:, 3:6] = rng.normal(scale=1e-4, size=(R, 3))
    return traj, init, dist


def run_both(ev, off, T, Cc, traj, init, dist, p, cap_log=None):
    log, summ = ev.simulate((off, T, Cc), traj, init, dist, p, cap_log=cap_log)
    rlog, rsumm = S.simulate(off, T, Cc, traj, init, dist, p, cap_log=cap_log)
    print("max |device - serial|:", agree(log, summ, rlog, rsumm))
    return log, summ


@pytest.mark.parametrize("ratio", [1, 10, 20])
@pytest.mark.parametrize("R", [1, 31, 33, 4097])
def test_rates_and_batch_edges(ev, ratio, R):
    # log_every 7 does not divide the 151 ticks; cap_log above n_log leaves a NaN tail; the attitude loop takes the odometry's yaw at
    # ratio 10 and its own R_to_ypr yaw at ratios 1 and 20
    off, T, Cc = trajectories()
    p = I.sim_default_params(sim_rate=100.0 * ratio, cmd_rate=100.0, t_end=1.5 if R < 4097 else 0.3, log_every=7,
                             use_external_yaw=int(ratio == 10))
    traj, init, dist = rollouts(off, Cc, R, p, seed=R)
    n_ticks, m, n_log = S.ticks(p)
    assert m == ratio and (n_ticks - 1) % p.log_every != 0
    if R < 4097:
        log, summ = run_both(ev, off, T, Cc, traj, init, dist, p, cap_log=n_log + 3)
        assert np.isnan(log[:, n_log:]).all() and np.isfinite(log[:, :n_log]).all()
    else:   # the last block holds one rollout: the batch against itself alone, and a sample against the serial restatement
        log, summ = ev.simulate((off, T, Cc), traj, init, dist, p)
        for r in (0, 2048, 4096):
            la, sa = ev.simulate((off, T, Cc), traj[r:r + 1], init[r:r + 1], dist[r:r + 1], p)
            assert np.array_equal(la[0].view(np.uint64), log[r].view(np.uint64))
            rl, rs = S.simulate(off, T, Cc, traj[r:r + 1], init[r:r + 1], dist[r:r + 1], p)
            agree(la, sa, rl, rs)
    assert all(s["accepted"] > 0 for s in summ)


def test_floor_clamps_and_command_hold(ev):
    off, T, Cc = trajectories()
    # past both trajectories' ends (2 s and 1 s), with an rpm ceiling the climb off the floor reaches
    p = I.sim_default_params(t_end=2.5, log_every=1, use_external_yaw=0, max_rpm=18000.0)
    traj, init, dist = rollouts(off, Cc, 4, p, rpm=0)
    init[:, 2], init[:, 5] = 0.0, -0.2   # zero rpm on the floor, moving down
    log, summ = run_both(ev, off, T, Cc, traj, init, dist, p)
    assert all(s["floor_contacts"] > 0 and s["clamped_steps"] > 0 for s in summ)
    # the command holds at the trajectory's end: the commanded position stops changing once t >= duration
    for r in range(4):
        dur = T[off[traj[r]]:off[traj[r] + 1]].sum()
        held = log[r, log[r, :, 0] >= dur]
        assert len(held) > 10 and (held[:, 18:21] == held[0, 18:21]).all()
    p.floor = 0
    log0, summ0 = run_both(ev, off, T, Cc, traj, init, dist, p)
    assert all(s["floor_contacts"] == 0 for s in summ0)


def test_divergence_branches(ev):
    off, T, Cc = trajectories()
    p = I.sim_default_params(t_end=0.5, log_every=1, diverge_dist=1.0)
    traj, init, dist = rollouts(off, Cc, 3, p)
    dist[1, 0] = 60.0          # a gust: the position error passes diverge_dist
    init[2, 10:13] = [1e150, -3e149, 2e149]   # each accepted try advances ~1e-152 s: the 100000-try bound of one step ends the rollout
    log, summ = run_both(ev, off, T, Cc, traj, init, dist, p)
    assert summ[0]["diverged"] == 0 and summ[1]["diverged"] == 1 and summ[2]["diverged"] == 1
    assert summ[2]["accepted"] + summ[2]["rejected"] >= 100000 and summ[2]["t_diverged"] == 1.0 / p.cmd_rate
    assert np.isnan(log[1, -1]).all() and np.isnan(log[2, 2:]).all()
    # Two ends of a step are reached by no case here. Both need a try's error to stay above 1 as h shrinks without bound, and the error
    # norm's floor stands in the way: a try's error is max_i |xe_i| / (1e-6 + 1e-6 (|x_i| + h |x'_i|)) with xe_i = h (e1 k1_i + e3 k3_i +
    # ... + e7 k7_i), so a rejection needs h |e . k_i| > 1e-6, which finite stage derivatives (below 1.8e308) cannot give once h < ~1e-314.
    # Only an infinite stage derivative keeps the error infinite, and in every overflowing state we tried (rpm, omega, velocity and an
    # external force of up to 1e300 or infinity) the infinities met weights of both signs, or an infinite h |x'_i|, and made the term
    # NaN, which the max skips: the try is accepted and step() rolls the NaN state back (test_nan_rollback). So:
    #   - the 1000-try rule would need 999 rejections in a row; each multiplies h by at most 0.9 (0.2 while err > 91). The thousands of
    #     tries in test_sim_reference_cpu.py's single steps are spread over many accepted substeps, fewer than 1000 in any one;
    #   - the no-progress test (h = 0, or t + h == t) would need h to underflow at a step's start, or ~23 rejections in a row right after
    #     an accepted substep with the error above 1 down to h ~ 1e-16 t.
    # Both rules are pinned by reading isdf_sim.cuh's integrate against its twin in tests/sim_serial.cpp, not by a test.


def test_nan_rollback(ev):
    # rpm^2 overflows: thrust is infinite, every step's integrated state has a NaN, and the step restores the state before it
    off, T, Cc = trajectories()
    p = I.sim_default_params(t_end=0.3, log_every=1)
    traj, init, dist = rollouts(off, Cc, 3, p, seed=4)
    init[1, 13:17] = 1e160
    init[2, 13:17] = [1e160, 16000.0, 16000.0, 16000.0]
    log, summ = run_both(ev, off, T, Cc, traj, init, dist, p)
    assert summ[0]["nan_rollbacks"] == 0
    for s in summ[1:]:
        assert s["nan_rollbacks"] > 0 and s["diverged"] == 0


def test_summary_against_the_log(ev):
    off, T, Cc = trajectories()
    p = I.sim_default_params(t_end=1.8, log_every=1)
    traj, init, dist = rollouts(off, Cc, 33, p, seed=9)
    init[:, 10:13] += np.random.default_rng(1).normal(scale=0.5, size=(33, 3))
    log, summ = ev.simulate((off, T, Cc), traj, init, dist, p)
    for r, s in enumerate(summ):
        L = log[r]
        err = np.linalg.norm(L[:, 1:4] - L[:, 18:21], axis=1)
        q = L[:, 7:11]
        R22 = 1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2)
        assert s["t_max_err"] == L[np.argmax(err), 0]
        assert abs(s["max_err"] - err.max()) <= 1e-12 and abs(s["rms_err"] - np.sqrt(np.mean(err ** 2))) <= 1e-12
        assert abs(s["max_tilt"] - np.arccos(np.clip(R22, -1, 1)).max()) <= 1e-7   # R22 rebuilt from the logged quaternion
        assert abs(s["max_omega"] - np.linalg.norm(L[:, 11:14], axis=1).max()) <= 1e-12
