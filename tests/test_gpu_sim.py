"""isdf_simulate / isdf_simulate_device on the GPU against the serial restatement tests/sim_serial.cpp, and its guarantees."""
import numpy as np
import pytest
import isdf_b200 as I
import sim_oracle as S
import workloads as W

pytestmark = pytest.mark.gpu


def ragged(seeds=(3, 5, 7), N=(4, 6, 3)):
    """three trajectories of different piece counts in isdf_plan_batch's ragged layout (2.5 s pieces: tracking far from the clamps)"""
    Ts, Cs = [], []
    for s, n in zip(seeds, N):
        T, Cc, _ = W.make_trajectory(n, [1, 1, 1], [4 + s % 3, 3, 2.5], seed=s, jitter=0.2)
        Ts.append(np.asarray(T, dtype=np.float64))
        Cs.append(np.asarray(Cc, dtype=np.float64).reshape(-1))
    off = np.zeros(len(Ts) + 1, dtype=np.int32)
    off[1:] = np.cumsum([t.size for t in Ts])
    return off, np.concatenate(Ts), np.concatenate(Cs)


def rollouts(off, Cc, R, seed=0):
    rng = np.random.default_rng(seed)
    traj = (np.arange(R) % (off.size - 1)).astype(np.int32)
    init = I.sim_init_from_trajectories(off, Cc, traj)
    init[:, 0:3] += rng.normal(scale=0.05, size=(R, 3))
    dist = np.zeros((R, 6))
    dist[:, 0:3] = rng.normal(scale=0.1, size=(R, 3))
    dist[:, 3:6] = rng.normal(scale=1e-4, size=(R, 3))
    return traj, init, dist


def same(a, b):
    """summary dicts equal bit for bit (NaN fields included)"""
    return [np.array(list(x.values()), dtype=np.float64).tobytes() for x in a] == [np.array(list(x.values()), dtype=np.float64).tobytes() for x in b]


@pytest.fixture(scope="module")
def ev():
    e = I.Evaluator(device=0)
    yield e
    e.close()


def test_device_matches_serial(ev):
    off, T, Cc = ragged()
    p = I.sim_default_params(floor=0, t_end=2.5, log_every=5)
    traj, init, dist = rollouts(off, Cc, 6)
    log, summ = ev.simulate((off, T, Cc), traj, init, dist, p)
    rlog, rsumm = S.simulate(off, T, Cc, traj, init, dist, p)
    assert np.isfinite(log).all()
    err = np.abs(log - rlog).max()
    print("max |device - serial| over the log:", err)
    assert err <= 1e-9
    for a, b in zip(summ, rsumm):
        assert a["diverged"] == b["diverged"] == 0
        for k in ("accepted", "rejected", "clamped_steps", "floor_contacts", "nan_rollbacks"):
            assert a[k] == b[k], k
        for k in ("max_err", "rms_err", "final_err", "max_tilt", "max_omega"):
            assert abs(a[k] - b[k]) <= 1e-9, k


def test_bit_identity_batch_and_entry_points(ev):
    import torch
    off, T, Cc = ragged()
    p = I.sim_default_params(floor=0, t_end=1.0, log_every=10)
    traj, init, dist = rollouts(off, Cc, 1024, seed=1)
    log1, s1 = ev.simulate((off, T, Cc), traj, init, dist, p)
    log2, s2 = ev.simulate((off, T, Cc), traj, init, dist, p)
    assert np.array_equal(log1.view(np.uint64), log2.view(np.uint64)) and same(s1, s2)
    for r in (0, 517, 1023):   # alone against inside the batch
        la, sa = ev.simulate((off, T, Cc), traj[r:r + 1], init[r:r + 1], dist[r:r + 1], p)
        assert np.array_equal(la[0].view(np.uint64), log1[r].view(np.uint64)) and same(sa, [s1[r]])
    dv = torch.device("cuda:0")
    out = ev.simulate_device(torch.from_numpy(off).to(dv), torch.from_numpy(T).to(dv), torch.from_numpy(Cc).to(dv), torch.from_numpy(traj).to(dv),
                             torch.from_numpy(init).to(dv), torch.from_numpy(dist).to(dv), p)
    torch.cuda.synchronize()
    assert np.array_equal(out["log"].cpu().numpy().view(np.uint64), log1.view(np.uint64))
    assert same(I.decode_sim_summaries(out["summary"]), s1)


def test_zero_rpm_start_and_divergence(ev):
    off, T, Cc = ragged()
    p = I.sim_default_params(floor=0, t_end=1.0, diverge_dist=0.5)
    traj = np.zeros(2, dtype=np.int32)
    init = I.sim_init_from_trajectories(off, Cc, traj, rpm=0)
    assert (init[:, 13:] == 0).all()
    dist = np.zeros((2, 6))
    dist[1, 0] = 50.0   # a gust no controller holds
    log, s = ev.simulate((off, T, Cc), traj, init, dist, p)
    rlog, rs = S.simulate(off, T, Cc, traj, init, dist, p)
    assert s[0]["diverged"] == 0 and s[1]["diverged"] == 1 and np.isfinite(s[1]["t_diverged"])
    assert s[1]["t_diverged"] == rs[1]["t_diverged"]
    assert np.isnan(log[1, -1]).all()


def test_errors_and_poisoning(ev):
    import torch
    off, T, Cc = ragged()
    traj, init, dist = rollouts(off, Cc, 4)
    for kw in (dict(cmd_rate=300.0), dict(sim_rate=-1.0), dict(log_every=0), dict(mass=float("nan")), dict(reserved_=1)):
        with pytest.raises(I.IsdfError):
            ev.simulate((off, T, Cc), traj, init, dist, I.sim_default_params(**kw))
    bad = traj.copy(); bad[2] = 7
    with pytest.raises(I.IsdfError):
        ev.simulate((off, T, Cc), bad, init, dist, I.sim_default_params(floor=0, t_end=0.1))
    with pytest.raises(I.IsdfError):
        ev.simulate((off, T, Cc), traj, init, dist, I.sim_default_params(floor=0, t_end=0.1), cap_log=2)
    # the device form poisons its summaries on a refused call and counts the launch
    dv = torch.device("cuda:0")
    sm = torch.zeros((4, 88), dtype=torch.uint8, device=dv)
    d = lambda a: torch.from_numpy(a).to(dv)
    o, t, c, tr, ini = d(off), d(T), d(Cc), d(traj), d(init)
    before = ev.stats().kernel_launches
    p = I.sim_default_params(cmd_rate=300.0)
    r = ev.simulate_device_raw(off.size - 1, o.data_ptr(), t.data_ptr(), c.data_ptr(), 4, tr.data_ptr(), ini.data_ptr(), 0, p, 0, 0, sm.data_ptr())
    torch.cuda.synchronize()
    assert r == -1 and ev.stats().kernel_launches == before + 1
    for s in I.decode_sim_summaries(sm):
        assert s["diverged"] == 1 and np.isnan(s["max_err"])
    # an index outside [0, B) on the device reads as diverged at t = NaN
    tr[1] = 99
    out = ev.simulate_device(o, t, c, tr, ini, None, I.sim_default_params(floor=0, t_end=0.2))
    torch.cuda.synchronize()
    s = I.decode_sim_summaries(out["summary"])
    assert s[1]["diverged"] == 1 and np.isnan(s[1]["t_diverged"]) and s[0]["diverged"] == 0
