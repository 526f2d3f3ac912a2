"""GPU: isdf_trajectory_states and isdf_pose_points.
  * every record bit-identical to the reference-compiled state of process() (tests/golden/states_reference.npz; where oracle/_ref/ travelled,
    also to the live reference trajectory evaluation and, up to signs of zero, its flatness map);
  * ragged independence: a record depends only on its own query and trajectory, zero-piece trajectories give NaN, plan_batch's output feeds in;
  * host form == device form bit for bit, across Q and B;
  * the argument contract: refusals leave outputs untouched, the device form's out-of-range indices give NaN, Q = 0 does nothing, no map or
    shape is needed;
  * pose_points bit-identical to the numpy restatement of Shape::Transform, host == device, identity attitude leaves points unchanged."""
import os
import numpy as np
import pytest
import torch
import isdf_b200 as I
import oracle_lib as O
import states_oracle as SO

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _ragged(trajs):
    """[(T, coeffs) or None] -> (piece_off, T, coeffs) in isdf_plan_batch's layout; None is a trajectory without pieces"""
    off = np.zeros(len(trajs) + 1, dtype=np.int32)
    Ts, Cs = [np.zeros(0)], [np.zeros(0)]
    for b, tc in enumerate(trajs):
        n = 0 if tc is None else tc[0].size
        off[b + 1] = off[b] + n
        if tc is not None:
            Ts.append(tc[0]); Cs.append(tc[1])
    return off, np.concatenate(Ts), np.concatenate(Cs)


def _device_states(ev, ragged, traj, times):
    off, T, Cc = ragged
    d = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()   # noqa: E731
    d_off, d_T, d_C, d_tr, d_tm = d(off, np.int32), d(T, np.float64), d(Cc, np.float64), d(traj, np.int32), d(times, np.float64)
    out = torch.full((len(times), 20), 3.0, dtype=torch.float64, device="cuda")
    ev.trajectory_states_device(off.size - 1, d_off.data_ptr(), d_T.data_ptr(), d_C.data_ptr(), len(times), d_tr.data_ptr(), d_tm.data_ptr(),
                                out.data_ptr(), 0)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("tag", SO.TAGS)
def test_records_equal_reference_compiled_process_state(tag):
    cases, _ = SO.load_golden()
    ev = I.Evaluator(SO.config_for(tag))
    ref = O.RefMinco() if os.path.exists(O.REF_MINCO) else None
    rflat = O.RefFlat(O.config_from(SO.config_for(tag))) if O.ref_flat_available() else None
    for c in cases:
        rg = (np.array([0, c["N"]], dtype=np.int32), c["T"], c["coeffs"])
        tr = np.zeros(c["times"].size, dtype=np.int32)
        rec = ev.trajectory_states(rg, tr, c["times"])
        assert SO.same_bits(rec, c["rec"][tag]), f"N={c['N']}: {np.argwhere(rec.view(np.uint64) != c['rec'][tag].view(np.uint64))[:5]}"
        assert SO.same_bits(_device_states(ev, rg, tr, c["times"]), rec)
        if ref is not None:   # the live reference-compiled trajectory.hpp fed by its own MINCO
            pvaj = ref.traj_eval(c["head"], c["tail"], c["inPs"], c["T"], c["times"])[0]
            assert SO.same_bits(rec[:, :12], pvaj), f"N={c['N']}: live reference pos/vel/acc/jer"
        if rflat is not None:  # optimizated_forward: forward at yaw 0 up to the signs of zero products
            q, o = rflat.forward(rec[:, 3:6], rec[:, 6:9], rec[:, 9:12])
            assert np.array_equal(q, rec[:, 12:16]) and np.array_equal(o, rec[:, 16:19])
    ev.close()


def _batch(B, seed):
    """B trajectories cycling through the golden ones, every 5th without pieces, and Q = 4 B queries at times before, inside and past each"""
    cases, _ = SO.load_golden()
    rng = np.random.default_rng(seed)
    trajs = [None if b % 5 == 3 else (cases[b % len(cases)]["T"], cases[b % len(cases)]["coeffs"]) for b in range(B)]
    traj = rng.integers(0, B, 4 * B).astype(np.int32)
    tot = np.array([0.0 if t is None else t[0].sum() for t in trajs])
    times = rng.uniform(-0.5, 1.1, traj.size) * np.maximum(tot[traj], 1.0)
    return trajs, traj, times


def test_ragged_records_are_independent_of_the_batch():
    trajs, traj, times = _batch(23, seed=3)
    rg = _ragged(trajs)
    ev = I.Evaluator()
    rec = ev.trajectory_states(rg, traj, times)
    empty = np.array([trajs[b] is None for b in traj])
    assert empty.any() and np.isnan(rec[empty]).all() and np.isfinite(rec[~empty]).all()
    for b, tc in enumerate(trajs):
        sel = traj == b
        if tc is None or not sel.any():
            continue
        alone = ev.trajectory_states(_ragged([tc]), np.zeros(sel.sum(), dtype=np.int32), times[sel])
        assert SO.same_bits(alone, rec[sel]), f"trajectory {b}"
    perm = np.random.default_rng(4).permutation(traj.size)
    assert SO.same_bits(ev.trajectory_states(rg, traj[perm], times[perm]), rec[perm])
    # the same trajectories as plan_batch-style dicts
    plans = [dict(T=np.zeros(0), coeffs=np.zeros(0)) if tc is None else dict(T=tc[0], coeffs=tc[1]) for tc in trajs]
    assert SO.same_bits(ev.trajectory_states(plans, traj, times), rec)
    ev.close()


def test_plan_batch_output_feeds_in_unchanged():
    from test_gpu_plan import _ev, _scene, _params
    occ, start, goals = _scene(4, seed=7)
    goals = np.concatenate([goals, np.argwhere(occ == 1)[:1] + 0.5])   # a goal in an obstacle: no path, no pieces
    ev = _ev("Ball", occ)
    plans, _ = ev.plan_batch(start, goals, _params(ev))
    B = len(plans)
    assert any(p["pieces"] > 0 for p in plans)
    rng = np.random.default_rng(5)
    traj = np.repeat(np.arange(B, dtype=np.int32), 50)
    times = np.concatenate([np.sort(rng.uniform(0, max(p["duration"], 1.0), 50)) for p in plans])
    rec = ev.trajectory_states(plans, traj, times)
    for b, p in enumerate(plans):
        sel = traj == b
        if p["pieces"] == 0:
            assert np.isnan(rec[sel]).all()
            continue
        alone = ev.trajectory_states((np.array([0, p["pieces"]], dtype=np.int32), p["T"], p["coeffs"]), np.zeros(50, dtype=np.int32), times[sel])
        assert SO.same_bits(alone, rec[sel])
        pvaj = O.traj_eval(p["T"], p["coeffs"], times[sel])[0]
        assert SO.same_bits(pvaj, rec[sel][:, :12])
        assert np.abs(rec[sel][:, 15]).max() == 0.0   # yaw 0: quat z is zero
    ev.close()


@pytest.mark.parametrize("B", [1, 1024])
def test_host_equals_device(B):
    trajs, _, _ = _batch(B, seed=B)
    if B == 1:
        trajs = [(SO.load_golden()[0][4]["T"], SO.load_golden()[0][4]["coeffs"])]
    rg = _ragged(trajs)
    tot = np.array([0.0 if t is None else t[0].sum() for t in trajs])
    ev = I.Evaluator()
    rng = np.random.default_rng(9)
    for Q in (1, 31, 32, 33, 100000):
        traj = rng.integers(0, B, Q).astype(np.int32)
        times = rng.uniform(-0.2, 1.2, Q) * np.maximum(tot[traj], 1.0)
        host = ev.trajectory_states(rg, traj, times)
        assert SO.same_bits(host, _device_states(ev, rg, traj, times)), f"B={B} Q={Q}"
    ev.close()


def test_argument_contract():
    c = SO.load_golden()[0][2]
    rg = (np.array([0, c["N"]], dtype=np.int32), c["T"], c["coeffs"])
    ev = I.Evaluator()                     # no map, no shape
    lib, h = ev.lib, ev.h
    import ctypes as C
    ip = C.POINTER(C.c_int32)
    tr, tm = np.zeros(3, dtype=np.int32), np.array([0.1, 0.5, 1.0])
    rec = ev.trajectory_states(rg, tr, tm)
    assert np.isfinite(rec).all()

    def call(B=1, off=None, T=None, Cc=None, Q=3, traj=None, times=None, out=True):
        o = np.full((3, 20), 7.0)
        a = [np.ascontiguousarray(x) for x in (rg[0] if off is None else off, rg[1] if T is None else T, rg[2] if Cc is None else Cc,
                                                tr if traj is None else traj, tm if times is None else times)]
        r = lib.isdf_trajectory_states(h, B, a[0].ctypes.data_as(ip), I._dp(a[1]), I._dp(a[2]), Q, a[3].ctypes.data_as(ip), I._dp(a[4]),
                                       I._dp(o) if out else None)
        return r, o

    bad_T, bad_C, inf_T = c["T"].copy(), c["coeffs"].copy(), c["T"].copy()
    bad_T[3], bad_C[40], inf_T[0] = 0.0, np.nan, np.inf
    neg_T = c["T"].copy(); neg_T[1] = -1.0
    for kw in (dict(B=0), dict(Q=-1), dict(off=np.array([1, c["N"]], dtype=np.int32)), dict(B=2, off=np.array([0, 3, 2], dtype=np.int32)),
               dict(traj=np.array([0, 1, 0], dtype=np.int32)), dict(traj=np.array([0, -1, 0], dtype=np.int32)), dict(T=bad_T), dict(T=inf_T),
               dict(T=neg_T), dict(Cc=bad_C), dict(out=False)):
        r, o = call(**kw)
        assert r == -1 and (o == 7.0).all(), kw
    r, o = call(Q=0)
    assert r == 0 and (o == 7.0).all()
    assert lib.isdf_trajectory_states(h, 1, rg[0].ctypes.data_as(ip), None, I._dp(rg[2]), 3, tr.ctypes.data_as(ip), I._dp(tm), I._dp(np.zeros(60))) == -1
    # the device form: indices outside [0, B) give NaN records, the rest is unchanged; Q = 0 leaves out alone
    traj = np.array([0, -1, 1, 0, 7], dtype=np.int32)
    times = np.array([0.1, 0.5, 1.0, 1.0, 0.2])
    got = _device_states(ev, rg, traj, times)
    assert np.isnan(got[[1, 2, 4]]).all() and SO.same_bits(got[[0, 3]], ev.trajectory_states(rg, traj[[0, 3]], times[[0, 3]]))
    out = torch.full((1, 20), 3.0, dtype=torch.float64, device="cuda")
    d = torch.zeros(1, dtype=torch.float64, device="cuda")
    ev.trajectory_states_device(1, d.data_ptr(), d.data_ptr(), d.data_ptr(), 0, d.data_ptr(), d.data_ptr(), out.data_ptr(), 0)
    torch.cuda.synchronize()
    assert (out == 3.0).all()
    with pytest.raises(I.IsdfError):
        ev.trajectory_states_device(0, d.data_ptr(), d.data_ptr(), d.data_ptr(), 1, d.data_ptr(), d.data_ptr(), out.data_ptr(), 0)
    # pose_points refusals
    st, body = np.tile(rec[:1], (2, 1)), np.ones((4, 3))
    o = np.full(24, 7.0)
    assert lib.isdf_pose_points(h, -1, I._dp(st), 4, I._dp(body), I._dp(o)) == -1
    assert lib.isdf_pose_points(h, 2, I._dp(st), -1, I._dp(body), I._dp(o)) == -1
    assert lib.isdf_pose_points(h, 2, None, 4, I._dp(body), I._dp(o)) == -1
    assert lib.isdf_pose_points(h, 2 ** 40, I._dp(st), 2 ** 30, I._dp(body), I._dp(o)) == -1
    assert lib.isdf_pose_points(h, 0, I._dp(st), 4, I._dp(body), I._dp(o)) == 0
    assert (o == 7.0).all()
    ev.close()


def _device_pose(ev, states, body):
    d_s = torch.from_numpy(np.ascontiguousarray(states)).cuda()
    d_b = torch.from_numpy(np.ascontiguousarray(body, dtype=np.float64)).cuda()
    out = torch.empty((states.shape[0], body.shape[0], 3), dtype=torch.float64, device="cuda")
    ev.pose_points_device(states.shape[0], d_s.data_ptr(), body.shape[0], d_b.data_ptr(), out.data_ptr(), 0)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("body", ["one", "drone", "odd"])
def test_pose_points_equal_numpy_transform(body):
    cases, _ = SO.load_golden()
    states = np.concatenate([c["rec"]["drag"] for c in cases])
    if body == "one":
        pts = np.array([[0.3, -0.2, 0.1]])
    elif body == "drone":
        pts = np.load(os.path.join(G, "ref_meshes.npz"))["drone_V"]
    else:
        pts = np.random.default_rng(2).normal(size=(1001, 3))   # 3003 doubles per state: not a multiple of the block
    states = np.concatenate([states, np.full((1, 20), np.nan)])
    ev = I.Evaluator()
    got = ev.pose_points(states, pts)
    assert got.shape == (states.shape[0], pts.shape[0], 3)
    assert SO.same_bits(got, SO.pose_points(states, pts))
    assert np.isnan(got[-1]).all()
    assert SO.same_bits(_device_pose(ev, states, pts), got)
    ident = np.zeros((3, 20)); ident[:, 12] = 1.0
    assert np.array_equal(ev.pose_points(ident, pts), np.broadcast_to(pts, (3,) + pts.shape))
    ev.close()
