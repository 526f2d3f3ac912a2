"""isdf_trajectory_brake / _device: every BRAKED stop bit for bit the restatement of tests/brake_oracle.py, its summaries bit for bit the
public certificates of the output, the chosen candidate the largest one that passes both (every candidate rebuilt by the restatement and
checked through isdf_trajectory_certify / isdf_trajectory_dynamics), host = device (also on a side stream), a trajectory alone = inside a
batch, a stop before a one-voxel wall flown to rest without touching it, and the argument contract."""
import numpy as np
import pytest
import isdf_b200 as I
import brake_oracle as BO
import host_lib as H
import navigate_oracle as NO
from test_gpu_plan import _cfg

pytestmark = pytest.mark.gpu

DIMS, BMIN, RES = (40, 24, 8), np.zeros(3), 1.0


def _ev(occ):
    ev = I.Evaluator(_cfg())
    ev.set_shape_named("Ball")
    ev.set_map_u8(occ, BMIN, RES)
    return ev


def _world(rng, density=0.02):
    return (rng.random(DIMS) < density).astype(np.uint8)


def _traj(rng, N):
    """a smooth N-piece MINCO trajectory inside the frame, moving and accelerating at its start"""
    p = rng.uniform([4, 4, 2], [36, 20, 6])
    head = np.stack([p, rng.normal(0, 1.5, 3), rng.normal(0, 1.0, 3)], 1)
    pts = [p]
    for _ in range(N):
        pts.append(np.clip(pts[-1] + rng.normal(0, 1.5, 3), [1.5, 1.5, 1.0], [38.5, 22.5, 7.0]))
    tail = np.stack([pts[-1], np.zeros(3), np.zeros(3)], 1)
    T = rng.uniform(0.5, 1.5, N)
    wps = np.stack(pts[1:-1], 1) if N > 1 else np.zeros((3, 0))
    return T, H.minco_forward(head, tail, wps, T)[0]


def _ragged(rng, counts):
    Ts, Cs = [], []
    for n in counts:
        if n:
            t, c = _traj(rng, n)
            Ts.append(t); Cs.append(c)
    off = np.zeros(len(counts) + 1, dtype=np.int32)
    off[1:] = np.cumsum(counts)
    return off, (np.concatenate(Ts) if Ts else np.zeros(0)), (np.concatenate(Cs) if Cs else np.zeros(0))


def _stop_times(rng, off, T):
    ts = []
    for b in range(len(off) - 1):
        D = float(np.sum(T[off[b]:off[b + 1]])) if off[b + 1] > off[b] else 1.0
        ts.append([np.inf, rng.uniform(0.05, 1.0) * D, 2 * D, np.inf, rng.uniform(0.3, 1.0) * D, 0.0, np.nan, -1.0][b % 8])
    return np.array(ts)


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    x, y = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    if x.dtype.kind == "f":
        return x.shape == y.shape and np.array_equal(x.astype(np.float64).view(np.uint64), y.astype(np.float64).view(np.uint64))
    return np.array_equal(x, y)


def _concat(blocks):
    """per-trajectory 6M x 3 blocks -> one concatenated block (piece q M + i), the certificates' layout"""
    return NO._unblock(np.concatenate([NO._block(c, c.size // 18) for c in blocks]))


def _checks(ev, bp, Ts, Cs):
    """the public certificates of trajectories of M pieces each, N0 = M -> (certify dicts, dynamics dicts)"""
    M = bp.pieces
    T, Cc = np.concatenate(Ts), _concat(Cs)
    cp = bp.certify.clearance
    cs = ev.trajectory_certify(T, Cc, cp.samples_per_piece, cp.reach, cp.margin, N0=M, max_depth=bp.certify.max_depth,
                               max_samples=bp.certify.max_samples_per_traj)
    dp = I.DynamicsParams.from_buffer_copy(bytes(bp.dynamics))
    dp.pieces_per_traj = M
    ds = ev.trajectory_dynamics(T, Cc, params=dp)
    return cs, ds


def _check_against_restatement(ev, bp, off, T, Cc, ts, out, summ):
    B, K, M = len(off) - 1, bp.candidates, bp.pieces
    oo, oT, oC = out
    cands, where = [], []
    for b in range(B):
        s = summ[b]
        if BO.tau_max(T[off[b]:off[b + 1]], ts[b]) is None:
            assert s["status"] == I.BRAKE_NO_INPUT and s["candidate"] == -1 and oo[b + 1] == oo[b]
            assert (s["certified"], s["feasible"]) == (0, 0) and np.isnan(s["tau_stop"]) and s["certify"]["verdict"] == 0
            continue
        for k in range(K):
            cands.append(BO.ragged_candidate(off, T, Cc, ts, b, k, K, M))
            where.append((b, k))
    cs, ds = _checks(ev, bp, [c["T"] for c in cands], [c["coeffs"] for c in cands])
    passed = {}
    for (b, k), c, x, y in zip(where, cands, cs, ds):
        passed.setdefault(b, []).append((x["verdict"] == I.CERTIFIED, y["verdict"] == I.FEASIBLE, c, x, y))
    n_braked = 0
    for b, lst in passed.items():
        s = summ[b]
        ok = [k for k, (ck, dk, *_ ) in enumerate(lst) if ck and dk]
        assert s["certified"] == sum(ck for ck, *_ in lst) and s["feasible"] == sum(dk for _, dk, *_ in lst), b
        if not ok:
            assert s["status"] == I.BRAKE_NONE and s["candidate"] == -1 and oo[b + 1] == oo[b], b
            continue
        n_braked += 1
        k = max(ok)
        _, _, c, x, y = lst[k]
        assert s["status"] == I.BRAKED and s["candidate"] == k and oo[b + 1] - oo[b] == M, (b, s["candidate"], k)
        a = int(oo[b])
        assert _same(oT[a:a + M], c["T"]) and _same(oC[18 * a:18 * (a + M)], c["coeffs"]), b
        assert s["tau_stop"] == c["tau"] and s["duration"] == sum(float(t) for t in c["T"]), b
        assert _same(s["certify"], x) and _same(s["dynamics"], y), b
    return n_braked


def _summaries_of_output(ev, bp, out, summ):
    """the summaries equal the public certificates of the output itself"""
    oo, oT, oC = out
    M = bp.pieces
    br = [b for b in range(len(summ)) if summ[b]["status"] == I.BRAKED]
    if not br:
        return
    cs, ds = _checks(ev, bp, [oT[oo[b]:oo[b] + M] for b in br], [oC[18 * oo[b]:18 * (oo[b] + M)] for b in br])
    for b, x, y in zip(br, cs, ds):
        assert _same(summ[b]["certify"], x) and _same(summ[b]["dynamics"], y), b


@pytest.mark.parametrize("B", [5, 1024])
def test_stops_equal_the_restatement_and_the_largest_passing_candidate(B):
    import torch
    rng = np.random.default_rng(100 + B)
    ev = _ev(_world(rng))
    counts = [int(rng.integers(1, 13)) for _ in range(B)]
    if B > 8:
        counts[7] = 0   # a trajectory without pieces
    off, T, Cc = _ragged(rng, counts)
    ts = _stop_times(rng, off, T)
    bp = ev.brake_params()
    host, summ = ev.trajectory_brake((off, T, Cc), ts, params=bp)
    d = ev.trajectory_brake_device(torch.as_tensor(off, device="cuda"), torch.as_tensor(T, device="cuda"), torch.as_tensor(Cc, device="cuda"),
                                   torch.as_tensor(ts, device="cuda"), params=bp)
    do = d["piece_off"].cpu().numpy()
    assert np.array_equal(do, host[0])
    assert _same(d["T"][:do[-1]].cpu().numpy(), host[1]) and _same(d["coeffs"][:18 * do[-1]].cpu().numpy(), host[2])
    assert _same(I.decode_brake_summaries(d["summary"]), summ)
    n = _check_against_restatement(ev, bp, off, T, Cc, ts, host, summ)
    _summaries_of_output(ev, bp, host, summ)
    st = [s["status"] for s in summ]
    print(B, {k: st.count(k) for k in set(st)})
    assert n > 0
    if B > 8:
        assert st.count(I.BRAKE_NONE) > 0 and st.count(I.BRAKE_NO_INPUT) > 0
    ev.close()


def test_host_device_side_stream_and_alone_in_a_batch():
    import torch
    rng = np.random.default_rng(7)
    ev = _ev(_world(rng))
    counts = [int(rng.integers(1, 13)) for _ in range(64)]
    off, T, Cc = _ragged(rng, counts)
    ts = _stop_times(rng, off, T)
    bp = ev.brake_params(candidates=5, pieces=3)
    host, summ = ev.trajectory_brake((off, T, Cc), ts, params=bp)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        args = [torch.as_tensor(x, device="cuda") for x in (off, T, Cc, ts)]
    d = ev.trajectory_brake_device(*args, params=bp, stream=side)
    side.synchronize()
    do = d["piece_off"].cpu().numpy()
    assert np.array_equal(do, host[0]) and _same(d["T"][:do[-1]].cpu().numpy(), host[1])
    assert _same(d["coeffs"][:18 * do[-1]].cpu().numpy(), host[2]) and _same(I.decode_brake_summaries(d["summary"]), summ)
    for b in (0, 1, 9, 33, 63):
        a, e = off[b], off[b + 1]
        (o1, t1, c1), s1 = ev.trajectory_brake((np.array([0, e - a], dtype=np.int32), T[a:e], Cc[18 * a:18 * e]), ts[b:b + 1], params=bp)
        assert _same(s1[0], summ[b]) and o1[1] == host[0][b + 1] - host[0][b]
        assert _same(t1, host[1][host[0][b]:host[0][b + 1]]) and _same(c1, host[2][18 * host[0][b]:18 * host[0][b + 1]])
    ev.close()


def test_a_stop_before_a_one_voxel_wall_is_flown_to_rest_clear_of_it():
    import torch
    occ = np.zeros(DIMS, np.uint8)
    occ[20, :, :] = 1   # the wall x in [20, 21]
    ev = _ev(occ)
    p0, v = np.array([5.5, 12.5, 4.5]), np.array([2.0, 0.0, 0.0])
    blk = np.zeros((1, 3, 6))
    blk[0, :, 0], blk[0, :, 1] = p0, v
    T, Cc = np.array([15.0]), NO._unblock(blk)
    bp = ev.brake_params()
    cp = bp.certify.clearance
    cert = ev.trajectory_certify(T, Cc, cp.samples_per_piece, cp.reach, cp.margin, max_depth=bp.certify.max_depth,
                                 max_samples=bp.certify.max_samples_per_traj)[0]
    assert cert["verdict"] == I.COLLIDING and 0 < cert["first_hit"] < 7.5
    off = np.array([0, 1], dtype=np.int32)
    (oo, oT, oC), summ = ev.trajectory_brake((off, T, Cc), [cert["first_hit"]], params=bp)
    s = summ[0]
    print(s["candidate"], s["tau_stop"], s["duration"], s["certified"], s["feasible"])
    assert s["status"] == I.BRAKED and s["certify"]["verdict"] == I.CERTIFIED and s["dynamics"]["verdict"] == I.FEASIBLE
    # the stop's end lies on the line before the wall, at rest
    pe, ve, ae = BO.pva(oT, oC, s["duration"])
    assert pe[0] < 20.0 and abs(pe[0] - (p0[0] + v[0] * s["tau_stop"])) < 1e-9 and np.abs(ve).max() < 1e-9
    # fly it from the moving state
    sp = I.sim_default_params(t_end=float(s["duration"]) + 1.0)
    init = I.sim_init_from_trajectories(oo, oC, [0], params=sp)
    init[0, 3:6] = v
    dev = "cuda"
    sim = ev.simulate_device(torch.as_tensor(oo, device=dev), torch.as_tensor(oT, device=dev), torch.as_tensor(oC, device=dev),
                             torch.zeros(1, dtype=torch.int32, device=dev), torch.as_tensor(init, device=dev), params=sp)
    log = sim["log"][0].cpu().numpy()
    speed = np.linalg.norm(log[-1, 4:7])
    clear = ev.pose_clearance(log, 1, 7)[0]
    print("final speed", speed, "min clearance", clear.min())
    assert speed < 0.2, speed
    assert clear.min() >= 0.0
    ev.close()


def test_argument_contract():
    rng = np.random.default_rng(3)
    off, T, Cc = _ragged(rng, [3, 2])
    ts = np.array([np.inf, 1.0])
    ev = I.Evaluator(_cfg())
    ev.set_shape_named("Ball")
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_brake((off, T, Cc), ts)
    assert e.value.code == -2   # no map
    ev.set_map_u8(np.zeros(DIMS, np.uint8), BMIN, RES)
    for kw, code in ((dict(candidates=0), -1), (dict(pieces=0), -1), (dict(pieces=I.BRAKE_MAX_PIECES + 1), -1)):
        with pytest.raises(I.IsdfError) as e:
            ev.trajectory_brake((off, T, Cc), ts, params=ev.brake_params(**kw))
        assert e.value.code == code, kw
    bp = ev.brake_params()
    bp.certify.clearance.pieces_per_traj = 4
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_brake((off, T, Cc), ts, params=bp)
    assert e.value.code == -1
    bp = ev.brake_params()
    bp.dynamics.pieces_per_traj = 4
    with pytest.raises(I.IsdfError):
        ev.trajectory_brake((off, T, Cc), ts, params=bp)
    bp = ev.brake_params()
    bp.reserved_[1] = 1
    with pytest.raises(I.IsdfError):
        ev.trajectory_brake((off, T, Cc), ts, params=bp)
    bp = ev.brake_params()
    bp.certify.max_depth = 65   # the certificate's own check
    with pytest.raises(I.IsdfError):
        ev.trajectory_brake((off, T, Cc), ts, params=bp)
    bad = T.copy()
    bad[1] = 0.0   # the host form checks as isdf_trajectory_states does
    with pytest.raises(I.IsdfError):
        ev.trajectory_brake((off, bad, Cc), ts)
    with pytest.raises(I.IsdfError):
        ev.trajectory_brake((np.array([0, 3, 2], dtype=np.int32), T, Cc), ts)
    before = ev.stats().kernel_launches
    ev.trajectory_brake((off, T, Cc), ts)
    assert ev.stats().kernel_launches > before + 5
    ev.set_shape_named("Torus")   # a shape the certificate refuses
    with pytest.raises(I.IsdfError) as e:
        ev.trajectory_brake((off, T, Cc), ts)
    assert e.value.code == -4
    ev.close()
