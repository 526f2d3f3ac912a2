"""The planning step in device memory: isdf_path_waypoints_device against the host selection, isdf_plan_pairs_device /
isdf_plan_batch_device against the host forms byte for byte, stream order, chaining into the trajectory states, caps, refusals and the
transfer budget (isdf_dbg_plan_transfers)."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
from test_gpu_plan import _ev, _cfg, _scene, _params
from test_gpu_plan_pairs import _pairs

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch


def _b(a):
    return np.ascontiguousarray(a).view(np.uint8)


# ---- waypoints -------------------------------------------------------------------------------------------------------------------------
def _ragged_paths(lengths, seed):
    rng = np.random.default_rng(seed)
    off = np.zeros(len(lengths) + 1, dtype=np.int32)
    off[1:] = np.cumsum(lengths)
    return off, rng.uniform(-50, 50, (int(off[-1]), 3))


def _wp_host(off, xyz, res, parlength, cap):
    B = len(off) - 1
    ip = C.POINTER(C.c_int32)
    wp, wo, pc = np.zeros((max(cap, 1), 3)), np.zeros(B + 1, dtype=np.int32), np.zeros(B, dtype=np.int32)
    lib = I.load_library()
    r = lib.isdf_path_waypoints(B, off.ctypes.data_as(ip), I._dp(xyz), res, parlength, cap, I._dp(wp), wo.ctypes.data_as(ip), pc.ctypes.data_as(ip))
    return r, wp, wo, pc


def _wp_device(ev, off, xyz, res, parlength, cap):
    torch = _torch()
    B = len(off) - 1
    d_off, d_xyz = torch.from_numpy(off).cuda(), torch.from_numpy(xyz).cuda()
    wp = torch.full((max(cap, 1), 3), -7.0, dtype=torch.float64, device="cuda")
    wo, pc = torch.full((B + 1,), -7, dtype=torch.int32, device="cuda"), torch.full((B,), -7, dtype=torch.int32, device="cuda")
    r = ev.path_waypoints_device(B, d_off.data_ptr(), d_xyz.data_ptr(), res, parlength, cap, wp.data_ptr() if cap else 0, wo.data_ptr(), pc.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return r, wp.cpu().numpy(), wo.cpu().numpy(), pc.cpu().numpy()


# (parlength, res): the /1.5 loop runs 0 times on long paths, once, many times, and res not dividing parlength
WP_PARAMS = [(3.0, 1.0), (3.0, 0.7), (1.6, 0.5), (40.0, 0.3), (1e6, 0.25)]


@pytest.mark.parametrize("B", [1, 4096])
def test_waypoints_device_equal_host(B):
    ev = I.Evaluator(_cfg())
    rng = np.random.default_rng(B)
    base = [1, 2, 3, 5000, 4, 7]
    lengths = (base + list(rng.integers(1, 40, B)))[:B] if B > 1 else [5000]
    off, xyz = _ragged_paths(lengths, B)
    for parlength, res in WP_PARAMS:
        r, wp, wo, pc = _wp_host(off, xyz, res, parlength, int(off[-1]))
        assert r == 0
        total = int(wo[-1])
        for cap in (total, total - 1):
            if cap < 0:
                continue
            hr, hwp, hwo, hpc = _wp_host(off, xyz, res, parlength, cap)
            dr, dwp, dwo, dpc = _wp_device(ev, off, xyz, res, parlength, cap)
            assert hr == dr == (0 if cap == total else -1), (parlength, res, cap)
            assert np.array_equal(hwo, dwo) and np.array_equal(hpc, dpc), (parlength, res, cap)
            n = min(cap, total)
            assert np.array_equal(_b(hwp[:n]), _b(dwp[:n])), (parlength, res, cap)
    # cap 0 with no waypoints: paths of 1 and 2 nodes
    off, xyz = _ragged_paths([1, 2] * (B // 2) if B > 1 else [2], 3)
    hr, _, hwo, hpc = _wp_host(off, xyz, 1.0, 3.0, 0)
    dr, _, dwo, dpc = _wp_device(ev, off, xyz, 1.0, 3.0, 0)
    assert hr == dr == 0 and np.array_equal(hwo, dwo) and np.array_equal(hpc, dpc) and (dpc == 1).all()
    ev.close()


# ---- planning ---------------------------------------------------------------------------------------------------------------------------
def _host(ev, p, starts, goals, pairs=True, max_fields=0, cap_nodes=100000, cap_pieces=100000):
    """the host form's raw outputs as numpy arrays"""
    B = len(goals)
    ip = C.POINTER(C.c_int32)
    st, gl = np.ascontiguousarray(starts, dtype=np.float64), np.ascontiguousarray(goals, dtype=np.float64)
    pf, po = np.zeros(B + 1, dtype=np.int32), np.zeros(B + 1, dtype=np.int32)
    xyz, T, Cc = np.zeros((max(cap_nodes, 1), 3)), np.zeros(max(cap_pieces, 1)), np.zeros(18 * max(cap_pieces, 1))
    res, cs, ds = (I.PlanResult * B)(), (I.CertifySummary * B)(), (I.DynamicsSummary * B)()
    args = (C.byref(p),) + ((max_fields,) if pairs else ()) + (cap_nodes, pf.ctypes.data_as(ip), I._dp(xyz), cap_pieces, po.ctypes.data_as(ip),
                                                                I._dp(T), I._dp(Cc), res, cs, ds)
    if pairs:
        r = ev.lib.isdf_plan_pairs(ev.h, B, I._dp(st), I._dp(gl), *args)
    else:
        r = ev.lib.isdf_plan_batch(ev.h, I._dp(st), B, I._dp(gl), *args)
    return r, dict(path_off=pf, path_xyz=xyz[:max(pf[-1], 0)], piece_off=po, T=T[:max(po[-1], 0)], coeffs=Cc[:18 * max(po[-1], 0)],
                   results=_b(res), certify=_b(cs), dynamics=_b(ds))


def _device(ev, p, starts, goals, pairs=True, max_fields=0, cap_nodes=100000, cap_pieces=100000, stream=None, d_goals=None):
    """the device form's raw outputs, copied to numpy after the call"""
    torch = _torch()
    B = len(goals)
    s = stream or torch.cuda.current_stream()
    gl = d_goals if d_goals is not None else torch.tensor(np.asarray(goals, dtype=np.float64), device="cuda")
    st = torch.tensor(np.asarray(starts, dtype=np.float64), device="cuda") if pairs else None
    pf, po = torch.full((B + 1,), -7, dtype=torch.int32, device="cuda"), torch.full((B + 1,), -7, dtype=torch.int32, device="cuda")
    xyz = torch.zeros((max(cap_nodes, 1), 3), dtype=torch.float64, device="cuda")
    T, Cc = torch.zeros(max(cap_pieces, 1), dtype=torch.float64, device="cuda"), torch.zeros(18 * max(cap_pieces, 1), dtype=torch.float64, device="cuda")
    res = torch.zeros((B, 64), dtype=torch.uint8, device="cuda")
    cs = torch.zeros((B, C.sizeof(I.CertifySummary)), dtype=torch.uint8, device="cuda")
    ds = torch.zeros((B, C.sizeof(I.DynamicsSummary)), dtype=torch.uint8, device="cuda")
    if stream is not None:   # the outputs' initial fills came first on the current stream; the goals' producer stays unsynchronised
        s.wait_stream(torch.cuda.current_stream())
    ptrs = (pf.data_ptr(), xyz.data_ptr(), cap_pieces, po.data_ptr(), T.data_ptr(), Cc.data_ptr(), res.data_ptr(), cs.data_ptr(), ds.data_ptr(),
            s.cuda_stream)
    if pairs:
        r = ev.plan_pairs_device_raw(B, st.data_ptr(), gl.data_ptr(), p, max_fields, cap_nodes, *ptrs)
    else:
        r = ev.plan_batch_device_raw(starts, B, gl.data_ptr(), p, cap_nodes, *ptrs)
    torch.cuda.synchronize()
    n, q = max(int(pf[-1]), 0), max(int(po[-1]), 0)
    return r, dict(path_off=pf.cpu().numpy(), path_xyz=xyz[:n].cpu().numpy(), piece_off=po.cpu().numpy(), T=T[:q].cpu().numpy(),
                   coeffs=Cc[:18 * q].cpu().numpy(), results=res.cpu().numpy().reshape(-1), certify=cs.cpu().numpy().reshape(-1),
                   dynamics=ds.cpu().numpy().reshape(-1))


def _same_outputs(a, b, what=""):
    for k in a:
        assert np.array_equal(_b(a[k]), _b(b[k])), (what, k)


def _parity(ev, p, starts, goals, pairs=True, max_fields=0):
    rh, h = _host(ev, p, starts, goals, pairs, max_fields)
    ih = ev.plan_info()
    rd, d = _device(ev, p, starts, goals, pairs, max_fields)
    idv = ev.plan_info()
    assert rh == rd == 0
    _same_outputs(h, d, (pairs, max_fields, p.flags))
    assert ih["groups"] == idv["groups"] and ih["backend_rounds"] == idv["backend_rounds"]
    return h


def _stages(h):
    return I.decode_plan_results(_torch().from_numpy(h["results"].copy()))["stage"].numpy()


def _batch_trajectories(ev, h):
    st = _stages(h)
    pieces = [int(h["piece_off"][b + 1] - h["piece_off"][b]) for b in range(len(st)) if st[b] == I.OPTIMISED]
    return ev.batch_trajectories_ragged(pieces) if pieces else None


def test_parity_stages_flags_and_fields():
    occ, _, goals = _scene(12)
    occ = occ.copy()
    occ[30:35, 30:35, 30:35] = 1
    occ[31:34, 31:34, 31:34] = 0                                 # NO_PATH: a free pocket no path reaches
    ev = _ev("Ball", occ)
    starts = _pairs(ev, occ, goals, 5)
    goals = np.concatenate([goals, [[32.5, 32.5, 32.5]]])
    starts = np.concatenate([starts, starts[:1]])
    seen = set()
    for flags in (0, I.PLAN_CERTIFY, I.PLAN_DYNAMICS, I.PLAN_CERTIFY | I.PLAN_DYNAMICS):
        p = _params(ev, flags=flags)
        h = _parity(ev, p, starts, goals)
        seen |= set(_stages(h).tolist())
        # isdf_get_batch_trajectories afterwards: the device call left what the host call left
        rh, h2 = _host(ev, p, starts, goals)
        th = _batch_trajectories(ev, h2)
        _device(ev, p, starts, goals)
        td = _batch_trajectories(ev, h2)
        if th is not None:
            for a, b in zip(th, td):
                for x, y in zip(a, b):
                    assert np.array_equal(_b(np.asarray(x)), _b(np.asarray(y)))
    p = _params(ev)
    for mf in (1, 2):
        _parity(ev, p, starts, goals, max_fields=mf)
    _parity(ev, p, starts[:1], goals[:1])                        # B = 1
    _parity(ev, p, starts[0], goals, pairs=False)                # isdf_plan_batch_device
    _parity(ev, p, starts[0], goals[3:4], pairs=False)
    q = _params(ev, midend_max_rounds=1)                         # MIDEND_FAILED
    h = _parity(ev, q, starts, goals)
    seen |= set(_stages(h).tolist())
    ev.close()
    # TOO_LONG: the 300-voxel corridor with parlength 1
    occ = np.zeros((300, 3, 3), dtype=np.uint8)
    ev = _ev("Ball", occ, _cfg(ks=5))
    p = _params(ev, parlength=1.0)
    h = _parity(ev, p, np.array([[0.5, 1.5, 1.5], [280.5, 1.5, 1.5]]), np.array([[298.5, 1.5, 1.5], [260.5, 1.5, 1.5]]))
    seen |= set(_stages(h).tolist())
    ev.close()
    assert {I.NO_PATH, I.TOO_LONG, I.MIDEND_FAILED, I.OPTIMISED} <= seen, seen


def test_stream_order_chaining_and_mixed_use():
    torch = _torch()
    occ, _, goals = _scene(10, seed=11)
    ev = _ev("Ball", occ)
    starts = _pairs(ev, occ, goals, 11)
    p = _params(ev)
    rh, h = _host(ev, p, starts, goals)
    assert rh == 0
    # goals produced by a torch kernel on a side stream, not synchronised before the call
    side = torch.cuda.Stream()
    base = torch.tensor(goals - 1.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        d_goals = base + 1.0
    rd, d = _device(ev, p, starts, goals, stream=side, d_goals=d_goals)
    assert rd == 0
    _same_outputs(h, d, "side stream")
    # chaining: the public wrapper's tensors straight into trajectory_states_device
    out = ev.plan_pairs_device(torch.tensor(starts, device="cuda"), torch.tensor(goals, device="cuda"), p)
    assert np.array_equal(_b(out["results"].cpu().numpy().reshape(-1)), h["results"])
    plans, _ = ev.plan_pairs(starts, goals, p)
    B = len(goals)
    rng = np.random.default_rng(3)
    traj = rng.integers(0, B, 500).astype(np.int32)
    times = rng.uniform(-0.5, 12.0, 500)
    ref = ev.trajectory_states(plans, traj, times)
    d_out = torch.empty((500, I.STATE_DOUBLES), dtype=torch.float64, device="cuda")
    d_traj, d_times = torch.from_numpy(traj).cuda(), torch.from_numpy(times).cuda()
    ev.trajectory_states_device(B, out["piece_off"].data_ptr(), out["T"].data_ptr(), out["coeffs"].data_ptr(), 500, d_traj.data_ptr(),
                                d_times.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(_b(ref), _b(d_out.cpu().numpy()))
    fields = I.decode_plan_results(out["results"])
    assert [int(x) for x in fields["stage"].cpu()] == [g["stage"] for g in plans]
    assert np.array_equal(fields["duration"].cpu().numpy(), np.array([g["duration"] for g in plans]))
    # mixed use: host and device calls alternated on one context
    for k in range(2):
        _, hk = _host(ev, p, starts, goals)
        _, dk = _device(ev, p, starts, goals)
        _same_outputs(h, hk, ("host", k))
        _same_outputs(h, dk, ("device", k))
    _, bh = _host(ev, p, starts[0], goals, pairs=False)
    _, bd = _device(ev, p, starts[0], goals, pairs=False)
    _same_outputs(bh, bd, "batch")
    ev.close()


def test_caps_refusals_and_state_left_behind():
    torch = _torch()
    occ, _, goals = _scene(4, seed=9)
    ev = _ev("Ball", occ)
    starts = _pairs(ev, occ, goals, 9)
    p = _params(ev)
    _, full = _host(ev, p, starts, goals)
    nodes, pieces = int(full["path_off"][-1]), int(full["piece_off"][-1])
    for cn, cp in ((nodes - 1, 100000), (100000, pieces - 1)):
        rh, h = _host(ev, p, starts, goals, cap_nodes=cn, cap_pieces=cp)
        rd, d = _device(ev, p, starts, goals, cap_nodes=cn, cap_pieces=cp)
        assert rh == rd == -1
        assert d["path_off"][-1] == nodes and d["piece_off"][-1] == pieces
        for k in ("path_off", "piece_off", "results", "certify", "dynamics"):
            assert np.array_equal(_b(h[k]), _b(d[k])), k
        assert (_stages(d) == I.PLAN_FAILED).all()
    # the public wrapper repeats a call whose caps are too small
    out = ev.plan_pairs_device(torch.tensor(starts, device="cuda"), torch.tensor(goals, device="cuda"), p, cap_nodes=1, cap_pieces=1)
    assert np.array_equal(out["T"].cpu().numpy(), full["T"]) and np.array_equal(out["path_xyz"].cpu().numpy(), full["path_xyz"])
    # refusals: the host form's codes, and the same poisoned outputs
    bad = starts.copy()
    bad[2] = [-1.0, 3.0, 3.0]
    cases = [("start outside", p, bad, goals, {}), ("goal outside", p, starts, bad, {}), ("max_fields", p, starts, goals, dict(max_fields=-1))]
    for field, value in (("reserved_", 1), ("flags", 4)):
        q = _params(ev)
        setattr(q, field, value)
        cases.append((field, q, starts, goals, {}))
    for what, q, s, g, kw in cases:
        rh, h = _host(ev, q, s, g, **kw)
        rd, d = _device(ev, q, s, g, **kw)
        assert rh == rd == -1, what
        for k in ("results", "certify", "dynamics"):
            assert np.array_equal(h[k], d[k]), (what, k)
    # NULL device pointers
    d_g = torch.tensor(goals, device="cuda")
    res = torch.zeros((4, 64), dtype=torch.uint8, device="cuda")
    po = torch.zeros(5, dtype=torch.int32, device="cuda")
    assert ev.plan_pairs_device_raw(4, 0, d_g.data_ptr(), p, 0, 10, 0, 0, 0, po.data_ptr(), 0, 0, res.data_ptr(), 0, 0) == -1
    assert ev.plan_batch_device_raw(starts[0], 4, 0, _params(ev, flags=0), 10, 0, 0, 0, po.data_ptr(), 0, 0, res.data_ptr(), 0, 0) == -1
    assert ev.plan_batch_device_raw(starts[0], 4, d_g.data_ptr(), _params(ev, flags=0), 10, 0, 0, 0, po.data_ptr(), 0, 0, 0, 0, 0) == -1
    assert ev.plan_batch_device_raw(starts[0], 4, d_g.data_ptr(), p, 10, 0, 0, 0, po.data_ptr(), 0, 0, res.data_ptr(), 0, 0) == -1   # no summaries
    # sharded context, no front-end kernels, no shape, no map
    ev.set_shard(0, 2)
    assert _host(ev, p, starts, goals)[0] == _device(ev, p, starts, goals)[0] == -4
    ev.set_shard(0, 1)
    ev.close()
    for kw, code in ((dict(kernels=False), -2),):
        e2 = _ev("Ball", occ, **kw)
        rh, h = _host(e2, p, starts, goals)
        rd, d = _device(e2, p, starts, goals)
        assert rh == rd == code and np.array_equal(h["results"], d["results"])
        e2.close()
    e3 = I.Evaluator(_cfg())
    e3.set_map_u8(occ, [0, 0, 0], 1.0)
    assert _host(e3, p, starts, goals)[0] == _device(e3, p, starts, goals)[0] == -2     # no shape
    e3.close()
    e4 = I.Evaluator(_cfg())
    assert _host(e4, p, starts, goals)[0] == _device(e4, p, starts, goals)[0] == -2     # no map
    e4.close()


def test_transfer_budget():
    occ, _, goals = _scene(16, seed=13)
    ev = _ev("Ball", occ)
    starts = _pairs(ev, occ, goals, 13)
    p = _params(ev, flags=0)
    B = len(goals)
    _device(ev, p, starts, goals)
    dev = ev.dbg_plan_transfers()
    _host(ev, p, starts, goals)
    host = ev.dbg_plan_transfers()
    print("device", dev, "host", host)
    assert dev["d2h_bytes"] <= 80 * B + 64 and dev["round_reads"] > 0
    assert host["d2h_bytes"] > dev["d2h_bytes"] + 24 * (B + 1)           # at least every path node and every piece's duration crossed
    ev.close()
    # paths several times longer: the same B plans in a corridor 4x as long give the same device-to-host bytes
    got = []
    for L in (40, 160):
        occ = np.zeros((L + 4, 12, 3), dtype=np.uint8)
        e = _ev("Ball", occ, _cfg(ks=5))
        s = np.array([[0.5 + k % 4, 1.5 + 2 * (k // 4), 1.5] for k in range(8)])
        g = s + [L, 0, 0]
        q = _params(e, flags=0, parlength=8.0)
        r, d = _device(e, q, s, g)
        assert r == 0
        got.append((e.dbg_plan_transfers()["d2h_bytes"], int(d["path_off"][-1])))
        e.close()
    # equal unless a plan's mid-end outcome differs between the two lengths (its gathered point count: 4 bytes)
    assert got[1][1] >= 3 * got[0][1] and got[1][0] <= got[0][0] + 4 * 8 and got[1][0] <= 80 * 8 + 64, got
