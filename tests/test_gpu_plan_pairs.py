"""(start, goal) pairs: the source-batched cost-to-come fields against the serial Dijkstra and the single-source field bit for bit, each
pair of isdf_frontend_path_pairs against isdf_frontend_path on that pair alone, and each plan of isdf_plan_pairs against isdf_plan_batch
on that pair alone; permutations, every max_fields, the host and device forms, the refusals and the state the planning call leaves."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W
import frontpath_oracle as FO
from test_gpu_frontend_path import _setup, _centre, _index, _field
from test_gpu_plan import _ev, _cfg, _scene, _params, _check_plan

pytestmark = pytest.mark.gpu

BMIN = np.array([-3.25, 1.5, 0.125])


def _pocket_map():
    """random clutter with one free voxel (5, 5, 5) inside a solid block: a start with no traversable neighbour"""
    occ = (np.random.default_rng(11).random((20, 18, 22)) < 0.04).astype(np.uint8)
    occ[4:7, 4:7, 4:7] = 1
    occ[5, 5, 5] = 0
    return occ


FIELD_CASES = {
    # name: (occupancy, robot, kernel_size, front_end_safeh)
    "random24_ball": (lambda: W.random_map(24, 24, 24, p=0.05, seed=3, slabs=1), "Ball", 5, 0.0),
    "slits_40x36x28_capped_cone": (lambda: W.three_slit_map(40, 36, 28, noise=0.003, seed=5), "CappedCone", 13, 0.0),
    "random_64_mesh": (lambda: (np.random.default_rng(6).random((64, 40, 37)) < 0.05).astype(np.uint8), "mesh", 9, 0.8),
    "pocket_20_ball": (_pocket_map, "Ball", 3, 0.0),
}


def _fields(ev, starts, shape):
    import torch
    S = len(starts)
    d_g = torch.empty(S * int(np.prod(shape)), dtype=torch.float64, device="cuda")
    ev.frontend_path_fields_device(starts, d_g.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_g.cpu().numpy().reshape((S,) + tuple(shape))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("case", list(FIELD_CASES))
def test_source_batched_fields_equal_dijkstra_and_the_single_field(case):
    mk, robot, ks, safeh = FIELD_CASES[case]
    occ = mk()
    X, Y, Z = occ.shape
    ev = _setup(occ, robot, ks, safeh=safeh)
    trav = FO.traversable(occ, ev.frontend_feasibility(X, Y, Z))
    rng = np.random.default_rng(sum(map(ord, case)))
    cand = np.argwhere(trav)
    a = cand[rng.integers(0, len(cand))]
    # the voxel with the fewest traversable neighbours (none in the pocket map)
    pad = np.pad(trav.astype(np.int32), 1)
    nb = sum(pad[1 + i:1 + i + X, 1 + j:1 + j + Y, 1 + k:1 + k + Z] for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)) - trav
    lonely = (5, 5, 5) if case == "pocket_20_ball" else np.unravel_index(np.argmin(np.where(occ == 0, nb, 99)), occ.shape)
    if case == "pocket_20_ball":
        assert nb[lonely] == 0
    voxels = [a, a, np.argwhere(occ)[0], np.array(lonely), cand[rng.integers(0, len(cand))]]   # two starts in one voxel, one occupied
    starts = np.array([_centre(v) + rng.uniform(-0.45, 0.45, 3) for v in voxels])
    for S in (1, 2, 5):
        g = _fields(ev, starts[:S], (X, Y, Z))
        info = ev.frontend_path_info()
        assert info["field_bytes"] == 8 * S * X * Y * Z and info["rounds"] >= 1
        for s in range(S):
            src = tuple(int(v) for v in voxels[s])
            ref = FO.dijkstra(trav.astype(np.uint8), src)
            assert np.array_equal(_bits(g[s]), _bits(ref)), (case, S, s, int((_bits(g[s]) != _bits(ref)).sum()))
            one = _field(ev, starts[s], (X, Y, Z))
            assert np.array_equal(_bits(g[s]), _bits(one)), (case, S, s)
    lone = FO.dijkstra(trav.astype(np.uint8), tuple(int(v) for v in voxels[3]))
    if nb[lonely] == 0:
        assert np.isfinite(lone).sum() == 1
    ev.close()


def _split_scene():
    """a map cut by a full wall at x = 20 and a wall at y = 18 with one hole: goals reachable from some starts and not from others"""
    occ = (np.random.default_rng(21).random((40, 36, 28)) < 0.02).astype(np.uint8)
    occ[20, :, :] = 1
    occ[:20, 18, :] = 1
    occ[:20, 18, 14] = 0
    occ[2:5, 2:5, 2:5] = 1
    occ[3, 3, 3] = 0                                     # an isolated free voxel
    ev = _setup(occ, "Ball", 3)
    X, Y, Z = occ.shape
    trav = FO.traversable(occ, ev.frontend_feasibility(X, Y, Z))
    rng = np.random.default_rng(22)
    left, right = np.argwhere(trav[:20]), np.argwhere(trav[21:]) + [21, 0, 0]
    sv = [left[rng.integers(0, len(left))], right[rng.integers(0, len(right))], left[rng.integers(0, len(left))],
          right[rng.integers(0, len(right))], np.array([3, 3, 3])]
    gv = [left[rng.integers(0, len(left))] for _ in range(4)] + [right[rng.integers(0, len(right))] for _ in range(4)] + [np.array([3, 3, 3])]
    si = [0, 1, 2, 3, 4, 0, 1, 2, 3, 0, 1, 4, 2, 0]
    gi = [0, 1, 4, 5, 8, 6, 2, 3, 7, 8, 0, 1, 2, 4]
    starts = np.array([_centre(sv[i]) + rng.uniform(-0.45, 0.45, 3) for i in si])
    starts[5] = _centre(sv[0]) + [0.3, -0.2, 0.1]         # another point of start 0's voxel
    goals = np.array([_centre(gv[i]) + rng.uniform(-0.45, 0.45, 3) for i in gi])
    return ev, occ, starts, goals


def _same_paths(a, b):
    for k in ("xyz", "rp", "offsets", "costs", "found"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def test_frontend_pairs_equal_each_pair_alone():
    import torch
    ev, occ, starts, goals = _split_scene()
    B = len(goals)
    res = ev.frontend_path_pairs(starts, goals)
    info = ev.frontend_path_info()
    X, Y, Z = occ.shape
    S = len({tuple(_index(s)) for s in starts})
    assert S == 5 and info["field_bytes"] == 8 * S * X * Y * Z and info["rounds"] >= 1
    assert 3 <= res["found"].sum() < B
    reach = set()
    for b in range(B):
        p, rp, c, f = ev.frontend_path(starts[b], goals[b])
        assert np.array_equal(p, res["paths"][b]) and np.array_equal(rp, res["roll_pitch"][b]) and f == res["found"][b], b
        assert np.float64(c).view(np.uint64) == res["costs"][b].view(np.uint64), b
        assert np.array_equal(_index(p[0]), _index(starts[b]))
        reach.add((tuple(_index(goals[b])), bool(f)))
    # a goal reachable from one start and not from another: a field leaking into another slice fails the comparison above
    assert any((g, True) in reach and (g, False) in reach for g, _ in reach)
    # every max_fields gives the same bits; the fields held at once follow it
    for mf in (1, 2, 3):
        again = ev.frontend_path_pairs(starts, goals, max_fields=mf)
        _same_paths(again, res)
        assert ev.frontend_path_info()["field_bytes"] == 8 * min(mf, S) * X * Y * Z
    # permuted pairs permute the outputs
    perm = np.random.default_rng(3).permutation(B)
    sh = ev.frontend_path_pairs(starts[perm], goals[perm], max_fields=2)
    for k, b in enumerate(perm):
        assert np.array_equal(sh["paths"][k], res["paths"][b]) and np.array_equal(sh["roll_pitch"][k], res["roll_pitch"][b])
        assert sh["costs"][k].view(np.uint64) == res["costs"][b].view(np.uint64) and sh["found"][k] == res["found"][b]
    # the device form on a side stream
    n = int(res["offsets"][-1])
    dev = torch.device("cuda", 0)
    d_s, d_t = torch.from_numpy(starts.reshape(-1)).to(dev), torch.from_numpy(goals.reshape(-1)).to(dev)
    d_xyz, d_rp = torch.zeros(3 * n, dtype=torch.float64, device=dev), torch.zeros(2 * n, dtype=torch.float64, device=dev)
    d_off, d_cost = torch.zeros(B + 1, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.float64, device=dev)
    d_found = torch.zeros(B, dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ev.frontend_path_pairs_device(B, d_s.data_ptr(), d_t.data_ptr(), n, d_xyz.data_ptr(), d_rp.data_ptr(), d_off.data_ptr(), d_cost.data_ptr(),
                                      d_found.data_ptr(), side.cuda_stream, max_fields=1)
    side.synchronize()
    assert np.array_equal(d_off.cpu().numpy(), res["offsets"])
    assert np.array_equal(d_xyz.cpu().numpy().reshape(-1, 3), res["xyz"]) and np.array_equal(d_rp.cpu().numpy().reshape(-1, 2), res["rp"])
    assert np.array_equal(d_cost.cpu().numpy().view(np.uint64), res["costs"].view(np.uint64))
    assert np.array_equal(d_found.cpu().numpy().astype(bool), res["found"])
    # one start for every pair: the batch call
    one = ev.frontend_path_pairs(np.repeat(starts[:1], B, axis=0), goals)
    _same_paths(one, ev.frontend_path_batch(starts[0], goals))
    # a cap one node short: ISDF_ERR_INVALID with every offset reported, for every max_fields
    for mf in (0, 1):
        r, off = ev.frontend_path_pairs_raw(starts, goals, n - 1, max_fields=mf)
        assert r == -1 and np.array_equal(off, res["offsets"])
        r, off = ev.frontend_path_pairs_raw(starts, goals, n, max_fields=mf)
        assert r == 0 and np.array_equal(off, res["offsets"])
    ev.close()


def test_frontend_pairs_refusals():
    ev, occ, starts, goals = _split_scene()
    bad = starts.copy()
    bad[3] = BMIN - [1e-9, 0, 0]
    for s, g, mf, what in ((bad, goals, 0, "starts[3]"), (starts, bad, 0, "goals[3]"), (starts, goals, -1, None)):
        r, off = ev.frontend_path_pairs_raw(s, g, 10000, max_fields=mf)
        assert r == -1
        if what:
            assert what in ev.lib.isdf_last_error().decode()
    nan = starts.copy()
    nan[2, 1] = np.nan
    with pytest.raises(I.IsdfError) as e:
        ev.frontend_path_pairs(nan, goals)
    assert e.value.code == -1 and "starts[2]" in str(e.value)
    import torch
    d_g = torch.empty(8, dtype=torch.float64, device="cuda")
    assert ev.lib.isdf_frontend_path_fields_device(ev.h, 0, I._dp(starts), None, d_g.data_ptr(), None) == -1
    with pytest.raises(I.IsdfError) as e:
        ev.frontend_path_fields_device(bad[:4], d_g.data_ptr())
    assert e.value.code == -1 and "starts[3]" in str(e.value)
    ev.set_shard(0, 2)
    with pytest.raises(I.IsdfError) as e:
        ev.frontend_path_pairs(starts, goals)
    assert e.value.code == -4
    ev.close()


def _pairs(ev, occ, goals, seed):
    """pairs from 6 distinct traversable starts of ev's map, each used in turn, to the given goals"""
    trav = np.argwhere(FO.traversable(occ, ev.frontend_feasibility(*occ.shape)))
    sv = trav[np.random.default_rng(seed + 100).choice(len(trav), 6, replace=False)] + 0.5
    return sv[np.arange(len(goals)) % 6]


def _raw_pairs(ev, p, starts, goals, max_fields=0, cap_nodes=100000, cap_pieces=100000):
    B = len(goals)
    ip = C.POINTER(C.c_int32)
    st, gl = np.ascontiguousarray(starts, dtype=np.float64), np.ascontiguousarray(goals, dtype=np.float64)
    pf, po = np.zeros(B + 1, dtype=np.int32), np.zeros(B + 1, dtype=np.int32)
    xyz, T, Cc = np.zeros((max(cap_nodes, 1), 3)), np.zeros(max(cap_pieces, 1)), np.zeros(18 * max(cap_pieces, 1))
    res, cs, ds = (I.PlanResult * B)(), (I.CertifySummary * B)(), (I.DynamicsSummary * B)()
    r = ev.lib.isdf_plan_pairs(ev.h, B, I._dp(st), I._dp(gl), C.byref(p), max_fields, cap_nodes, pf.ctypes.data_as(ip), I._dp(xyz), cap_pieces,
                               po.ctypes.data_as(ip), I._dp(T), I._dp(Cc), res, cs, ds)
    return r, pf, po, res, cs, ds


@pytest.mark.parametrize("robot", ["Ball", "mesh"])
def test_plan_pairs_equal_each_pair_alone(robot):
    occ, _, goals = _scene(12)
    ev = _ev(robot, occ)
    starts = _pairs(ev, occ, goals, 5)
    p = _params(ev)
    assert p.flags == I.PLAN_CERTIFY | I.PLAN_DYNAMICS
    got, info = ev.plan_pairs(starts, goals, p)
    assert len({tuple(s) for s in starts}) >= 5
    assert sum(g["stage"] == I.OPTIMISED for g in got) >= 2 and info["groups"] >= 1 and info["backend_rounds"] > 0
    for b in range(len(goals)):
        alone, _ = ev.plan_batch(starts[b], goals[b:b + 1], p)
        _check_plan(got[b], alone[0], b)
        assert np.array_equal(got[b]["path"][0], starts[b])            # the head: the start voxel's cube centre
    # max_fields = 1 gives the same bits as 0, permuted pairs the permuted outputs
    one, info1 = ev.plan_pairs(starts, goals, p, max_fields=1)
    perm = np.random.default_rng(2).permutation(len(goals))
    sh, _ = ev.plan_pairs(starts[perm], goals[perm], p)
    for b in range(len(goals)):
        _check_plan(one[b], got[b], b)
    for k, b in enumerate(perm):
        _check_plan(sh[k], got[b], b)
    assert info1["groups"] == info["groups"] and info1["backend_rounds"] == info["backend_rounds"]
    # isdf_get_batch_trajectories: every back-end plan's final trajectory, in pair order
    be = [g for g in sh if g["stage"] == I.OPTIMISED]
    T, Cc, _ = ev.batch_trajectories_ragged([g["pieces"] for g in be])
    for g, t, c in zip(be, T, Cc):
        assert np.array_equal(g["T"], t) and np.array_equal(g["coeffs"], np.asarray(c).reshape(-1))
    print(robot, "stages", [g["stage"] for g in got], "N", [g["pieces"] for g in got], "info", info)
    ev.close()


def test_plan_pairs_with_one_start_equal_plan_batch():
    occ, start, goals = _scene(12)
    ev = _ev("Ball", occ)
    p = _params(ev)
    starts = np.repeat(start[None], len(goals), axis=0)
    got, info = ev.plan_pairs(starts, goals, p)
    ref, rinfo = ev.plan_batch(start, goals, p)
    for b in range(len(goals)):
        _check_plan(got[b], ref[b], b)
    assert info["groups"] == rinfo["groups"] and info["backend_rounds"] == rinfo["backend_rounds"]
    from test_gpu_plan import _raw_plan
    r0, pf0, po0, _, _, _ = _raw_plan(ev, p, start, goals)
    r1, pf1, po1, _, _, _ = _raw_pairs(ev, p, starts, goals, max_fields=1)
    assert r0 == 0 and r1 == 0 and np.array_equal(pf0, pf1) and np.array_equal(po0, po1)
    ev.close()


def test_plan_pairs_stages():
    # NO_PATH: a free pocket no path reaches, from two starts; the plan's path is its own start alone
    occ, _, goals = _scene(4, seed=7)
    occ = occ.copy()
    occ[30:35, 30:35, 30:35] = 1
    occ[31:34, 31:34, 31:34] = 0
    ev = _ev("Ball", occ)
    starts = _pairs(ev, occ, goals, 7)
    p = _params(ev)
    goals = np.concatenate([[[32.5, 32.5, 32.5]], goals[1:], [[32.5, 32.5, 32.5]]])
    starts = np.concatenate([starts, starts[2:3]])
    got, _ = ev.plan_pairs(starts, goals, p)
    for b in (0, len(goals) - 1):
        assert got[b]["stage"] == I.NO_PATH and got[b]["path_nodes"] == 1 and np.array_equal(got[b]["path"][0], starts[b])
    for b in range(len(goals)):
        alone, _ = ev.plan_batch(starts[b], goals[b:b + 1], p)
        _check_plan(got[b], alone[0], b)
    # MIDEND_FAILED (-1008: the mid-end's round cap)
    q = _params(ev, midend_max_rounds=1)
    got, info = ev.plan_pairs(starts, goals, q)
    assert info["backend_rounds"] == 0 and sum(g["stage"] == I.MIDEND_FAILED for g in got) >= 1
    for b, g in enumerate(got):
        if g["stage"] != I.NO_PATH:
            assert g["stage"] == I.MIDEND_FAILED and g["midend_ret"] == -1008 and np.isnan(g["backend_f"])
        alone, _ = ev.plan_batch(starts[b], goals[b:b + 1], q)
        _check_plan(g, alone[0], b)
    ev.close()
    # TOO_LONG: the 300-voxel corridor with parlength 1, next to a short pair from another start
    occ = np.zeros((300, 3, 3), dtype=np.uint8)
    ev = _ev("Ball", occ, _cfg(ks=5))
    p = _params(ev, parlength=1.0)
    starts, goals = np.array([[0.5, 1.5, 1.5], [280.5, 1.5, 1.5]]), np.array([[298.5, 1.5, 1.5], [260.5, 1.5, 1.5]])
    got, info = ev.plan_pairs(starts, goals, p)
    assert got[0]["stage"] == I.TOO_LONG and got[0]["pieces"] > 290 and got[0]["T"].size == 0
    assert got[1]["stage"] in (I.OPTIMISED, I.MIDEND_FAILED) and got[1]["pieces"] == 20 and info["groups"] == 1
    for b in range(2):
        alone, _ = ev.plan_batch(starts[b], goals[b:b + 1], p)
        _check_plan(got[b], alone[0], b)
    ev.close()


def test_plan_pairs_refusals_and_state_left_behind():
    occ, _, goals = _scene(4, seed=9)
    ev = _ev("Ball", occ)
    starts = _pairs(ev, occ, goals, 9)
    p = _params(ev)
    bad = starts.copy()
    bad[2] = [-1.0, 3.0, 3.0]
    for s, g, mf, what in ((bad, goals, 0, "starts[2]"), (starts, bad, 0, "goals[2]"), (starts, goals, -1, "max_fields")):
        r, _, _, res, cs, ds = _raw_pairs(ev, p, s, g, max_fields=mf)
        assert r == -1 and what in ev.lib.isdf_last_error().decode()
        assert all(x.stage == -1 and np.isnan(x.midend_f) and np.isnan(x.backend_f) for x in res)
        assert all(x.verdict == 0 and np.isnan(x.lower_bound) for x in cs) and all(x.samples == -1 for x in ds)
    full, _ = ev.plan_pairs(starts, goals, p)                  # caps too small: the sizes needed are reported
    nodes, pieces = sum(g["path_nodes"] for g in full), sum(g["T"].size for g in full)
    r, pf, po, res, _, _ = _raw_pairs(ev, p, starts, goals, cap_nodes=nodes - 1)
    assert r == -1 and pf[-1] == nodes and po[-1] == pieces and all(x.stage == -1 for x in res)
    # both point sets given up after the call, also after a failure past the argument checks
    for s in (starts, bad):
        ev.set_points(np.argwhere(occ)[:50] + 0.5)
        _raw_pairs(ev, p, s, goals)
        dp = C.POINTER(C.c_double)
        T, Cc = np.ones(2), np.zeros(36)
        assert ev.lib.isdf_eval_swept(ev.h, 2, T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(C.c_double(0.0)),
                                      np.zeros(36).ctypes.data_as(dp), np.zeros(2).ctypes.data_as(dp)) == -2
    ev.close()


def test_full_size_fields_past_2_31_elements():
    """129 fields of a 256^3 map in one relaxation: 2^31 + 2^24 elements; slices 0, 64 and 128 (which starts at element 2^31) equal the
    single-source field bit for bit"""
    import torch
    X = 256
    occ = W.random_map(X, X, X, p=0.05, seed=1, slabs=3)
    ev = _setup(occ, "Ball", 5, bmin=np.zeros(3))
    d1 = torch.empty(X ** 3, dtype=torch.float64, device="cuda")
    ev.frontend_path_field_device([0.5, 0.5, 0.5], d1.data_ptr())
    cand = np.argwhere(ev.dbg_frontpath_traversable())
    rng = np.random.default_rng(4)
    S = 129
    starts = cand[rng.choice(len(cand), S, replace=False)] + 0.5
    d_g = torch.empty(S * X ** 3, dtype=torch.float64, device="cuda")
    assert d_g.numel() > 2 ** 31
    ev.frontend_path_fields_device(starts, d_g.data_ptr())
    torch.cuda.synchronize()
    info = ev.frontend_path_info()
    print("256^3 x 129 fields:", info)
    assert info["field_bytes"] == 8 * S * X ** 3
    for s in (0, 64, 128):
        ev.frontend_path_field_device(starts[s], d1.data_ptr())
        torch.cuda.synchronize()
        sl = d_g[s * X ** 3:(s + 1) * X ** 3]
        assert torch.equal(sl.view(torch.int64), d1.view(torch.int64)), s
        assert torch.isfinite(sl).sum().item() > 1
    del d_g
    ev.close()
