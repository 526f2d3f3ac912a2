"""The occupancy grid from a point cloud (isdf_set_map_cloud / isdf_set_map_cloud_device) on the GPU: every case of
tests/golden/cloud_reference.npz (reference-compiled voxelisation) bit for bit through both entry points and both readbacks; skipped
non-finite records; refusals that leave the previous map in place; a 20 M-point cloud built twice and shuffled; and downstream
bit-identity of the evaluation, gather, clearance and front-end entry points with the same occupancy given to isdf_set_map_u8."""
import numpy as np
import pytest
import torch
import cloud_oracle as CO
import isdf_b200 as I
import workloads as W

pytestmark = pytest.mark.gpu
FIX = CO.load_fixture()


def evaluator(collision=True):
    cfg = I.default_config_values()
    if collision:
        cfg.flags = I.WITH_DYNAMICS | I.WITH_COLLISION
        cfg.integral_intervs = 16
    return I.Evaluator(cfg, device=0)


def check_map(ev, f, thr, n_used, n_skipped=0):
    info = ev.map_info()
    assert info["dims"] == f["dims"] and info["res"] == f["res"]
    assert np.array_equal(info["bmin"], f["bmin"]) and np.array_equal(info["bmax"], f["bmax"])
    assert info["points_used"] == n_used and info["points_skipped"] == n_skipped
    occ = f["occ"][thr]
    assert info["occupied_voxels"] == int(occ.sum())
    u8 = ev.get_map_u8()
    assert np.array_equal(u8, occ), f"{int((u8 != occ).sum())} voxels differ"
    f64 = ev.get_map_f64()
    assert f64.dtype == np.float64 and np.array_equal(f64, occ.astype(np.float64))


@pytest.mark.parametrize("name", sorted(FIX))
def test_fixture_cases_bit_identical_through_both_entry_points(name):
    f = FIX[name]
    n = f["raw"].size // f["stride"]
    ev = evaluator(collision=False)
    d_raw = torch.from_numpy(f["raw"].copy()).cuda()
    for thr in CO.THRESHOLDS:
        s0 = ev.stats()
        ev.set_map_cloud(f["raw"], f["res"], thr, stride_bytes=f["stride"])
        s1 = ev.stats()
        assert s1.kernel_launches > s0.kernel_launches
        assert (s1.evals_discrete, s1.evals_swept, s1.last_pairs, s1.last_sdf_evals, s1.last_kernel_ms) == \
               (s0.evals_discrete, s0.evals_swept, s0.last_pairs, s0.last_sdf_evals, s0.last_kernel_ms)
        check_map(ev, f, thr, n)
        ev.set_map_cloud_device(d_raw.data_ptr(), n=n, stride_bytes=f["stride"], res=f["res"], sta_threshold=thr,
                                stream=torch.cuda.current_stream().cuda_stream)
        check_map(ev, f, thr, n)
    # a negative threshold behaves as 0 (every voxel occupied), as in the reference
    ev.set_map_cloud(f["raw"], f["res"], -3, stride_bytes=f["stride"])
    check_map(ev, f, 0, n)
    # float32 (n, k) arrays and tensors: PointXYZ-style rows
    if f["stride"] in (12, 16):
        rows = f["raw"].view(np.float32).reshape(n, f["stride"] // 4)
        ev.set_map_cloud(rows, f["res"], 2)
        check_map(ev, f, 2, n)
        ev.set_map_cloud_device(torch.from_numpy(rows.copy()).cuda(), res=f["res"], sta_threshold=2)
        check_map(ev, f, 2, n)
    ev.close()


def test_non_finite_records_are_skipped_and_counted():
    f = FIX["uniform_r04_stride32"]
    rec = f["raw"].view(np.float32).reshape(-1, 8)
    bad = np.zeros((5, 8), dtype=np.float32)
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3, :3], bad[4, 0] = np.nan, np.inf, -np.inf, [1e30, np.nan, 0], -np.inf
    allrec = np.concatenate([bad[:2], rec[:100], bad[2:], rec[100:]])
    ev = evaluator(collision=False)
    for thr in (1, 3):
        ev.set_map_cloud(allrec, f["res"], thr)
        check_map(ev, f, thr, rec.shape[0], 5)
        ev.set_map_cloud_device(torch.from_numpy(allrec.copy()).cuda(), res=f["res"], sta_threshold=thr)
        check_map(ev, f, thr, rec.shape[0], 5)
    ev.close()


def test_refusals_leave_the_previous_map_usable_and_unchanged():
    f = FIX["faces_r1_xyz16"]
    ev = evaluator()
    ev.set_shape_named("Ball")
    ev.set_map_cloud(f["raw"], f["res"], 1, stride_bytes=f["stride"])
    before, occ = ev.map_info(), ev.get_map_u8()
    T, Cc, _ = W.make_trajectory(3, f["bmin"], f["bmax"], seed=4, jitter=0.2)
    c0, g0, t0 = ev.eval_discrete(T, Cc)
    rng = np.random.default_rng(7)
    flat = np.concatenate([rng.random((50, 2)) * 5, np.full((50, 1), 1.5)], 1).astype(np.float32)           # every z equal
    huge = np.array([[0, 0, 0], [5000, 5000, 3000]], dtype=np.float32)                                   # X*Y*ceil(Z/32) >= 2^31
    fine = (rng.random((100, 3)) * 2).astype(np.float32)                                                 # a pose window > 1023 voxels
    nan = np.full((10, 3), np.nan, dtype=np.float32)
    tall = np.array([[0, 0, 0], [1, 1, 70000]], dtype=np.float32)                                        # Z > 65535
    for pts, res, code, msg in ((flat, 1.0, -1, "degenerate"), (huge, 0.05, -1, "map too large"), (fine, 0.01, -4, "resolution too fine"),
                                (nan, 1.0, -1, "no point with finite"), (tall, 1.0, -4, "Z > 65535")):
        for dev in (False, True):
            with pytest.raises(I.IsdfError) as e:
                if dev:
                    ev.set_map_cloud_device(torch.from_numpy(pts).cuda(), res=res)
                else:
                    ev.set_map_cloud(pts, res)
            assert e.value.code == code and msg in str(e.value), str(e.value)
            if msg not in ("degenerate", "no point with finite"):
                assert "the cloud asks for" in str(e.value)
            after = ev.map_info()
            assert after["dims"] == before["dims"] and np.array_equal(after["bmax"], before["bmax"])
            assert after["occupied_voxels"] == before["occupied_voxels"] and np.array_equal(ev.get_map_u8(), occ)
            c1, g1, t1 = ev.eval_discrete(T, Cc)
            assert c1 == c0 and np.array_equal(g1, g0) and np.array_equal(t1, t0)
    ev.close()


def test_large_cloud_is_order_independent_and_matches_the_cpu():
    rng = np.random.default_rng(11)
    occ = W.random_map(96, 80, 64, p=0.06, seed=5)
    idx = np.argwhere(occ)
    k = max(1, -(-20_000_000 // idx.shape[0]))
    pts = (np.repeat(idx, k, axis=0) + rng.random((idx.shape[0] * k, 3))) * 0.25 + np.array([-7.3, 2.15, -0.6])
    pts = np.concatenate([pts, [[-7.3, 2.15, -0.6], [-7.3 + 24.0, 2.15 + 20.0, -0.6 + 16.0]]]).astype(np.float32)
    assert pts.shape[0] >= 20_000_000
    ev = evaluator(collision=False)
    for thr in (1, 3):
        ref = CO.numpy_map(pts, 12, 0.25, thr)
        ev.set_map_cloud(pts, 0.25, thr)
        a = ev.get_map_u8()
        assert np.array_equal(a, ref["occ"]) and ev.map_info()["dims"] == ref["dims"]
        d = torch.from_numpy(pts).cuda()
        ev.set_map_cloud_device(d, res=0.25, sta_threshold=thr)
        assert np.array_equal(ev.get_map_u8(), a)
        d = d[torch.randperm(d.shape[0], device=d.device)].contiguous()
        ev.set_map_cloud_device(d, res=0.25, sta_threshold=thr)
        assert np.array_equal(ev.get_map_u8(), a)
        del d
    ev.close()


def border_cloud(res, seed):
    """a cloud whose maximum lies off the bmin + X*res lattice, with obstacles in the far corner: k jittered points per occupied voxel"""
    rng = np.random.default_rng(seed)
    occ = W.three_slit_map(40, 36, 30, noise=0.05, seed=seed)
    occ[-6:, -6:, -6:] |= (rng.random((6, 6, 6)) < 0.5).astype(occ.dtype)
    bmin = np.array([-3.25, 1.5, -0.75])
    idx = np.argwhere(occ)
    pts = (np.repeat(idx, 3, axis=0) + 0.05 + 0.9 * rng.random((idx.shape[0] * 3, 3))) * res + bmin
    top = bmin + (np.array(occ.shape) - 0.35) * res
    pts = np.concatenate([pts, [bmin, top]]).astype(np.float32)
    return pts, occ


@pytest.mark.parametrize("res", [1.0, 0.4])
def test_downstream_bit_identical_to_set_map_u8(res):
    pts, _ = border_cloud(res, seed=2)
    ev_c, ev_u = evaluator(), evaluator()
    ev_c.set_map_cloud(pts, res, 1)
    info = ev_c.map_info()
    occ = ev_c.get_map_u8()
    X, Y, Z = info["dims"]
    assert np.all(info["bmax"] < info["bmin"] + np.array(info["dims"]) * res)      # the cloud's maximum, not the lattice
    ev_u.set_map_u8(occ, info["bmin"], res)
    assert np.array_equal(ev_u.get_map_u8(), occ)
    far = info["bmin"] + np.array(info["dims"]) * res
    wp = np.array([info["bmin"] + [4.0, 5.0, 3.0], far - [8.0, 6.0, 5.0], far - [2.0, 1.5, 1.0], far + [1.5, 1.0, 0.5], far + [3.0, -2.0, 1.0]])
    T = np.full(wp.shape[0] - 1, 2.0)
    Cc = W.minco_s3(wp, T)
    for shape in ("Ball", "RoundedCone"):
        for ev in (ev_c, ev_u):
            ev.set_shape_named(shape)
        a, b = ev_c.eval_discrete(T, Cc), ev_u.eval_discrete(T, Cc)
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        assert np.array_equal(ev_c.piece_costs(T.size), ev_u.piece_costs(T.size))
        ga, gb = ev_c.gather_obstacle_points(wp, 3.0), ev_u.gather_obstacle_points(wp, 3.0)
        assert ga[1] == gb[1] > 0 and np.array_equal(ga[0], gb[0])
        pa, pb = ev_c.points_in_aabb(far - 1.0, 2.5), ev_u.points_in_aabb(far - 1.0, 2.5)
        assert pa[1] == pb[1] > 0 and np.array_equal(pa[0], pb[0])
        ca, cb = ev_c.trajectory_clearance(T, Cc, 8, 2.0, 0.866), ev_u.trajectory_clearance(T, Cc, 8, 2.0, 0.866)
        assert np.array_equal(ca[0], cb[0]) and np.array_equal(ca[1], cb[1]) and ca[2] == cb[2]
    assert ev_c.frontend_build_kernels() == ev_u.frontend_build_kernels()
    fa, fb = ev_c.frontend_feasibility(X, Y, Z), ev_u.frontend_feasibility(X, Y, Z)
    assert np.array_equal(fa, fb)
    ev_c.close(); ev_u.close()


@pytest.mark.parametrize("dims", [(7, 5, 33), (3, 4, 1), (17, 9, 70), (40, 30, 31)])
def test_readback_round_trips_set_map_u8(dims):
    rng = np.random.default_rng(sum(dims))
    occ = (rng.random(dims) < 0.3).astype(np.uint8)
    ev = evaluator(collision=False)
    ev.set_map_u8(occ * rng.integers(1, 255, size=dims).astype(np.uint8), [0.5, -1.0, 2.0], 0.7)
    assert np.array_equal(ev.get_map_u8(), occ)
    assert np.array_equal(ev.get_map_f64(), occ.astype(np.float64))
    info = ev.map_info()
    assert info["occupied_voxels"] == int(occ.sum()) and info["points_used"] == 0 and info["points_skipped"] == 0
    assert np.array_equal(info["bmax"], np.array([0.5, -1.0, 2.0]) + np.array(dims) * 0.7)
    ev.set_map_f64(occ.astype(np.float64), [0.5, -1.0, 2.0], 0.7)
    assert np.array_equal(ev.get_map_u8(), occ)
    short = np.zeros(occ.size - 1, dtype=np.uint8)
    assert ev.lib.isdf_get_map_u8(ev.h, short.ctypes.data_as(I.C.POINTER(I.C.c_uint8)), short.size) == -1
    ev.close()


def test_no_map_is_a_state_error():
    ev = evaluator(collision=False)
    with pytest.raises(I.IsdfError) as e:
        ev.map_info()
    assert e.value.code == -2
    ev.close()
