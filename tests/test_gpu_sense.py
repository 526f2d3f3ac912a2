"""Depth sensing on the GPU (isdf_sense_*): depth images bit-identical to the reference's own renderer (live when
oracle/_ref/libref_depth.so exists, and against tests/golden/sense_reference.npz always), images and sensed clouds bit-identical to the
serial restatement tests/sense_serial.cpp at the cull boundaries, independence of Q, pose order and chunking, host and device forms, poses
read in place from a simulate log and from trajectory-state records, the chain plan -> simulate -> sense -> map against the serial chain,
the cloud's replacement, errors and the cap."""
import numpy as np
import pytest
import isdf_b200 as I
import sense_oracle as SO

pytestmark = pytest.mark.gpu


def _torch():
    import torch
    return torch


def _ev(xyz=None):
    ev = I.Evaluator(I.default_config_values())
    if xyz is not None:
        ev.set_sense_cloud(xyz)
    return ev


def _records(pos, quat):
    return np.ascontiguousarray(np.column_stack([pos, quat]))


def _boundary_scene(pos, quat, p, seed=11):
    """a room plus points placed at pose 0's cull boundaries: centres just inside and just outside each image edge, and points on the
    optical axis just within and just beyond the horizon at depth"""
    rng = np.random.default_rng(seed)
    c2w = SO.pose(pos[0], quat[0], np.array(p.cam_to_body[:]))[0].reshape(4, 4)
    cam = []
    for z in (1.0, 2.5, 4.0):
        for e in (-1e-6, 0.0, 1e-6, 1e-4):
            for px in (-1.0 + e, -0.5 + e, p.width - 0.5 + e, p.width + e):   # centre values around the rule's edges
                cam.append(((px - 0.5 - p.cx) / p.fx * z, rng.uniform(-0.3, 0.3) * z, z))
            for py in (-1.0 + e, -0.5 + e, p.height - 0.5 + e, p.height + e):
                cam.append((rng.uniform(-0.3, 0.3) * z, (py - 0.5 - p.cy) / p.fy * z, z))
    if np.isfinite(p.sensing_horizon):
        for dz in (-2e-3, -5e-4, -1e-4, 0.0, 1e-4, 4e-4, 6e-4, 1e-3, 2e-3, 3e-3):
            cam.append((0.0, 0.0, p.sensing_horizon + dz))
    cam = np.array(cam)
    world = cam @ c2w[:3, :3].T + c2w[:3, 3]
    return np.concatenate([SO.room_scene(120000, seed), world.astype(np.float32)])


def _same_cloud(got, ref):
    (gp, go), (rp, ro) = got, ref
    assert np.array_equal(go, ro), "offsets differ"
    assert np.array_equal(gp.view(np.uint32), rp.view(np.uint32)), "points differ"


# ---- against the reference's own kernel ----
def test_depth_matches_reference_golden():
    p = I.sense_params()
    for name, g in SO.load_golden().items():
        ev = _ev(g["xyz"])
        got = ev.sense_depth(_records(g["pos"], g["quat"]), params=p)
        assert np.array_equal(got, g["depth"]), name
        ev.close()


@pytest.mark.skipif(not SO.ref_available(), reason="oracle/_ref/libref_depth.so not built (no reference tree)")
def test_depth_matches_reference_live():
    p = I.sense_params()
    for name, (xyz, pos, quat) in SO.golden_cases().items():
        T = [SO.pose(pos[q], quat[q], np.array(p.cam_to_body[:]))[1] for q in range(len(pos))]
        ref = SO.ref_render(xyz, T, p)
        ev = _ev(xyz)
        assert np.array_equal(ev.sense_depth(_records(pos, quat), params=p), ref), name
        ev.close()
    # more poses in a denser room, the near-wall ones among them
    xyz0 = SO.room_scene(200000, 7)
    pos, quat = SO.room_poses(12, 8)
    pos = np.concatenate([pos, [[4.7, 0.0, 1.5], [0.0, -4.75, 1.0]]])
    quat = np.concatenate([quat, [SO.yaw_pitch_quat(0.0), SO.yaw_pitch_quat(-np.pi / 2, 0.2)]])
    xyz = SO.keep_ahead(xyz0, pos, quat, 0.15)
    T = [SO.pose(pos[q], quat[q], np.array(p.cam_to_body[:]))[1] for q in range(len(pos))]
    ev = _ev(xyz)
    assert np.array_equal(ev.sense_depth(_records(pos, quat), params=p), SO.ref_render(xyz, T, p))
    ev.close()


# ---- against the serial restatement ----
@pytest.mark.parametrize("horizon", [5.0, 2.0])
def test_depth_and_cloud_match_serial(horizon):
    p = I.sense_params(sensing_horizon=horizon)
    pos, quat = SO.room_poses(24, 21)
    xyz = _boundary_scene(pos, quat, p)
    assert len(xyz) >= 100000
    ev = _ev(xyz)
    rec = _records(pos, quat)
    depth = ev.sense_depth(rec, params=p)
    ref_depth = SO.depth(xyz, pos, quat, p)
    assert np.array_equal(depth, ref_depth)
    _same_cloud(ev.sense_cloud(rec, params=p), SO.cloud(xyz, pos, quat, p, images=ref_depth))
    # the boundary points themselves are seen where the definition sees them: pose 0's image differs from the room's alone
    ev2 = _ev(SO.room_scene(120000, 11))
    assert not np.array_equal(ev2.sense_depth(rec[:1], params=p)[0], depth[0])
    ev.close(); ev2.close()


def test_cloud_with_a_camera_offset_and_non_finite_records():
    C = np.array([[0, 0, 1, 0.3], [-1, 0, 0, 0.05], [0, -1, 0, -0.1], [0, 0, 0, 1.0]])
    p = I.sense_params(sensing_horizon=3.0, cam_to_body=C, width=320, height=200, fx=200.0, fy=210.0, cx=158.3, cy=101.9)
    pos, quat = SO.room_poses(16, 5)
    xyz = SO.room_scene(100000, 4)
    rec = np.zeros((len(xyz) + 3, 4), np.float32)   # 16-byte records, three of them non-finite
    rec[:len(xyz), :3] = xyz
    rec[len(xyz):, :3] = [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf]]
    ev = _ev()
    ev.set_sense_cloud(rec)
    assert ev.sense_info()["points_used"] == len(xyz) and ev.sense_info()["points_skipped"] == 3
    ref_depth = SO.depth(rec, pos, quat, p)
    assert np.array_equal(ev.sense_depth(_records(pos, quat), params=p), ref_depth)
    _same_cloud(ev.sense_cloud(_records(pos, quat), params=p), SO.cloud(rec, pos, quat, p, images=ref_depth))
    ev.close()


# ---- guarantees ----
def test_independent_of_q_order_chunking_and_entry_point():
    torch = _torch()
    p = I.sense_params(sensing_horizon=4.0)
    pos, quat = SO.room_poses(40, 31)
    xyz = SO.room_scene(150000, 30)
    ev = _ev(xyz)
    rec = _records(pos, quat)
    depth = ev.sense_depth(rec, params=p)
    cloud = ev.sense_cloud(rec, params=p)
    perm = np.random.default_rng(1).permutation(40)
    assert np.array_equal(ev.sense_depth(rec[perm], params=p), depth[perm])
    pp, po = ev.sense_cloud(rec[perm], params=p)
    for i, q in enumerate(perm):
        assert np.array_equal(pp[po[i]:po[i + 1]], cloud[0][cloud[1][q]:cloud[1][q + 1]])
    for q in (0, 17, 39):
        assert np.array_equal(ev.sense_depth(rec[q:q + 1], params=p)[0], depth[q])
    for chunk in (1, 7, 40):
        ev.dbg_sense_chunk(chunk)
        assert np.array_equal(ev.sense_depth(rec, params=p), depth), chunk
        _same_cloud(ev.sense_cloud(rec, params=p), cloud)
    ev.dbg_sense_chunk(0)
    d_rec = torch.from_numpy(rec).cuda()
    assert np.array_equal(ev.sense_depth_device(d_rec, params=p).cpu().numpy(), depth)
    dp_, do_ = ev.sense_cloud_device(d_rec, params=p)
    torch.cuda.synchronize()
    _same_cloud((dp_.cpu().numpy(), do_.cpu().numpy()), cloud)
    ev.close()


def test_log_and_state_records_read_in_place():
    p = I.sense_params(sensing_horizon=5.0)
    pos, quat = SO.room_poses(10, 41)
    ev = _ev(SO.room_scene(60000, 40))
    log = np.full((10, I.SIM_DOUBLES), np.nan)
    log[:, 1:4], log[:, 7:11] = pos, quat
    st = np.full((10, I.STATE_DOUBLES), np.nan)
    st[:, 0:3], st[:, 12:16] = pos, quat
    a, b = ev.sense_depth(log, 1, 7, params=p), ev.sense_depth(st, 0, 12, params=p)
    assert np.array_equal(a, b) and np.array_equal(a, ev.sense_depth(_records(pos, quat), params=p))
    _same_cloud(ev.sense_cloud(log, 1, 7, params=p), ev.sense_cloud(st, 0, 12, params=p))
    ev.close()


def test_plan_simulate_sense_map_chain():
    """plan_pairs_device -> simulate_device -> sense_cloud_device on the log -> set_map_cloud_device, against the serial chain"""
    torch = _torch()
    import cloud_oracle as CLO
    from test_gpu_plan import _ev as plan_ev, _scene, _params
    occ, start, goals = _scene(4, seed=5)
    ev = plan_ev("Ball", occ)
    out = ev.plan_pairs_device(torch.tensor(np.tile(start, (4, 1)), device="cuda"), torch.tensor(goals, device="cuda"), _params(ev))
    off, T, Cc = out["piece_off"], out["T"], out["coeffs"]
    B = off.shape[0] - 1
    traj = torch.arange(B, dtype=torch.int32, device="cuda")
    init = torch.tensor(I.sim_init_from_trajectories(off.cpu().numpy(), Cc.cpu().numpy(), traj.cpu().numpy()), device="cuda")
    sim = ev.simulate_device(off, T, Cc, traj, init, None, I.sim_default_params(t_end=3.0, log_every=10))
    log = sim["log"].reshape(-1, I.SIM_DOUBLES)
    log = log[torch.isfinite(log[:, 0])].contiguous()
    # the scene: the map's occupied voxel centres
    xyz = (np.argwhere(occ != 0) + 0.5).astype(np.float32)
    ev.set_sense_cloud(xyz)
    p = I.sense_params(sensing_horizon=5.0)
    pts, po = ev.sense_cloud_device(log, 1, 7, params=p)
    ev.set_map_cloud_device(pts, stride_bytes=12, res=1.0)
    got, info = ev.get_map_u8(), ev.map_info()
    lg = log.cpu().numpy()
    rp, ro = SO.cloud(xyz, lg[:, 1:4], lg[:, 7:11], p)
    _same_cloud((pts.cpu().numpy(), po.cpu().numpy()), (rp, ro))
    ref = CLO.serial(rp, 12, 1.0, 1)
    assert tuple(info["dims"]) == ref["dims"] and np.array_equal(info["bmin"], ref["bmin"]) and np.array_equal(got, ref["occ"])
    ev.close()


def test_new_cloud_releases_the_old():
    torch = _torch()
    p = I.sense_params()
    pos, quat = SO.room_poses(3, 51)
    rec = _records(pos, quat)
    a, b = SO.room_scene(400000, 50), SO.room_scene(30000, 52)
    ev = _ev(a)
    ev.sense_depth(rec, params=p)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        ev.set_sense_cloud(a)
        ev.sense_depth(rec, params=p)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] >= free0 - (64 << 20)
    ev.set_sense_cloud(b)
    assert ev.sense_info()["points_used"] == len(b)
    assert np.array_equal(ev.sense_depth(rec, params=p), SO.depth(b, pos, quat, p))
    ev.close()


def test_errors_and_cap():
    torch = _torch()
    pos, quat = SO.room_poses(4, 61)
    rec = _records(pos, quat)
    ev = _ev()
    with pytest.raises(I.IsdfError) as e:
        ev.sense_depth(rec)
    assert e.value.code == -2 and "scene cloud" in str(e.value)
    with pytest.raises(I.IsdfError):
        ev.set_sense_cloud(np.zeros((0, 3), np.float32))
    ev.set_sense_cloud(SO.room_scene(50000, 60))
    for bad in (dict(width=0), dict(height=-3), dict(fx=-1.0), dict(cy=np.inf), dict(sensing_horizon=-1.0), dict(sensing_horizon=np.nan),
                dict(cam_to_body=np.diag([1, 1, 1, 2.0])), dict(width=10000, height=10000)):
        with pytest.raises(I.IsdfError) as e:
            ev.sense_depth(rec, **bad)
        assert e.value.code == -1, bad
    p = I.sense_params(sensing_horizon=5.0)
    full, off = ev.sense_cloud(rec, params=p)
    assert off[-1] > 1000
    # too small a cap: ISDF_ERR_INVALID, offsets written, the rows below cap written; the wrapper's retry gets everything
    cap = int(off[-1]) // 2
    pts, o2 = np.full((cap, 3), -7, np.float32), np.zeros(5, np.int64)
    import ctypes as C
    base = rec.ctypes.data
    r = ev.lib.isdf_sense_cloud(ev.h, 4, C.c_void_p(base), C.c_void_p(base + 24), 7, C.byref(p), cap, pts.ctypes.data_as(C.c_void_p),
                                o2.ctypes.data_as(C.c_void_p))
    assert r == -1 and np.array_equal(o2, off) and np.array_equal(pts, full[:cap])
    got, go = ev.sense_cloud(rec, params=p, cap=3)
    assert np.array_equal(go, off) and np.array_equal(got, full)
    d_rec = torch.from_numpy(rec).cuda()
    dp_, do_ = ev.sense_cloud_device(d_rec, params=p, cap=5)
    assert np.array_equal(do_.cpu().numpy(), off) and np.array_equal(dp_.cpu().numpy(), full)
    ev.close()
