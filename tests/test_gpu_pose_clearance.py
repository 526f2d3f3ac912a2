"""isdf_pose_clearance: the clearance check's definition over caller-given poses (the pose source of k_clearance_scan), against
isdf_trajectory_clearance on the same poses, on a flown rollout, and its guarantees and refusals."""
import numpy as np
import pytest
import isdf_b200 as I
import workloads as W

pytestmark = pytest.mark.gpu
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]


def dyadic_cfg():
    # no drag and gravity 4: with horizontal accelerations of 3 m/s^2 every pose quantity below is exact or computed by the same
    # operations in both pose pipelines, so trajectory samples and states records pose the robot identically, bit for bit
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION
    cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
    cfg.grav_acc = 4.0
    return cfg


def dyadic_trajectory():
    """four 2 s pieces of constant horizontal acceleration (+x, +y, -x, -y) at 3 m/s^2 from dyadic starts (not joined: each is checked as
    a trajectory of its own)"""
    starts = [(6.0, 8.0, 10.0), (12.0, 8.0, 11.0), (12.0, 14.0, 12.0), (6.0, 14.0, 12.5)]
    acc = [(1.5, 0.0), (0.0, 1.5), (-1.5, 0.0), (0.0, -1.5)]   # c2 = a / 2
    N = len(starts)
    Cc = np.zeros((3, N, 6))
    for i, (s, a) in enumerate(zip(starts, acc)):
        Cc[:, i, 0] = s
        Cc[0, i, 2], Cc[1, i, 2] = a
    return np.full(N, 2.0), Cc.reshape(-1)


def set_robot(ev, robot):
    if robot == "Ball":
        ev.set_shape_named("Ball")
    elif robot == "exact_mesh":
        V, F = W.rounded_cone_mesh()
        ev.set_shape_mesh(V, F, PP)
    else:
        V, F = W.box_mesh(1.2, 0.7, 0.4)
        ev.set_shape_mesh(V, F[2:], PP, I.MESH_SIGN_WINDING)


@pytest.mark.parametrize("robot", ["Ball", "exact_mesh", "winding_mesh"])
def test_states_poses_equal_the_trajectory_samples(robot):
    occ = W.random_map(24, 24, 24, p=0.05, seed=1, slabs=0)
    ev = I.Evaluator(dyadic_cfg())
    ev.set_map_u8(occ, [0.0, 0.0, 0.0], 1.0)
    set_robot(ev, robot)
    T, Cc = dyadic_trajectory()
    K, reach, margin = 16, 2.5, 0.866
    # each piece is its own trajectory (N0 = 1), so every sample, piece starts included, is a (trajectory, local time) states query
    clear, vox, summ = ev.trajectory_clearance(T, Cc, K, reach, margin, N0=1)
    N = T.size
    off = np.arange(N + 1, dtype=np.int32)
    traj = np.repeat(np.arange(N, dtype=np.int32), K + 1)
    times = np.array([j * (T[i] * (1.0 / K)) for i in range(N) for j in range(K + 1)])
    Cr = Cc.reshape(3, N, 6).transpose(1, 0, 2).reshape(-1)   # the ragged layout: each trajectory's own 6 x 3 column-major block
    rec = ev.trajectory_states((off, T, Cr), traj, times)
    pc, pv, ps = ev.pose_clearance(rec, 0, 12, reach, margin, poses_per_group=K + 1)
    assert np.array_equal(pc.view(np.uint64), clear.view(np.uint64))
    assert np.array_equal(pv, vox)
    assert (vox >= 0).any() and (clear < reach).any()
    for s, t in zip(ps, summ):
        assert s["min_clearance"] == t["min_clearance"] and s["voxel_min"] == t["voxel_min"]
        assert s["piece_min"] == t["sample_min"] and s["t_min"] == t["sample_min"]
        assert s["colliding_samples"] == t["colliding_samples"] and s["collision_free"] == t["collision_free"]
    ev.close()


def quintic_line(p0, p1, T):
    """one rest-to-rest piece from p0 to p1: p0 + (p1 - p0) (10 s^3 - 15 s^4 + 6 s^5), s = t / T"""
    d = np.asarray(p1, float) - np.asarray(p0, float)
    Cc = np.zeros((3, 6))
    Cc[:, 0] = p0
    Cc[:, 3], Cc[:, 4], Cc[:, 5] = 10 * d / T ** 3, -15 * d / T ** 4, 6 * d / T ** 5
    return np.array([T]), Cc.reshape(-1)


def test_flown_rollout_hits_a_wall_the_plan_clears():
    res = 0.5
    occ = np.zeros((40, 40, 20), dtype=np.uint8)
    occ[:, 24:, :] = 1   # a wall: every voxel centre with y >= 12.25
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0.0, 0.0, 0.0], res)
    ev.set_shape_named("Ball")
    T, Cc = quintic_line([4.0, 10.0, 5.0], [16.0, 10.0, 5.0], 8.0)
    cert = ev.trajectory_certify(T, Cc, 16, 2 * cfg.safety_hor, cfg.safety_hor)
    assert cert[0]["verdict"] == I.CERTIFIED
    p = I.sim_default_params(t_end=10.0, floor=0)
    off = np.array([0, 1], dtype=np.int32)
    init = I.sim_init_from_trajectories(off, Cc, [0], p)
    dist = np.array([[0.0, 12.0, 0.0, 0.0, 0.0, 0.0]])   # a steady side wind towards the wall
    log, summ = ev.simulate((off, T, Cc), [0], init, dist, p)
    assert summ[0]["diverged"] == 0
    rows = log[0]
    clear, vox, ps = ev.pose_clearance(rows, 1, 7, 2 * cfg.safety_hor, cfg.safety_hor)
    s = ps[0]
    assert s["collision_free"] == 0 and s["colliding_samples"] > 0 and s["first_hit"] >= 0
    w = s["voxel_min"]
    ix, iy, iz = w // (40 * 20), (w // 20) % 40, w % 20
    assert occ[ix, iy, iz] == 1 and iy >= 24
    # the commanded poses of the same log are clear: the hit is the flight's, not the plan's
    cmd = np.zeros((rows.shape[0], 7)); cmd[:, 0:3] = rows[:, 18:21]; cmd[:, 3] = 1.0
    cc, _, cs = ev.pose_clearance(cmd, 0, 3, 2 * cfg.safety_hor, cfg.safety_hor)
    assert cs[0]["collision_free"] == 1
    ev.close()


def test_groups_repeat_device_and_refusals():
    import torch
    occ = W.random_map(24, 24, 24, p=0.05, seed=1, slabs=0)
    ev = I.Evaluator(dyadic_cfg())
    ev.set_map_u8(occ, [0.0, 0.0, 0.0], 1.0)
    V, F = W.rounded_cone_mesh()
    ev.set_shape_mesh(V, F, PP)
    rng = np.random.default_rng(3)
    Q = 96
    rec = np.zeros((Q, 9))
    rec[:, 1:4] = 4.0 + 16.0 * rng.random((Q, 3))
    q = rng.normal(size=(Q, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    rec[:, 5:9] = q
    c1, v1, s1 = ev.pose_clearance(rec, 1, 5, 2.0, 0.866, poses_per_group=32)
    c2, v2, s2 = ev.pose_clearance(rec, 1, 5, 2.0, 0.866, poses_per_group=32)
    assert np.array_equal(c1.view(np.uint64), c2.view(np.uint64)) and np.array_equal(v1, v2) and s1 == s2
    ca, va, sa = ev.pose_clearance(rec[32:64], 1, 5, 2.0, 0.866)   # a group alone
    assert np.array_equal(ca.view(np.uint64), c1[32:64].view(np.uint64)) and sa[0] == s1[1]
    dv = torch.device("cuda:0")
    d = torch.from_numpy(rec).to(dv)
    dc, dvx = torch.empty(Q, dtype=torch.float64, device=dv), torch.empty(Q, dtype=torch.int64, device=dv)
    ds = torch.empty((3, 48), dtype=torch.uint8, device=dv)
    p = ev.pose_clearance_params(2.0, 0.866, 32)
    ev.pose_clearance_device(Q, d.data_ptr() + 8, d.data_ptr() + 40, 9, p, dc.data_ptr(), dvx.data_ptr(), ds.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dc.cpu().numpy().view(np.uint64), c1.view(np.uint64)) and np.array_equal(dvx.cpu().numpy(), v1)
    # a non-finite pose reports NaN and counts as colliding
    bad = rec.copy(); bad[5, 1] = np.nan
    cb, _, sb = ev.pose_clearance(bad, 1, 5, 2.0, 0.866)
    assert np.isnan(cb[5]) and np.isnan(sb[0]["min_clearance"]) and sb[0]["collision_free"] == 0
    for kw in (dict(reach=-1.0), dict(reach=1.0, margin=2.0), dict(poses_per_group=7)):
        with pytest.raises(I.IsdfError):
            ev.pose_clearance(rec, 1, 5, **{k: v for k, v in dict(dict(reach=2.0, margin=0.866), **kw).items()})
    ev.close()
