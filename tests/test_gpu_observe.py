"""Known space on the GPU (isdf_map_observe, isdf_map_mark_known, isdf_get_map_known_u8, isdf_set_unknown_policy):
  observe   the known bits equal tests/observe_oracle.py applied to isdf_sense_depth's images, on the navigation wall scene at 1 m and 0.5 m
            with poses at the wall, the image edges and the horizon; the same bits under forced chunking, reversed pose order, other Q and
            from the device form on a side stream; exact info counts;
  invariant after 256 poses in mockamap's box world and in a Perlin world no scene point lies in the closed cube of a known voxel (every
            cube a point touches, by brute force);
  policy    under ISDF_UNKNOWN_OCCUPIED, clearance, pose clearance, certify, brake and the planning certificate equal the same calls under
            ISDF_UNKNOWN_FREE on a context whose map is occ | ~known; under FREE every output equals a context that never observed;
  lifecycle set_map_* clears known, fusion keeps it and the next certificate sees the fused voxel, mark_known and the readback round-trip."""
import numpy as np
import pytest
import isdf_b200 as I
import navigate_oracle as NO
import observe_oracle as OO
import sense_oracle as SO
from test_gpu_navigate import _wall_cloud
from test_gpu_brake import _traj, _ragged, _stop_times
from test_gpu_plan import _cfg, _scene, _params

pytestmark = pytest.mark.gpu


def _records(pos, quat):
    return np.ascontiguousarray(np.column_stack([pos, quat]))


def _wall_poses(Q, seed):
    """poses across the 40 x 24 x 8 m frame, some facing the wall from 0.8 m, some at its edges and corners"""
    rng = np.random.default_rng(seed)
    pos = np.column_stack([rng.uniform(1, 39, Q), rng.uniform(1, 23, Q), rng.uniform(0.5, 7.5, Q)])
    yaw, pitch = rng.uniform(-np.pi, np.pi, Q), rng.uniform(-0.4, 0.4, Q)
    pos[:6] = [[17.2, 7.0, 4.0], [17.2, 12.0, 4.0], [17.2, 17.5, 1.0], [21.8, 12.0, 4.0], [19.5, 5.3, 4.0], [10.0, 12.0, 4.0]]
    yaw[:6], pitch[:6] = [0.0, 0.3, 0.0, np.pi, np.pi / 2, 0.0], [0.0, 0.0, 0.3, 0.0, 0.0, 0.0]
    quat = np.array([SO.yaw_pitch_quat(a, b) for a, b in zip(yaw, pitch)])
    return pos, quat


def _oracle(ev, rec, p, bmin, res, dims):
    imgs = ev.sense_depth(rec, params=p)
    cws = [SO.pose(r[:3], r[3:7], np.array(p.cam_to_body[:]))[1] for r in rec]
    return OO.observe_many(imgs, cws, rec[:, :3], p, bmin, res, dims)


@pytest.mark.parametrize("res", [1.0, 0.5])
def test_observe_equals_the_restatement_in_any_order_chunking_and_form(res):
    import torch
    dims = (int(40 / res), int(24 / res), int(8 / res))
    bmin = np.zeros(3)
    p = I.sense_params(sensing_horizon=12.0)
    pos, quat = _wall_poses(32, seed=int(7 / res))
    rec = _records(pos, quat)
    ev = I.Evaluator(I.default_config_values())
    ev.set_sense_cloud(_wall_cloud())
    ev.set_map_u8(np.zeros(dims, np.uint8), bmin, res)
    want = _oracle(ev, rec, p, bmin, res, dims)
    info = ev.map_observe(rec, params=p)
    got = ev.get_map_known_u8().astype(bool)
    assert want.sum() > 1000 and np.array_equal(got, want)
    assert info == dict(poses=32, voxels_tested=OO.tested(pos, 12.0, bmin, res, dims), voxels_added=int(want.sum()))
    # a second pass adds nothing; set_map_* forgets what was known
    assert ev.map_observe(rec, params=p)["voxels_added"] == 0
    ev.set_map_u8(np.zeros(dims, np.uint8), bmin, res)
    assert not ev.get_map_known_u8().any()
    # forced chunking, reversed order, Q split in two calls, and the device form on a side stream
    for chunk in (1, 5):
        ev.set_map_u8(np.zeros(dims, np.uint8), bmin, res)
        ev.dbg_sense_chunk(chunk)
        assert ev.map_observe(rec, params=p)["voxels_added"] == want.sum()
        assert np.array_equal(ev.get_map_known_u8().astype(bool), want), chunk
    ev.dbg_sense_chunk(0)
    ev.set_map_u8(np.zeros(dims, np.uint8), bmin, res)
    ev.map_observe(rec[::-1].copy(), params=p)
    assert np.array_equal(ev.get_map_known_u8().astype(bool), want)
    ev.set_map_u8(np.zeros(dims, np.uint8), bmin, res)
    a = ev.map_observe(rec[:11], params=p)["voxels_added"]
    b = ev.map_observe(rec[11:], params=p)["voxels_added"]
    assert a + b == want.sum() and np.array_equal(ev.get_map_known_u8().astype(bool), want)
    ev.set_map_u8(np.zeros(dims, np.uint8), bmin, res)
    side = torch.cuda.Stream()
    d_rec = torch.from_numpy(rec).cuda()
    torch.cuda.synchronize()
    dinfo = ev.map_observe_device(d_rec, params=p, stream=side)
    assert dinfo == info and np.array_equal(ev.get_map_known_u8().astype(bool), want)
    ev.close()


def _touched(pts, bmin, res, dims):
    """for every point, the voxels whose closed padded cube contains it (up to 2 per axis) -> flat indices"""
    pts = pts.astype(np.float64)
    cand = []
    for a in range(3):
        f = np.floor((pts[:, a] - bmin[a]) / res).astype(np.int64)
        opts = []
        for d in (-1, 0, 1):
            i = f + d
            lo, hi = OO.voxel_span(float(bmin[a]), res, i.astype(np.float64))
            opts.append((i, (i >= 0) & (i < dims[a]) & (lo <= pts[:, a]) & (pts[:, a] <= hi)))
        cand.append(opts)
    out = []
    for ix, mx in cand[0]:
        for iy, my in cand[1]:
            for iz, mz in cand[2]:
                m = mx & my & mz
                out.append((ix[m] * dims[1] + iy[m]) * dims[2] + iz[m])
    return np.concatenate(out)


@pytest.mark.parametrize("kind", ["boxes", "perlin"])
def test_no_scene_point_lies_in_a_known_voxel(kind):
    ev = I.Evaluator(I.default_config_values())
    cloud = ev.world_cloud(kind=kind)
    ev.set_map_cloud(cloud[:, :3].copy(), 0.1, 1)
    ev.set_sense_cloud(cloud)
    mi = ev.map_info()
    bmin, dims = mi["bmin"], mi["dims"]
    rng = np.random.default_rng(5)
    Q = 256
    lo, hi = mi["bmin"], mi["bmax"]
    pos = rng.uniform(lo, hi, (Q, 3))
    quat = np.array([SO.yaw_pitch_quat(a, b) for a, b in zip(rng.uniform(-np.pi, np.pi, Q), rng.uniform(-0.6, 0.6, Q))])
    p = I.sense_params(sensing_horizon=5.0)
    info = ev.map_observe(_records(pos, quat), params=p)
    known = ev.get_map_known_u8().astype(bool)
    assert info["voxels_added"] == known.sum() > 0.05 * known.size
    idx = _touched(cloud[:, :3], bmin, 0.1, dims)
    assert len(idx) >= len(cloud)
    assert not known.reshape(-1)[idx].any()
    ev.close()


# ---- the unknown policy ----
def _policy_setup(seed):
    occ, start, goals = _scene(4, seed=seed)
    rng = np.random.default_rng(seed)
    boxes = []
    for _ in range(60):
        c, h = rng.uniform(0, 48, 3), rng.uniform(2, 7, 3)
        boxes.append(np.concatenate([c - h, c + h]))
    boxes = np.array(boxes)
    known = OO.mark_boxes(boxes, np.zeros(3), 1.0, occ.shape)
    evs = []
    for m in (occ, occ, (occ.astype(bool) | ~known).astype(np.uint8)):
        ev = I.Evaluator(_cfg())
        ev.set_map_u8(m, [0, 0, 0], 1.0)
        ev.set_shape_named("Ball")
        ev.frontend_build_kernels(45.0, 45.0, 9.0, 0.0)
        evs.append(ev)
    evs[0].map_mark_known(boxes)
    assert np.array_equal(evs[0].get_map_known_u8().astype(bool), known)
    return evs, occ, start, goals, rng


def _outputs(ev, rng_seed, start, goals):
    """every clearance-family output on fixed inputs"""
    rng = np.random.default_rng(rng_seed)
    out = {}
    T, Cc = _traj(rng, 6)
    out["clearance"] = ev.trajectory_clearance(T, Cc, 8, 2.0, 0.866)
    out["certify"] = ev.trajectory_certify(T, Cc, 8, 2.0, 0.866)
    pos = rng.uniform(2, 46, (64, 3))
    quat = np.array([SO.yaw_pitch_quat(a) for a in rng.uniform(-np.pi, np.pi, 64)])
    out["pose"] = ev.pose_clearance(_records(pos, quat), reach=2.0, margin=0.866, poses_per_group=8)
    off, Tb, Cb = _ragged(rng, [3, 5, 1, 4, 6, 2, 7, 3])
    out["brake"] = ev.trajectory_brake((off, Tb, Cb), _stop_times(rng, off, Tb))
    heads = np.zeros((len(goals), 9))
    heads[:, :3] = start
    plans = ev.plan_states(heads, goals, _params(ev, flags=I.PLAN_CERTIFY))[0]
    out["plan"] = [{k: r[k] for k in ("stage", "pieces", "path", "T", "coeffs", "certify")} for r in plans]
    return out


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if a is None or isinstance(a, (str, int, float, bool, np.integer, np.floating)):
        return a == b or (a != a and b != b)
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def test_occupied_policy_equals_free_on_the_blocked_map():
    evs, occ, start, goals, rng = _policy_setup(31)
    a, never, blocked = evs
    free_a = _outputs(a, 9, start, goals)
    assert _same(free_a, _outputs(never, 9, start, goals))   # FREE: the known grid changes nothing
    a.set_unknown_policy(I.UNKNOWN_OCCUPIED)
    assert a.unknown_policy() == I.UNKNOWN_OCCUPIED
    got, want = _outputs(a, 9, start, goals), _outputs(blocked, 9, start, goals)
    for k in ("clearance", "certify", "pose", "brake"):
        assert _same(got[k], want[k]), k
    # planning stays optimistic: the plans are FREE's, and their certificates are the blocked map's
    p = _params(a, flags=I.PLAN_CERTIFY)
    cp = p.certify
    for g, f in zip(got["plan"], free_a["plan"]):
        assert all(_same(g[k], f[k]) for k in ("stage", "path", "T", "coeffs"))
        if g["pieces"] > 0:
            s = blocked.trajectory_certify(g["T"], g["coeffs"], cp.clearance.samples_per_piece, cp.clearance.reach, cp.clearance.margin,
                                           max_depth=cp.max_depth, max_samples=cp.max_samples_per_traj)[0]
            assert _same(g["certify"], s)
    assert not _same(got["pose"], free_a["pose"])   # the unknown voxels count
    for ev in evs:
        ev.close()


def test_lifecycle_set_map_fuse_and_readback():
    ev = I.Evaluator(_cfg())
    ev.set_shape_named("Ball")
    dims = (40, 24, 8)
    ev.set_map_u8(np.zeros(dims, np.uint8), [0, 0, 0], 1.0)
    assert not ev.get_map_known_u8().any()
    box = np.array([[1.0, 1.0, 1.0, 30.0, 20.0, 7.0]])
    ev.map_mark_known(box)
    known = ev.get_map_known_u8().astype(bool)
    assert np.array_equal(known, OO.mark_boxes(box, np.zeros(3), 1.0, dims))
    ev.set_unknown_policy(I.UNKNOWN_OCCUPIED)
    # a straight line through the known box: CERTIFIED; a voxel fused onto it: the next certificate sees it, the known grid is kept
    def line(p0, v):
        blk = np.zeros((1, 3, 6))
        blk[0, :, 0], blk[0, :, 1] = p0, v
        return NO._unblock(blk)
    T, Cc = np.array([4.0]), line([6.0, 10.0, 4.0], [4.0, 0.0, 0.0])
    assert ev.trajectory_certify(T, Cc, 8, 2.0, 0.866)[0]["verdict"] == I.CERTIFIED
    ev.map_fuse_cloud(np.array([[14.5, 10.5, 4.5]], np.float32))
    assert np.array_equal(ev.get_map_known_u8().astype(bool), known)
    assert ev.trajectory_certify(T, Cc, 8, 2.0, 0.866)[0]["verdict"] == I.COLLIDING
    # leaving the known box: COLLIDING under OCCUPIED, CERTIFIED under FREE
    Cc2 = line([20.0, 5.0, 4.0], [4.0, 0.0, 0.0])
    assert ev.trajectory_certify(T, Cc2, 8, 2.0, 0.866)[0]["verdict"] == I.COLLIDING
    ev.set_unknown_policy(I.UNKNOWN_FREE)
    assert ev.trajectory_certify(T, Cc2, 8, 2.0, 0.866)[0]["verdict"] == I.CERTIFIED
    # a cloud map clears known too
    ev.set_map_cloud(np.array([[0, 0, 0], [10, 10, 5]], np.float32), 1.0, 1)
    assert not ev.get_map_known_u8().any()
    ev.close()


def test_errors():
    ev = I.Evaluator(I.default_config_values())
    rec = _records(np.array([[1.0, 1.0, 1.0]]), np.array([[1.0, 0, 0, 0]]))
    with pytest.raises(RuntimeError):
        ev.map_observe(rec, params=I.sense_params(sensing_horizon=5.0))   # no scene
    ev.set_sense_cloud(_wall_cloud())
    with pytest.raises(RuntimeError):
        ev.map_observe(rec, params=I.sense_params(sensing_horizon=5.0))   # no map
    with pytest.raises(RuntimeError):
        ev.map_mark_known([[0, 0, 0, 1, 1, 1]])                          # no map
    ev.set_map_u8(np.zeros((40, 24, 8), np.uint8), [0, 0, 0], 1.0)
    with pytest.raises(RuntimeError):
        ev.map_observe(rec, params=I.sense_params())                      # infinite horizon
    with pytest.raises(RuntimeError):
        ev.map_mark_known([[0, 0, 0, -1, 1, 1]])                         # lo > hi
    with pytest.raises(RuntimeError):
        ev.set_unknown_policy(2)
    assert ev.unknown_policy() == I.UNKNOWN_FREE
    ev.close()
