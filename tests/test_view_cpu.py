"""CPU checks of the view gain (include/isdf.h, isdf_view_gain) through its numpy restatement (tests/view_oracle.py): an occupied slab hides
what lies behind it; known, occupied and out-of-view voxels never count; the line of sight is an integer 26-connected line from the pose's
voxel to the voxel; a rig counts the union of its cameras' voxels; after isdf_map_observe's restatement of a pose, every voxel the gain
still counts there failed observe's rule 4. Also the argument checks that need no device and the isdf_frontier_goal layout."""
import ctypes as C
from fractions import Fraction
import numpy as np
import pytest
import isdf_b200 as I
import observe_oracle as OO
import sense_oracle as SO
import view_oracle as VO
from test_plan_cpu import _probe, _fields

RES = 0.25
BMIN = np.array([-1.0, -4.0, -3.0])
DIMS = (32, 32, 24)
POS = np.array([0.1, 0.05, 0.02])
LEVEL = np.array([1.0, 0.0, 0.0, 0.0])
SLAB_X = 12   # voxel index of the slab: x in [2.0, 2.25]


def _cam(**kw):
    # the reference camera (looking along the body's x axis) with a 5 m horizon
    return I.sense_params(sensing_horizon=kw.pop("sensing_horizon", 5.0), **kw)


def _yawed(deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    c0 = np.array([[0, 0, 1, 0], [-1, 0, 0, 0], [0, -1, 0, 0], [0, 0, 0, 1]], dtype=np.float64)
    Rz = np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    return _cam(cam_to_body=(Rz @ c0).reshape(-1))


def _slab():
    occ = np.zeros(DIMS, dtype=bool)
    occ[SLAB_X] = True
    return occ


def test_an_occupied_slab_hides_what_lies_behind_it():
    occ = _slab()
    free = VO.view_set(np.zeros(DIMS, bool), None, POS, LEVEL, _cam(), BMIN, RES)
    got = VO.view_set(occ, None, POS, LEVEL, _cam(), BMIN, RES)
    assert free[SLAB_X + 1:].sum() > 1000 and free[:SLAB_X].sum() > 100
    assert not got[SLAB_X:].any()                                # nothing on or behind the slab
    assert np.array_equal(got[:SLAB_X], free[:SLAB_X])          # everything in front of it, as without the slab


def test_known_occupied_and_out_of_view_voxels_do_not_count():
    rng = np.random.default_rng(4)
    occ = rng.random(DIMS) < 0.02
    known = rng.random(DIMS) < 0.3
    cam = _cam()
    got = VO.view_set(occ, known, POS, LEVEL, cam, BMIN, RES)
    seen = VO.in_view(POS, LEVEL, cam, BMIN, RES, DIMS)
    assert got.sum() > 100
    assert not (got & (occ | known | ~seen)).any()
    # an unknown, free, in-view voxel with a clear line counts
    s = VO.pose_voxel(POS, BMIN, RES)
    for v in np.argwhere(seen & ~occ & ~known)[:200]:
        assert got[tuple(v)] == (not occ[tuple(VO.line(s, v).T)].any() if len(VO.line(s, v)) else True)


@pytest.mark.parametrize("seed", range(4))
def test_the_line_is_integer_26_connected_and_reaches_v(seed):
    rng = np.random.default_rng(seed)
    for _ in range(200):
        s = rng.integers(-20, 20, 3)
        v = s + rng.integers(-15, 16, 3)
        L = VO.line(s, v)
        d = v - s
        m = int(np.abs(d).max())
        assert L.dtype == np.int64 and len(L) == max(m - 1, 0)
        chain = np.concatenate([[s], L, [v]]) if m else np.array([s])
        assert (np.abs(np.diff(chain, axis=0)).max(axis=1) == 1).all() if m else True
        for k, p in enumerate(L, 1):   # exact: the nearest voxel to s + k d / m, halves rounded up
            for a in range(3):
                assert p[a] == s[a] + int(np.floor(Fraction(k * int(d[a]), m) + Fraction(1, 2)))


def test_a_rig_counts_the_union_of_its_cameras():
    rng = np.random.default_rng(8)
    occ = rng.random(DIMS) < 0.01
    known = rng.random(DIMS) < 0.2
    cams = [_yawed(a) for a in (0.0, 90.0, 180.0, 270.0)]
    sets = [VO.view_set(occ, known, POS, LEVEL, c, BMIN, RES) for c in cams]
    for k in (2, 4):
        rig = VO.view_set(occ, known, POS, LEVEL, cams[:k], BMIN, RES)
        assert np.array_equal(rig, np.logical_or.reduce(sets[:k]))
        n = [int(x.sum()) for x in sets[:k]]
        assert max(n) <= rig.sum() <= sum(n) and rig.sum() > max(n)
        assert VO.gain(occ, known, POS, LEVEL, cams[:k], BMIN, RES) == int(rig.sum())


def test_after_observing_a_pose_what_still_counts_failed_rule_4():
    occ = _slab()
    cam = _cam()
    # the scene: points on the slab's near face and a post in front of it
    yy, zz = np.meshgrid(np.arange(-3.9, 3.9, 0.05), np.arange(-2.9, 2.9, 0.05), indexing="ij")
    face = np.stack([np.full(yy.size, 2.01), yy.ravel(), zz.ravel()], 1)
    post = np.stack([np.full(40, 1.0), np.full(40, 0.3), np.linspace(-0.5, 0.5, 40)], 1)
    pts = np.concatenate([face, post]).astype(np.float32)
    occ[int(np.floor((1.0 - BMIN[0]) / RES)), int(np.floor((0.3 - BMIN[1]) / RES)), 10:15] = True
    c2w, cw = SO.pose(POS, LEVEL, np.array(cam.cam_to_body[:]))
    img, _ = SO.render(pts, cw, cam)
    obs = OO.observe(img, cw, POS, cam, BMIN, RES, DIMS)
    before = VO.view_set(occ, None, POS, LEVEL, cam, BMIN, RES)
    after = VO.view_set(occ, obs, POS, LEVEL, cam, BMIN, RES)
    seen = VO.in_view(POS, LEVEL, cam, BMIN, RES, DIMS)
    assert obs.sum() > 50 and after.sum() > 0 and after.sum() < before.sum()
    # rules 2, 1 and 3 hold (in view) and the voxel was not marked: rule 4 failed for it
    assert not (after & ~seen).any() and not (after & obs).any()
    assert np.array_equal(after, before & ~obs)


def test_argument_checks_without_a_device():
    lib = I.load_library()
    rec = np.zeros((1, 7))
    rec[0, 3] = 1.0
    dp = rec.ctypes.data
    cams = (I.SenseParams * 1)(_cam())
    g = np.zeros(1, dtype=np.int64)
    assert lib.isdf_view_gain(None, 1, C.c_void_p(dp), C.c_void_p(dp + 24), 7, 1, cams, g.ctypes.data) == -1
    assert b"ctx" in lib.isdf_last_error()
    assert lib.isdf_view_gain(None, 1, C.c_void_p(dp), C.c_void_p(dp + 24), 7, 0, cams, g.ctypes.data) == -1
    assert b"n_cams" in lib.isdf_last_error()
    assert lib.isdf_view_gain_device(None, 0, C.c_void_p(dp), C.c_void_p(dp + 24), 7, 1, cams, g.ctypes.data, None) == -1
    assert b"Q" in lib.isdf_last_error()
    inf = (I.SenseParams * 1)(_cam(sensing_horizon=np.inf))
    assert lib.isdf_view_gain(None, 1, C.c_void_p(dp), C.c_void_p(dp + 24), 7, 1, inf, g.ctypes.data) == -1
    assert b"finite sensing_horizon" in lib.isdf_last_error()
    out = np.zeros(1, dtype=I.FRONTIER_GOAL_DTYPE)
    assert lib.isdf_frontier_goals_view(None, 1, I._dp(POS), I._dp(POS), None, 1, cams, 0, 0, out.ctypes.data, None) == -1
    ev = object.__new__(I.Evaluator)   # the refusals come before any device work
    with pytest.raises(ValueError, match="explore=True"):
        ev.navigate(np.zeros((1, 3)), np.ones((1, 3)), rounds=1, horizon=0.5, min_gain=5)
    with pytest.raises(ValueError, match="needs a rig"):
        ev.frontier_goals(np.zeros((1, 3)), np.ones((1, 3)), min_gain=3)


def test_frontier_goal_layout():
    got = _probe([("isdf_frontier_goal", I.FrontierGoal)])
    size, offs = got["isdf_frontier_goal"]
    assert size == C.sizeof(I.FrontierGoal) == 64 and offs == dict(_fields(I.FrontierGoal))
    assert I.FrontierGoal.gain.offset == 4 and I.FRONTIER_GOAL_DTYPE.fields["gain"][1] == 4
