"""CPU checks of known space (include/isdf.h, isdf_map_observe / isdf_map_mark_known) through its numpy restatement
(tests/observe_oracle.py) on synthetic depth images: an empty image marks the in-image frustum within the horizon, one near pixel blocks
the voxels whose mip cells cover it, voxels across the image edge, z = 0 and the horizon stay unknown; the box rule of mark_known; the
argument checks that need no device; isdf_observe_info against a g++ probe of include/isdf.h."""
import ctypes as C
import numpy as np
import isdf_b200 as I
import observe_oracle as OO
from test_plan_cpu import _probe, _fields

RES = 0.25
BMIN = np.array([-4.0, -4.0, -1.0])
DIMS = (32, 32, 32)


def _cam(horizon=5.0):
    # a small camera looking along world +z from the origin (camera frame = world frame)
    return I.sense_params(width=64, height=48, fx=40.0, fy=40.0, cx=31.5, cy=23.5, sensing_horizon=horizon)


CW = np.eye(4).reshape(16)
BODY = np.zeros(3)


def _corners(ix, iy, iz):
    lo = [OO.voxel_span(BMIN[a], RES, i)[0] for a, i in enumerate((ix, iy, iz))]
    hi = [OO.voxel_span(BMIN[a], RES, i)[1] for a, i in enumerate((ix, iy, iz))]
    return np.array([[hi[0] if k & 1 else lo[0], hi[1] if k & 2 else lo[1], hi[2] if k & 4 else lo[2]] for k in range(8)])


def _frustum(p, inner=0.0, zmin=0.0):
    """voxels whose 8 corners lie in front of the camera (z > zmin), within the horizon, and project inner pixels inside the image"""
    out = np.zeros(DIMS, dtype=bool)
    for ix in range(DIMS[0]):
        for iy in range(DIMS[1]):
            for iz in range(DIMS[2]):
                c = _corners(ix, iy, iz)
                if not (c[:, 2] > zmin).all() or not (np.linalg.norm(c, axis=1) <= p.sensing_horizon).all():
                    continue
                u = c[:, 0] / c[:, 2] * p.fx + p.cx
                v = c[:, 1] / c[:, 2] * p.fy + p.cy
                out[ix, iy, iz] = u.min() >= -0.5 + inner and u.max() < p.width - 0.5 - inner and v.min() >= -0.5 + inner \
                    and v.max() < p.height - 0.5 - inner
    return out


def test_empty_image_marks_the_frustum_within_the_horizon():
    p = _cam()
    img = np.full((p.height, p.width), 999999, dtype=np.int32)
    k = OO.observe(img, CW, BODY, p, BMIN, RES, DIMS)
    outer, inner = _frustum(p), _frustum(p, inner=0.01, zmin=1e-3)
    assert k.sum() > 1000
    assert not (k & ~outer).any()       # nothing outside the exact frustum
    assert not (inner & ~k).any()       # everything strictly inside it
    # the index box: floor((0 -+ 5 - bmin) / 0.25) - 1 + [0, 43) per axis, cut to the map: all of x and y, z indices 0 .. 25
    assert OO.tested([BODY], p.sensing_horizon, BMIN, RES, DIMS) == 32 * 32 * 26


def test_one_near_pixel_blocks_exactly_the_voxels_whose_cells_cover_it():
    p = _cam()
    empty = np.full((p.height, p.width), 999999, dtype=np.int32)
    img = empty.copy()
    u0, v0 = 40, 30
    img[v0, u0] = 2000   # a point 2 m deep
    k0 = OO.observe(empty, CW, BODY, p, BMIN, RES, DIMS)
    k1 = OO.observe(img, CW, BODY, p, BMIN, RES, DIMS)
    assert not (k1 & ~k0).any()
    lost = k0 & ~k1
    assert lost.any()
    # the voxels holding the pixel's ray at 1.9 m (in front of the point, but reaching behind it) and at 3.1 m (behind it) are no longer
    # known; every lost voxel reaches behind the point, and its corners' rectangle, grown to its mip cells, covers the pixel
    for z in (1.9, 3.1):
        pt = np.array([(u0 - p.cx) / p.fx * z, (v0 - p.cy) / p.fy * z, z])
        idx = tuple(int(np.floor((pt[a] - BMIN[a]) / RES)) for a in range(3))
        assert k0[idx] and not k1[idx]
    for ix, iy, iz in zip(*np.nonzero(lost)):
        c = _corners(ix, iy, iz)
        assert c[:, 2].max() > 2.0 - 1e-3
        u = c[:, 0] / c[:, 2] * p.fx + p.cx
        v = c[:, 1] / c[:, 2] * p.fy + p.cy
        x0, x1, y0, y1 = int(np.floor(u.min() + 0.5)), int(np.floor(u.max() + 0.5)), int(np.floor(v.min() + 0.5)), int(np.floor(v.max() + 0.5))
        l = 0
        while (x1 >> l) - (x0 >> l) > 1 or (y1 >> l) - (y0 >> l) > 1:
            l += 1
        assert (x0 >> l) <= (u0 >> l) <= (x1 >> l) + 1 and (y0 >> l) <= (v0 >> l) <= (y1 >> l) + 1
    # voxels wholly in front of the point stay known
    assert k1[:, :, :int(np.floor((1.99 - BMIN[2]) / RES))].sum() == k0[:, :, :int(np.floor((1.99 - BMIN[2]) / RES))].sum()


def test_voxels_across_the_edge_z0_and_horizon_stay_unknown():
    p = _cam(horizon=3.0)
    img = np.full((p.height, p.width), 999999, dtype=np.int32)
    k = OO.observe(img, CW, BODY, p, BMIN, RES, DIMS)
    iz0 = int(round((0.0 - BMIN[2]) / RES))   # voxels [iz0 - 1] straddle nothing: their top face is z = 0
    assert not k[:, :, :iz0 + 1].any()        # z in [0, 0.25] touches z = 0: every corner must be in front by the margin
    for ix in range(DIMS[0]):
        for iy in range(DIMS[1]):
            for iz in range(DIMS[2]):
                if not k[ix, iy, iz]:
                    continue
                c = _corners(ix, iy, iz)
                assert (np.linalg.norm(c, axis=1) <= 3.0).all()
                u = c[:, 0] / c[:, 2] * p.fx + p.cx
                assert u.min() >= -0.5 and u.max() < p.width - 0.5
    # a voxel crossing the horizon sphere along the axis, and one crossing the image's right edge at 2 m
    iz_h = int(np.floor((3.0 - BMIN[2]) / RES))
    assert not k[16, 16, iz_h] and not k[16, 16, iz_h - 1] and k[16, 16, iz_h - 2]
    x_edge = (p.width - 0.5 - p.cx) / p.fx * 2.0
    ix_e = int(np.floor((x_edge - BMIN[0]) / RES))
    assert not k[ix_e, 16, int(np.floor((2.0 - BMIN[2]) / RES))]


def test_mip_levels_are_clipped_minima():
    rng = np.random.default_rng(3)
    img = rng.integers(100, 999999, (13, 21)).astype(np.int32)
    L = OO.mip(img)
    assert L[-1].shape == (1, 1) and L[-1][0, 0] == img.min()
    for l in range(1, len(L)):
        s = 1 << l
        for j in range(L[l].shape[0]):
            for i in range(L[l].shape[1]):
                assert L[l][j, i] == img[j * s:(j + 1) * s, i * s:(i + 1) * s].min()


def test_mark_known_box_rule():
    boxes = np.array([[-1.0, -1.0, -1.0, 0.5, 0.5, 0.5], [1.1, 1.1, 1.1, 1.2, 1.2, 1.2], [2.1, 2.0, 2.0, 2.4999, 2.75, 2.75]])
    k = OO.mark_boxes(boxes, BMIN, RES, DIMS)
    # the closed box [-1, 0.5] holds the voxels whose cubes [bmin + i res, bmin + (i + 1) res] lie in it, faces on its faces included
    sel = lambda lo, hi, b: (np.arange(DIMS[0]) >= round((lo - b) / RES)) & (np.arange(DIMS[0]) < round((hi - b) / RES))
    want = sel(-1.0, 0.5, -4.0)[:, None, None] & sel(-1.0, 0.5, -4.0)[None, :, None] & sel(-1.0, 0.5, -1.0)[None, None, :]
    # the second box is thinner than a voxel; the third holds three voxels in y and z but none in x ([2.1, 2.4999] holds no cube)
    assert np.array_equal(k, want) and k.sum() == 6 * 6 * 6


def test_constants_and_info_layout():
    assert (I.UNKNOWN_FREE, I.UNKNOWN_OCCUPIED) == (0, 1)
    got = _probe([("isdf_observe_info", I.ObserveInfo)])
    size, offs = got["isdf_observe_info"]
    assert size == C.sizeof(I.ObserveInfo) == 24 and offs == dict(_fields(I.ObserveInfo))


def test_argument_checks_without_a_device():
    lib = I.load_library()
    rec = np.zeros((1, 7))
    rec[0, 3] = 1.0
    dp = rec.ctypes.data
    p = I.sense_params(sensing_horizon=10.0)
    info = I.ObserveInfo()
    assert lib.isdf_map_observe(None, 1, C.c_void_p(dp), C.c_void_p(dp + 24), 7, C.byref(p), C.byref(info)) == -1
    assert lib.isdf_map_observe_device(None, 1, C.c_void_p(dp), C.c_void_p(dp + 24), 7, C.byref(p), C.byref(info), None) == -1
    assert lib.isdf_map_observe(None, 0, C.c_void_p(dp), C.c_void_p(dp + 24), 7, C.byref(p), None) == -1 and b"Q" in lib.isdf_last_error()
    assert lib.isdf_map_mark_known(None, 0, None) == -1
    assert lib.isdf_get_map_known_u8(None, None, 0) == -1
    assert lib.isdf_set_unknown_policy(None, 0) == -1
    v = C.c_int(5)
    assert lib.isdf_get_unknown_policy(None, C.byref(v)) == -1


def test_navigate_refuses_occupied_without_brake_and_infinite_horizons():
    import pytest
    ev = object.__new__(I.Evaluator)   # the refusals come before any device work
    s, g = np.zeros((1, 3)), np.ones((1, 3))
    with pytest.raises(ValueError, match="fallback='brake'"):
        ev.navigate(s, g, rounds=1, horizon=0.5, unknown="occupied", fallback="keep", sense_params=_cam())
    with pytest.raises(ValueError, match="finite sensing_horizon"):
        ev.navigate(s, g, rounds=1, horizon=0.5, unknown="occupied", fallback="brake", sense_params=[_cam(), I.sense_params()])
    with pytest.raises(ValueError, match="unknown must be"):
        ev.navigate(s, g, rounds=1, horizon=0.5, unknown="maybe")
    with pytest.raises(ValueError, match="empty camera list"):
        ev.navigate(s, g, rounds=1, horizon=0.5, sense_params=[])
