"""The serial depth-sensing restatement (tests/sense_serial.cpp) on cases computed by hand: one point's centre and splat, occlusion, the
centre rule at the image's edges, points behind the camera, the 500 m rule, the horizon, the node's pixel order and non-finite records."""
import numpy as np
import pytest
import isdf_b200 as I
import sense_oracle as SO

IDENT = np.eye(4)


def cam(**kw):
    return I.sense_params(**kw)


def test_default_camera():
    p = cam()
    assert (p.width, p.height) == (640, 480)
    assert (p.fx, p.fy, p.cx, p.cy) == (387.229248046875, 387.229248046875, 321.04638671875, 243.44969177246094)
    assert list(p.cam_to_body) == [0, 0, 1, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 1]
    assert p.sensing_horizon == np.inf


def test_single_point_centre_and_splat():
    # camera frame = world frame; a point 2 m ahead at the optical axis of a 64 x 48 camera with fx = 100 at (31.6, 23.2)
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2)
    img, sk = SO.render(np.array([[0.0, 0.0, 2.0]], np.float32), IDENT, p)
    assert sk == 0
    # px = trunc(31.6 + 0.5) = 32, py = trunc(23.2 + 0.5) = 23; r = trunc(0.0573 * 100 / 2 + 0.5) = trunc(3.365) = 3; 2000 mm
    seen = np.argwhere(img != 999999)
    assert seen[:, 0].min() == 20 and seen[:, 0].max() == 26 and seen[:, 1].min() == 29 and seen[:, 1].max() == 35
    assert len(seen) == 49 and (img[img != 999999] == 2000).all()


def test_occlusion_takes_the_minimum():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2)
    img, _ = SO.render(np.array([[0.0, 0.0, 2.0], [0.0, 0.0, 1.5], [0.0, 0.0, 3.0]], np.float32), IDENT, p)
    assert img[23, 32] == 1500
    # r at 1.5 m is trunc(4.32) = 4, so the 2 m point's square lies inside the 1.5 m point's
    assert (img[19:28, 28:37] == 1500).all() and (img != 999999).sum() == 81


def test_centre_outside_is_rejected_though_its_splat_would_reach_in():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=0.0, cy=23.2)
    # x / z fx + cx + 0.5 = -1.2: trunc -> -1, outside; r = trunc(0.0573 100 / 0.5 + 0.5) = 11 would reach the image
    img, _ = SO.render(np.array([[-0.017, 0.0, 0.5]], np.float32), IDENT, p)
    assert (img == 999999).all()
    # the right edge: centre at 64.1 -> 64 = width
    img, _ = SO.render(np.array([[0.321, 0.0, 0.5]], np.float32), IDENT, p)
    assert (img == 999999).all()


def test_centre_in_minus_one_to_zero_is_kept():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=0.0, cy=23.2)
    # x / z fx + 0.5 = -0.7: truncates to 0, kept at column 0
    img, _ = SO.render(np.array([[-0.006, 0.0, 0.5]], np.float32), IDENT, p)
    assert img[23, 0] == 500 and (img[:, 0] == 500).sum() == 23 and (img[23, :] == 500).sum() == 12


def test_points_behind_the_camera():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2)
    img, _ = SO.render(np.array([[0.0, 0.0, -2.0], [0.0, 0.0, 0.0]], np.float32), IDENT, p)
    assert (img == 999999).all()


def test_depth_beyond_500_m_is_not_sensed():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2)
    img, _ = SO.render(np.array([[0.0, 0.0, 600.0]], np.float32), IDENT, p)
    assert img[23, 32] == 600000
    assert len(SO.backproject(img, IDENT.reshape(16), np.zeros(3), p)) == 0
    img, _ = SO.render(np.array([[0.0, 0.0, 499.0]], np.float32), IDENT, p)
    assert len(SO.backproject(img, IDENT.reshape(16), np.zeros(3), p)) == 1


def test_horizon_drop():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2, sensing_horizon=2.001)
    img, _ = SO.render(np.array([[0.0, 0.0, 2.0]], np.float32), IDENT, p)   # a 7 x 7 square at 2 m
    pts = SO.backproject(img, IDENT.reshape(16), np.zeros(3), p)
    # pixel (u, v) back-projects to ((u - cx) 2 / 100, (v - cy) 2 / 100, 2): kept where its distance is <= 2.001
    u, v = np.meshgrid(np.arange(29, 36), np.arange(20, 27), indexing="ij")
    d = np.sqrt(((u - 31.6) * 0.02) ** 2 + ((v - 23.2) * 0.02) ** 2 + 4.0)
    assert len(pts) == int((d <= 2.001).sum()) and 0 < len(pts) < 49


def test_pixel_order_is_u_outer_v_inner():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2)
    img = np.full((48, 64), 999999, np.int32)
    img[10, 5] = 1000    # u 5, v 10
    img[3, 7] = 2000     # u 7, v 3
    img[30, 5] = 3000    # u 5, v 30
    pts = SO.backproject(img, IDENT.reshape(16), np.zeros(3), p)
    assert pts[:, 2].tolist() == [1.0, 3.0, 2.0]
    assert np.isclose(pts[0, 0], (5 - 31.6) * 1.0 / 100) and np.isclose(pts[1, 1], (30 - 23.2) * 3.0 / 100)


def test_non_finite_records_are_skipped():
    p = cam(width=64, height=48, fx=100.0, fy=100.0, cx=31.6, cy=23.2)
    rec = np.array([[np.nan, 0, 1], [0, np.inf, 1], [0, 0, -np.inf], [0.0, 0.0, 2.0]], np.float32)
    img, sk = SO.render(rec, IDENT, p)
    ref, _ = SO.render(rec[3:], IDENT, p)
    assert sk == 3 and np.array_equal(img, ref)


def test_pose_matrices_with_the_default_camera():
    # body at (1, 2, 3) yawed by 90 degrees: the camera looks along world +y
    q = np.array([np.cos(np.pi / 4), 0, 0, np.sin(np.pi / 4)])
    c2w, cw = SO.pose(np.array([1.0, 2.0, 3.0]), q, np.array(cam().cam_to_body[:]))
    assert np.allclose(c2w.reshape(4, 4)[:3, 2], [0, 1, 0]) and np.array_equal(c2w.reshape(4, 4)[:3, 3], [1.0, 2.0, 3.0])
    T = cw.reshape(4, 4)
    assert np.allclose(T[:3, :3] @ c2w.reshape(4, 4)[:3, :3], np.eye(3), atol=1e-7)
    assert (T[:3] == T[:3].astype(np.float32)).all()   # rounded to FP32
    # a point 5 m ahead of the body is at camera depth 5
    assert np.isclose(T[2, :3] @ [1.0, 7.0, 3.0] + T[2, 3], 5.0, atol=1e-6)


@pytest.mark.parametrize("bad", [dict(width=0), dict(fx=0.0), dict(fx=np.nan), dict(sensing_horizon=0.0), dict(sensing_horizon=np.nan)])
def test_param_refusals_need_no_device(bad):
    ev = I.Evaluator.__new__(I.Evaluator)   # the checks run before the context is looked at
    ev.lib, ev.h = I.load_library(), None
    recs = np.zeros((1, 7))
    recs[0, 3] = 1
    with pytest.raises(I.IsdfError) as e:
        ev.sense_depth(recs, 0, 3, **bad)
    assert e.value.code != 0


def test_serial_matches_reference_golden():
    """the restatement reproduces the reference-compiled kernel's stored images from the same double[16] transforms"""
    p = cam()
    for name, g in SO.load_golden().items():
        for q in range(len(g["T"])):
            img, _ = SO.render(g["xyz"], g["T"][q], p)
            assert np.array_equal(img, g["depth"][q]), (name, q)
        # and the transforms are the ones the library defines for the stored poses
        for q in range(len(g["pos"])):
            assert np.array_equal(SO.pose(g["pos"][q], g["quat"][q], np.array(p.cam_to_body[:]))[1], g["T"][q])
