"""CPU-only checks of the continuous clearance certificate's restatement (tests/certify_oracle.py): the motion bound against the dense
displacement of mesh vertices and Box corners on aggressive pieces, the pose pad against the rounding of the pose, soundness of the
oracle's CERTIFIED verdicts against a dense clearance, the thin wall that sampling misses, and the C ABI without a GPU."""
import ctypes as C
import math
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import clearance_oracle as CO
import certify_oracle as CE

BOX_HALF = [0.9, 0.5, 0.3]


def cfg_with(drag):
    cfg = I.default_config_values()
    if not drag:
        cfg.horiz_drag = cfg.paras_drag = 0.0
    return cfg


def aggressive_pieces():
    """(name, T (1,), coeffs (18,)) single pieces: hover, an 80-degree tilt with large jerk, random quintics"""
    g = 9.8
    out = []
    c = np.zeros((3, 6)); c[:, 0] = [1.0, 2.0, 3.0]; c[0, 1] = 2.0
    out.append(("cruise", 2.0, c))
    c = np.zeros((3, 6)); c[0, 2] = 0.5 * g * math.tan(math.radians(80.0)); c[0, 3] = 40.0; c[1, 3] = -30.0; c[2, 1] = 1.0
    out.append(("tilt80_jerk", 0.25, c))
    rng = np.random.default_rng(3)
    for k in range(4):
        c = rng.normal(0, 1, (3, 6)) * np.array([5, 4, 3, 2, 1.5, 1.0])
        out.append((f"random{k}", 0.6 + 0.2 * k, c))
    return [(n, np.array([T]), c.reshape(-1)) for n, T, c in out]


def max_tilt(cfg, T, Cc):
    _, R = CE.pose_at(cfg, T, Cc, np.zeros(201, int), np.linspace(0, T[0], 201))
    return float(np.degrees(np.arccos(np.clip(R[:, 2, 2], -1, 1))).max())


def bodies():
    V, _ = W.rounded_cone_mesh(n_theta=16, n_prof=12)
    return {"mesh": V, "box": CE.box_corners(BOX_HALF)}


@pytest.mark.parametrize("drag", [True, False])
def test_bound_covers_dense_displacement(drag):
    cfg = cfg_with(drag)
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + 2.0
    tilts = []
    for name, T, Cc in aggressive_pieces():
        tilts.append(max_tilt(cfg, T, Cc))
        if tilts[-1] > 85.0:
            continue
        c = CE.piece_coeffs(Cc, 1, 0)
        Ti = T[0]
        ivs = [(0.0, Ti), (0.3 * Ti, 0.3 * Ti + 1e-6), (Ti - Ti / 64, Ti), (0.0, Ti / 64), (Ti - 1e-6, Ti)]
        for bname, body in bodies().items():
            r = CE.body_radius(body)
            for ta, tb in ivs:
                for te in (ta, tb):
                    D = CE.bound(cfg, r, H, c, ta, tb, te)
                    dense = CE.displacement(cfg, T, Cc, 0, ta, tb, te, body)
                    assert D >= dense, (name, bname, ta, tb, te, D, dense)
                    assert D < math.inf or tb - ta > Ti / 2      # a whole piece may enclose |zu| = 0: no bound, refine
    assert max(tilts) >= 75.0, tilts                                  # the aggressive case is aggressive


def test_bound_at_piece_ends_of_a_multi_piece_trajectory():
    cfg = cfg_with(True)
    T, Cc, _ = W.make_trajectory(3, [0, 0, 0], [20, 20, 20], seed=4, jitter=0.3)
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + 1.0
    body = bodies()["mesh"]
    r = CE.body_radius(body)
    for i in range(3):
        c = CE.piece_coeffs(Cc, 3, i)
        for ta, tb in [(0.0, T[i] / 16), (T[i] - T[i] / 16, T[i]), (0.0, T[i])]:
            for te in (ta, tb):
                assert CE.bound(cfg, r, H, c, ta, tb, te) >= CE.displacement(cfg, T, Cc, i, ta, tb, te, body)


def test_pose_pad_covers_the_rounding_of_the_pose():
    """eps_e against the difference between the double pose and an extended-precision one, scaled as in the definition: position
    error plus (r + 2H) times the rotation error must stay far below eps_e"""
    cfg = cfg_with(True)
    body = bodies()["mesh"]
    r = CE.body_radius(body)
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + 2.0
    for name, T, Cc in aggressive_pieces():
        c = CE.piece_coeffs(Cc, 1, 0)
        for te in np.linspace(0, T[0], 7):
            p64, R64 = CE.pose_at(cfg, T, Cc, [0], [te])
            pl, Rl = CE.pose_closed_form(cfg, c, te, np.longdouble)
            err = float(np.abs(p64[0] - pl.astype(float)).max() + (r + 2 * H) * np.abs(R64[0] - Rl.astype(float)).max())
            eps = CE.eps_pad(cfg, r, H, c, te)
            assert err * 1e3 <= eps, (name, te, err, eps)


def thin_wall():
    """a one-voxel wall across a straight rest-to-rest piece: the samples at K_c = 3 lie 4 m and more from it"""
    occ = np.zeros((20, 9, 9), dtype=np.uint8)
    occ[10, :, :] = 1
    wp = np.array([[2.0, 4.5, 4.5], [18.0, 4.5, 4.5]])
    T = np.array([4.0])
    return occ, [0.0, 0.0, 0.0], 1.0, T, W.minco_s3(wp, T)


def crossing_window(cfg, T, Cc, radius, margin):
    """times at which the ball's centre is closer than radius + margin to the wall's voxel centres (x = 10.5)"""
    t = np.linspace(0, T[0], 40001)
    pos, _ = CE.pose_at(cfg, T, Cc, np.zeros(t.size, int), t)
    inside = np.abs(pos[:, 0] - 10.5) < radius + margin
    return t[inside].min(), t[inside].max()


def test_thin_wall_is_colliding_in_the_oracle():
    cfg = I.default_config_values()
    occ, bmin, res, T, Cc = thin_wall()
    ball = O.Shape.named("Ball")
    reach, margin, K = 2.0, 0.5, 3
    sampled = CO.clearance(O.config_from(cfg), occ, bmin, res, ball, T, Cc, K, reach, margin)
    assert sampled["summary"][0]["collision_free"] == 1 and sampled["clear"].min() >= margin + 0.1
    out = CE.certify(cfg, occ, bmin, res, ball, 0.0, T, Cc, K, reach, margin)
    s = out["summary"][0]
    lo, hi = crossing_window(cfg, T, Cc, 1.0, margin)
    assert s["verdict"] == -1 and lo <= s["first_hit"] <= hi, (s, lo, hi)
    assert s["lower_bound"] <= s["min_clearance"] < margin


@pytest.mark.parametrize("shape", ["Ball", "Box"])
def test_oracle_certified_means_dense_clear(shape):
    cfg = I.default_config_values()
    cfg.kernel_size = 7
    occ = W.random_map(14, 14, 14, p=0.01, seed=5, slabs=0)
    if shape == "Ball":
        osh, r = O.Shape.named("Ball"), 0.0
    else:
        osh, r = O.Shape.analytic(I.SHAPE_KINDS["BOX"], BOX_HALF), CE.body_radius(CE.box_corners(BOX_HALF))
    reach, K = 2.0, 4
    verdicts = []
    for seed in range(4):
        rng = np.random.default_rng(seed)
        wp = 3.0 + 8.0 * rng.random((3, 3))
        T = 1.5 + rng.random(2)
        Cc = W.minco_s3(wp, T)
        dense = CO.clearance(O.config_from(cfg), occ, [0, 0, 0], 1.0, osh, T, Cc, 4096, reach, 0.0)["clear"].min()
        for margin in (0.2, 0.6):
            s = CE.certify(cfg, occ, [0, 0, 0], 1.0, osh, r, T, Cc, K, reach, margin, max_depth=8, max_samples=512)["summary"][0]
            verdicts.append(s["verdict"])
            assert s["lower_bound"] <= dense + 1e-12
            if s["verdict"] == 1:
                assert dense >= s["lower_bound"] >= margin
    assert 1 in verdicts, verdicts


def test_struct_layouts_and_defaults_without_a_gpu():
    assert C.sizeof(I.CertifyParams) == 40 and C.sizeof(I.CertifySummary) == 56 and I.CERT_LEAF_DTYPE.itemsize == 56
    lib = I.load_library()
    p = I.CertifyParams()
    assert lib.isdf_certify_default_params(C.byref(p)) == 0
    d = I.default_config_values()
    q = p.clearance
    assert (q.samples_per_piece, q.pieces_per_traj, q.margin, q.reach) == (d.integral_intervs, 0, d.safety_hor, 2 * d.safety_hor)
    assert (p.max_depth, p.max_samples_per_traj, p.reserved_[0], p.reserved_[1]) == (16, 2048, 0, 0)
    assert lib.isdf_certify_default_params(None) == -1
    summ = (I.CertifySummary * 2)()
    dp = C.POINTER(C.c_double)
    T, Cc = np.ones(4), np.zeros(72)
    p.clearance.pieces_per_traj = 2
    assert lib.isdf_trajectory_certify(None, 4, T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(p), summ) == -1
    for s in summ:
        assert s.verdict == 0 and np.isnan(s.lower_bound) and np.isnan(s.min_clearance)
