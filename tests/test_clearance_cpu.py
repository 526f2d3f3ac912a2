"""CPU-only checks of the trajectory clearance check: the brute-force restatement (tests/clearance_oracle.py) against an independent
numpy closed form for the Ball robot, and the C ABI's struct layouts and argument validation without a GPU."""
import ctypes as C
import numpy as np
import pytest
import isdf_b200 as I
import oracle_lib as O
import workloads as W
import clearance_oracle as CO


def closed_form_ball(cfg, occ, bmin, res, radius, T, Cc, K, reach, margin):
    """the definition restated for Ball: Horner-evaluated positions, the oracle's flatness quaternion, an explicit triple loop over the
    voxel index box of each sample's H ball-of-infinity (clipped to the map), sdf = |c - x| - radius (rotation-invariant)"""
    T = np.asarray(T, float)
    N = T.size
    Cm = np.asarray(Cc, float).reshape(3, 6 * N)
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + reach
    X, Y, Z = occ.shape
    bmin = np.asarray(bmin, float)
    clear, vox = [], []
    oc = O.config_from(cfg)
    for i in range(N):
        c = Cm[:, 6 * i:6 * i + 6]
        step = T[i] * (1.0 / K)
        for j in range(K + 1):
            s = j * step
            p = np.zeros(3); v = np.zeros(3); a = np.zeros(3)
            for k in range(5, -1, -1):
                p = p * s + c[:, k]
            for k in range(5, 0, -1):
                v = v * s + k * c[:, k]
            for k in range(5, 1, -1):
                a = a * s + k * (k - 1) * c[:, k]
            q, _ = O.flat_forward(oc, v, a, np.zeros(3))
            w, x, y, z = q
            R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                          [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                          [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
            r = H * np.sqrt(3.0) + res                           # every candidate lies within the circumscribed ball of the H box
            lo = np.maximum(np.floor((p - r - bmin) / res).astype(int), 0)
            hi = np.minimum(np.ceil((p + r - bmin) / res).astype(int), np.array([X, Y, Z]) - 1)
            best, bid = reach, -1
            for ix in range(lo[0], hi[0] + 1):
                for iy in range(lo[1], hi[1] + 1):
                    zs = np.arange(lo[2], hi[2] + 1)
                    zs = zs[occ[ix, iy, zs] != 0] if zs.size else zs
                    for iz in zs:
                        ctr = (np.array([ix, iy, iz]) + 0.5) * res + bmin
                        d = ctr - p
                        if np.any(np.abs(R.T @ d) > H):
                            continue
                        sd = np.sqrt(d @ d) - radius
                        a_ = (ix * Y + iy) * Z + iz
                        if sd < best or (sd == best and bid >= 0 and a_ < bid):
                            best, bid = sd, a_
            clear.append(best); vox.append(bid)
    return np.array(clear), np.array(vox, dtype=np.int64)


def test_oracle_matches_ball_closed_form_with_a_pose_outside_the_map():
    cfg = I.default_config_values()
    cfg.kernel_size = 5
    occ = W.random_map(14, 12, 10, p=0.08, seed=2, slabs=0)
    bmin, res = [0.25, -0.5, 0.125], 0.8
    wp = np.array([[2.0, 2.0, 2.0], [8.0, 6.0, 5.0], [22.0, 4.0, 7.5]])   # the last piece leaves the map (x > 0.25 + 14 * 0.8)
    T = np.array([2.0, 2.5])
    Cc = W.minco_s3(wp, T)
    K, reach, margin = 6, 1.2, 0.6
    oc = O.config_from(cfg)
    ball = O.Shape.named("Ball")
    radius = ball.params()[0]
    got = CO.clearance(oc, occ, bmin, res, ball, T, Cc, K, reach, margin)
    exp_c, exp_v = closed_form_ball(cfg, occ, bmin, res, radius, T, Cc, K, reach, margin)
    assert np.max(np.abs(got["clear"] - exp_c)) <= 1e-12
    assert np.array_equal(got["voxel"], exp_v)
    assert (exp_v >= 0).sum() >= 4 and (exp_v < 0).sum() >= 1      # both outcomes occur
    s = got["summary"][0]
    assert s["colliding_samples"] == int((exp_c < margin).sum())
    assert abs(s["min_clearance"] - exp_c.min()) <= 1e-12 and s["voxel_min"] == exp_v[int(np.argmin(exp_c))]


def test_struct_layouts_match_the_header():
    assert C.sizeof(I.ClearanceParams) == 24
    assert C.sizeof(I.ClearanceSummary) == 48
    assert [n for n, _ in I.ClearanceSummary._fields_] == ["min_clearance", "t_min", "first_hit", "voxel_min", "piece_min", "sample_min",
                                                           "colliding_samples", "collision_free"]


def test_default_params_without_a_gpu():
    lib = I.load_library()
    p = I.ClearanceParams()
    assert lib.isdf_clearance_default_params(C.byref(p)) == 0
    d = I.default_config_values()
    assert (p.samples_per_piece, p.pieces_per_traj, p.reach, p.margin) == (d.integral_intervs, 0, d.safety_hor, d.safety_hor)
    assert lib.isdf_clearance_default_params(None) == -1


@pytest.mark.parametrize("N0,B", [(0, 1), (2, 3)])
def test_argument_validation_poisons_every_summary_without_gpu_calls(N0, B):
    lib = I.load_library()
    N = 6
    T, Cc = np.ones(N), np.zeros(18 * N)
    p = I.ClearanceParams(8, N0, 1.0, 0.5)
    summ = (I.ClearanceSummary * B)()
    dp = C.POINTER(C.c_double)
    r = lib.isdf_trajectory_clearance(None, N, T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), C.byref(p), None, None, summ)
    assert r == -1 and b"ctx" in lib.isdf_last_error()
    for s in summ:                                               # never reads as collision-free
        assert np.isnan(s.min_clearance) and s.collision_free == 0 and s.voxel_min == -1
    assert lib.isdf_trajectory_clearance(None, N, None, None, None, None, None, None) == -1
    assert lib.isdf_trajectory_clearance_device(None, N, None, None, C.byref(p), None, None, None, None) == -1
