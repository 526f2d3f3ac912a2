"""CPU checks of the closed-loop navigation calls: the fusion restatement's inside test, index and counts; the shift restatement against
exact rational re-expansion and at junctions and ends; the log -> initial state conversion; refusals of every new entry point without a
context; and isdf_fuse_info's layout against a g++ probe of include/isdf.h."""
import ctypes as C
from fractions import Fraction
import numpy as np
import isdf_b200 as I
import navigate_oracle as NO
from test_plan_cpu import _probe, _fields


def test_fuse_inside_test_at_the_bounds_and_exact_multiples():
    bmin, res, dims = np.array([-1.0, 0.0, 2.0]), 0.5, (4, 4, 4)
    bmax = bmin + np.array(dims) * res
    occ = np.zeros(dims, dtype=np.uint8)
    pts = np.array([bmin, bmax, bmin + 0.5, bmin + [1.0, 1.5, 0.0],   # on bmin, on bmax (top layer), exact multiples
                    bmin - [1e-6, 0, 0], bmax + [0, 0, 1e-6],         # just outside
                    [np.nan, 0, 3], [0, np.inf, 3]], dtype=np.float32)
    out, cnt = NO.fuse(occ, bmin, bmax, res, pts)
    assert cnt == dict(points_used=4, points_outside=2, points_skipped=2, voxels_added=4)
    assert out[0, 0, 0] and out[3, 3, 3] and out[1, 1, 1] and out[2, 3, 0]
    # bits only grow, and a second fusion of the same points adds nothing
    out2, cnt2 = NO.fuse(out, bmin, bmax, res, pts)
    assert np.array_equal(out, out2) and cnt2["voxels_added"] == 0 and cnt2["points_used"] == 4


def test_fuse_is_order_and_split_free():
    rng = np.random.default_rng(3)
    bmin, res, dims = np.zeros(3), 0.25, (12, 10, 8)
    bmax = bmin + np.array(dims) * res
    pts = rng.uniform(-0.5, 3.5, (500, 3)).astype(np.float32)
    whole, cw = NO.fuse(np.zeros(dims, np.uint8), bmin, bmax, res, pts)
    perm = pts[rng.permutation(len(pts))]
    acc, added = np.zeros(dims, np.uint8), 0
    for part in np.array_split(perm, 7):
        acc, c = NO.fuse(acc, bmin, bmax, res, part)
        added += c["voxels_added"]
    assert np.array_equal(acc, whole) and added == cw["voxels_added"] == int(whole.sum())


def _random_traj(rng, N):
    T = rng.uniform(0.2, 1.5, N)
    Cc = rng.normal(0, 2, 18 * N)
    return T, Cc


def test_shift_matches_exact_reexpansion():
    rng = np.random.default_rng(5)
    for _ in range(50):
        c = rng.normal(0, 3, 6)
        tau = float(rng.uniform(0, 2))
        got = NO.reexpand(c, tau)
        ref = NO.reexpand_exact(c, tau)
        scale = float(sum(abs(Fraction(float(x))) * Fraction(tau) ** j for j, x in enumerate(c)))
        for g, r in zip(got, ref):
            assert abs(Fraction(g) - r) <= Fraction(1e-13) * max(scale, 1.0)
        # the polynomial about tau at s equals the original at tau + s (exactly, in rationals)
        s = Fraction(0.3)
        orig = sum(Fraction(float(x)) * (Fraction(tau) + s) ** j for j, x in enumerate(c))
        assert sum(d * s ** k for k, d in enumerate(ref)) == orig


def test_shift_junctions_ends_and_ragged():
    rng = np.random.default_rng(7)
    T1, C1 = _random_traj(rng, 3)
    T2, C2 = _random_traj(rng, 1)
    T1[:] = [0.5, 0.25, 1.0]   # exact binary times: junctions are exact
    off = np.array([0, 3, 3, 4], dtype=np.int32)
    T, Cc = np.concatenate([T1, T2]), np.concatenate([C1, C2])
    # t0 = 0: piece 0 re-expanded about 0 is itself, every piece kept
    oo, oT, oC = NO.shift(off, T, Cc, [0.0, 0.0, 0.0])
    assert list(oo) == [0, 3, 3, 4] and np.array_equal(oT, T) and np.array_equal(oC, Cc)
    # t0 on the first junction: locatePieceIdx keeps it in piece 0 with tau = T_0, so piece 0 is dropped and the rest copied
    oo, oT, oC = NO.shift(off, T, Cc, [0.5, 1.0, T2[0] / 2])
    assert list(oo) == [0, 2, 2, 3]
    assert np.array_equal(oT[:2], T1[1:]) and np.array_equal(oC[:36], NO._unblock(NO._block(C1, 3)[1:]))
    assert oT[2] == T2[0] - T2[0] / 2
    # the end and beyond, negative and non-finite times: no piece
    for t0 in (1.75, 2.0, -1e-9, np.nan, np.inf):
        oo, oT, oC = NO.shift(off[:2], T1, C1, [t0])
        assert list(oo) == [0, 0] and oT.size == 0
    # inside a piece: one re-expanded piece, then the copies
    oo, oT, oC = NO.shift(off[:2], T1, C1, [0.6])
    i, tau = NO.locate(list(T1), 0.6)
    assert (i, list(oo)) == (1, [0, 2]) and oT[0] == T1[1] - tau and oT[1] == T1[2]
    blk = NO._block(oC, 2)
    for a in range(3):
        assert blk[0, a].tolist() == NO.reexpand(NO._block(C1, 3)[1, a], tau)


def test_log_to_init():
    rec = np.arange(2 * 21, dtype=np.float64).reshape(2, 21)
    init = NO.log_to_init(rec)
    assert init.shape == (2, I.SIM_INIT_DOUBLES) and np.array_equal(init, rec[:, 1:18])
    assert np.array_equal(I.sim_init_from_log(rec), init)


def test_new_entry_points_refuse_a_null_context():
    lib = I.load_library()
    pts = np.zeros((4, 3), dtype=np.float32)
    vp = C.c_void_p(pts.ctypes.data)
    info = I.FuseInfo()
    assert lib.isdf_map_fuse_cloud(None, vp, 4, 12, C.byref(info)) == -1
    assert lib.isdf_map_fuse_cloud_device(None, vp, 4, 12, C.byref(info), None) == -1
    assert lib.isdf_map_fuse_cloud(None, vp, 4, 10, None) == -1 and b"stride" in lib.isdf_last_error()
    st, gl = np.zeros(9), np.zeros(3)
    dp = C.POINTER(C.c_double)
    p = I.PlanParams()
    assert lib.isdf_plan_default_params(None, C.byref(p)) == 0
    res = (I.PlanResult * 1)()
    po = np.zeros(2, dtype=np.int32)
    args = (None, 1, st.ctypes.data_as(dp), gl.ctypes.data_as(dp), C.byref(p), 0, 0, None, None, 0, po.ctypes.data_as(C.POINTER(C.c_int32)),
            None, None, res, None, None)
    assert lib.isdf_plan_states(*args) == -1 and res[0].stage == I.PLAN_FAILED
    assert lib.isdf_plan_states_device(*args, None) == -1
    off, T, Cc, t0 = np.array([0, 1], dtype=np.int32), np.ones(1), np.zeros(18), np.zeros(1)
    ip = C.POINTER(C.c_int32)
    sargs = (None, 1, off.ctypes.data_as(ip), T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), t0.ctypes.data_as(dp), off.ctypes.data_as(ip),
             T.ctypes.data_as(dp), Cc.ctypes.data_as(dp))
    assert lib.isdf_trajectory_shift(*sargs) == -1
    dargs = [a.ctypes.data for a in (off, T, Cc, t0, off, T, Cc)]
    assert lib.isdf_trajectory_shift_device(None, 1, *dargs, None) == -1


def test_fuse_info_layout_matches_the_header():
    got = _probe([("isdf_fuse_info", I.FuseInfo)])
    size, offs = got["isdf_fuse_info"]
    assert size == C.sizeof(I.FuseInfo) == 32 and offs == dict(_fields(I.FuseInfo))
