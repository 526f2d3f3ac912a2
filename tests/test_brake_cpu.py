"""CPU checks of isdf_trajectory_brake's definition (tests/brake_oracle.py): the constant-deceleration schedule on a straight line, the
single-piece and single-candidate cases, tau_max clamped by the trajectory's duration, the NO_INPUT cases, the candidate's MINCO solve
against the reference-compiled minco.hpp when it is built, the argument checks that need no device, and isdf_brake_params /
isdf_brake_summary against a g++ probe of include/isdf.h."""
import ctypes as C
import math
import os
import numpy as np
import pytest
import isdf_b200 as I
import brake_oracle as BO
import navigate_oracle as NO
import oracle_lib as O
from test_plan_cpu import _probe, _fields


def _line(p0, v, D):
    """one piece of duration D: x(t) = p0 + v t"""
    blk = np.zeros((1, 3, 6))
    blk[0, :, 0], blk[0, :, 1] = p0, v
    return np.array([D]), NO._unblock(blk)


def _random_traj(rng, N):
    T = rng.uniform(0.3, 1.2, N)
    blk = rng.normal(0, 1.5, (N, 3, 6))
    return T, NO._unblock(blk)


def _end_state(cand):
    D = 0.0
    for x in cand["T"]:
        D += x
    return BO.pva(cand["T"], cand["coeffs"], D)


def test_schedule_is_the_constant_deceleration_profile():
    # at time t of a stop of duration 2 tau the remaining path is covered up to f = 1 - (1 - t / (2 tau))^2 of tau
    for M in (1, 2, 4, 7):
        tau, dur, times = BO.schedule(3.0, 1, 4, M)
        assert tau == 3.0 * (2.0 / 4.0) and dur.size == M and np.all(dur == (tau + tau) / M)
        for j, s in enumerate(times, 1):
            t = j * (2 * tau / M)
            assert s == pytest.approx(tau * (1 - (1 - t / (2 * tau)) ** 2), rel=1e-15)
        assert len(times) == M - 1


def test_constant_velocity_line_stops_at_x_tau_with_zero_v_and_a():
    p0, v = np.array([1.0, -2.0, 0.5]), np.array([2.0, 1.0, -0.5])
    T, Cc = _line(p0, v, 6.0)
    K, M = 5, 4
    for k in range(K):
        cand = BO.candidate(T, Cc, 4.0, k, K, M)
        tau = cand["tau"]
        assert tau == 4.0 * (float(k + 1) / float(K))
        # the head is the input's state at 0, bit for bit
        assert np.array_equal(cand["head"][:, 0], p0) and np.array_equal(cand["head"][:, 1], v) and np.all(cand["head"][:, 2] == 0)
        h = BO.pva(cand["T"], cand["coeffs"], 0.0)
        scale = np.abs(p0).max() + np.abs(v).max() * tau
        assert np.abs(h[0] - p0).max() <= 1e-12 * scale and np.abs(h[1] - v).max() <= 1e-11 * scale
        # the end: x(tau) at rest
        pe, ve, ae = _end_state(cand)
        assert np.abs(pe - (p0 + v * tau)).max() <= 1e-11 * scale
        assert np.abs(ve).max() <= 1e-10 * scale and np.abs(ae).max() <= 1e-9 * scale
        # on a line the constant-deceleration profile is what MINCO S3 interpolates: position at each waypoint time of the stop
        for j, s in enumerate(cand["times"], 1):
            pj = BO.pva(cand["T"], cand["coeffs"], j * cand["T"][0])[0]
            assert np.abs(pj - (p0 + v * s)).max() <= 1e-11 * scale


def test_single_piece_and_single_candidate():
    rng = np.random.default_rng(11)
    T, Cc = _random_traj(rng, 3)
    c = BO.candidate(T, Cc, 1.1, 0, 1, 1)   # K = 1: tau = tau_max; M = 1: no waypoint
    assert c["tau"] == 1.1 and c["T"].tolist() == [2.2] and c["waypoints"].shape == (3, 0) and c["coeffs"].size == 18
    assert np.array_equal(c["tail"][:, 0], BO.pva(T, Cc, 1.1)[0]) and np.all(c["tail"][:, 1:] == 0)
    pe, ve, ae = _end_state(c)
    assert np.abs(pe - c["tail"][:, 0]).max() <= 1e-10 * max(1.0, np.abs(pe).max()) and np.abs(ve).max() <= 1e-9 and np.abs(ae).max() <= 1e-8
    c2 = BO.candidate(T, Cc, 1.1, 2, 3, 5)
    assert c2["tau"] == 1.1 * (3.0 / 3.0) and len(c2["times"]) == 4


def test_tau_max_is_clamped_by_the_duration():
    rng = np.random.default_rng(12)
    T, Cc = _random_traj(rng, 4)
    D = 0.0
    for x in T:
        D += x
    for ts in (D, D + 1.0, np.inf, 1e300):
        assert BO.tau_max(T, ts) == D
    c = BO.candidate(T, Cc, np.inf, 3, 4, 3)
    assert c["tau"] == D and np.array_equal(c["tail"][:, 0], BO.pva(T, Cc, D)[0])
    # the position at D is the last piece at its end (locatePieceIdx clamps into it)
    i, tl = NO.locate(list(T), D)
    assert i == 3 and tl == pytest.approx(T[3], rel=1e-12)
    assert BO.tau_max(T, 0.5 * D) == 0.5 * D


def test_no_input_cases():
    rng = np.random.default_rng(13)
    T, Cc = _random_traj(rng, 2)
    for ts in (0.0, -1.0, -np.inf, np.nan, -0.0):
        assert BO.tau_max(T, ts) is None and BO.candidate(T, Cc, ts, 0, 8, 4) is None
    assert BO.tau_max(np.zeros(0), 1.0) is None
    off = np.array([0, 2, 2], dtype=np.int32)
    assert BO.ragged_candidate(off, T, Cc, [1.0, 1.0], 1, 0, 8, 4) is None
    assert BO.ragged_candidate(off, T, Cc, [1.0, 1.0], 0, 7, 8, 4)["tau"] == BO.tau_max(T, 1.0)


@pytest.mark.skipif(not os.path.exists(O.REF_MINCO), reason="oracle/_ref not built (needs the reference tree)")
def test_candidates_against_reference_compiled_minco():
    rng = np.random.default_rng(14)
    rm = O.RefMinco()
    for N, M in ((1, 1), (3, 4), (6, 4), (12, 8)):
        T, Cc = _random_traj(rng, N)
        c = BO.candidate(T, Cc, float(rng.uniform(0.2, 3.0)), int(rng.integers(0, 8)), 8, M)
        rc = rm.forward(c["head"], c["tail"], c["waypoints"], c["T"])[0]
        assert np.abs(c["coeffs"] - rc).max() <= 1e-12 * np.abs(rc).max(), f"N={N} M={M}"


def _args(B=1, K=8, M=4, **over):
    p = I.BrakeParams()
    assert I.load_library().isdf_brake_default_params(None, C.byref(p)) == 0
    p.candidates, p.pieces = K, M
    for k, v in over.items():
        setattr(p, k, v)
    return p


def test_default_params():
    lib = I.load_library()
    p = I.BrakeParams()
    assert lib.isdf_brake_default_params(None, C.byref(p)) == 0
    cp, dp = I.CertifyParams(), I.DynamicsParams()
    lib.isdf_certify_default_params(C.byref(cp))
    lib.isdf_dynamics_default_params(None, C.byref(dp))
    assert (p.candidates, p.pieces, list(p.reserved_)) == (8, 4, [0, 0]) and I.BRAKE_MAX_PIECES == 64
    assert bytes(p.certify) == bytes(cp) and bytes(p.dynamics) == bytes(dp)
    assert lib.isdf_brake_default_params(None, None) == -1


def test_argument_checks_without_a_device():
    """refusals that come before any device work: a NULL context or pointer, and every summary poisoned"""
    lib = I.load_library()
    off, T, Cc, ts = np.array([0, 1], dtype=np.int32), np.ones(1), np.zeros(18), np.ones(1)
    oo, oT, oC = np.zeros(2, dtype=np.int32), np.zeros(4), np.zeros(72)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    summ = (I.BrakeSummary * 1)()
    summ[0].status, summ[0].candidate = 7, 7
    p = _args()
    args = [None, 1, off.ctypes.data_as(ip), T.ctypes.data_as(dp), Cc.ctypes.data_as(dp), ts.ctypes.data_as(dp), C.byref(p),
            oo.ctypes.data_as(ip), oT.ctypes.data_as(dp), oC.ctypes.data_as(dp), summ]
    assert lib.isdf_trajectory_brake(*args) == -1
    s = summ[0]
    assert (s.status, s.candidate, s.certified, s.feasible) == (I.BRAKE_NONE, -1, -1, -1)
    assert math.isnan(s.tau_stop) and math.isnan(s.duration) and s.certify.verdict == 0 and math.isnan(s.certify.first_hit)
    assert s.dynamics.samples == -1 and math.isnan(s.dynamics.upper[0])
    dargs = [None, 1] + [a.ctypes.data for a in (off, T, Cc, ts)] + [C.byref(p)] + [a.ctypes.data for a in (oo, oT, oC)] + [C.addressof(summ), None]
    assert lib.isdf_trajectory_brake_device(*dargs) == -1


def test_struct_layouts_match_the_header():
    got = _probe([("isdf_brake_params", I.BrakeParams), ("isdf_brake_summary", I.BrakeSummary)])
    for cname, py in (("isdf_brake_params", I.BrakeParams), ("isdf_brake_summary", I.BrakeSummary)):
        size, offs = got[cname]
        assert size == C.sizeof(py) and offs == dict(_fields(py)), cname
    assert C.sizeof(I.BrakeSummary) == 256
