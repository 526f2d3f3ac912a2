"""CPU-only anchors of the exact restatement (tests/exact_oracle.py) the certificates are held to: its directed rounding against
math.nextafter and the correctly rounded sqrt, its pose and channels against the pinned restatements (certify_oracle.pose_at,
dynlimits_oracle.dense) and the reference-compiled FlatnessMap::forward golden, its body rate against a finite difference of R(z(t)), and
its extrema against the polynomial maxima of dynlimits_oracle."""
import math
import os
import sys
from fractions import Fraction as Fr
import numpy as np
import mpmath as mp
from mpmath import mpf
import isdf_b200 as I
import exact_oracle as E
import certify_oracle as CE
import dynlimits_oracle as DO
import vehicles as VH

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flat_forward_reference.npz")
DMAX = sys.float_info.max


def doubles(seed, n=3000):
    rng = np.random.default_rng(seed)
    m = rng.uniform(1, 2, n) * rng.choice([-1, 1], n)
    x = [float(v) for v in np.ldexp(m, rng.integers(-1074, 1023, n))]
    return x + [5e-324, -5e-324, 2.2250738585072014e-308, math.nextafter(2.2250738585072014e-308, 0), 1.0, -1.0, DMAX, -DMAX,
                math.nextafter(DMAX, 0), 0.1, 1 / 3]


def test_directed_rounding_against_nextafter():
    for x in doubles(1):
        if math.isinf(x) or x == 0:
            continue
        up = math.nextafter(x, math.inf)
        X = Fr(x)
        assert E.rd(X) == x and E.ru(X) == x
        if math.isinf(up):                       # beyond DBL_MAX: RD stays, RU overflows
            q = X + Fr(1, 2 ** 60) * X
            assert E.rd(q) == DMAX and E.ru(q) == math.inf
            assert E.rd(-q) == -math.inf and E.ru(-q) == -DMAX
            continue
        U = Fr(up)
        for f in (Fr(1, 3), Fr(1, 2), Fr(2 ** 60 - 1, 2 ** 60), Fr(1, 2 ** 70)):
            q = X + f * (U - X)
            assert E.rd(q) == x and E.ru(q) == up, (x, f)
            assert E.rd(-q) == -up and E.ru(-q) == -x
    # below the smallest subnormal
    t = Fr(1, 2 ** 1080)
    assert E.rd(t) == 0.0 and E.ru(t) == 5e-324 and E.rd(-t) == -5e-324 and E.ru(-t) == 0.0
    assert E.rd(0) == 0.0 and E.ru(0) == 0.0


def test_sqrt_rounding_brackets_the_correctly_rounded_root():
    for x in doubles(2):
        x = abs(x)
        if x == 0 or math.isinf(x):
            continue
        lo, hi, rn = E.sqrt_rd(Fr(x)), E.sqrt_ru(Fr(x)), math.sqrt(x)
        assert lo <= rn <= hi and (lo == rn or hi == rn)
        assert Fr(lo) ** 2 <= Fr(x) <= Fr(hi) ** 2
        assert hi == lo or hi == math.nextafter(lo, math.inf)
    for q in (Fr(2), Fr(1, 3), Fr(10 ** 40 + 1, 7), Fr(1, 2 ** 1074)):
        lo, hi = E.sqrt_rd(q), E.sqrt_ru(q)
        assert Fr(lo) ** 2 <= q < Fr(math.nextafter(lo, math.inf)) ** 2
        assert Fr(hi) ** 2 >= q > Fr(math.nextafter(hi, 0)) ** 2


def aggressive_pieces():
    g = 9.8
    out = []
    c = np.zeros((3, 6)); c[:, 0] = [1.0, 2.0, 3.0]; c[0, 1] = -1.0; c[0, 2] = 1.0
    out.append((1.0, c))
    c = np.zeros((3, 6)); c[0, 2] = 0.5 * g * math.tan(math.radians(80.0)); c[0, 3] = 40.0; c[1, 3] = -30.0; c[2, 1] = 1.0
    out.append((0.25, c))
    rng = np.random.default_rng(3)
    for k in range(4):
        out.append((0.6 + 0.2 * k, rng.normal(0, 1, (3, 6)) * np.array([5, 4, 3, 2, 1.5, 1.0])))
    return [(np.array([T]), c.reshape(-1)) for T, c in out]


def cfgs():
    out = [I.default_config_values(), VH.config("heavy")]
    nod = I.default_config_values()
    nod.horiz_drag = nod.vert_drag = nod.paras_drag = 0.0
    out.append(nod)
    return out


def test_pose_and_channels_agree_with_the_pinned_restatements():
    import workloads as W
    pieces = aggressive_pieces()
    T4, C4, _ = W.make_trajectory(4, [0, 0, 0], [30, 30, 20], seed=7, jitter=0.3)
    n = 0
    for cfg in cfgs():
        fp = E.Flat.of_cfg(cfg)
        for T, Cc in pieces + [(T4, C4)]:
            N = len(T)
            for i in range(N):
                t = np.linspace(0.0, T[i], 7)
                pos, R = CE.pose_at(cfg, T, Cc, np.full(t.size, i), t)
                dense, _ = DO.dense(cfg, T, Cc, i, t)
                c = E.piece(Cc, N, i)
                for k, tk in enumerate(t):
                    x, v, a, j = E.state(c, tk)
                    assert max(abs(float(x[ax]) - pos[k, ax]) for ax in range(3)) <= 1e-12 * max(1.0, np.abs(pos[k]).max())
                    att = E.attitude(fp, v, a)
                    assert np.abs(np.array([[float(e) for e in row] for row in att[1]]) - R[k]).max() <= 1e-12
                    ch = E.channels(fp, v, a, j)
                    for q, nm in enumerate(("speed", "acc", "omega", "tilt", "thrust")):
                        ref = dense[k, q]
                        tol = 1e-9 if nm == "tilt" else 1e-12      # the reference's tilt is acos of a quaternion product
                        assert abs(float(ch[nm]) - ref) <= tol * max(1.0, abs(ref)), (nm, float(ch[nm]), ref)
                    n += 1
    assert n >= 100


def test_thrust_body_rate_and_tilt_equal_the_reference_compiled_golden():
    g = np.load(GOLDEN)
    for tag, drag in (("drag", True), ("nodrag", False)):
        cfg = I.default_config_values()
        if not drag:
            cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
        par = np.array([cfg.vehicle_mass, cfg.grav_acc, cfg.horiz_drag, cfg.vert_drag, cfg.paras_drag, cfg.speed_eps])
        assert np.array_equal(par, g[f"{tag}_par"])
        fp = E.Flat.of_cfg(cfg)
        v, a, j, thr, omg, quat = (g[f"{tag}_{x}"] for x in ("v", "a", "j", "thr", "omg", "quat"))
        for k in range(0, len(thr), 4):
            ch = E.channels(fp, v[k], a[k], j[k])
            assert abs(float(ch["thrust"]) - thr[k]) <= 1e-12 * max(1.0, abs(thr[k]))
            assert abs(float(ch["omega"]) - np.linalg.norm(omg[k])) <= 1e-12 * max(1.0, np.linalg.norm(omg[k]))
            cz = 1 - 2 * (quat[k, 1] ** 2 + quat[k, 2] ** 2)
            assert abs(float(mp.cos(ch["tilt"])) - cz) <= 1e-12


def test_body_rate_is_the_derivative_of_the_attitude():
    """omega = vee(R^T dR/dt) for R(z(t)) along a piece, by a central difference at 60 digits"""
    for cfg in cfgs():
        fp = E.Flat.of_cfg(cfg)
        for T, Cc in aggressive_pieces()[1:4]:
            c = E.piece(Cc, 1, 0)
            for t in (mpf(T[0]) / 3, mpf(T[0]) * 0.71):
                eps = mpf(10) ** -25
                Rs = []
                for tt in (t - eps, t + eps):
                    _, v, a, _ = E.state(c, tt)
                    Rs.append(E.attitude(fp, v, a)[1])
                _, v, a, j = E.state(c, t)
                R = E.attitude(fp, v, a)[1]
                dR = [[(Rs[1][r][q] - Rs[0][r][q]) / (2 * eps) for q in range(3)] for r in range(3)]
                W = [[sum(R[k][r] * dR[k][q] for k in range(3)) for q in range(3)] for r in range(3)]   # R^T dR
                w = [W[2][1], W[0][2], W[1][0]]
                assert abs(E.norm(w) - E.channels(fp, v, a, j)["omega"]) <= mpf(10) ** -20


def test_polynomial_extrema_agree_with_roots_and_refinement():
    for T, Cc in aggressive_pieces():
        vm, am = DO.poly_max_va(T, Cc, 0)
        c = E.piece(Cc, 1, 0)
        P1 = [E.deriv_coeffs(c[ax], 1) for ax in range(3)]
        P2 = [E.deriv_coeffs(c[ax], 2) for ax in range(3)]
        mv, tv, _, _ = E.max_norm_poly(P1, 0, T[0])
        ma, ta, _, _ = E.max_norm_poly(P2, 0, T[0])
        assert abs(float(mv) - vm) <= 1e-12 * max(1.0, vm) and abs(float(ma) - am) <= 1e-12 * max(1.0, am)
        # the grid-and-golden-section search finds the same maximum of the speed
        gv, gt = E.extremum(lambda t: E.norm(E.state(c, t)[1]), 0, T[0])
        assert abs(gv - mv) <= mpf(10) ** -25 * max(1, mv)
