"""The certificates end to end on the GPU against the exact quantities they bound (tests/exact_oracle.py, mpmath at 60 digits), through
the library's own entry points and with no slack:

  * motion bound (isdf_dbg_certify_bound): D_e >= the exact largest displacement of the origin, and of body points |p| <= r along the
    singular directions of R(t) - R(t_e), for Ball, Box and the bench mesh, every interval kind, long pieces whose coefficients cancel
    and pieces near free fall
  * dynamic limits (isdf_trajectory_dynamics): upper >= the exact maximum, attained <= the exact value at its (piece, local time),
    thrust_lower <= the exact minimum; with each limit at exact max x (1 +- {1e-6, 1e-9, 1e-12}), FEASIBLE only when the exact maximum
    is within the limit and VIOLATING only when the exact value at the witness is past it
  * clearance (isdf_trajectory_certify), Ball and Point: grazing passes whose exact minimum is margin -+ delta at an irrational time
    between samples are never CERTIFIED / COLLIDING, and lower_bound <= the exact minimum
  * swept volume (isdf_swept_volume_sdf), Ball and Point: lower <= SV(p) exactly and value >= SV(p) - the rounding of one sampled SDF
    (SV_ROUND, stated below), at points 1e-9 .. 1e-3 from the swept surface and at the band edge
Each test prints the largest bound / exact ratio it met, a record of how tight the bounds are."""
import math
import numpy as np
import pytest
from mpmath import mpf
import isdf_b200 as I
import workloads as W
import exact_oracle as E

pytestmark = pytest.mark.gpu
BOX_HALF = [0.9, 0.5, 0.3]
PP = [0.0, 0.0, 0.0, 120.0, 0.0, 0.0]
# value is one sampled SDF, |p - x(t)| - r in FP64 round to nearest at |p|, |x| <= 40: a few dozen roundings of at most 40 * 2^-53 each
SV_ROUND = 1e-12


def single(c):
    return np.asarray(c, float).reshape(-1)


def long_piece():
    """T = 60: x = 1e-5 (t - 30)^5 + t expanded in t^k, y = -2e-6 (t - 45.25)^5, z = 5 + 0.01 t^2"""
    c = np.zeros((3, 6))
    for ax, (s, t0) in enumerate(((1e-5, 30.0), (-2e-6, 45.25))):
        c[ax] = [s * math.comb(5, k) * (-t0) ** (5 - k) for k in range(6)]
    c[0, 1] += 1.0
    c[2, 0], c[2, 2] = 5.0, 0.01
    return np.array([60.0]), single(c)


def near_free_fall(eps):
    """one piece, T = 0.5: a_z = -g + eps, a small sideways jerk"""
    c = np.zeros((3, 6))
    c[2, 0], c[2, 2] = 10.0, 0.5 * (-9.8 + eps)
    c[0, 3] = 0.2
    return np.array([0.5]), single(c)


# ---- 1. motion bound ----------------------------------------------------------------------------------------------------------------
def rot_lower_candidates(u, M, r):
    """body points p with |p| <= r (mpf vectors) where |u + M p| is largest in the directions that matter: +- r times each right
    singular vector of M (from float64; any unit direction is a valid candidate), and r (M^T u) / |M^T u|"""
    Mf = np.array([[float(x) for x in row] for row in M])
    _, _, Vt = np.linalg.svd(Mf)
    dirs = [Vt[k] for k in range(3)] + [-Vt[k] for k in range(3)]
    mu = Mf.T @ np.array([float(x) for x in u])
    if np.linalg.norm(mu) > 0:
        dirs.append(mu)
    out = []
    for d in dirs:
        dm = [mpf(float(x)) for x in d]
        n = E.norm(dm)
        if n > 0:
            out.append([x * (mpf(r) / n) for x in dm])
    return out


def displacement_lower(fp, c, te, t, r):
    """an attained displacement at time t from t_e: max over the candidates of |x(t) + R(t) p - x(t_e) - R(t_e) p|"""
    x0, v0, a0, _ = E.state(c, te)
    x1, v1, a1, _ = E.state(c, t)
    u = [x1[k] - x0[k] for k in range(3)]
    best = E.norm(u)
    if r > 0:
        A0, A1 = E.attitude(fp, v0, a0), E.attitude(fp, v1, a1)
        if A0 is None or A1 is None:
            return best
        M = [[A1[1][i][k] - A0[1][i][k] for k in range(3)] for i in range(3)]
        for p in rot_lower_candidates(u, M, r):
            w = [u[i] + sum(M[i][k] * p[k] for k in range(3)) for i in range(3)]
            best = max(best, E.norm(w))
    return best


def intervals_of(T, rng):
    piece, ta, tb = [], [], []
    for i in range(len(T)):
        for h in (T[i], T[i] / 16, T[i] / 64, 1e-6):
            a = float(rng.uniform(0, T[i] - h))
            for x, y in ((a, a + h), (T[i] - h, T[i]), (0.0, h)):
                piece.append(i); ta.append(x); tb.append(y)
    return piece, ta, tb


@pytest.mark.parametrize("shape", ["Ball", "Box", "bench_mesh"])
def test_motion_bound_against_exact_displacement(shape):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION
    ev = I.Evaluator(cfg)
    if shape == "Box":
        ev.set_shape_analytic(I.SHAPE_KINDS["BOX"], BOX_HALF)
    elif shape == "bench_mesh":
        V, F = W.rounded_cone_mesh(n_theta=24, n_prof=16)
        ev.set_shape_mesh(V, F, PP, I.MESH_SIGN_EXACT)
    else:
        ev.set_shape_named("Ball")
    fp = E.Flat.of_cfg(cfg)
    rng = np.random.default_rng(1)
    T4, C4, _ = W.make_trajectory(4, [0, 0, 0], [30, 30, 30], seed=6, jitter=0.4)
    cases = [(T4, C4), long_piece(), near_free_fall(1e-3), near_free_fall(0.0)]
    ratios, infinite = [], 0
    for T, Cc in cases:
        piece, ta, tb = intervals_of(T, rng)
        D, r = ev.dbg_certify_bound(T, Cc, 2.0, piece, ta, tb)
        N = len(T)
        for k in range(len(piece)):
            c = E.piece(Cc, N, piece[k])
            for e, te in enumerate((ta[k], tb[k])):
                if D[k, e] == math.inf:
                    infinite += 1
                    continue
                assert math.isfinite(D[k, e]), (k, e, D[k, e])
                Dm = mpf(D[k, e])
                # the origin: exact sup over [ta, tb] of |x(t) - x(te)| (roots of its derivative)
                x0 = E.state(c, te)[0]
                P = [E.shift_poly(c[ax], x0[ax]) for ax in range(3)]
                mx, targ, _, _ = E.max_norm_poly(P, ta[k], tb[k])
                assert Dm >= mx, (shape, k, e, D[k, e], mx)
                # body points within r: a time grid, the translation's argmax, and the singular directions of Delta R there
                best = mx
                for t in [mpf(ta[k]) + (mpf(tb[k]) - mpf(ta[k])) * q / 12 for q in range(13)] + [targ]:
                    best = max(best, displacement_lower(fp, c, mpf(te), t, r))
                assert Dm >= best, (shape, k, e, D[k, e], best)
                if best > 0:
                    ratios.append(float(Dm / best))
    assert ratios
    assert infinite >= 1     # the free-fall piece: |zu| vanishes, no finite bound
    print(f"    {shape}: r = {r:.4g}, {len(ratios)} finite bounds, D / exact displacement: median {np.median(ratios):.4g}, max "
          f"{max(ratios):.4g}, min {min(ratios):.12g}; {infinite} infinite")
    ev.close()


# ---- 2. dynamic limits ------------------------------------------------------------------------------------------------------------
NAMES = ("speed", "acc", "omega", "tilt", "thrust")
LIMIT_FIELD = ("vmax", "amax", "omgmax", "thetamax", "thrust_max")


def speed_bump(V0, A):
    c = np.zeros((3, 6))
    c[0, 1], c[0, 2], c[0, 3], c[0, 4] = V0, 0.25 * A, -0.5 * A, 0.25 * A
    c[2, 0] = 5.0
    return np.array([1.0]), single(c)


def jerk_bump(B, T):
    c = np.zeros((3, 6))
    c[1, 4], c[1, 5] = -B * T / 24.0, B / 60.0
    c[2, 0] = 5.0
    return np.array([T]), single(c)


def dyn_pieces():
    out = [("speed_bump", *speed_bump(9.5, 30.0)), ("jerk_bump", *jerk_bump(-600.0 / 0.04 ** 2, 0.04))]
    g = 9.8
    c = np.zeros((3, 6)); c[0, 2] = 0.5 * g * math.tan(math.radians(80.0)); c[0, 3] = 40.0; c[1, 3] = -30.0; c[2, 1] = 1.0
    out.append(("tilt80", np.array([0.25]), single(c)))
    rng = np.random.default_rng(3)
    for k in range(3):
        out.append((f"random{k}", np.array([0.6 + 0.2 * k]), single(rng.normal(0, 1, (3, 6)) * np.array([5, 4, 3, 2, 1.5, 1.0]))))
    return out


class Piece:
    """exact channel values of one piece, memoised by time"""

    def __init__(self, fp, Cc):
        self.fp, self.c, self.memo = fp, E.piece(Cc, 1, 0), {}

    def at(self, t):
        t = mpf(t)
        if t not in self.memo:
            _, v, a, j = E.state(self.c, t)
            self.memo[t] = E.channels(self.fp, v, a, j)
        return self.memo[t]

    def extrema(self, T):
        """exact max per channel and the thrust minimum"""
        c = self.c
        mv = E.max_norm_poly([E.deriv_coeffs(c[ax], 1) for ax in range(3)], 0, T)[0]
        ma = E.max_norm_poly([E.deriv_coeffs(c[ax], 2) for ax in range(3)], 0, T)[0]
        mo = E.extremum(lambda t: self.at(t)["omega"], 0, T)[0]
        mt = E.extremum(lambda t: self.at(t)["tilt"], 0, T)[0]
        mth = E.extremum(lambda t: self.at(t)["thrust"], 0, T)[0]
        mnth = -E.extremum(lambda t: -self.at(t)["thrust"], 0, T)[0]
        return [mv, ma, mo, mt, mth], mnth


def check_summary(P, s, mx, mn):
    """upper >= exact max, attained <= the exact value at its time, thrust_lower <= exact min <= the exact thrust at its witness"""
    ratios = {}
    for q, nm in enumerate(NAMES):
        assert mpf(s["upper"][q]) >= mx[q], (nm, s["upper"][q], mx[q])
        assert mpf(s["attained"][q]) <= P.at(s["t_attained"][q])[nm], (nm, s["attained"][q])
        if mx[q] > 0:
            ratios[nm] = float(mpf(s["upper"][q]) / mx[q])
    assert mpf(s["thrust_lower"]) <= mn
    assert mpf(s["thrust_attained_min"]) >= P.at(s["t_thrust_attained_min"])["thrust"]
    return ratios


@pytest.mark.parametrize("vehicle", ["default", "heavy", "nodrag_veps0"])
def test_dynamic_limits_against_exact_extrema(vehicle):
    import vehicles as VH
    if vehicle == "heavy":
        cfg = VH.config("heavy")
    else:
        cfg = I.default_config_values()
        if vehicle == "nodrag_veps0":
            cfg.horiz_drag = cfg.vert_drag = 0.0
            cfg.paras_drag, cfg.speed_eps = 0.05, 0.0      # parasitic drag alone, s = |v| reaches 0 at rest
    fp = E.Flat.of_cfg(cfg)
    ev = I.Evaluator(cfg, device=0)
    off = dict(vmax=math.inf, amax=math.inf, omgmax=math.inf, thetamax=math.inf, thrust_max=math.inf, thrust_min=-math.inf)
    worst = {}
    decided = dict(feasible=0, violating=0, undecided=0)
    for name, T, Cc in dyn_pieces():
        P = Piece(fp, Cc)
        mx, mn = P.extrema(T[0])
        s = ev.trajectory_dynamics(T, Cc, K=8, max_depth=24, max_samples=4000, **off)[0]
        for nm, x in check_summary(P, s, mx, mn).items():
            worst[nm] = max(worst.get(nm, 0.0), x)
        # adversarial limits around the exact extremum, one channel at a time
        for q, field in enumerate(LIMIT_FIELD + ("thrust_min",)):
            ex = mx[q] if q < 5 else mn
            if q in (0, 1, 2) and ex == 0:
                continue
            for rel in (1e-6, 1e-9, 1e-12):
                for sgn in (1, -1):
                    lim = float(ex * (1 + sgn * rel)) if q < 5 else float(ex - sgn * rel * abs(ex))
                    kw = dict(off)
                    kw[field] = lim
                    s =ev.trajectory_dynamics(T, Cc, K=8, max_depth=30, max_samples=4000, **kw)[0]
                    check_summary(P, s, mx, mn)
                    if s["verdict"] == I.FEASIBLE:
                        decided["feasible"] += 1
                        assert (mx[q] <= mpf(lim)) if q < 5 else (mn >= mpf(lim)), (name, field, lim, ex)
                    elif s["verdict"] == I.VIOLATING:
                        decided["violating"] += 1
                        assert s["violated"] == 1 << q, (name, field, s["violated"])
                        if q < 5:
                            assert P.at(s["t_attained"][q])[NAMES[q]] > mpf(lim), (name, field, lim)
                        else:
                            assert P.at(s["t_thrust_attained_min"])["thrust"] < mpf(lim), (name, field, lim)
                    else:
                        decided["undecided"] += 1
    print(f"    {vehicle}: upper / exact max per channel (largest): {{{', '.join(f'{k}: {v:.6g}' for k, v in worst.items())}}}; "
          f"adversarial verdicts {decided}")
    assert decided["feasible"] > 0 and decided["violating"] > 0
    ev.close()


def test_dynamic_limits_multi_piece_bounds():
    cfg = I.default_config_values()
    fp = E.Flat.of_cfg(cfg)
    ev = I.Evaluator(cfg, device=0)
    for seed in (5, 6):
        T, Cc, _ = W.make_trajectory(5, [0, 0, 0], [30, 30, 20], seed=seed, piece_time=1.2, jitter=0.3)
        s = ev.trajectory_dynamics(T, Cc, K=8, max_depth=20, max_samples=4000, vmax=math.inf, amax=math.inf, omgmax=math.inf,
                                   thetamax=math.inf, thrust_max=math.inf, thrust_min=-math.inf)[0]
        N = len(T)
        for i in range(N):
            c = E.piece(Cc, N, i)
            mv = E.max_norm_poly([E.deriv_coeffs(c[ax], 1) for ax in range(3)], 0, T[i])[0]
            ma = E.max_norm_poly([E.deriv_coeffs(c[ax], 2) for ax in range(3)], 0, T[i])[0]
            assert mpf(s["upper"][0]) >= mv and mpf(s["upper"][1]) >= ma

            def ch(t, nm):
                _, v, a, j = E.state(c, t)
                return E.channels(fp, v, a, j)[nm]
            for q, nm in ((2, "omega"), (3, "tilt"), (4, "thrust")):
                assert mpf(s["upper"][q]) >= E.extremum(lambda t: ch(t, nm), 0, T[i], n=24)[0], (seed, i, nm)
            assert mpf(s["thrust_lower"]) <= -E.extremum(lambda t: -ch(t, "thrust"), 0, T[i], n=24)[0]
    ev.close()


# ---- 3. clearance: grazing passes ---------------------------------------------------------------------------------------------------
def grazing(dy, s=3.1, T=2.0):
    """one piece: x = 4 + s t^2, y = 12.5 + dy, z = 12.5; the voxel centre (12.5, 12.5, 12.5) is passed at t* = sqrt(8.5 / s), irrational"""
    c = np.zeros((3, 6))
    c[0, 0], c[0, 2] = 4.0, s
    c[1, 0] = 12.5 + dy
    c[2, 0] = 12.5
    return np.array([T]), single(c)


@pytest.mark.parametrize("shape,radius", [("Ball", 1.0), ("Point", 0.0)])
def test_grazing_clearance_never_certified_or_colliding_wrongly(shape, radius):
    cfg = I.default_config_values()
    cfg.flags = I.WITH_COLLISION
    occ = np.zeros((24, 24, 24), np.uint8)
    occ[12, 12, 12] = 1
    ev = I.Evaluator(cfg)
    ev.set_map_u8(occ, [0, 0, 0], 1.0)
    ev.set_shape_named(shape)
    reach, margin, K = 2.0, 0.5, 8
    out = []
    for delta in (1e-4, 1e-8, 1e-11):
        for sgn in (-1, 1):
            dyf = 12.5 + (radius + margin + sgn * delta)          # the centre line's y, as a double
            T, Cc = grazing(dyf - 12.5)
            y = Cc[6]                                            # the y coefficient c_0 actually used
            exact = abs(mpf(y) - mpf(12.5)) - radius             # the exact minimum clearance, attained at t*
            assert (exact < margin) == (sgn < 0)
            s = ev.trajectory_certify(T, Cc, K, reach, margin, max_depth=40, max_samples=100000)[0]
            assert mpf(s["lower_bound"]) <= exact, (shape, delta, sgn, s)
            if sgn < 0:
                assert s["verdict"] != I.CERTIFIED, (shape, delta, s)
            else:
                assert s["verdict"] != I.COLLIDING, (shape, delta, s)
            out.append((delta, sgn, s["verdict"], s["samples"]))
    print(f"    {shape}: (delta, side, verdict, samples) {out}")
    ev.close()


# ---- 4. swept volume --------------------------------------------------------------------------------------------------------------
class SweptExact:
    """SV(p) = min over t of |p - x(t)| - radius, exactly: the roots of d/dt |x(t) - p|^2 on every piece that can hold the minimum.
    A piece is skipped only when a 64-cell sample of it, less its largest speed times half a cell (and 1e-6 for the samples' rounding),
    stays above the exact minimum found so far."""

    def __init__(self, T, Cc, radius, cells=64):
        self.T, self.N, self.radius = T, len(T), radius
        self.c = [E.piece(Cc, self.N, i) for i in range(self.N)]
        self.vmax = [float(E.max_norm_poly([E.deriv_coeffs(ci[ax], 1) for ax in range(3)], 0, T[i])[0]) for i, ci in enumerate(self.c)]
        cf = np.asarray(Cc, float).reshape(3, self.N, 6)
        self.ts = [np.linspace(0, T[i], cells + 1) for i in range(self.N)]
        self.xs = [np.stack([np.polynomial.polynomial.polyval(self.ts[i], cf[ax, i]) for ax in range(3)], 1) for i in range(self.N)]
        self.half = [0.5 * T[i] / cells for i in range(self.N)]

    def __call__(self, p):
        lb = [float(np.linalg.norm(self.xs[i] - p, axis=1).min()) - self.vmax[i] * self.half[i] - 1e-6 for i in range(self.N)]
        best = None
        for i in np.argsort(lb):
            if best is not None and lb[i] > best:
                continue
            P = [E.shift_poly(self.c[i][ax], mpf(float(p[ax]))) for ax in range(3)]
            mn = E.max_norm_poly(P, 0, self.T[i])[2]
            best = mn if best is None else min(best, mn)
        return best - self.radius


@pytest.mark.parametrize("shape,radius", [("Ball", 1.0), ("Point", 0.0)])
def test_swept_volume_encloses_the_exact_field(shape, radius):
    cfg = I.default_config_values()
    ev = I.Evaluator(cfg)
    ev.set_shape_named(shape)
    T, Cc, _ = W.make_trajectory(3, [2, 2, 2], [14, 12, 10], seed=8, jitter=0.3, piece_time=1.5)
    p = ev.swept_params()
    band = p.band
    rng = np.random.default_rng(2)
    N = len(T)
    pts = []
    for _ in range(12):
        i = int(rng.integers(N))
        t = float(rng.uniform(0, T[i]))
        c = E.piece(Cc, N, i)
        x, v, _, _ = E.state(c, t)
        vf = np.array([float(w) for w in v])
        u = np.cross(vf, rng.normal(size=3))                      # perpendicular to the velocity: the surface point nearest is x(t)
        u /= np.linalg.norm(u)
        xf = np.array([float(w) for w in x])
        for d in (1e-9, -1e-9, 1e-6, -1e-6, 1e-3, -1e-3):
            pts.append(xf + (radius + d) * u if radius + d > 0 else xf + d * u)
        for d in (band - 1e-9, band + 1e-9, band - 1e-3):          # the band edge
            pts.append(xf + (radius + d) * u)
    pts = np.array(pts)
    value, lower, tstar, dec = ev.swept_volume_sdf(T, Cc, pts, p)
    gap = []
    sv = SweptExact(T, Cc, radius)
    for k, q in enumerate(pts):
        ex = sv(q)
        assert mpf(lower[k]) <= ex, (k, lower[k], ex)
        assert mpf(value[k]) >= min(ex, mpf(band)) - SV_ROUND, (k, value[k], ex)
        gap.append(float(min(ex, mpf(band)) - mpf(lower[k])))
    print(f"    {shape}: {len(pts)} points, SV - lower: max {max(gap):.3g}, median {np.median(gap):.3g}; decided {int(dec.sum())}")
    ev.close()
