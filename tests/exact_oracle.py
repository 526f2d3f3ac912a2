"""Exact restatement of what the certificates bound — TEST INFRASTRUCTURE for test_gpu_interval_exact.py and test_gpu_certify_exact.py.

The certificates (include/isdf.h: isdf_trajectory_certify, isdf_trajectory_dynamics, isdf_swept_volume_sdf) claim proven bounds of
real-valued quantities. certify_oracle.py and dynlimits_oracle.py restate their algorithms in round-to-nearest FP64; this module
restates the quantities themselves, with nothing rounded that a claim depends on:

  rd(q), ru(q)               a rational (fractions.Fraction) rounded down / up to a double: subnormals, and overflow to +-inf exactly as
                             IEEE directed rounding does it (RD of a value above DBL_MAX is DBL_MAX, RU is +inf)
  sqrt_rd(q), sqrt_ru(q)     the neighbouring doubles of the square root of a rational (integer square root, then exact squares)
  X, ext_*                   extended reals: a Fraction, or the float +-inf
  pose / vaj / zu / R(z)     mpmath at DPS digits: x(t) and its derivatives from the piece polynomial, the flatness map
                             zu = a + dh_over_m kap v + g e_z, z = zu / |zu| and R(z) of the zero-yaw attitude as include/isdf.h writes it
  channels(fp, v, a, j)      |v|, |a|, |omega|, tilt, thrust at one state (omega: the zero-yaw attitude's body rate, the time
                             derivative of R(z) restated through dz; the CPU test holds it to the reference-compiled flatness map and to a
                             finite difference of R)
  max_norm_poly(P, ta, tb)   the exact maximum (and minimum) over [ta, tb] of |P(t)| for a vector polynomial P: the interval ends and the
                             real roots of d/dt |P|^2 (mpmath.polyroots)
  extremum(f, ta, tb)        max of a smooth scalar f over [ta, tb]: a grid, then golden-section refinement in every cell that brackets a
                             local maximum

A double end is compared with an mpf exactly (mpf(double) is exact at this precision). Every value these functions return is either
exact (rationals) or within 10^-(DPS-5) relative of the exact real, far below one ulp of a double."""
import math
import sys
from fractions import Fraction as Fr
import mpmath as mp
from mpmath import mpf

DPS = 60
mp.mp.dps = DPS
DBL_MAX = sys.float_info.max
INF = math.inf


# ---- directed rounding of rationals -------------------------------------------------------------------------------------------------
def rd(q):
    """the largest double <= q (q a Fraction or int); -inf below -DBL_MAX"""
    q = Fr(q)
    if q == 0:
        return 0.0
    try:
        f = q.numerator / q.denominator          # correctly rounded to nearest (CPython's integer true division)
    except OverflowError:
        return DBL_MAX if q > 0 else -INF
    if Fr(f) > q:
        f = math.nextafter(f, -INF)
    return f


def ru(q):
    """the smallest double >= q; +inf above DBL_MAX"""
    return -rd(-Fr(q))


def _isqrt_floor(q, bits=160):
    """a Fraction F with F <= sqrt(q) < F + 2^-bits sqrt(q) (roughly), q > 0"""
    n, d = q.numerator, q.denominator
    k = max(0, (2 * bits - (n * d).bit_length()) // 2 + 1)
    return Fr(math.isqrt(n * d * 4 ** k), d * 2 ** k)


def sqrt_rd(q):
    """the largest double f >= 0 with f^2 <= q (q >= 0)"""
    q = Fr(q)
    if q <= 0:
        return 0.0
    f = rd(_isqrt_floor(q))
    while Fr(math.nextafter(f, INF)) ** 2 <= q:
        f = math.nextafter(f, INF)
    while f > 0 and Fr(f) ** 2 > q:
        f = math.nextafter(f, -INF)
    return f


def sqrt_ru(q):
    """the smallest double f >= 0 with f^2 >= q (q >= 0); +inf when no finite double is large enough"""
    q = Fr(q)
    if q <= 0:
        return 0.0
    f = sqrt_rd(q)
    if Fr(f) ** 2 < q:
        f = math.nextafter(f, INF)
    return f


# ---- extended reals: a Fraction or +-inf ----------------------------------------------------------------------------------------------
def X(x):
    """a double as an extended real"""
    return x if math.isinf(x) else Fr(x)


def ext_add(a, b):
    if isinstance(a, float) or isinstance(b, float):
        s = (a if isinstance(a, float) else 0.0) + (b if isinstance(b, float) else 0.0)
        assert s == s, "inf - inf"
        return s
    return a + b


def ext_mul(a, b):
    """set-based product: 0 * inf = 0 (the limit of the products inside the intervals)"""
    if a == 0 or b == 0:
        return Fr(0)
    if isinstance(a, float) or isinstance(b, float):
        return INF if (a > 0) == (b > 0) else -INF
    return a * b


def ext_div(a, b):
    """a / b for b > 0 (b may be +inf: a / inf = 0 for finite a)"""
    if isinstance(b, float):
        assert not isinstance(a, float), "inf / inf"
        return Fr(0)
    if isinstance(a, float):
        return a
    return a / b


def xrd(x):
    return x if isinstance(x, float) else rd(x)


def xru(x):
    return x if isinstance(x, float) else ru(x)


# ---- the pose and the flatness map in mpmath ------------------------------------------------------------------------------------------
def piece(coeffs, N, i):
    """(3, 6) t^k coefficients of piece i as mpf (coeffs: 6N x 3 column-major, as floats)"""
    flat = [float(x) for x in coeffs]
    return [[mpf(flat[6 * N * ax + 6 * i + k]) for k in range(6)] for ax in range(3)]


def deriv_coeffs(c, der):
    """t^k coefficients of the der-th derivative of one axis"""
    return [c[k] * math.perm(k, der) for k in range(der, 6)]


def polyval(cs, t):
    r = mpf(0)
    for x in reversed(cs):
        r = r * t + x
    return r


def vaj(c, t):
    """position, v, a, j (lists of 3 mpf) of one piece at local time t"""
    t = mpf(t)
    return [[polyval(deriv_coeffs(c[ax], der), t) for ax in range(3)] for der in range(4)]


class Flat:
    """the flatness map's parameters: FlatParams {mass, grav, dh_over_m, cp, veps} and the thrust's mass and vert_drag"""

    def __init__(self, mass, grav, dh_over_m, cp, veps, dv=0.0):
        self.mass, self.grav, self.dh, self.cp, self.veps, self.dv = (mpf(float(x)) for x in (mass, grav, dh_over_m, cp, veps, dv))
        self.raw = (float(mass), float(grav), float(dh_over_m), float(cp), float(veps))
        self.dv_raw = float(dv)

    @staticmethod
    def of_cfg(cfg):
        return Flat(cfg.vehicle_mass, cfg.grav_acc, cfg.horiz_drag / cfg.vehicle_mass, cfg.paras_drag, cfg.speed_eps, cfg.vert_drag)


def dot(u, w):
    return u[0] * w[0] + u[1] * w[1] + u[2] * w[2]


def norm(u):
    return mp.sqrt(dot(u, u))


def flat(fp, v, a):
    """(s, kap, zu, n) at one state: s = sqrt(|v|^2 + veps), kap = 1 + cp s, zu = a + dh kap v + g e_z, n = |zu|"""
    v, a = [mpf(x) for x in v], [mpf(x) for x in a]
    s = mp.sqrt(dot(v, v) + fp.veps)
    kap = 1 + fp.cp * s
    zu = [a[k] + fp.dh * (kap * v[k]) for k in range(3)]
    zu[2] += fp.grav
    return s, kap, zu, norm(zu)


def rot_of_z(z):
    """R(z) of the zero-yaw attitude (include/isdf.h, certificate): rows of the 3 x 3 matrix"""
    zx, zy, zz = z
    op = 1 + zz
    return [[1 - zx * zx / op, -zx * zy / op, zx], [-zx * zy / op, 1 - zy * zy / op, zy], [-zx, -zy, zz]]


def attitude(fp, v, a):
    """(z, R(z)) at one state; None where |zu| or 1 + z_z vanishes"""
    _, _, zu, n = flat(fp, v, a)
    if n == 0:
        return None
    z = [w / n for w in zu]
    if 1 + z[2] == 0:
        return None
    return z, rot_of_z(z)


def channels(fp, v, a, j):
    """{speed, acc, omega, tilt, thrust} at one state; omega is None where |zu|, 1 + z_z (or s with cp != 0) vanishes, tilt and thrust
    None where |zu| does. s = 0 with cp != 0 takes lam v = 0, its limit."""
    v, a, j = [mpf(x) for x in v], [mpf(x) for x in a], [mpf(x) for x in j]
    s, kap, zu, n = flat(fp, v, a)
    out = dict(speed=norm(v), acc=norm(a), omega=None, tilt=None, thrust=None)
    if n == 0:
        return out
    z = [w / n for w in zu]
    F = [fp.mass * a[k] + fp.dv * (kap * v[k]) for k in range(3)]
    F[2] += fp.mass * fp.grav
    out["thrust"] = dot(z, F)
    out["tilt"] = mp.acos(max(min(z[2], mpf(1)), mpf(-1)))
    od = 1 + z[2]
    if od == 0:
        return out
    lamv = [mpf(0)] * 3 if (fp.cp == 0 or s == 0) else [fp.cp * dot(v, a) / s * v[k] for k in range(3)]
    xi = [j[k] + fp.dh * (kap * a[k] + lamv[k]) for k in range(3)]
    zxi = dot(z, xi)
    dz = [(xi[k] - z[k] * zxi) / n for k in range(3)]
    ot = dz[2] / od
    om = [-dz[1] + z[1] * ot, dz[0] - z[0] * ot, (z[1] * dz[0] - z[0] * dz[1]) / od]
    out["omega"] = norm(om)
    return out


def state(c, t):
    """(x, v, a, j) of one piece (c: piece()) at local time t"""
    return vaj(c, t)


# ---- extrema over a piece -----------------------------------------------------------------------------------------------------------
def _poly_mul(p, q):
    r = [mpf(0)] * (len(p) + len(q) - 1)
    for i, x in enumerate(p):
        for k, y in enumerate(q):
            r[i + k] += x * y
    return r


def _poly_add(p, q):
    n = max(len(p), len(q))
    return [(p[k] if k < len(p) else 0) + (q[k] if k < len(q) else 0) for k in range(n)]


def real_roots(cs, ta, tb):
    """real roots in [ta, tb] of the polynomial with t^k coefficients cs (mpf)"""
    cs = list(cs)
    while cs and cs[-1] == 0:
        cs.pop()
    if len(cs) <= 1:
        return []
    hi = [x for x in reversed(cs)]
    try:
        rts = mp.polyroots(hi, maxsteps=400, extraprec=100)
    except mp.libmp.libhyper.NoConvergence:
        rts = mp.polyroots(hi, maxsteps=2000, extraprec=1200, error=False)
    if not isinstance(rts, (list, tuple)):
        rts = [rts]
    scale = max(mpf(1), abs(mpf(ta)), abs(mpf(tb)))
    out = []
    for r in rts:
        r = mp.mpc(r)
        if abs(r.imag) <= mpf(10) ** (-DPS // 3) * scale:
            x = r.real
            if mpf(ta) <= x <= mpf(tb):
                out.append(x)
    return out


def max_norm_poly(P, ta, tb):
    """(max, argmax, min, argmin) over [ta, tb] of |P(t)|, P a list of 3 coefficient lists (t^k, mpf): ends and roots of d/dt |P|^2"""
    sq = [mpf(0)]
    for ax in range(3):
        sq = _poly_add(sq, _poly_mul(P[ax], P[ax]))
    d = [sq[k] * k for k in range(1, len(sq))]
    cand = [mpf(ta), mpf(tb)] + real_roots(d, ta, tb)
    vals = [(mp.sqrt(max(polyval(sq, t), mpf(0))), t) for t in cand]
    mx = max(vals, key=lambda x: x[0])
    mn = min(vals, key=lambda x: x[0])
    return mx[0], mx[1], mn[0], mn[1]


def shift_poly(cs, c0):
    """t^k coefficients of P(t) - c0 (constant term shifted)"""
    out = list(cs)
    out[0] = out[0] - c0
    return out


def golden_max(f, a, b, iters=90):
    """the maximum of a unimodal f on [a, b] (golden section; the bracket shrinks by 0.618 per step)"""
    a, b = mpf(a), mpf(b)
    g = (mp.sqrt(5) - 1) / 2
    x1, x2 = b - g * (b - a), a + g * (b - a)
    f1, f2 = f(x1), f(x2)
    for _ in range(iters):
        if f1 < f2:
            a, x1, f1 = x1, x2, f2
            x2 = a + g * (b - a)
            f2 = f(x2)
        else:
            b, x2, f2 = x2, x1, f1
            x1 = b - g * (b - a)
            f1 = f(x1)
    return (f1, x1) if f1 >= f2 else (f2, x2)


def extremum(f, ta, tb, n=48, iters=90):
    """(max, argmax) of f over [ta, tb]: the ends, an n-cell grid and golden-section refinement of every grid local maximum"""
    ta, tb = mpf(ta), mpf(tb)
    ts = [ta + (tb - ta) * k / n for k in range(n + 1)]
    fs = [f(t) for t in ts]
    best = max(zip(fs, ts), key=lambda x: x[0])
    for k in range(n + 1):
        if (k == 0 or fs[k] >= fs[k - 1]) and (k == n or fs[k] >= fs[k + 1]):
            lo, hi = ts[max(k - 1, 0)], ts[min(k + 1, n)]
            if hi > lo:
                cand = golden_max(f, lo, hi, iters)
                if cand[0] > best[0]:
                    best = cand
    return best
