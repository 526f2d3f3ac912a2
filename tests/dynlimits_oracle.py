"""Serial FP64 restatement of the dynamic-limit certificate (include/isdf.h, isdf_trajectory_dynamics) — TEST INFRASTRUCTURE.

  enclose(cfg, c, te, h)        (lo, hi) of the six channels over |t - te| <= h for pieces with coefficients c: the device's interval
                                algorithm (Taylor re-expansion, then the flatness map in interval arithmetic), in round-to-nearest
  point(cfg, c, t) / bound(...) the sample and interval forms the rounds use
  certify(cfg, T, coeffs, p)    the rounds (folds, split rule, per-trajectory budgets, leaves) and the summaries
  dense(cfg, T, coeffs, i, t)   the reference values: v, a, j from the polynomial in np.longdouble, omega and the quaternion from the
                                reference-compiled flatness map (oracle_lib.RefFlat), the thrust from thrust_exact
  thrust_exact(cfg, v, a)       FlatnessMap::forward's thrust in np.longdouble, held to the reference-compiled golden
  poly_max_va(T, coeffs, i)     exact maxima of |v| and |a| over a piece from the roots of d/dt |v|^2 and d/dt |a|^2

Channels: 0 |v|, 1 |a|, 2 |omega|, 3 tilt, 4 thrust, 5 -thrust. The device rounds every operation outward; here every operation rounds to
nearest, so the device's upper ends are never below these by more than a few ulps per operation."""
import math
import numpy as np
import oracle_lib as O

CH = 6
ACOS_PAD = 2.0 ** -49
BINOM = [[math.comb(m, k) for k in range(6)] for m in range(6)]
INF = math.inf


class Iv:
    """interval over numpy arrays, the device's operation structure without directed rounding"""

    def __init__(self, lo, hi=None):
        self.lo = np.asarray(lo, float)
        self.hi = self.lo if hi is None else np.asarray(hi, float)

    def __add__(a, b):
        b = b if isinstance(b, Iv) else Iv(b)
        return Iv(a.lo + b.lo, a.hi + b.hi)

    def __sub__(a, b):
        b = b if isinstance(b, Iv) else Iv(b)
        return Iv(a.lo - b.hi, a.hi - b.lo)

    def __neg__(a):
        return Iv(-a.hi, -a.lo)

    def __mul__(a, b):
        b = b if isinstance(b, Iv) else Iv(b)
        with np.errstate(invalid="ignore"):
            p = [a.lo * b.lo, a.lo * b.hi, a.hi * b.lo, a.hi * b.hi]
        return Iv(np.fmin(np.fmin(p[0], p[1]), np.fmin(p[2], p[3])), np.fmax(np.fmax(p[0], p[1]), np.fmax(p[2], p[3])))

    def sqr(a):
        m = np.fmax(np.abs(a.lo), np.abs(a.hi))
        n = np.where(a.lo > 0, a.lo, np.where(a.hi < 0, -a.hi, 0.0))
        return Iv(n * n, m * m)

    def divp(a, b):
        """a / b for b.lo > 0 (elsewhere the result is not used)"""
        with np.errstate(divide="ignore", invalid="ignore"):
            return Iv(np.where(a.lo >= 0, a.lo / b.hi, a.lo / b.lo), np.where(a.hi >= 0, a.hi / b.lo, a.hi / b.hi))

    def sqrt(a):
        with np.errstate(invalid="ignore"):
            return Iv(np.sqrt(np.fmax(a.lo, 0.0)), np.sqrt(a.hi))

    def mag(a):
        return np.fmax(np.abs(a.lo), np.abs(a.hi))

    def widen(a, r):
        return Iv(a.lo - r, a.hi + r)


def norm3(w):
    return (w[0].sqr() + w[1].sqr() + w[2].sqr()).sqrt()


def piece_coeffs(coeffs, N):
    """(N, 3, 6): t^k coefficients per piece and axis (coeffs: 6N x 3 column-major)"""
    return np.asarray(coeffs, float).reshape(3, N, 6).transpose(1, 0, 2)


def vaj(c, te, h):
    """enclosures (lists of 3 Iv) of v, a, j of pieces c (n, 3, 6) over |t - te| <= h"""
    te, h = np.asarray(te, float), np.asarray(h, float)
    hp = [np.ones_like(h)]
    for k in range(1, 5):
        hp.append(hp[-1] * h)
    tp = [Iv(np.ones_like(te))]
    for k in range(1, 6):
        tp.append(tp[-1] * Iv(te))
    v, a, j = [], [], []
    for ax in range(3):
        cc = c[:, ax, :]
        d = [None]
        for k in range(1, 6):
            s = Iv(np.zeros_like(te))
            for q in range(k, 6):
                s = s + (Iv(float(BINOM[q][k])) * Iv(cc[:, q])) * tp[q - k]
            d.append(s)
        vr = ar = jr = 0.0
        for k in range(2, 6):
            m = d[k].mag()
            vr = vr + (k * m) * hp[k - 1]
            if k >= 3:
                ar = ar + (k * (k - 1) * m) * hp[k - 2]
            if k >= 4:
                jr = jr + (k * (k - 1) * (k - 2) * m) * hp[k - 3]
        v.append(d[1].widen(vr))
        a.append((Iv(2.0) * d[2]).widen(ar))
        j.append((Iv(6.0) * d[3]).widen(jr))
    return v, a, j


def channels(cfg, v, a, j):
    """(lo, hi), each (n, 6), of |v|, |a|, |omega|, tilt, thrust, -thrust over the boxes v, a, j"""
    dhm, cp, veps, g = cfg.horiz_drag / cfg.vehicle_mass, cfg.paras_drag, cfg.speed_eps, cfg.grav_acc
    mass, dv = cfg.vehicle_mass, cfg.vert_drag
    n_ = v[0].lo.shape
    lo, hi = np.zeros(n_ + (CH,)), np.zeros(n_ + (CH,))
    sv = v[0].sqr() + v[1].sqr() + v[2].sqr()
    spd, acc = sv.sqrt(), norm3(a)
    lo[..., 0], hi[..., 0], lo[..., 1], hi[..., 1] = spd.lo, spd.hi, acc.lo, acc.hi
    s = (sv + Iv(veps)).sqrt()
    kap = Iv(1.0) + Iv(cp) * s
    zu, F = [], []
    for k in range(3):
        w = kap * v[k]
        zu.append(a[k] + Iv(dhm) * w)
        F.append(Iv(mass) * a[k] + Iv(dv) * w)
    zu[2] = zu[2] + Iv(g)
    F[2] = F[2] + Iv(mass) * Iv(g)
    n = norm3(zu)
    Fm = norm3(F).hi
    ok = n.lo > 0
    z = [zu[k].divp(n) for k in range(3)]
    th = z[0] * F[0] + z[1] * F[1] + z[2] * F[2]
    th_lo = np.where(ok, np.fmax(-Fm, th.lo), -Fm)
    th_hi = np.where(ok, np.fmin(Fm, th.hi), Fm)
    zl, zh = np.clip(z[2].lo, -1, 1), np.clip(z[2].hi, -1, 1)
    with np.errstate(invalid="ignore"):
        ti_lo = np.where(ok, np.arccos(zh) * (1 - ACOS_PAD), 0.0)
        ti_hi = np.where(ok, np.arccos(zl) * (1 + ACOS_PAD), math.pi * (1 + ACOS_PAD))
    od = Iv(1.0) + z[2]
    ok2 = ok & (od.lo > 0) & ((cp == 0.0) | (s.lo > 0))
    vda = v[0] * a[0] + v[1] * a[1] + v[2] * a[2]
    lam = Iv(np.zeros(n_)) if cp == 0.0 else (Iv(cp) * vda).divp(s)
    xi = [j[k] + Iv(dhm) * (kap * a[k] + lam * v[k]) for k in range(3)]
    zxi = z[0] * xi[0] + z[1] * xi[1] + z[2] * xi[2]
    dz = [(xi[k] - z[k] * zxi).divp(n) for k in range(3)]
    ot = dz[2].divp(od)
    om = [-dz[1] + z[1] * ot, dz[0] - z[0] * ot, (z[1] * dz[0] - z[0] * dz[1]).divp(od)]
    o = norm3(om)
    lo[..., 2], hi[..., 2] = np.where(ok2, o.lo, 0.0), np.where(ok2, o.hi, INF)
    lo[..., 3], hi[..., 3] = ti_lo, ti_hi
    lo[..., 4], hi[..., 4], lo[..., 5], hi[..., 5] = th_lo, th_hi, -th_hi, -th_lo
    return lo, hi


def enclose(cfg, c, te, h):
    return channels(cfg, *vaj(c, te, h))


def point(cfg, c, t):
    """lower ends (n, 6) of the point enclosures at local times t; rows NaN where v, a or j is not finite"""
    v, a, j = vaj(c, t, np.zeros_like(np.asarray(t, float)))
    with np.errstate(invalid="ignore", over="ignore"):
        fin = np.ones(np.shape(t), bool)
        for w in v + a + j:
            fin &= np.isfinite(w.lo + w.hi)
        lo, _ = channels(cfg, v, a, j)
    lo[~fin] = np.nan
    return lo


def bound(cfg, c, ta, tb):
    """upper ends (n, 6) of the interval enclosures over [ta, tb] about the midpoint; NaN reads +inf"""
    ta, tb = np.asarray(ta, float), np.asarray(tb, float)
    te = ta + 0.5 * (tb - ta)
    h = np.fmax(np.fmax(tb - te, te - ta), 0.0)
    with np.errstate(invalid="ignore", over="ignore"):
        _, hi = enclose(cfg, c, te, h)
    return np.where(np.isnan(hi), INF, hi)


def limits(p):
    lim = np.array([p.vmax, p.amax, p.omgmax, p.thetamax, p.thrust_max, -p.thrust_min], float)
    tol = np.array([p.tol_v, p.tol_a, p.tol_omg, p.tol_theta, p.tol_thrust, p.tol_thrust], float)
    return lim, tol


def _more(v, t, bv, bt):
    return v > bv or (v == bv and t < bt)


def certify(cfg, T, coeffs, p):
    """the rounds of include/isdf.h for every trajectory: (summaries as dicts like isdf_b200.DynamicsSummary.as_dict, leaves per
    trajectory as lists of (piece, ta, tb, depth, hi))"""
    T = np.asarray(T, float).reshape(-1)
    N = T.size
    N0 = p.pieces_per_traj or N
    K, M = p.samples_per_piece, p.max_samples_per_traj
    c = piece_coeffs(coeffs, N)
    lim, tol = limits(p)
    out, leaves_all = [], []
    for b in range(N // N0):
        pcs = range(b * N0, b * N0 + N0)
        toff, t = {}, 0.0
        for i in pcs:
            toff[i] = t
            t += T[i]
        smp_t, smp_p = [], []
        ivs = []
        for i in pcs:
            step = T[i] * (1.0 / K)
            base = len(smp_t)
            for jj in range(K + 1):
                smp_t.append(jj * step); smp_p.append(i)
            for jj in range(K):
                ivs.append((jj * step, T[i] if jj + 1 == K else (jj + 1) * step, base + jj, base + jj + 1, i, 0,
                            1 | (2 if jj + 1 == K else 0)))
        smp_q = list(point(cfg, c[np.array(smp_p)], np.array(smp_t)))
        up, att, tatt = [-INF] * CH, [-INF] * CH, [INF] * CH
        bad, used, und, dep = False, 0, 0, 0
        leaves = []
        while True:
            for (ta, tb, sa, sb, i, d, fl) in ivs:
                for s in ([sa] if fl & 1 else []) + ([sb] if fl & 2 else []):
                    ts = toff[smp_p[s]] + smp_t[s]
                    for ch in range(CH):
                        v = smp_q[s][ch]
                        if v != v:
                            bad = True
                        elif _more(v, ts, att[ch], tatt[ch]):
                            att[ch], tatt[ch] = v, ts
            if not ivs:
                break
            hi = bound(cfg, c[np.array([I[4] for I in ivs])], [I[0] for I in ivs], [I[1] for I in ivs])
            allowed = max(M - used, 0)
            nxt, new_t, new_p = [], [], []
            for k, (ta, tb, sa, sb, i, d, fl) in enumerate(ivs):
                h = hi[k]
                over = h > lim
                need = bool(np.any((over & (np.array(att) <= lim)) | (h > np.array(att) + tol)))
                m = ta + 0.5 * (tb - ta)
                wants = need and not bad and d < p.max_depth and ta < m < tb
                if wants and len(new_t) < allowed:
                    s = len(smp_t) + len(new_t)
                    new_t.append(m); new_p.append(i)
                    nxt.append((ta, m, sa, s, i, d + 1, 0))
                    nxt.append((m, tb, s, sb, i, d + 1, 1))
                else:
                    up = list(np.fmax(up, h))
                    und += bool(np.any(over))
                    dep = max(dep, d)
                    leaves.append((i - b * N0, ta, tb, d, h))
            used += len(new_t)
            if new_t:
                q = point(cfg, c[np.array(new_p)], np.array(new_t))
                smp_t += new_t; smp_p += new_p; smp_q += list(q)
            ivs = nxt
            if not new_t:
                break
        viol = sum(1 << ch for ch in range(CH) if att[ch] > lim[ch])
        undm = sum(1 << ch for ch in range(CH) if not att[ch] > lim[ch] and not up[ch] <= lim[ch])
        s = dict(upper=np.array(up[:5]), attained=np.array(att[:5]), t_attained=np.array(tatt[:5]), thrust_lower=-up[5],
                 thrust_attained_min=-att[5], t_thrust_attained_min=tatt[5], verdict=-1 if (bad or viol) else (1 if undm == 0 else 0),
                 violated=viol, undecided=0 if bad else undm, samples=N0 * (K + 1) + used, undecided_intervals=und, depth=dep)
        if bad:
            s["upper"][:] = np.nan; s["attained"][:] = np.nan; s["thrust_lower"] = s["thrust_attained_min"] = np.nan
        out.append(s)
        leaves_all.append(leaves)
    return out, leaves_all


# ---- dense references ----------------------------------------------------------------------------------------------------------
def vaj_exact(c, t):
    """v, a, j (n, 3) of one piece's coefficients c (3, 6) at times t, in np.longdouble"""
    t = np.asarray(t, np.longdouble)
    cl = np.asarray(c, np.longdouble)
    out = []
    for der in (1, 2, 3):
        r = np.zeros((t.size, 3), np.longdouble)
        for k in range(der, 6):
            f = np.longdouble(math.perm(k, der))
            r += (f * cl[:, k])[None, :] * (t[:, None] ** (k - der))
        out.append(r)
    return out


def thrust_exact(cfg, v, a):
    """the thrust of FlatnessMap::forward at psi = dpsi = 0 (flatness.hpp:150-207), z . (mass a + dv w + mass g e_z) with
    w = (1 + cp sqrt(|v|^2 + veps)) v and z = zu / |zu|, evaluated in np.longdouble; tests/golden/flat_forward_reference.npz holds what the
    reference-compiled function returns, and the CPU tests hold this restatement to it"""
    v, a = np.asarray(v, np.longdouble).reshape(-1, 3), np.asarray(a, np.longdouble).reshape(-1, 3)
    L = np.longdouble
    mass, g = L(cfg.vehicle_mass), L(cfg.grav_acc)
    w = (1 + L(cfg.paras_drag) * np.sqrt((v * v).sum(1) + L(cfg.speed_eps)))[:, None] * v
    zu = a + (L(cfg.horiz_drag) / mass) * w
    zu[:, 2] += g
    F = mass * a + L(cfg.vert_drag) * w
    F[:, 2] += mass * g
    return np.asarray((zu * F).sum(1) / np.sqrt((zu * zu).sum(1)), float)


def dense(cfg, T, coeffs, i, t):
    """(n, 5) of speed, acceleration (np.longdouble, as float), body rate (reference optimizated_forward), tilt (acos of the reference
    quaternion's 1 - 2 (q1^2 + q2^2)), thrust (thrust_exact), and cos(tilt), at local times t of piece i"""
    T = np.asarray(T, float).reshape(-1)
    c = piece_coeffs(coeffs, T.size)[i]
    v, a, j = vaj_exact(c, t)
    vd, ad, jd = (np.asarray(x, float) for x in (v, a, j))
    q, o = O.RefFlat(cfg).forward(vd, ad, jd)
    thr = thrust_exact(cfg, v, a)
    cz = 1 - 2 * (q[:, 1] ** 2 + q[:, 2] ** 2)
    vals = np.stack([np.asarray(np.sqrt((v * v).sum(1)), float), np.asarray(np.sqrt((a * a).sum(1)), float),
                     np.linalg.norm(o, axis=1), np.arccos(np.clip(cz, -1, 1)), thr], axis=1)
    return vals, cz


def poly_max_va(T, coeffs, i):
    """exact max over [0, T_i] of |v| and |a| of piece i: the endpoints and the real roots of d/dt |v|^2 = 2 v.a and d/dt |a|^2 = 2 a.j
    in [0, T_i], each root polished by Newton steps in np.longdouble"""
    T = np.asarray(T, float).reshape(-1)
    c = piece_coeffs(coeffs, T.size)[i]
    Ti = T[i]
    res = []
    for der in (1, 2):
        P = [np.polynomial.Polynomial(c[ax]).deriv(der) for ax in range(3)]
        D = sum(P[ax] * P[ax].deriv() for ax in range(3))
        cand = [0.0, Ti]
        for r in D.roots():
            if abs(r.imag) <= 1e-6 * max(1.0, abs(r.real)) and -1e-9 <= r.real <= Ti + 1e-9:
                x = np.longdouble(min(max(r.real, 0.0), Ti))
                dc = [np.longdouble(z) for z in D.coef]
                for _ in range(8):
                    f = sum(dc[k] * x ** k for k in range(len(dc)))
                    df = sum(k * dc[k] * x ** (k - 1) for k in range(1, len(dc)))
                    if df == 0:
                        break
                    x = x - f / df
                    x = min(max(x, np.longdouble(0.0)), np.longdouble(Ti))
                cand.append(x)
        vals = []
        for x in cand:
            v, a, _ = vaj_exact(c, [x])
            w = v if der == 1 else a
            vals.append(np.sqrt((w * w).sum()))
        res.append(float(max(vals)))
    return res[0], res[1]
