"""The certificates' interval arithmetic on the GPU against exact arithmetic: tests/interval_probe.cu runs csrc/isdf_interval.cuh,
isdf_certify.cuh and isdf_dynlimits.cuh unchanged, built twice (with FMA contraction, as the clearance unit is, and with -fmad=false),
and the two builds must agree to the bit.

  * primitives (iadd, isub, ineg, imul, isqr, idivp, iwiden): EQUAL to the exact result rounded down / up (fractions.Fraction), over
    signed zeros, subnormals, the smallest normal, DBL_MAX, overflowing and underflowing products, straddling, degenerate and one-ulp
    intervals, infinite ends; isqrt: the neighbouring doubles of the exact roots; the 0 * inf products imul's fmin / fmax drop
  * taylor_coeff / taylor_axis: the exact Taylor coefficients, displacement and derivatives of the piece polynomial inside the
    enclosures, at every h from 0 to 60 s and on long pieces whose coefficients cancel
  * flat_enclose, cert_rot, dyn_channels: the exact flatness map, attitude and the six channels (tests/exact_oracle.py, mpmath) at the
    corners and inside the boxes, near free fall, near inversion, through zero speed and at tilts near 0 and pi, on three vehicles
  * what the callers make of a result that is no bound: cert_bound reads a non-finite piece as +inf, dyn_bound never returns NaN,
    dyn_point makes the samples of a piece with non-finite v, a or j NaN (so the trajectory is VIOLATING with no bound reported)
No comparison here has a tolerance."""
import math
import os
import shutil
import subprocess
import sys
from fractions import Fraction as Fr
import numpy as np
import pytest
from mpmath import mpf
import exact_oracle as E
import vehicles as VH

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIN, POUT = 32, 48
TINY, NORM_MIN, DMAX = 5e-324, 2.2250738585072014e-308, sys.float_info.max
INF, NAN = math.inf, math.nan
OPS = dict(iadd=0, isub=1, ineg=2, imul=3, isqr=4, idivp=5, isqrt=6, iwiden=7, inorm=8, taylor=9, flat=10, rot=11, channels=12,
           cert_bound=13, dyn_bound=14, dyn_point=15)


def _unit_flags():
    """the clearance unit's nvcc flags (FMA contraction on), as build() compiles it"""
    sys.path.insert(0, ROOT)
    import __graft_entry__ as GE
    flags = [f for f in GE.NVCC_COMMON if f not in ("-Xcompiler", "-fPIC")]
    return flags + list(dict(GE.TUS)["isdf_clearance_tu.cu"])


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.fail("nvcc not available: the probe is compiled at test time")
    d = tmp_path_factory.mktemp("interval_probe")
    exes = []
    for tag, extra in (("fma", []), ("nofma", ["-fmad=false"])):
        exe = str(d / f"probe_{tag}")
        r = subprocess.run(["nvcc"] + _unit_flags() + extra + ["-o", exe, os.path.join(ROOT, "tests", "interval_probe.cu")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        exes.append(exe)

    def run(op, recs):
        recs = np.asarray(recs, dtype=np.float64)
        n = recs.shape[0]
        full = np.full((n, PIN), np.nan)
        full[:, :recs.shape[1]] = recs
        fin = str(d / "in.bin")
        full.tofile(fin)
        outs = []
        for exe in exes:
            fout = str(d / "out.bin")
            r = subprocess.run([exe, str(OPS[op]), fin, fout, str(n)], capture_output=True, text=True, timeout=300)
            assert r.returncode == 0 and "INTERVAL PROBE OK" in r.stdout, (r.stdout, r.stderr)
            outs.append(np.fromfile(fout, dtype=np.float64).reshape(n, POUT))
        assert outs[0].tobytes() == outs[1].tobytes(), f"{op}: FMA contraction changed a bit"
        return outs[0]
    return run


# ---- inputs ----------------------------------------------------------------------------------------------------------------------------
def edge_values():
    base = [0.0, TINY, 2 * TINY, 3 * TINY, NORM_MIN, math.nextafter(NORM_MIN, 0), math.nextafter(NORM_MIN, 1), 1e-300, 1.5e-162,
            1e-154, 1e-20, 1e-8, 0.1, 1 / 3, 0.5, 1.0, math.nextafter(1.0, 2), math.nextafter(1.0, 0), 2.0, 3.0, math.pi, 7.0, 1e8,
            2 ** 52 + 1, 1e20, 1e154, 1.4e154, 1e160, 1e300, math.nextafter(DMAX, 0), DMAX]
    return sorted(set(base + [-x for x in base] + [-0.0]), key=lambda x: (x, math.copysign(1, x)))


def random_doubles(rng, n, emin=-330, emax=310):
    m = rng.uniform(1, 2, n) * rng.choice([-1, 1], n)
    e = rng.integers(emin, emax, n).astype(float)
    with np.errstate(over="ignore", under="ignore"):
        x = np.ldexp(m, e.astype(int))
    return np.where(np.isfinite(x), x, np.sign(x) * DMAX)


def intervals(seed, n_random=1500, inf_ends=True):
    """(lo, hi) pairs: every ordered pair of edge values, one-ulp and degenerate intervals, random ones, infinite ends"""
    ev = edge_values()
    out = [(a, b) for i, a in enumerate(ev) for b in ev[i:] if a <= b]
    out += [(x, math.nextafter(x, INF)) for x in ev if x < DMAX] + [(x, x) for x in ev]
    rng = np.random.default_rng(seed)
    for x, y in zip(random_doubles(rng, n_random), random_doubles(rng, n_random)):
        out.append((min(x, y), max(x, y)))
    for x in rng.normal(0, 3, n_random // 3):
        out.append((x, x + abs(rng.normal(0, 1)) * 10.0 ** rng.integers(-16, 1)))
    if inf_ends:
        for x in (-DMAX, -1.0, -TINY, -0.0, 0.0, TINY, 1.0, DMAX):
            out += [(-INF, x), (x, INF)]
        out.append((-INF, INF))
    return out


def pairs(seed, k=6000):
    """pairs of intervals: edge x edge subsets, random, and the ones with infinite or zero ends together"""
    iv = intervals(seed)
    rng = np.random.default_rng(seed + 1)
    idx = rng.integers(0, len(iv), (k, 2))
    out = [(iv[i], iv[j]) for i, j in idx]
    special = [(0.0, 0.0), (-0.0, 0.0), (0.0, 1.0), (-1.0, 0.0), (-INF, INF), (1.0, INF), (-INF, -1.0), (0.0, INF), (-INF, 0.0), (TINY, TINY),
               (-DMAX, DMAX), (DMAX, DMAX), (1e200, 1e201), (1e-200, 1e-199)]
    out += [(a, b) for a in special for b in special]
    return out


# ---- 1. primitives, to the bit -------------------------------------------------------------------------------------------------------
def exact_add(a, b):
    return E.xrd(E.ext_add(E.X(a[0]), E.X(b[0]))), E.xru(E.ext_add(E.X(a[1]), E.X(b[1])))


def exact_sub(a, b):
    return E.xrd(E.ext_add(E.X(a[0]), -E.X(b[1]))), E.xru(E.ext_add(E.X(a[1]), -E.X(b[0])))


def exact_mul(a, b):
    p = [E.ext_mul(E.X(x), E.X(y)) for x in a for y in b]
    return E.xrd(min(p)), E.xru(max(p))


def test_add_sub_neg_exact(probe):
    P = pairs(1)
    recs = [(a[0], a[1], b[0], b[1]) for a, b in P]
    for op, f in (("iadd", exact_add), ("isub", exact_sub)):
        out = probe(op, recs)
        for k, (a, b) in enumerate(P):
            assert (out[k, 0], out[k, 1]) == f(a, b), (op, a, b, out[k, :2])
    iv = intervals(2)
    out = probe("ineg", iv)
    for k, (lo, hi) in enumerate(iv):
        assert (out[k, 0], out[k, 1]) == (-hi, -lo)
    print(f"    iadd / isub: {len(P)} pairs each, ineg: {len(iv)}")


def test_mul_exact_and_dropped_nan(probe):
    P = pairs(3)
    out = probe("imul", [(a[0], a[1], b[0], b[1]) for a, b in P])
    nan_cases = 0
    for k, (a, b) in enumerate(P):
        got = (out[k, 0], out[k, 1])
        if got[0] != got[0] or got[1] != got[1]:
            # fmin / fmax drop the NaN of 0 * inf; only when all four products are 0 * inf is nothing left: [0, 0] times an interval
            # with two infinite ends. Every caller reads such an end as "no bound" (test_non_finite_pieces_give_no_bound).
            assert all(math.isnan(x * y) for x in a for y in b), (a, b, got)
            nan_cases += 1
            continue
        assert got == exact_mul(a, b), (a, b, got, exact_mul(a, b))
    assert nan_cases >= 1
    print(f"    imul: {len(P)} pairs, {nan_cases} all-(0 x inf) NaN")


def test_sqr_and_widen_exact(probe):
    iv = intervals(4)
    out = probe("isqr", iv)
    for k, (lo, hi) in enumerate(iv):
        n = lo if lo > 0 else (-hi if hi < 0 else 0.0)
        m = max(abs(lo), abs(hi))
        exp = (E.xrd(E.ext_mul(E.X(n), E.X(n))), E.xru(E.ext_mul(E.X(m), E.X(m))))
        assert (out[k, 0], out[k, 1]) == exp, (lo, hi, out[k, :2], exp)
    rng = np.random.default_rng(5)
    rads = [0.0, TINY, NORM_MIN, 1e-300, 1e-16, 1.0, 1e300, DMAX, INF]
    recs = [(lo, hi, rads[rng.integers(len(rads))] if rng.random() < 0.5 else abs(float(random_doubles(rng, 1)[0]))) for lo, hi in iv]
    out = probe("iwiden", recs)
    for k, (lo, hi, r) in enumerate(recs):
        exp = (E.xrd(E.ext_add(E.X(lo), -E.X(r))), E.xru(E.ext_add(E.X(hi), E.X(r))))
        assert (out[k, 0], out[k, 1]) == exp, (lo, hi, r, out[k, :2])
    print(f"    isqr / iwiden: {len(iv)} records each")


def test_divp_exact(probe):
    iv = intervals(6)
    rng = np.random.default_rng(7)
    pos = [b for b in iv if b[0] > 0]
    pos += [(TINY, TINY), (TINY, 1.0), (2 * TINY, DMAX), (math.nextafter(NORM_MIN, 0), NORM_MIN), (TINY, INF), (1.0, INF)]   # b.lo subnormal
    recs = []
    for k in range(6000):
        a = iv[rng.integers(len(iv))]
        b = pos[rng.integers(len(pos))]
        recs.append((a[0], a[1], b[0], b[1]))
    out = probe("idivp", recs)
    for k, (alo, ahi, blo, bhi) in enumerate(recs):
        lo = E.ext_div(E.X(alo), E.X(bhi)) if alo >= 0 else E.ext_div(E.X(alo), E.X(blo))
        hi = E.ext_div(E.X(ahi), E.X(blo)) if ahi >= 0 else E.ext_div(E.X(ahi), E.X(bhi))
        assert (out[k, 0], out[k, 1]) == (E.xrd(lo), E.xru(hi)), (recs[k], out[k, :2])
        # and the rule is the hull of the exact quotients
        qs = [E.ext_div(E.X(x), E.X(y)) for x in (alo, ahi) for y in (blo, bhi) if not (math.isinf(x) and math.isinf(y))]
        if qs and not any(math.isinf(v) for v in (alo, ahi, bhi)):
            assert E.X(out[k, 0]) <= min(qs) and max(qs) <= E.X(out[k, 1])
    print(f"    idivp: {len(recs)} records")


def test_sqrt_neighbouring_doubles(probe):
    iv = intervals(8)
    out = probe("isqrt", iv)
    neg = 0
    for k, (lo, hi) in enumerate(iv):
        glo, ghi = out[k, 0], out[k, 1]
        x = max(lo, 0.0)
        if hi < 0:
            assert math.isnan(ghi), (lo, hi, ghi)      # no root: the upper end is NaN, which no caller reads as a bound
            neg += 1
            continue
        assert glo == E.sqrt_rd(E.X(x)) if not math.isinf(x) else glo == INF, (lo, hi, glo)
        if math.isinf(hi):
            assert ghi == INF
        else:
            assert ghi == E.sqrt_ru(Fr(hi)), (lo, hi, ghi)
            assert Fr(glo) ** 2 <= Fr(x) and Fr(hi) <= Fr(ghi) ** 2
    assert neg >= 10
    print(f"    isqrt: {len(iv)} records, {neg} with hi < 0")


def test_norm_contains_the_exact_range(probe):
    rng = np.random.default_rng(9)
    iv = intervals(10, n_random=300, inf_ends=False)
    recs = [sum((iv[i] for i in rng.integers(0, len(iv), 3)), ()) for _ in range(3000)]
    out = probe("inorm", recs)
    for k, r in enumerate(recs):
        w = [(r[2 * a], r[2 * a + 1]) for a in range(3)]
        n2 = sum(Fr(lo if lo > 0 else (-hi if hi < 0 else 0.0)) ** 2 for lo, hi in w)
        m2 = sum(max(Fr(abs(lo)), Fr(abs(hi))) ** 2 for lo, hi in w)
        lo, hi = out[k, 0], out[k, 1]
        assert Fr(lo) ** 2 <= n2 and lo >= 0, (w, lo)
        assert hi == INF or Fr(hi) ** 2 >= m2, (w, hi)


# ---- 2. Taylor form -----------------------------------------------------------------------------------------------------------------
def taylor_cases():
    rng = np.random.default_rng(11)
    out = []
    hs = [0.0, 1e-12, 1e-9, 1e-6, 1e-3, 0.05, 0.5, 2.0, 10.0, 60.0]
    for T in (0.3, 2.0, 60.0):
        for _ in range(4):
            c = rng.normal(0, 1, 6) * np.array([5, 4, 3, 2, 1.5, 1.0]) / np.maximum(1.0, T) ** np.arange(6)
            for te in (0.0, T, float(rng.uniform(0, T))):
                for h in hs:
                    out.append((list(c), te, h))
    # long pieces whose monomial coefficients cancel: s (t - t0)^5 expanded, and a sum of two such
    for t0, s in ((30.0, 1e-5), (59.5, 3e-7), (45.25, -2e-6)):
        c = [s * math.comb(5, k) * (-t0) ** (5 - k) for k in range(6)]
        for te in (0.0, t0, 60.0, float(rng.uniform(0, 60))):
            for h in (0.0, 1e-12, 1e-3, 1.0, 30.0, 60.0):
                out.append((c, te, h))
    return out


def exact_taylor(c, te):
    """exact d_k (k = 0..5) of sum c_q t^q about te"""
    cq, t = [Fr(x) for x in c], Fr(te)
    return [sum(math.comb(q, k) * cq[q] * t ** (q - k) for q in range(k, 6)) for k in range(6)]


def test_taylor_encloses_exact_coefficients_and_derivatives(probe):
    cases = taylor_cases()
    out = probe("taylor", [tuple(c) + (te, h) for c, te, h in cases])
    U = 64
    for k, (c, te, h) in enumerate(cases):
        y = out[k]
        d = exact_taylor(c, te)
        assert np.array_equal(y[:10], y[17:27])            # taylor_coeff alone is what taylor_axis reports
        for q in range(1, 6):
            assert Fr(y[2 * q - 2]) <= d[q] <= Fr(y[2 * q - 1]), (k, q)
        H = Fr(h)
        assert Fr(y[10]) >= sum(abs(d[q]) * H ** q for q in range(1, 6)), k
        encl = [(Fr(y[11]), Fr(y[12])), (Fr(y[13]), Fr(y[14])), (Fr(y[15]), Fr(y[16]))]
        dv = [q * d[q] for q in range(1, 6)]                 # p'(te + s) = sum_q q d_q s^(q-1)
        da = [q * (q - 1) * d[q] for q in range(2, 6)]
        dj = [q * (q - 1) * (q - 2) * d[q] for q in range(3, 6)]
        for u in range(U + 1):
            s = H * Fr(2 * u - U, U)                         # both ends and 63 dyadic times between
            for (lo, hi), poly in zip(encl, (dv, da, dj)):
                val = sum(x * s ** m for m, x in enumerate(poly))
                assert lo <= val <= hi, (k, c, te, h, u)
    print(f"    taylor: {len(cases)} records, {U + 1} times each")


# ---- 3. flatness enclosures against mpmath -----------------------------------------------------------------------------------------
def vehicles():
    cfgs = {"default": VH.I.default_config_values()}
    for tag in ("heavy", "hdrag_lowg"):
        cfgs[tag] = VH.config(tag)
    nod = VH.I.default_config_values()
    nod.horiz_drag = nod.vert_drag = nod.paras_drag = 0.0
    cfgs["nodrag"] = nod
    for veps in (0.0, 1e-4):
        c = VH.I.default_config_values()
        c.speed_eps = veps
        c.paras_drag = 0.2
        cfgs[f"cp0.2_veps{veps}"] = c
    return cfgs


def box_cases():
    """(cfg tag, v box, a box, j box); boxes as (lo, hi) per axis"""
    rng = np.random.default_rng(13)
    out = []

    def box(c, r):
        return [(float(x - rr), float(x + rr)) for x, rr in zip(c, np.broadcast_to(r, 3))]

    cfgs = vehicles()
    for tag, cfg in cfgs.items():
        g = cfg.grav_acc
        for rad in (0.0, 1e-12, 1e-6, 1e-3, 0.1):
            for _ in range(3):
                out.append((tag, box(rng.normal(0, 4, 3), rad), box(rng.normal(0, 4, 3), rad), box(rng.normal(0, 30, 3), rad)))
        dh = cfg.horiz_drag / cfg.vehicle_mass
        for eps in (0.0, 1e-9, 1e-4, 1e-1):
            # near free fall: |zu| -> 0 (v = 0: zu = a + g e_z)
            out.append((tag, box([0, 0, 0], 1e-6), box([eps, 0, -g], 1e-7), box([3, -2, 1], 0.5)))
            out.append((tag, box([0, 0, 0], 0.0), box([0, eps, -g + eps], 0.0), box([1, 1, 1], 0.0)))
            # near inversion: 1 + z_z -> 0 (zu pointing down)
            out.append((tag, box([0.1, 0, 0], 1e-6), box([eps, -eps, -2 * g - dh * 0.1], 1e-6), box([0, 5, 0], 1.0)))
            # tilt near 0 and near pi exactly on the axis
            out.append((tag, box([0, 0, 0], 0.0), box([eps, 0, 0], 0.0), box([0, 0, 0], 0.0)))
            out.append((tag, box([0, 0, 0], 0.0), box([eps, 0, -3 * g], 0.0), box([0, 0, 0], 0.0)))
            # level thrust axis: z_z = 0 exactly, tilt exactly pi / 2 (acos(0) in double is below it)
            out.append((tag, box([0, 0, 0], 0.0), box([5 * eps + 1e-3, 0, -g], 0.0), box([0, 1, 0], 0.0)))
        # a speed box containing 0 (speed_eps = 0 divides by s)
        for rad in (1e-9, 1e-3, 0.5):
            out.append((tag, box([0, 0, 0], rad), box(rng.normal(0, 3, 3), 1e-3), box(rng.normal(0, 10, 3), 1e-2)))
            out.append((tag, box([rad / 2, 0, 0], rad), box([1, 2, 3], rad), box([4, 5, 6], rad)))
    return out, cfgs


def points_of(boxes, rng, n_corner=12, n_in=6):
    """corners (random subset) and random interior points of the boxes, as double states; the centre too"""
    lo = np.array([b[0] for bx in boxes for b in bx])
    hi = np.array([b[1] for bx in boxes for b in bx])
    pts = [lo + 0.5 * (hi - lo)]
    for _ in range(n_corner):
        pts.append(np.where(rng.random(lo.size) < 0.5, lo, hi))
    for _ in range(n_in):
        pts.append(lo + rng.random(lo.size) * (hi - lo))
    pts.append(lo); pts.append(hi)
    return [np.clip(p, lo, hi) for p in pts]


def inside(lo, hi, x):
    return mpf(lo) <= x <= mpf(hi)


def test_flatness_rotation_and_channels_contain_exact_values(probe):
    cases, cfgs = box_cases()
    fps = {t: E.Flat.of_cfg(c) for t, c in cfgs.items()}
    recs_f, recs_c = [], []
    for tag, v, a, j in cases:
        fp = fps[tag]
        fv = [x for b in v for x in b]
        fa = [x for b in a for x in b]
        fj = [x for b in j for x in b]
        recs_f.append(list(fp.raw) + fv + fa)
        recs_c.append(list(fp.raw) + [cfgs[tag].vehicle_mass, cfgs[tag].vert_drag] + fv + fa + fj)
    of = probe("flat", recs_f)
    orot = probe("rot", recs_f)
    och = probe("channels", recs_c)
    rng = np.random.default_rng(17)
    names = ("speed", "acc", "omega", "tilt", "thrust")
    checked = dict.fromkeys(names, 0)
    unbounded = 0
    for k, (tag, v, a, j) in enumerate(cases):
        fp = fps[tag]
        yf, yr, yc = of[k], orot[k], och[k]
        for p in points_of((v, a, j), rng):
            pv, pa, pj = p[0:3], p[3:6], p[6:9]
            s, kap, zu, n = E.flat(fp, pv, pa)
            if yf[0] == 1.0:
                assert inside(yf[1], yf[2], kap), (k, "kap")
                for ax in range(3):
                    assert inside(yf[3 + 2 * ax], yf[4 + 2 * ax], zu[ax]), (k, "zu", ax)
                assert inside(yf[9], yf[10], n) and n > 0, (k, "n")
            if yr[0] == 1.0:
                att = E.attitude(fp, pv, pa)
                assert att is not None, k
                z, R = att
                for q in range(9):
                    assert inside(yr[1 + 2 * q], yr[2 + 2 * q], R[q // 3][q % 3]), (k, "R", q)
                num = E.norm([mpf(x) for x in pa]) + fp.dh * kap * E.norm([mpf(x) for x in pv]) + abs(fp.grav)
                assert num / n <= mpf(yr[19]) and mpf(yr[20]) <= 1 + z[2], (k, "kappa/delta")
            ch = E.channels(fp, pv, pa, pj)
            for q, nm in enumerate(names):
                x = ch[nm]
                if x is None:
                    continue
                assert inside(yc[q], yc[6 + q], x), (k, tag, nm, yc[q], yc[6 + q], x, v, a, j)
                checked[nm] += 1
            if ch["thrust"] is not None:
                assert inside(yc[5], yc[11], -ch["thrust"]), (k, "-thrust")
            unbounded += yc[8] == INF
    print(f"    {len(cases)} boxes: exact values checked per channel {checked}, body rate unbounded in {unbounded} point checks")
    assert min(checked.values()) > 1000


# ---- 4. what the callers make of a result that is no bound ---------------------------------------------------------------------------
def test_non_finite_pieces_give_no_bound(probe):
    cfg = VH.I.default_config_values()
    fp = E.Flat.of_cfg(cfg)
    base = np.zeros(18); base[12] = 5.0; base[1] = 1.0
    recs_c, recs_d, recs_p = [], [], []
    for pos, val in ((0, INF), (3, -INF), (5, NAN), (11, INF), (17, NAN), (14, 1e300)):
        c = base.copy(); c[pos] = val
        recs_c.append(list(fp.raw) + [1.0, 3.0] + list(c) + [0.0, 0.5, 0.0])
        recs_d.append(list(fp.raw) + [cfg.vehicle_mass, cfg.vert_drag] + list(c) + [0.0, 0.5])
        recs_p.append(list(fp.raw) + [cfg.vehicle_mass, cfg.vert_drag] + list(c) + [0.25])
    D = probe("cert_bound", recs_c)[:, 0]
    hi = probe("dyn_bound", recs_d)[:, :6]
    q = probe("dyn_point", recs_p)[:, :6]
    for k in range(len(recs_c)):
        c = np.array(recs_c[k][7:25]).reshape(3, 6)
        if not np.all(np.isfinite(c)):
            assert D[k] == INF, (k, D[k])                                   # NaN and overflow read as no bound
        else:
            assert not np.isnan(D[k])
        assert not np.any(np.isnan(hi[k])), (k, hi[k])                     # dyn_bound reads NaN as +inf
        if not np.all(np.isfinite(c[:, 1:])):
            # v, a or j not finite: every piece's end samples come out NaN, so the trajectory is VIOLATING with no bound reported,
            # whatever its intervals' enclosures say (they are not bounds of anything then)
            assert np.all(np.isnan(q[k])), (k, q[k])
        else:
            # finite, even where squares overflow: every lower end that is a number is attained (v, a, j do not see c_0)
            x, v, a, j = E.state(E.piece(c.reshape(-1), 1, 0), 0.25)
            ch = E.channels(fp, v, a, j)
            for n_, nm in enumerate(("speed", "acc", "omega", "tilt", "thrust")):
                if not math.isnan(q[k, n_]) and ch[nm] is not None:
                    assert mpf(q[k, n_]) <= ch[nm], (k, nm, q[k, n_])
