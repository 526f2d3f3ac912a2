"""CPU references of the certified swept volume (include/isdf.h, isdf_swept_volume_*) — TEST INFRASTRUCTURE.

  exact_sv_point(T, coeffs, p, radius)    min_t |p - x(t)| - radius for Point (radius 0) and Ball: per piece, the real roots in [0, T_i] of
                                          the degree-9 derivative of |p - x(t)|^2, plus the piece ends
  dense_sv(cfg, T, coeffs, p, sdf, n)     min over n times per piece of sd(R^T (p - x)) (oracle poses), polished by golden section
  dense_lower(cfg, T, coeffs, p, sdf, r, H, n)
                                          a lower bound of SV(p): n intervals per piece, max(sd_a - D_a, sd_b - D_b) with
                                          certify_oracle.bound
  box_sdf(half)                           the Box's SDF (body frame) as a callable
  sv_refine(cfg, T, coeffs, p, sdf, r_rot, r_body, params)
                                          the per-point refinement of include/isdf.h (steps 1-5) restated serially, with the smallest
                                          margin of any of its decisions (near-tie guard)
  node_cull_bound / brick_cull_bound      the sphere cull's node and brick (without its slack) bounds with the device's directed
                                          rounding, exactly (fractions)
  marching_tets(value, tstar, bmin, res)  the library's marching tetrahedra restated in NumPy (same vertex order, rounding and triangles)
  marching_tets_np(value, tstar, bmin, res)
                                          the same, vectorised over nodes and cells (large grids)
  mesh_checks(V, F)                       edge-manifold / orientation / Euler characteristic / signed volume"""
import math
from fractions import Fraction
import numpy as np
import certify_oracle as CE

# ---- exact SV for Point and Ball -----------------------------------------------------------------------------------------------------
def exact_sv_point(T, coeffs, p, radius=0.0):
    T = np.asarray(T, float).reshape(-1)
    N = T.size
    p = np.asarray(p, float)
    best = math.inf
    for i in range(N):
        c = CE.piece_coeffs(coeffs, N, i)                         # (3, 6), ascending powers
        d = c.copy()
        d[:, 0] -= p                                              # x(t) - p
        dv = np.array([[k * d[a, k] for k in range(1, 6)] for a in range(3)])   # derivative, ascending powers 0..4
        g = np.zeros(10)                                          # (x - p) . x', ascending powers 0..9
        for a in range(3):
            g += np.convolve(d[a], dv[a])
        roots = np.roots(g[::-1]) if np.any(g) else np.array([])
        ts = [0.0, T[i]] + [r.real for r in roots if abs(r.imag) <= 1e-9 * max(1.0, abs(r)) and -1e-12 <= r.real <= T[i] + 1e-12]
        for t in ts:
            t = min(max(t, 0.0), T[i])
            x = c @ (t ** np.arange(6))
            best = min(best, float(np.linalg.norm(x - p)))
    return best - radius


# ---- dense references for any distance shape -----------------------------------------------------------------------------------------
def box_sdf(half):
    h = np.asarray(half, float)

    def f(q):
        q = np.atleast_2d(q)
        d = np.abs(q) - h
        return np.linalg.norm(np.maximum(d, 0.0), axis=1) + np.minimum(d.max(axis=1), 0.0)
    return f


def _sd(cfg, T, coeffs, piece, t, p, sdf):
    pos, R = CE.pose_at(cfg, T, coeffs, piece, t)
    q = np.einsum("nji,nj->ni", R, np.asarray(p, float)[None, :] - pos)   # R^T (p - x)
    return sdf(q)


def dense_sv(cfg, T, coeffs, p, sdf, n=20001, polish=60):
    """(value, trajectory time) of the smallest sd over n times per piece, polished by golden section around the best time"""
    T = np.asarray(T, float).reshape(-1)
    best, arg = math.inf, (0, 0.0)
    for i in range(T.size):
        t = np.linspace(0.0, T[i], n)
        v = _sd(cfg, T, coeffs, np.full(n, i), t, p, sdf)
        k = int(np.argmin(v))
        if v[k] < best:
            best, arg = float(v[k]), (i, float(t[k]))
    i, t0 = arg
    h = T[i] / (n - 1)
    a, b = max(t0 - h, 0.0), min(t0 + h, T[i])
    g = (math.sqrt(5) - 1) / 2
    for _ in range(polish):
        x1, x2 = b - g * (b - a), a + g * (b - a)
        f1, f2 = _sd(cfg, T, coeffs, [i, i], [x1, x2], p, sdf)
        if f1 < f2:
            b = x2
        else:
            a = x1
        best = min(best, float(f1), float(f2))
    return best, float(np.sum(T[:i])) + t0


def dense_lower(cfg, T, coeffs, p, sdf, r, H, n=64):
    """min over n intervals per piece of max(sd_a - D_a, sd_b - D_b): a lower bound of SV(p) (up to the bound's rounding)"""
    T = np.asarray(T, float).reshape(-1)
    N = T.size
    lo = math.inf
    for i in range(N):
        t = np.linspace(0.0, T[i], n + 1)
        v = _sd(cfg, T, coeffs, np.full(n + 1, i), t, p, sdf)
        c = CE.piece_coeffs(coeffs, N, i)
        for k in range(n):
            Da = CE.bound(cfg, r, H, c, t[k], t[k + 1], t[k])
            Db = CE.bound(cfg, r, H, c, t[k], t[k + 1], t[k + 1])
            lo = min(lo, max(v[k] - Da, v[k + 1] - Db))
    return lo


# ---- the per-point refinement, restated ----------------------------------------------------------------------------------------------
class SvPrep:
    """what the refinement uses that does not depend on p (k_sv_prep): the initial intervals, piece start times, and caches of the poses
    and motion bounds every point of one (trajectory, r_rot, band, K) shares"""

    def __init__(self, cfg, T, coeffs, r_rot, params):
        self.cfg = cfg
        self.T = np.asarray(T, float).reshape(-1)
        self.coeffs = np.asarray(coeffs, float).reshape(-1)
        N = self.N = self.T.size
        K = self.K = int(params.samples_per_piece)
        self.r_rot, self.band = float(r_rot), float(params.band)
        self.toff, t = [], 0.0
        for i in range(N):                        # piece start times, summed left to right
            self.toff.append(t)
            t += float(self.T[i])
        self.cs = [CE.piece_coeffs(self.coeffs, N, i) for i in range(N)]
        self._pose, self._bound = {}, {}
        self.iv = []                              # (piece, j, ta, tb, tbs) in interval order
        for i in range(N):
            step = float(self.T[i]) * (1.0 / K)
            for j in range(K):
                ta, tbs = j * step, (j + 1) * step
                self.iv.append((i, j, ta, float(self.T[i]) if j + 1 == K else tbs, tbs))
        self.poses([(i, j * (float(self.T[i]) * (1.0 / K))) for i in range(N) for j in range(K + 1)])

    def poses(self, keys):
        """(pos, R) at (piece, local time) keys, through certify_oracle.pose_at, cached"""
        miss = sorted({k for k in keys if k not in self._pose})
        if miss:
            pos, R = CE.pose_at(self.cfg, self.T, self.coeffs, [k[0] for k in miss], [k[1] for k in miss])
            for k, x, r in zip(miss, pos, R):
                self._pose[k] = (x, r)
        return [self._pose[k] for k in keys]

    def bound(self, i, ta, tb, te):
        key = (i, ta, tb, te)
        if key not in self._bound:
            self._bound[key] = CE.bound(self.cfg, self.r_rot, self.band, self.cs[i], ta, tb, te)
        return self._bound[key]


def _lb(fa, fb, Da, Db):
    a = -math.inf if fa != fa else fa - Da
    b = -math.inf if fb != fb else fb - Db
    return max(a, b)


def sv_refine(cfg, T, coeffs, p, sdf, r_rot, r_body, params, prep=None):
    """include/isdf.h's per-point refinement (steps 1-5), serially, with this module's poses and bounds (round to nearest).
    sdf: body-frame points (n, 3) -> (n,). params: an isdf_swept_params (samples_per_piece, max_depth, max_samples_per_point, tol, band).
    prep: an SvPrep of the same trajectory, r_rot and params, to share poses and bounds across points.
    Returns dict(value, lower, tstar, decided, evals (counted as the kernel counts them: a sample shared by two kept intervals once),
    deepest, leaves [(piece, ta, tb, lb, depth)], margin (the smallest distance of any decision from its threshold: the sphere cull
    against band, lb against hi0 - tol where the split is otherwise possible, lower against value - tol, value against band), tgap (the
    smallest difference between value and a sample value other than it), near (the times of the samples within 1e-12 of value: where
    t* may go when tgap is below the rounding of the two sides), ties (how many sample times attain value exactly), shared (the
    intervals whose first endpoint is the previous kept interval's last, evaluated once), max_wanting (most intervals wanting a split in one round),
    budget_cut (an interval wanted a split the budget refused), partial (a round in which the budget left granted some splits and refused
    others), depth_cut (an interval wanted a split at max_depth))."""
    P = prep if prep is not None else SvPrep(cfg, T, coeffs, r_rot, params)
    K, band, tol = P.K, float(params.band), float(params.tol)
    max_depth, max_samples = int(params.max_depth), int(params.max_samples_per_point)
    p = np.asarray(p, float)
    margin = math.inf
    samples = []                                  # (value, trajectory time) of every evaluated sample

    def sd(keys):
        if not keys:
            return []
        ps = P.poses(keys)
        pos = np.array([x for x, _ in ps])
        R = np.array([r for _, r in ps])
        q = np.einsum("nji,nj->ni", R, p[None, :] - pos)
        return [float(v) for v in np.asarray(sdf(q), float).reshape(-1)]

    # steps 1-2: initial intervals, sphere cull
    kept = []
    for q, (i, j, ta, tb, tbs) in enumerate(P.iv):
        Da, Db = P.bound(i, ta, tb, ta), P.bound(i, ta, tb, tbs)
        (xa, _), (xb, _) = P.poses([(i, ta), (i, tbs)])
        L = max(float(np.linalg.norm(p - xa)) - r_body - Da, float(np.linalg.norm(p - xb)) - r_body - Db)
        if L == L and abs(L) < math.inf:
            margin = min(margin, abs(L - band))
        if not L >= band:
            kept.append((q, i, j, ta, tb, tbs, Da, Db))
    # step 3: round 0, a sample shared by two kept intervals evaluated once
    keys, evals, shared = [], 0, []
    kq = {k[0] for k in kept}
    for (q, i, j, ta, tb, tbs, Da, Db) in kept:
        need_a = not (j != 0 and (q - 1) in kq)
        if not need_a:
            shared.append(q)
        keys += ([(i, ta)] if need_a else []) + [(i, tbs)]
        evals += 1 + need_a
    val = dict(zip(keys, sd(keys)))
    for (i, t) in keys:
        samples.append((val[(i, t)], P.toff[i] + t))
    cur = [dict(ta=ta, tb=tb, tbs=tbs, fa=val[(i, ta)], fb=val[(i, tbs)], Da=Da, Db=Db, piece=i, depth=0)
           for (q, i, j, ta, tb, tbs, Da, Db) in kept]

    def key_min():
        v, t = band, math.inf
        for sv, st in samples:
            if sv < v or (sv == v and st < t):
                v, t = sv, st
        return v, t

    # step 4: level-synchronous rounds
    leaves, used, max_wanting, budget_cut, depth_cut = [], 0, 0, False, False
    partial = False
    while cur:
        hi0 = key_min()[0]
        allowed = max(max_samples - used, 0)
        nxt, splits, nwant = [], [], 0
        for I in cur:
            lb = _lb(I["fa"], I["fb"], I["Da"], I["Db"])
            m = I["ta"] + 0.5 * (I["tb"] - I["ta"])
            open_ = I["ta"] < m < I["tb"]
            below = lb < hi0 - tol
            if open_ and I["depth"] < max_depth and abs(lb) < math.inf:
                margin = min(margin, abs(lb - (hi0 - tol)))
            depth_cut |= below and open_ and I["depth"] >= max_depth
            wants = below and I["depth"] < max_depth and open_
            nwant += wants
            if wants and used < max_samples:
                used += 1
                splits.append((I, m))
            else:
                budget_cut |= wants
                leaves.append((I["piece"], I["ta"], I["tb"], lb, I["depth"]))
        max_wanting = max(max_wanting, nwant)
        partial |= 0 < allowed < nwant
        fm = sd([(I["piece"], m) for I, m in splits])
        evals += len(splits)
        for (I, m), f in zip(splits, fm):
            samples.append((f, P.toff[I["piece"]] + m))
            i, d = I["piece"], I["depth"] + 1
            nxt.append(dict(ta=I["ta"], tb=m, tbs=m, fa=I["fa"], fb=f, Da=P.bound(i, I["ta"], m, I["ta"]), Db=P.bound(i, I["ta"], m, m),
                            piece=i, depth=d))
            nxt.append(dict(ta=m, tb=I["tb"], tbs=I["tbs"], fa=f, fb=I["fb"], Da=P.bound(i, m, I["tb"], m),
                            Db=P.bound(i, m, I["tb"], I["tbs"]), piece=i, depth=d))
        cur = nxt
    # step 5
    hv, ht = key_min()
    hi = min(hv, band)
    lo_leaf = min([-math.inf if lb != lb else lb for (_, _, _, lb, _) in leaves], default=math.inf)
    lo = min(hi, lo_leaf)
    if lo != hi and abs(lo) < math.inf:   # lower == value is decided whatever the rounding
        margin = min(margin, abs(lo - (hi - tol)))
    if hv < band:
        margin = min(margin, band - hv)
    tgap = min([abs(v - hv) for v, _ in samples if v == v and v != hv], default=math.inf)
    near = sorted({t for v, t in samples if abs(v - hv) <= 1e-12}) if hi < band else [-1.0]
    ties = len({t for v, t in samples if v == hv}) if hi < band else 0
    return dict(value=hi, lower=lo, tstar=-1.0 if hi == band else ht, decided=bool(lo >= hi - tol), evals=evals, near=near, ties=ties, shared=shared,
                deepest=max([l[4] for l in leaves], default=0), leaves=leaves, margin=margin, tgap=tgap, max_wanting=max_wanting,
                budget_cut=budget_cut, partial=partial, depth_cut=depth_cut)


# ---- the sphere cull's bounds with the device's directed rounding ----------------------------------------------------------------------
def _rd(x):
    f = float(x)   # Fraction -> nearest double
    return f if Fraction(f) <= x else math.nextafter(f, -math.inf)


def _ru(x):
    f = float(x)
    return f if Fraction(f) >= x else math.nextafter(f, math.inf)


def _sqrt_rd(x):
    s = math.sqrt(x)
    return s if Fraction(s) ** 2 <= Fraction(x) else math.nextafter(s, -math.inf)


def _sqrt_ru(x):
    s = math.sqrt(x)
    return s if Fraction(s) ** 2 >= Fraction(x) else math.nextafter(s, math.inf)


def _dist_rd(p, x):
    d = [_rd(abs(Fraction(float(p[k])) - Fraction(float(x[k])))) for k in range(3)]
    s = _rd(Fraction(_rd(Fraction(d[0]) ** 2)) + Fraction(_rd(Fraction(d[1]) ** 2)))
    return _sqrt_rd(_rd(Fraction(s) + Fraction(_rd(Fraction(d[2]) ** 2))))


def node_cull_bound(p, x, r_body, D):
    """|p - x| - r_body - D with every operation rounded down, as the node test of the sphere cull (sv_cull_bound) computes it"""
    return _rd(Fraction(_rd(Fraction(_dist_rd(p, x)) - Fraction(r_body))) - Fraction(D))


def brick_cull_bound(bmin, res, lo, hi, x, r_body, D):
    """the brick test of the sphere cull (k_sv_bricks) before its relative slack: |c - x| - (r_body + rho) - D, with c the centre of
    the nodes lo..hi and rho their half-diagonal rounded up, the distance and the differences rounded down"""
    c, rho2 = [], 0.0
    for a in range(3):
        plo, phi = float(bmin[a] + float(lo[a]) * res), float(bmin[a] + float(hi[a]) * res)
        c.append(0.5 * (plo + phi))
        h = max(_ru(Fraction(phi) - Fraction(c[a])), _ru(Fraction(c[a]) - Fraction(plo)))
        rho2 = _ru(Fraction(rho2) + Fraction(_ru(Fraction(h) ** 2)))
    rb = _ru(Fraction(r_body) + Fraction(_sqrt_ru(rho2)))
    return _rd(Fraction(_rd(Fraction(_dist_rd(c, x)) - Fraction(rb))) - Fraction(D))


# ---- marching tetrahedra, restated ---------------------------------------------------------------------------------------------------
DIR_BITS = [1, 2, 4, 3, 5, 6, 7]
BITS_DIR = {b: d for d, b in enumerate(DIR_BITS)}
TETS = [[0, 1, 3, 7], [0, 1, 5, 7], [0, 2, 3, 7], [0, 2, 6, 7], [0, 4, 5, 7], [0, 4, 6, 7]]
TET_POS = [True, False, False, True, True, False]
EVEN = [[0, 1, 2, 3], [1, 0, 3, 2], [2, 3, 0, 1], [3, 2, 1, 0]]


def _off(b):
    return np.array([b & 1, (b >> 1) & 1, (b >> 2) & 1])


def marching_tets(value, tstar, bmin, res):
    """(V, vtime, F) of include/isdf.h's marching tetrahedra on node values (X, Y, Z); tstar may be None (vtime then empty)"""
    f = np.asarray(value, float)
    X, Y, Z = f.shape
    inside = f < 0.0
    ts = np.zeros_like(f) if tstar is None else np.asarray(tstar, float)
    ax = [np.float64(bmin[a]) + np.arange(n, dtype=np.float64) * np.float64(res) for a, n in enumerate((X, Y, Z))]
    vid = {}
    V, vt = [], []
    # vertices in (node address, direction) order
    for ix in range(X):
        for iy in range(Y):
            for iz in range(Z):
                for d, b in enumerate(DIR_BITS):
                    jx, jy, jz = (ix, iy, iz) + _off(b)
                    if jx >= X or jy >= Y or jz >= Z or inside[ix, iy, iz] == inside[jx, jy, jz]:
                        continue
                    f0, f1 = f[ix, iy, iz], f[jx, jy, jz]
                    s = f0 / (f0 - f1)
                    p0 = np.array([ax[0][ix], ax[1][iy], ax[2][iz]])
                    p1 = np.array([ax[0][jx], ax[1][jy], ax[2][jz]])
                    vid[(ix, iy, iz, d)] = len(V)
                    V.append(p0 + s * (p1 - p0))
                    vt.append(ts[ix, iy, iz] if abs(f0) <= abs(f1) else ts[jx, jy, jz])
    F = []
    for ix in range(X - 1):
        for iy in range(Y - 1):
            for iz in range(Z - 1):
                cin = [bool(inside[ix + (c & 1), iy + ((c >> 1) & 1), iz + ((c >> 2) & 1)]) for c in range(8)]
                for t, tv in enumerate(TETS):
                    ins = [q for q in range(4) if cin[tv[q]]]
                    k = len(ins)
                    if k in (0, 4):
                        continue

                    def E(x, y):
                        u, w = (tv[x], tv[y]) if x < y else (tv[y], tv[x])
                        o = _off(u)
                        return vid[(ix + o[0], iy + o[1], iz + o[2], BITS_DIR[w & ~u])]
                    if k in (1, 3):
                        i = ins[0] if k == 1 else [q for q in range(4) if q not in ins][0]
                        e = EVEN[i]
                        tris = [[E(i, e[1]), E(i, e[2]), E(i, e[3])]] if k == 1 else [[E(i, e[1]), E(i, e[3]), E(i, e[2])]]
                    else:
                        i, j = ins
                        kk, l = [q for q in range(4) if q not in ins]
                        perm = [i, j, kk, l]
                        inv = sum(perm[a] > perm[b] for a in range(4) for b in range(a + 1, 4))
                        if inv % 2:
                            kk, l = l, kk
                        tris = [[E(i, l), E(j, l), E(j, kk)], [E(i, l), E(j, kk), E(i, kk)]]
                    for tr in tris:
                        F.append(tr if TET_POS[t] else [tr[0], tr[2], tr[1]])
    return (np.array(V, float).reshape(-1, 3), np.array(vt, float), np.array(F, dtype=np.int32).reshape(-1, 3))


def _tet_cases():
    """per (tetrahedron, inside mask of its 4 vertices): the triangles as (corner u, corner w) pairs of their vertices' edges, in the
    order and orientation of marching_tets"""
    out = {}
    for t, tv in enumerate(TETS):
        for m in range(16):
            ins = [q for q in range(4) if (m >> q) & 1]
            k = len(ins)
            if k in (0, 4):
                out[(t, m)] = []
                continue

            def E(x, y):
                return (tv[x], tv[y]) if x < y else (tv[y], tv[x])
            if k in (1, 3):
                i = ins[0] if k == 1 else [q for q in range(4) if q not in ins][0]
                e = EVEN[i]
                tris = [[E(i, e[1]), E(i, e[2]), E(i, e[3])]] if k == 1 else [[E(i, e[1]), E(i, e[3]), E(i, e[2])]]
            else:
                i, j = ins
                kk, l = [q for q in range(4) if q not in ins]
                perm = [i, j, kk, l]
                if sum(perm[a] > perm[b] for a in range(4) for b in range(a + 1, 4)) % 2:
                    kk, l = l, kk
                tris = [[E(i, l), E(j, l), E(j, kk)], [E(i, l), E(j, kk), E(i, kk)]]
            out[(t, m)] = [tr if TET_POS[t] else [tr[0], tr[2], tr[1]] for tr in tris]
    return out


def marching_tets_np(value, tstar, bmin, res):
    """marching_tets vectorised over nodes and cells: the same (V, vtime, F), bit for bit"""
    f = np.asarray(value, float)
    X, Y, Z = f.shape
    n = f.size
    inside = (f < 0.0).reshape(-1)
    fl = f.reshape(-1)
    ts = np.zeros(n) if tstar is None else np.asarray(tstar, float).reshape(-1)
    ax = [np.float64(bmin[a]) + np.arange(m, dtype=np.float64) * np.float64(res) for a, m in enumerate((X, Y, Z))]
    ix, iy, iz = (g.reshape(-1) for g in np.meshgrid(np.arange(X), np.arange(Y), np.arange(Z), indexing="ij"))
    # crossed edges per (node, direction), numbered in (node address, direction) order
    cross = np.zeros((n, 7), bool)
    nbr = np.zeros((n, 7), np.int64)
    for d, b in enumerate(DIR_BITS):
        o = _off(b)
        jx, jy, jz = ix + o[0], iy + o[1], iz + o[2]
        ok = (jx < X) & (jy < Y) & (jz < Z)
        a1 = np.where(ok, (jx * Y + jy) * Z + jz, 0)
        nbr[:, d] = a1
        cross[:, d] = ok & (inside != inside[a1])
    vid = np.cumsum(cross.reshape(-1)).reshape(n, 7) - 1
    a0, d = np.nonzero(cross)
    a1 = nbr[a0, d]
    f0, f1 = fl[a0], fl[a1]
    s = f0 / (f0 - f1)
    P0 = np.stack([ax[0][ix[a0]], ax[1][iy[a0]], ax[2][iz[a0]]], 1)
    P1 = np.stack([ax[0][ix[a1]], ax[1][iy[a1]], ax[2][iz[a1]]], 1)
    V = P0 + s[:, None] * (P1 - P0)
    vt = np.where(np.abs(f0) <= np.abs(f1), ts[a0], ts[a1])
    # triangles in (cell address, tetrahedron, local) order, over the cells whose corners are not all on one side
    cell = (ix < X - 1) & (iy < Y - 1) & (iz < Z - 1)
    cin = np.zeros(n, np.int64)
    for c in range(8):
        o = _off(c)
        ac = np.where(cell, ((ix + o[0]) * Y + iy + o[1]) * Z + iz + o[2], 0)
        cin |= inside[ac].astype(np.int64) << c
    cells = np.flatnonzero(cell & (cin != 0) & (cin != 255))
    cases = _tet_cases()
    out = np.full((cells.size, 6, 2, 3), -1, np.int64)
    for t, tv in enumerate(TETS):
        m = np.zeros(cells.size, np.int64)
        for q in range(4):
            m |= ((cin[cells] >> tv[q]) & 1) << q
        for mm in range(16):
            sel = np.flatnonzero(m == mm)
            for l, tri in enumerate(cases[(t, mm)]):
                for v, (u, w) in enumerate(tri):
                    o = _off(u)
                    node = ((ix[cells[sel]] + o[0]) * Y + iy[cells[sel]] + o[1]) * Z + iz[cells[sel]] + o[2]
                    out[sel, t, l, v] = vid[node, BITS_DIR[w & ~u]]
    F = out.reshape(-1, 3)
    F = F[F[:, 0] >= 0].astype(np.int32)
    return V.reshape(-1, 3), vt, F


def mesh_checks(V, F):
    """dict(manifold, oriented, euler, volume): every undirected edge in exactly two triangles; every directed edge once (so the two
    triangles of an edge traverse it in opposite directions); chi = V_used - E + F; signed volume by the divergence theorem"""
    F = np.asarray(F)
    used = np.unique(F)
    und, dire = {}, {}
    for a, b, c in F:
        for u, w in ((a, b), (b, c), (c, a)):
            dire[(u, w)] = dire.get((u, w), 0) + 1
            key = (min(u, w), max(u, w))
            und[key] = und.get(key, 0) + 1
    manifold = all(v == 2 for v in und.values())
    oriented = all(v == 1 for v in dire.values()) and all((w, u) in dire for (u, w) in dire)
    P = np.asarray(V, float)
    vol = float(np.sum(np.einsum("ij,ij->i", P[F[:, 0]], np.cross(P[F[:, 1]], P[F[:, 2]])))) / 6.0 if len(F) else 0.0
    return dict(manifold=manifold, oriented=oriented, euler=len(used) - len(und) + len(F), volume=vol)
