"""CPU references of the certified swept volume (include/isdf.h, isdf_swept_volume_*) — TEST INFRASTRUCTURE.

  exact_sv_point(T, coeffs, p, radius)    min_t |p - x(t)| - radius for Point (radius 0) and Ball: per piece, the real roots in [0, T_i] of
                                          the degree-9 derivative of |p - x(t)|^2, plus the piece ends
  dense_sv(cfg, T, coeffs, p, sdf, n)     min over n times per piece of sd(R^T (p - x)) (oracle poses), polished by golden section
  dense_lower(cfg, T, coeffs, p, sdf, r, H, n)
                                          a lower bound of SV(p): n intervals per piece, max(sd_a - D_a, sd_b - D_b) with
                                          certify_oracle.bound
  box_sdf(half)                           the Box's SDF (body frame) as a callable
  marching_tets(value, tstar, bmin, res)  the library's marching tetrahedra restated in NumPy (same vertex order, rounding and triangles)
  mesh_checks(V, F)                       edge-manifold / orientation / Euler characteristic / signed volume"""
import math
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
