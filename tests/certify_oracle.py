"""Serial FP64 restatement of the continuous clearance certificate (include/isdf.h, isdf_trajectory_certify) — TEST INFRASTRUCTURE.

  pose_at(cfg, T, coeffs, piece, t)   the pose at any local time, built the way grazing.sample_poses builds the clearance samples' poses
  bound(cfg, r, H, c, ta, tb, te)     D_e of the definition: the same interval algorithm as the device, in round-to-nearest
  displacement(...)                   the dense reference: largest displacement of given body points over 2001 times of an interval
  certify(...)                        the refinement (rounds, per-trajectory budgets, leaves, summaries) on top of clearance_oracle's
                                      brute-force clearance of a pose

The device bound rounds every operation outward; here every operation rounds to nearest, so the two agree to a few ulps per operation
(the device's is never smaller than this one's by more than that)."""
import ctypes as C
import math
import numpy as np
import oracle_lib as O
import grazing as G
import clearance_oracle as CO

EPS_REL = 1e-10
BINOM = [[math.comb(m, k) for k in range(6)] for m in range(6)]


def flat_params(cfg):
    """FlatParams of the library from an isdf_config: (dh_over_m, cp, veps, grav)"""
    return cfg.horiz_drag / cfg.vehicle_mass, cfg.paras_drag, cfg.speed_eps, cfg.grav_acc


def piece_coeffs(coeffs, N, i):
    """(3, 6): t^k coefficients of piece i per axis (coeffs: 6N x 3 column-major)"""
    return np.asarray(coeffs, float).reshape(3, 6 * N)[:, 6 * i:6 * i + 6]


def pose_at(cfg, T, coeffs, piece, t):
    """pos (n,3), R (n,3,3) at local times t of pieces `piece`: the piece polynomial evaluated directly, the oracle's flatness
    quaternion, Eigen's quaternion formula (grazing.sample_poses at arbitrary times)"""
    T = np.asarray(T, float).reshape(-1)
    N = T.size
    piece, t = np.atleast_1d(piece).astype(int), np.atleast_1d(np.asarray(t, float))
    pos, vel, acc, jer = [], [], [], []
    k = np.arange(6)
    for i, s in zip(piece, t):
        c = piece_coeffs(coeffs, N, i)
        pos.append(c @ (s ** k))
        vel.append(c @ np.array([0, 1, 2 * s, 3 * s ** 2, 4 * s ** 3, 5 * s ** 4]))
        acc.append(c @ np.array([0, 0, 2, 6 * s, 12 * s ** 2, 20 * s ** 3]))
        jer.append(c @ np.array([0, 0, 0, 6, 24 * s, 60 * s ** 2]))
    q, _ = O.flat_forward_batch(O.config_from(cfg), np.array(vel), np.array(acc), np.array(jer))
    return np.array(pos), G.quat_to_R(q)


def pose_closed_form(cfg, c, t, dtype=np.float64):
    """(pos, R) of one piece (c: (3,6)) at time t in the given float type, from the closed form R(z) of the definition"""
    dh, cp, veps, g = (dtype(x) for x in flat_params(cfg))
    c = np.asarray(c, dtype=dtype)
    t = dtype(t)
    p = np.array([sum(c[a, k] * t ** k for k in range(6)) for a in range(3)], dtype=dtype)
    v = np.array([sum(k * c[a, k] * t ** (k - 1) for k in range(1, 6)) for a in range(3)], dtype=dtype)
    a_ = np.array([sum(k * (k - 1) * c[a, k] * t ** (k - 2) for k in range(2, 6)) for a in range(3)], dtype=dtype)
    s = np.sqrt(v @ v + veps)
    zu = a_ + dh * (1 + cp * s) * v + np.array([0, 0, g], dtype=dtype)
    z = zu / np.sqrt(zu @ zu)
    return p, rot_of_z(z)


def rot_of_z(z):
    zx, zy, zz = z
    op = 1 + zz
    return np.array([[1 - zx * zx / op, -zx * zy / op, zx], [-zx * zy / op, 1 - zy * zy / op, zy], [-zx, -zy, zz]])


# ---- the bound, interval by interval (round to nearest) ---------------------------------------------------------------------------
def _add(a, b): return (a[0] + b[0], a[1] + b[1])
def _sub(a, b): return (a[0] - b[1], a[1] - b[0])
def _neg(a): return (-a[1], -a[0])
def _mag(a): return max(abs(a[0]), abs(a[1]))


def _mul(a, b):
    p = (a[0] * b[0], a[0] * b[1], a[1] * b[0], a[1] * b[1])
    return (min(p), max(p))


def _sqr(a):
    m = _mag(a)
    n = a[0] if a[0] > 0 else (-a[1] if a[1] < 0 else 0.0)
    return (n * n, m * m)


def _divp(a, b):
    return (a[0] / b[1] if a[0] >= 0 else a[0] / b[0], a[1] / b[0] if a[1] >= 0 else a[1] / b[1])


def _sqrt(a): return (math.sqrt(max(a[0], 0.0)), math.sqrt(a[1]))


def _rot(fp, v, a):
    dh, cp, veps, g = fp
    s = _sqrt(_add(_add(_add(_sqr(v[0]), _sqr(v[1])), _sqr(v[2])), (veps, veps)))
    kap = _add((1.0, 1.0), _mul((cp, cp), s))
    zu = [_add(a[k], _mul((dh, dh), _mul(kap, v[k]))) for k in range(3)]
    zu[2] = _add(zu[2], (g, g))
    n = _sqrt(_add(_add(_sqr(zu[0]), _sqr(zu[1])), _sqr(zu[2])))
    if not n[0] > 0:
        return None
    zx, zy, zz = (_divp(zu[k], n) for k in range(3))
    op = _add((1.0, 1.0), zz)
    if not op[0] > 0:
        return None
    xx, yy, xy = _divp(_sqr(zx), op), _divp(_sqr(zy), op), _divp(_mul(zx, zy), op)
    R = [_sub((1.0, 1.0), xx), _neg(xy), zx, _neg(xy), _sub((1.0, 1.0), yy), zy, _neg(zx), _neg(zy), zz]
    nrm = lambda w: math.sqrt(_mag(w[0]) ** 2 + _mag(w[1]) ** 2 + _mag(w[2]) ** 2)
    kappa = (nrm(a) + dh * kap[1] * nrm(v) + abs(g)) / n[0]
    return R, kappa, op[0]


def bound(cfg, r, H, c, ta, tb, te):
    """D_e for one piece (c: (3,6) coefficients) over [ta, tb] measured from t_e, restating isdf_certify.cuh::cert_bound"""
    fp = flat_params(cfg)
    h = max(tb - te, te - ta, 0.0)
    hp = [h ** k for k in range(6)]
    tp = [(1.0, 1.0)]
    for k in range(1, 6):
        tp.append(_mul(tp[-1], (te, te)))
    P2 = A = 0.0
    ve, vi, ae, ai = [], [], [], []
    for ax in range(3):
        cc = [float(x) for x in c[ax]]
        m, dd = [0.0] * 6, [None] * 6
        for k in range(1, 6):
            d = (0.0, 0.0)
            for q in range(k, 6):
                d = _add(d, _mul(_mul((BINOM[q][k], BINOM[q][k]), (cc[q], cc[q])), tp[q - k]))
            m[k], dd[k] = _mag(d), d
        disp = sum(m[k] * hp[k] for k in range(1, 6))
        vr = sum(k * m[k] * hp[k - 1] for k in range(2, 6))
        ar = sum(k * (k - 1) * m[k] * hp[k - 2] for k in range(3, 6))
        A += abs(cc[0]) + sum(abs(cc[k]) * _mag(tp[k]) for k in range(1, 6))
        P2 += disp * disp
        ve.append(dd[1]); vi.append((dd[1][0] - vr, dd[1][1] + vr))
        a2 = _mul((2.0, 2.0), dd[2])
        ae.append(a2); ai.append((a2[0] - ar, a2[1] + ar))
    P = math.sqrt(P2)
    ri, re = _rot(fp, vi, ai), _rot(fp, ve, ae)
    if ri is None or re is None:
        return math.inf
    Q = math.sqrt(sum(_mag(_sub(x, y)) ** 2 for x, y in zip(ri[0], re[0])))
    eps = EPS_REL * (1 + A + 2 * H + (r + 2 * H) * re[1] / re[2])
    D = P + r * Q + eps
    return D if D < math.inf else math.inf


def eps_pad(cfg, r, H, c, te):
    """the pose pad eps_e alone (bound with h = 0 minus P and Q, which vanish there)"""
    return bound(cfg, r, H, c, te, te, te)


def displacement(cfg, T, coeffs, piece, ta, tb, te, body, n=2001):
    """max over n times of [ta, tb] and the body points (m,3) of |x(t) + R(t) p - x(t_e) - R(t_e) p| (oracle poses)"""
    t = np.linspace(ta, tb, n)
    pos, R = pose_at(cfg, T, coeffs, np.full(n, piece), t)
    p0, R0 = pose_at(cfg, T, coeffs, [piece], [te])
    body = np.asarray(body, float).reshape(-1, 3)
    q = pos[:, None, :] + np.einsum("tij,mj->tmi", R, body)
    q0 = p0[0][None, :] + body @ R0[0].T
    return float(np.linalg.norm(q - q0[None], axis=2).max())


def body_radius(points):
    return float(np.linalg.norm(np.asarray(points, float).reshape(-1, 3), axis=1).max()) * (1.0 + 1e-12)


def box_corners(half, rot=None, trans=None):
    """body-frame corners of ISDF_SHAPE_BOX {hx, hy, hz} with Rotate / trans (the inverse of shape_pre: p_in = Rotate q + trans)"""
    rot = np.eye(3) if rot is None else np.asarray(rot, float).reshape(3, 3)
    trans = np.zeros(3) if trans is None else np.asarray(trans, float)
    q = np.array([[sx * half[0], sy * half[1], sz * half[2]] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
    return q @ rot.T + trans


# ---- refinement ---------------------------------------------------------------------------------------------------------------------
def _clear_at(cfg, scene, T, coeffs, piece, t, reach):
    occ_ids, ctr, f = scene
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + reach
    pos, R = pose_at(cfg, T, coeffs, piece, t)
    out_c, out_v = np.full(len(piece), float(reach)), np.full(len(piece), -1, dtype=np.int64)
    for s in range(len(piece)):
        if not np.all(np.isfinite(pos[s])):
            out_c[s] = np.nan
            continue
        prel = (ctr - pos[s]) @ R[s]
        m = ~np.any(np.abs(prel) > H, axis=1)
        if m.any():
            v = f(prel[m])
            if v.min() < reach:
                out_c[s] = v.min()
                out_v[s] = occ_ids[m][v == v.min()].min()
    return out_c, out_v


def certify(cfg, occ, bmin, res, sdf, r, T, coeffs, K_c, reach, margin, N0=0, max_depth=16, max_samples=2048):
    """dict(summary=[per trajectory], leaves=[(traj, piece in block, ta, tb, ca, cb, Da, Db, state)]) — the device's refinement with
    this module's bound (round to nearest) and the brute-force clearance. sdf: an oracle Shape or callable prel -> sdf."""
    f = sdf if callable(sdf) else (lambda p: sdf.query(p, what=0)[0])
    ids, ctr = CO.occupied(occ, bmin, res)
    scene = (ids, ctr, f)
    T = np.asarray(T, float).reshape(-1)
    N, K = T.size, int(K_c)
    N0 = N if N0 == 0 else N0
    B = N // N0
    H = cfg.kernel_size * cfg.occupancy_resolution / 2 + reach
    cs = [piece_coeffs(coeffs, N, i) for i in range(N)]
    toff = np.zeros(N)
    for b in range(B):
        t = 0.0
        for q in range(N0):
            toff[b * N0 + q] = t
            t += T[b * N0 + q]
    # samples: (piece, t) -> clearance, witness
    sp = [i for i in range(N) for j in range(K + 1)]
    st = [j * (T[i] * (1.0 / K)) for i in range(N) for j in range(K + 1)]
    sc, sv = _clear_at(cfg, scene, T, coeffs, sp, st, reach)
    sc, sv = list(sc), list(sv)
    active = []   # per trajectory: list of [ta, tb, sa, sb, piece, depth, fold_a, fold_b]
    for b in range(B):
        lst = []
        for i in range(b * N0, (b + 1) * N0):
            step = T[i] * (1.0 / K)
            for j in range(K):
                lst.append([j * step, T[i] if j + 1 == K else (j + 1) * step, i * (K + 1) + j, i * (K + 1) + j + 1, i, 0, True, j + 1 == K])
        active.append(lst)
    state = [dict(lb=math.inf, key=(math.inf, math.inf, 2 ** 64 - 1), fh=math.inf, used=0, und=0, depth=0) for _ in range(B)]
    hit = [False] * B
    leaves = []

    def fold(b, s):
        v = sc[s] if sc[s] == sc[s] else -math.inf
        t = toff[sp[s]] + st[s]
        key = (v, t, int(sv[s]) % 2 ** 64)
        if key < state[b]["key"]:
            state[b]["key"] = key
        if not v >= margin:
            state[b]["fh"] = min(state[b]["fh"], t)

    for b in range(B):
        for s in range(b * N0 * (K + 1), (b + 1) * N0 * (K + 1)):
            hit[b] |= not (sc[s] >= margin)
    while any(active):
        new_s = []
        nxt = [[] for _ in range(B)]
        for b in range(B):
            stt = state[b]
            for I in active[b]:
                ta, tb, sa, sb, i, dep, fa, fb = I
                Da = bound(cfg, r, H, cs[i], ta, tb, st[sa])
                Db = bound(cfg, r, H, cs[i], ta, tb, st[sb])
                ca, cb = sc[sa], sc[sb]
                lb = max(-math.inf if ca != ca else ca - Da, -math.inf if cb != cb else cb - Db)
                if fa:
                    fold(b, sa)
                if fb:
                    fold(b, sb)
                safe = lb >= margin
                m = ta + 0.5 * (tb - ta)
                wants = (not safe) and (not hit[b]) and dep < max_depth and ta < m < tb
                if wants and stt["used"] < max_samples:
                    stt["used"] += 1
                    s = len(sp) + len(new_s)
                    new_s.append((i, m))
                    nxt[b].append([ta, m, sa, s, i, dep + 1, False, False])
                    nxt[b].append([m, tb, s, sb, i, dep + 1, True, False])
                else:
                    stl = 1 if safe else (-1 if hit[b] else 0)
                    leaves.append((b, i - b * N0, ta, tb, ca, cb, Da, Db, stl))
                    stt["lb"] = min(stt["lb"], lb)
                    stt["und"] += stl == 0
                    stt["depth"] = max(stt["depth"], dep)
        if new_s:
            c_, v_ = _clear_at(cfg, scene, T, coeffs, [p for p, _ in new_s], [t for _, t in new_s], reach)
            for (p, t), cc, vv in zip(new_s, c_, v_):
                sp.append(p); st.append(t); sc.append(cc); sv.append(vv)
                hit[p // N0] |= not (cc >= margin)
        active = nxt
    summ = []
    for b in range(B):
        s = state[b]
        v, t, x = s["key"]
        summ.append(dict(verdict=-1 if hit[b] else (1 if s["und"] == 0 else 0), lower_bound=s["lb"], min_clearance=math.nan if v == -math.inf else v,
                         t_min=t, voxel_min=x - 2 ** 64 if x >= 2 ** 63 else x, first_hit=-1.0 if s["fh"] == math.inf else s["fh"],
                         samples=N0 * (K + 1) + s["used"], undecided_intervals=s["und"], depth=s["depth"]))
    return dict(summary=summ, leaves=leaves)
