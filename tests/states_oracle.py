"""numpy restatements of isdf_trajectory_states' attitude half and of isdf_pose_points, in float64 one rounded operation at a time (numpy
never contracts a product and a sum into an FMA), and the fixture tests/golden/states_reference.npz."""
import os
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "states_reference.npz")
TAGS = ("drag", "nodrag")


def load_golden():
    z = np.load(GOLDEN)
    n = len([f for f in z.files if f.endswith("_times")])
    cases = [dict(N=z[f"c{k}_T"].size, head=z[f"c{k}_head"], tail=z[f"c{k}_tail"], inPs=z[f"c{k}_inPs"], T=z[f"c{k}_T"], coeffs=z[f"c{k}_coeffs"],
                  times=z[f"c{k}_times"], rec={t: z[f"c{k}_{t}_rec"] for t in TAGS}) for k in range(n)]
    return cases, {t: z[f"{t}_par"] for t in TAGS}


def config_for(tag):
    import isdf_b200 as I
    cfg = I.default_config_values()
    if tag == "nodrag":
        cfg.horiz_drag = cfg.vert_drag = cfg.paras_drag = 0.0
    return cfg


def flat_forward_yaw0(par, v, a, j):
    """FlatnessMap::forward(v, a, j, 0, 0, thr, quat, omg) (flatness.hpp:150-228) on (n, 3) arrays -> quat (n, 4), omg (n, 3), thr (n,)"""
    mass, grav, dh, dv, cp, veps = (float(x) for x in par)
    dh_over_m = dh / mass
    c_half, s_half, c_psi, s_psi, dpsi = 1.0, 0.0, 1.0, 0.0, 0.0
    v0, v1, v2, a0, a1, a2 = v[:, 0], v[:, 1], v[:, 2], a[:, 0], a[:, 1], a[:, 2]
    cp_term = np.sqrt(v0 * v0 + v1 * v1 + v2 * v2 + veps)
    w_term = 1.0 + cp * cp_term
    w0, w1, w2 = w_term * v0, w_term * v1, w_term * v2
    zu0, zu1, zu2 = a0 + dh_over_m * w0, a1 + dh_over_m * w1, a2 + dh_over_m * w2 + grav
    s0, s1, s2 = zu0 * zu0, zu1 * zu1, zu2 * zu2
    zu01, zu12, zu02 = zu0 * zu1, zu1 * zu2, zu0 * zu2
    sn = s0 + s1 + s2
    n = np.sqrt(sn)
    z0, z1, z2 = zu0 / n, zu1 / n, zu2 / n
    den = sn * n
    ng00, ng01, ng02 = (s1 + s2) / den, -zu01 / den, -zu02 / den
    ng11, ng12, ng22 = (s0 + s2) / den, -zu12 / den, (s0 + s1) / den
    vda = v0 * a0 + v1 * a1 + v2 * a2
    dw_term = cp * vda / cp_term
    dw0, dw1, dw2 = w_term * a0 + dw_term * v0, w_term * a1 + dw_term * v1, w_term * a2 + dw_term * v2
    d0, d1, d2 = j[:, 0] + dh_over_m * dw0, j[:, 1] + dh_over_m * dw1, j[:, 2] + dh_over_m * dw2
    dz0 = ng00 * d0 + ng01 * d1 + ng02 * d2
    dz1 = ng01 * d0 + ng11 * d1 + ng12 * d2
    dz2 = ng02 * d0 + ng12 * d1 + ng22 * d2
    f0, f1, f2 = mass * a0 + dv * w0, mass * a1 + dv * w1, mass * (a2 + grav) + dv * w2
    thr = z0 * f0 + z1 * f1 + z2 * f2
    td = np.sqrt(2.0 * (1.0 + z2))
    t0, t1, t2 = 0.5 * td, -z1 / td, z0 / td
    quat = np.stack([t0 * c_half, t1 * c_half + t2 * s_half, t2 * c_half - t1 * s_half, t0 * s_half], axis=1)
    od = z2 + 1.0
    ot = dz2 / od
    omg = np.stack([dz0 * s_psi - dz1 * c_psi - (z0 * s_psi - z1 * c_psi) * ot,
                    dz0 * c_psi + dz1 * s_psi - (z0 * c_psi + z1 * s_psi) * ot,
                    (z1 * dz0 - z0 * dz1) / od + dpsi], axis=1)
    return quat, omg, thr


def quat_rot(q):
    """Eigen's Quaternion::toRotationMatrix on (n, 4) (w, x, y, z) -> (n, 3, 3)"""
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.stack([np.stack([1.0 - (tyy + tzz), txy - twz, txz + twy], axis=1),
                     np.stack([txy + twz, 1.0 - (txx + tzz), tyz - twx], axis=1),
                     np.stack([txz - twy, tyz + twx, 1.0 - (txx + tyy)], axis=1)], axis=1)


def pose_points(states, body):
    """((R_k0 b0 + R_k1 b1) + R_k2 b2) + pos_k for every state and body point -> (Q, P, 3)"""
    R = quat_rot(np.asarray(states)[:, 12:16])
    pos = np.asarray(states)[:, 0:3]
    b = np.asarray(body, dtype=np.float64).reshape(-1, 3)
    out = np.empty((R.shape[0], b.shape[0], 3))
    for k in range(3):
        out[:, :, k] = ((R[:, k, 0, None] * b[None, :, 0] + R[:, k, 1, None] * b[None, :, 1]) + R[:, k, 2, None] * b[None, :, 2]) + pos[:, k, None]
    return out


def same_bits(a, b):
    """identical float64 bit patterns, every NaN counting as the same (x86 and the GPU spell a generated NaN differently)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64)))
