// Device-side FP64 vector math, MINCO basis, quadrotor flatness map + adjoint, hinge.
// Written for sm_90a; every function is __device__ __forceinline__ so the fused kernels keep state in registers.
// Reference semantics: flatness.hpp:53-148, 230-406; back_end_optimizer.hpp:127-173, 332-356, 472-488.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

#define ISDF_HD __host__ __device__ __forceinline__

namespace isdf {

struct d3 { double x, y, z; };

ISDF_HD d3 mk3(double x, double y, double z) { d3 r; r.x = x; r.y = y; r.z = z; return r; }
ISDF_HD d3 operator+(d3 a, d3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
ISDF_HD d3 operator-(d3 a, d3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
ISDF_HD d3 operator*(double s, d3 a) { return mk3(s * a.x, s * a.y, s * a.z); }
ISDF_HD d3 operator-(d3 a) { return mk3(-a.x, -a.y, -a.z); }
ISDF_HD double dot3(d3 a, d3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
ISDF_HD d3 cross3(d3 a, d3 b) {
    return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
ISDF_HD double len3(d3 a) { return sqrt(dot3(a, a)); }
// Eigen normalized(): divide by the norm when the squared norm is positive
ISDF_HD d3 unit3(d3 a) {
    const double n2 = dot3(a, a);
    if (n2 > 0.0) { const double n = sqrt(n2); return mk3(a.x / n, a.y / n, a.z / n); }
    return a;
}

// rotation as three rows
struct rot3 { d3 r0, r1, r2; };
__device__ __forceinline__ d3 rot_apply(const rot3 &R, d3 v) { return mk3(dot3(R.r0, v), dot3(R.r1, v), dot3(R.r2, v)); }
__device__ __forceinline__ d3 rot_applyT(const rot3 &R, d3 v) {
    return mk3(R.r0.x * v.x + R.r1.x * v.y + R.r2.x * v.z,
               R.r0.y * v.x + R.r1.y * v.y + R.r2.y * v.z,
               R.r0.z * v.x + R.r1.z * v.y + R.r2.z * v.z);
}

struct quat4 { double w, x, y, z; };

// unnormalised quaternion -> rotation matrix, Eigen's formula (back_end_optimizer.hpp:492)
__device__ __forceinline__ rot3 quat_rot(quat4 q) {
    const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    rot3 R;
    R.r0 = mk3(1.0 - (tyy + tzz), txy - twz, txz + twy);
    R.r1 = mk3(txy + twz, 1.0 - (txx + tzz), tyz - twx);
    R.r2 = mk3(txz - twy, tyz + twx, 1.0 - (txx + tyy));
    return R;
}

// smooth hinge (back_end_optimizer.hpp:332-356). Returns f (0 when x <= 0 contributes nothing) and df.
// The reference leaves its outputs untouched for x < 0 and its callers test f > 0, so "x <= 0 -> inactive" is exact.
__device__ __forceinline__ bool hinge(double x, double mu, double &f, double &df) {
    if (x < 0.0) { f = 0.0; df = 0.0; return false; }
    if (x > mu) { f = x - 0.5 * mu; df = 1.0; return true; }
    const double r = x / mu, r2 = r * r, m = mu - 0.5 * x;
    f = m * r2 * r;
    df = r2 * ((-0.5) * r + 3.0 * m / mu);
    return true;
}

// -g^T (dR^T/dq_k) d for the four quaternion components (back_end_optimizer.hpp:127-173, 816-820).
// Expanded by hand from the four constant-pattern matrices so no 3x3 temporaries are formed.
__device__ __forceinline__ void quat_pull(quat4 q, d3 g, d3 d, double out[4]) {
    const double w = q.w, x = q.x, y = q.y, z = q.z;
    out[0] = g.x * (2 * z * d.y - 2 * y * d.z) + g.y * (-2 * z * d.x + 2 * x * d.z) + g.z * (2 * y * d.x - 2 * x * d.y);
    out[1] = g.x * (2 * y * d.y + 2 * z * d.z) + g.y * (2 * y * d.x - 4 * x * d.y + 2 * w * d.z) + g.z * (2 * z * d.x - 2 * w * d.y - 4 * x * d.z);
    out[2] = g.x * (-4 * y * d.x + 2 * x * d.y - 2 * w * d.z) + g.y * (2 * x * d.x + 2 * z * d.z) + g.z * (2 * w * d.x + 2 * z * d.y - 4 * y * d.z);
    out[3] = g.x * (-4 * z * d.x + 2 * w * d.y + 2 * x * d.z) + g.y * (-2 * w * d.x - 4 * z * d.y + 2 * y * d.z) + g.z * (2 * x * d.x + 2 * y * d.y);
}

struct FlatParams { double mass, grav, dh_over_m, cp, veps; };

// Shared forward state of the flatness map. Everything the adjoint needs is kept so it is never recomputed.
struct FlatState {
    double s, kap, lam, n2, n, td, od, ot;
    d3 zu, z, xi, dz;
};

__device__ __forceinline__ void flat_state(const FlatParams &fp, d3 v, d3 a, d3 j, FlatState &m) {
    m.s = sqrt(v.x * v.x + v.y * v.y + v.z * v.z + fp.veps);
    m.kap = 1.0 + fp.cp * m.s;
    m.zu = mk3(a.x + fp.dh_over_m * (m.kap * v.x), a.y + fp.dh_over_m * (m.kap * v.y), a.z + fp.dh_over_m * (m.kap * v.z) + fp.grav);
    const double s0 = m.zu.x * m.zu.x, s1 = m.zu.y * m.zu.y, s2 = m.zu.z * m.zu.z;
    m.n2 = s0 + s1 + s2;
    m.n = sqrt(m.n2);
    m.z = mk3(m.zu.x / m.n, m.zu.y / m.n, m.zu.z / m.n);
    m.td = sqrt(2.0 * (1.0 + m.z.z));
    const double den = m.n2 * m.n;
    const double p00 = (s1 + s2) / den, p11 = (s0 + s2) / den, p22 = (s0 + s1) / den;
    const double p01 = -(m.zu.x * m.zu.y) / den, p02 = -(m.zu.x * m.zu.z) / den, p12 = -(m.zu.y * m.zu.z) / den;
    const double vda = v.x * a.x + v.y * a.y + v.z * a.z;
    m.lam = fp.cp * vda / m.s;
    m.xi = mk3(j.x + fp.dh_over_m * (m.kap * a.x + m.lam * v.x),
               j.y + fp.dh_over_m * (m.kap * a.y + m.lam * v.y),
               j.z + fp.dh_over_m * (m.kap * a.z + m.lam * v.z));
    m.dz = mk3(p00 * m.xi.x + p01 * m.xi.y + p02 * m.xi.z,
               p01 * m.xi.x + p11 * m.xi.y + p12 * m.xi.z,
               p02 * m.xi.x + p12 * m.xi.y + p22 * m.xi.z);
    m.od = m.z.z + 1.0;
    m.ot = m.dz.z / m.od;
}
__device__ __forceinline__ quat4 flat_quat(const FlatState &m) {
    quat4 q; q.w = 0.5 * m.td; q.x = -m.z.y / m.td; q.y = m.z.x / m.td; q.z = 0.0; return q;
}
__device__ __forceinline__ d3 flat_omega(const FlatState &m) {
    return mk3(-m.dz.y + m.z.y * m.ot, m.dz.x - m.z.x * m.ot, (m.z.y * m.dz.x - m.z.x * m.dz.y) / m.od);
}
// quaternion-only forward (flatness.hpp:53-86): skips the body-rate half
__device__ __forceinline__ quat4 flat_quat_only(const FlatParams &fp, d3 v, d3 a) {
    const double s = sqrt(v.x * v.x + v.y * v.y + v.z * v.z + fp.veps);
    const double kap = 1.0 + fp.cp * s;
    const double zx = a.x + fp.dh_over_m * (kap * v.x), zy = a.y + fp.dh_over_m * (kap * v.y), zz = a.z + fp.dh_over_m * (kap * v.z) + fp.grav;
    const double n = sqrt(zx * zx + zy * zy + zz * zz);
    const double z0 = zx / n, z1 = zy / n, z2 = zz / n;
    const double td = sqrt(2.0 * (1.0 + z2));
    quat4 q; q.w = 0.5 * td; q.x = -z1 / td; q.y = z0 / td; q.z = 0.0; return q;
}

// Reverse-mode adjoint of (quat, omega) with respect to (vel, acc, jer) — the contract of
// FlatnessMap::backwardthreadsafe (flatness.hpp:230-406): total grads = pulled-back (qb, ob) + direct (vel_grad).
// Derived in vector form: dz = P xi with P = I/n - zu zu^T/n^3 (symmetric), z = zu/n.
__device__ __forceinline__ void flat_adjoint(const FlatParams &fp, const FlatState &m, d3 v, d3 a,
                                             const double qb[4], d3 ob, d3 vel_grad, d3 &gv, d3 &ga, d3 &gj) {
    const d3 z = m.z, dz = m.dz, zu = m.zu, xi = m.xi;
    const double iod = 1.0 / m.od;
    d3 dzb = mk3(ob.y + ob.z * z.y * iod, -ob.x - ob.z * z.x * iod, 0.0);
    const double otb = ob.x * z.y - ob.y * z.x;
    dzb.z = otb * iod;
    d3 zb = mk3(-ob.y * m.ot - ob.z * dz.y * iod, ob.x * m.ot + ob.z * dz.x * iod, 0.0);
    const double odb = -(ob.z * (z.y * dz.x - z.x * dz.y) + otb * dz.z) * iod * iod;
    const double itd = 1.0 / m.td;
    const double tdb = 0.5 * qb[0] + (qb[1] * z.y - qb[2] * z.x) * itd * itd;
    zb.x += qb[2] * itd;
    zb.y -= qb[1] * itd;
    zb.z = odb + tdb * itd;
    const double in = 1.0 / m.n, in3 = in / m.n2, in5 = in3 / m.n2;
    const double zu_xi = dot3(zu, xi), zu_dzb = dot3(zu, dzb), dzb_xi = dot3(dzb, xi);
    const d3 xib = mk3(dzb.x * in - zu.x * zu_dzb * in3, dzb.y * in - zu.y * zu_dzb * in3, dzb.z * in - zu.z * zu_dzb * in3);
    const double c_zu = -dzb_xi * in3 + 3.0 * zu_dzb * zu_xi * in5;
    const double zb_z = dot3(zb, z);
    d3 zub = mk3(c_zu * zu.x - (zu_xi * dzb.x + zu_dzb * xi.x) * in3 + (zb.x - zb_z * z.x) * in,
                 c_zu * zu.y - (zu_xi * dzb.y + zu_dzb * xi.y) * in3 + (zb.y - zb_z * z.y) * in,
                 c_zu * zu.z - (zu_xi * dzb.z + zu_dzb * xi.z) * in3 + (zb.z - zb_z * z.z) * in);
    const d3 wb = fp.dh_over_m * zub;
    const d3 dwb = fp.dh_over_m * xib;
    gj = xib;
    const double kapb = dot3(a, dwb) + dot3(v, wb);
    const double lamb = dot3(v, dwb);
    const double lc = lamb * fp.cp / m.s;
    const double sb = -lamb * m.lam / m.s + fp.cp * kapb;
    const double sv = sb / m.s;
    ga = mk3(zub.x + m.kap * dwb.x + lc * v.x, zub.y + m.kap * dwb.y + lc * v.y, zub.z + m.kap * dwb.z + lc * v.z);
    gv = mk3(m.lam * dwb.x + m.kap * wb.x + lc * a.x + sv * v.x + vel_grad.x,
             m.lam * dwb.y + m.kap * wb.y + lc * a.y + sv * v.y + vel_grad.y,
             m.lam * dwb.z + m.kap * wb.z + lc * a.z + sv * v.z + vel_grad.z);
}

// Quintic piece evaluated through the beta basis (back_end_optimizer.hpp:472-488). c: 6 coefficients per axis.
struct PieceEval { d3 pos, vel, acc, jer, sna; double b0[6], b1[6], b2[6], b3[6]; };

__device__ __forceinline__ void piece_eval(const double *cx, const double *cy, const double *cz, double s1, PieceEval &e) {
    const double s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2, s5 = s4 * s1;
    e.b0[0] = 1.0; e.b0[1] = s1; e.b0[2] = s2; e.b0[3] = s3; e.b0[4] = s4; e.b0[5] = s5;
    e.b1[0] = 0.0; e.b1[1] = 1.0; e.b1[2] = 2.0 * s1; e.b1[3] = 3.0 * s2; e.b1[4] = 4.0 * s3; e.b1[5] = 5.0 * s4;
    e.b2[0] = 0.0; e.b2[1] = 0.0; e.b2[2] = 2.0; e.b2[3] = 6.0 * s1; e.b2[4] = 12.0 * s2; e.b2[5] = 20.0 * s3;
    e.b3[0] = 0.0; e.b3[1] = 0.0; e.b3[2] = 0.0; e.b3[3] = 6.0; e.b3[4] = 24.0 * s1; e.b3[5] = 60.0 * s2;
    const double b44 = 24.0, b45 = 120.0 * s1;
    double p[3], v[3], a[3], j[3], sn[3];
    const double *c[3] = {cx, cy, cz};
#pragma unroll
    for (int ax = 0; ax < 3; ax++) {
        double sp = 0, sv = 0, sa = 0, sj = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) {
            const double ck = c[ax][k];
            sp += ck * e.b0[k]; sv += ck * e.b1[k]; sa += ck * e.b2[k]; sj += ck * e.b3[k];
        }
        p[ax] = sp; v[ax] = sv; a[ax] = sa; j[ax] = sj;
        sn[ax] = c[ax][4] * b44 + c[ax][5] * b45;  // beta4 = [0,0,0,0,24,120 s]
    }
    e.pos = mk3(p[0], p[1], p[2]); e.vel = mk3(v[0], v[1], v[2]); e.acc = mk3(a[0], a[1], a[2]);
    e.jer = mk3(j[0], j[1], j[2]); e.sna = mk3(sn[0], sn[1], sn[2]);
}

// warp-wide sum of a double, result valid in every lane (xor butterfly: same order on every launch => deterministic)
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace isdf
