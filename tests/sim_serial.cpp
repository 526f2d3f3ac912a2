// TEST INFRASTRUCTURE ONLY: the serial CPU restatement of the closed loop that isdf_simulate is held against (include/isdf.h, DESIGN
// §3.17). Written from the reference's src/uav_simulator: Quadrotor.cpp (model, step), quadrotor_simulator_so3.cpp (getControl, setInput),
// SO3Control.cpp (calculateControl), so3_control_nodelet.cpp (odometry / command order), traj_server.cpp (the 100 Hz command) and the
// vendored odeint's integrate_adaptive + controlled_runge_kutta<runge_kutta_dopri5>. Built with g++ -O3 -ffp-contract=off; the attitude
// loop is float code as the reference writes it.
#include "../include/isdf.h"
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>

namespace {

const double NaN = std::numeric_limits<double>::quiet_NaN();

struct Traj { const double *T, *C; int N; double dur; };

// locatePieceIdx + Piece::getPos / getVel / getAcc (the library's coefficient layout: 6N x 3 column-major, ascending powers)
void traj_pva(const Traj &tr, double t, double p[3], double v[3], double a[3]) {
    int i = 0;
    for (; i < tr.N; i++) {
        if (!(t > tr.T[i])) break;
        t -= tr.T[i];
    }
    if (i == tr.N) { i--; t += tr.T[i]; }
    for (int d = 0; d < 3; d++) {
        const double *c = tr.C + 6 * tr.N * d + 6 * i;
        double pp = 0, vv = 0, aa = 0, ptn = 1.0, vtn = 1.0, atn = 1.0;
        int vn = 1, am = 1, an = 2;
        for (int k = 0; k < 6; k++) {
            pp += ptn * c[k]; ptn *= t;
            if (k >= 1) { vv += (vn * vtn) * c[k]; vtn *= t; vn++; }
            if (k >= 2) { aa += ((am * an) * atn) * c[k]; atn *= t; am++; an++; }
        }
        p[d] = pp; v[d] = vv; a[d] = aa;
    }
}

// Eigen's 3x3 inverse: adjugate from cofactors, det along column 0; m and out row-major
void inv3(const double m[9], double out[9]) {
    auto M = [&](int i, int j) { return m[3 * i + j]; };
    auto cof = [&](int i, int j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        return M(i1, j1) * M(i2, j2) - M(i1, j2) * M(i2, j1);
    };
    const double c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
    const double det = c00 * M(0, 0) + c10 * M(1, 0) + c20 * M(2, 0);
    const double invdet = 1.0 / det;
    out[0] = c00 * invdet; out[1] = c10 * invdet; out[2] = c20 * invdet;
    out[3] = cof(0, 1) * invdet; out[4] = cof(1, 1) * invdet; out[5] = cof(2, 1) * invdet;
    out[6] = cof(0, 2) * invdet; out[7] = cof(1, 2) * invdet; out[8] = cof(2, 2) * invdet;
}

// R (row-major) from the state's column-major block x[6..14], re-orthonormalised as R L^-1 with L L^T = R^T R (Eigen's LLT)
void polar(const double *xs, double Rn[9]) {
    double R[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) R[3 * i + j] = xs[3 * j + i];
    double Mt[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Mt[3 * i + j] = R[i] * R[j] + R[3 + i] * R[3 + j] + R[6 + i] * R[6 + j];
    double L[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    L[0] = std::sqrt(Mt[0]);
    L[3] = Mt[3] / L[0]; L[6] = Mt[6] / L[0];
    L[4] = std::sqrt(Mt[4] - L[3] * L[3]);
    L[7] = (Mt[7] - L[6] * L[3]) / L[4];
    L[8] = std::sqrt(Mt[8] - (L[6] * L[6] + L[7] * L[7]));
    double Li[9];
    inv3(L, Li);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rn[3 * i + j] = R[3 * i] * Li[j] + R[3 * i + 1] * Li[3 + j] + R[3 * i + 2] * Li[6 + j];
}

struct Vehicle {
    const isdf_sim_params *p;
    double J[9], Jinv[9];
    double F[3], Mx[3];
    double input[4];
    double acc[3];
};

void vehicle_init(Vehicle &q, const isdf_sim_params *p, const double *dist) {
    q.p = p;
    for (int i = 0; i < 9; i++) q.J[i] = 0.0;
    q.J[0] = p->J[0]; q.J[4] = p->J[1]; q.J[8] = p->J[2];
    inv3(q.J, q.Jinv);
    for (int i = 0; i < 3; i++) { q.F[i] = dist ? dist[i] : 0.0; q.Mx[i] = dist ? dist[3 + i] : 0.0; q.acc[i] = 0.0; }
    for (int i = 0; i < 4; i++) q.input[i] = 0.0;
}

// Quadrotor::operator()
void rhs(Vehicle &q, const double x[22], double dx[22]) {
    const isdf_sim_params *p = q.p;
    double R[9];
    polar(x + 6, R);
    const double o0 = x[15], o1 = x[16], o2 = x[17];
    double sq[4];
    for (int i = 0; i < 4; i++) sq[i] = x[18 + i] * x[18 + i];
    const double thrust = p->kf * (((sq[0] + sq[1]) + sq[2]) + sq[3]);
    const double mom0 = p->kf * (sq[2] - sq[3]) * p->arm;
    const double mom1 = p->kf * (sq[1] - sq[0]) * p->arm;
    const double mom2 = p->km * (sq[0] + sq[1] - sq[2] - sq[3]);
    const double vn2 = x[3] * x[3] + x[4] * x[4] + x[5] * x[5];
    const double vn = std::sqrt(vn2);
    const double resistance = 0.1 * 3.14159265 * p->arm * p->arm * vn * vn;
    double vh[3] = {x[3], x[4], x[5]};
    if (vn != 0) for (int i = 0; i < 3; i++) vh[i] = x[3 + i] / vn;
    const double g3[3] = {-0.0, -0.0, -p->grav};
    double vd[3];
    for (int i = 0; i < 3; i++) vd[i] = g3[i] + thrust * R[3 * i + 2] / p->mass + q.F[i] / p->mass - resistance * vh[i] / p->mass;
    for (int i = 0; i < 3; i++) q.acc[i] = vd[i];
    // R_dot = R [omega]x ; column j of R_dot into dx[6 + 3 j + i]
    const double W[9] = {0.0, -o2, o1, o2, 0.0, -o0, -o1, o0, 0.0};
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) dx[6 + 3 * j + i] = R[3 * i] * W[j] + R[3 * i + 1] * W[3 + j] + R[3 * i + 2] * W[6 + j];
    double Jo[3];
    for (int i = 0; i < 3; i++) Jo[i] = q.J[3 * i] * o0 + q.J[3 * i + 1] * o1 + q.J[3 * i + 2] * o2;
    const double cr[3] = {o1 * Jo[2] - o2 * Jo[1], o2 * Jo[0] - o0 * Jo[2], o0 * Jo[1] - o1 * Jo[0]};
    const double tq[3] = {mom0 - cr[0] + q.Mx[0], mom1 - cr[1] + q.Mx[1], mom2 - cr[2] + q.Mx[2]};
    for (int i = 0; i < 3; i++) dx[15 + i] = q.Jinv[3 * i] * tq[0] + q.Jinv[3 * i + 1] * tq[1] + q.Jinv[3 * i + 2] * tq[2];
    for (int i = 0; i < 3; i++) { dx[i] = x[3 + i]; dx[3 + i] = vd[i]; }
    for (int i = 0; i < 4; i++) dx[18 + i] = (q.input[i] - x[18 + i]) / p->motor_tau;
    for (int i = 0; i < 22; i++) if (std::isnan(dx[i])) dx[i] = 0;
}

// Dormand-Prince 5(4) tableau
const double a21 = 1.0 / 5;
const double a31 = 3.0 / 40, a32 = 9.0 / 40;
const double a41 = 44.0 / 45, a42 = -56.0 / 15, a43 = 32.0 / 9;
const double a51 = 19372.0 / 6561, a52 = -25360.0 / 2187, a53 = 64448.0 / 6561, a54 = -212.0 / 729;
const double a61 = 9017.0 / 3168, a62 = -355.0 / 33, a63 = 46732.0 / 5247, a64 = 49.0 / 176, a65 = -5103.0 / 18656;
const double c1 = 35.0 / 384, c3 = 500.0 / 1113, c4 = 125.0 / 192, c5 = -2187.0 / 6784, c6 = 11.0 / 84;
const double e1 = c1 - 5179.0 / 57600, e3 = c3 - 7571.0 / 16695, e4 = c4 - 393.0 / 640, e5 = c5 - -92097.0 / 339200,
             e6 = c6 - 187.0 / 2100, e7 = -1.0 / 40;

// one try of the controlled stepper from (x, dxdt) with step h: out, dout and the error norm
double dopri5_try(Vehicle &q, const double x[22], const double k1[22], double h, double out[22], double k7[22]) {
    double k2[22], k3[22], k4[22], k5[22], k6[22], t[22];
    for (int i = 0; i < 22; i++) t[i] = 1.0 * x[i] + h * a21 * k1[i];
    rhs(q, t, k2);
    for (int i = 0; i < 22; i++) t[i] = 1.0 * x[i] + h * a31 * k1[i] + h * a32 * k2[i];
    rhs(q, t, k3);
    for (int i = 0; i < 22; i++) t[i] = 1.0 * x[i] + h * a41 * k1[i] + h * a42 * k2[i] + h * a43 * k3[i];
    rhs(q, t, k4);
    for (int i = 0; i < 22; i++) t[i] = 1.0 * x[i] + h * a51 * k1[i] + h * a52 * k2[i] + h * a53 * k3[i] + h * a54 * k4[i];
    rhs(q, t, k5);
    for (int i = 0; i < 22; i++) t[i] = 1.0 * x[i] + h * a61 * k1[i] + h * a62 * k2[i] + h * a63 * k3[i] + h * a64 * k4[i] + h * a65 * k5[i];
    rhs(q, t, k6);
    for (int i = 0; i < 22; i++) out[i] = 1.0 * x[i] + h * c1 * k1[i] + h * c3 * k3[i] + h * c4 * k4[i] + h * c5 * k5[i] + h * c6 * k6[i];
    rhs(q, out, k7);
    double err = 0.0;
    for (int i = 0; i < 22; i++) {
        const double xe = h * e1 * k1[i] + h * e3 * k3[i] + h * e4 * k4[i] + h * e5 * k5[i] + h * e6 * k6[i] + h * e7 * k7[i];
        const double r = std::fabs(xe) / (1e-6 + 1e-6 * (1.0 * std::fabs(x[i]) + (1.0 * h) * std::fabs(k1[i])));
        err = (std::fabs(err) < std::fabs(r)) ? std::fabs(r) : std::fabs(err);
    }
    return err;
}

// integrate_adaptive(controlled_runge_kutta<dopri5>, sys, x, 0, dt, dt); returns false after 1000 rejections in a row
bool integrate(Vehicle &q, double x[22], double dt, long long &acc, long long &rej) {
    double k1[22], out[22], k7[22];
    rhs(q, x, k1);
    double t = 0.0, h = dt;
    const long long tries_cap = acc + rej + 100000;   // this library's bound on the tries of one step (odeint has none)
    while (t < dt) {
        if (dt < t + h) h = dt - t;
        int trials = 0;
        for (;;) {
            if (!(h > 0) || t + h == t || acc + rej >= tries_cap) return false;   // no progress: the step cannot finish
            const double err = dopri5_try(q, x, k1, h, out, k7);
            trials++;
            if (err > 1.0) {
                rej++;
                h *= std::fmax(0.9 * std::pow(err, -1.0 / 3.0), 0.2);
                if (trials == 1000) return false;
                continue;
            }
            acc++;
            if (trials == 1000) return false;   // odeint throws when its 1000th try ends the loop, accepted or not
            t += h;
            if (err < 0.5) {
                const double e = std::fmax(std::pow(5.0, -5.0), err);
                h *= 0.9 * std::pow(e, -1.0 / 5.0);
            }
            std::memcpy(x, out, sizeof(out));
            std::memcpy(k1, k7, sizeof(k7));
            break;
        }
    }
    return true;
}

struct Counters { long long acc = 0, rej = 0; int clamped = 0, floor = 0, rollbacks = 0; };

// Quadrotor::step(dt); false when the integrator gave up
bool model_step(Vehicle &q, double x[22], double dt, int floor_on, Counters &c) {
    double save[22];
    std::memcpy(save, x, sizeof(save));
    if (!integrate(q, x, dt, c.acc, c.rej)) return false;
    for (int i = 0; i < 22; i++) if (std::isnan(x[i])) { std::memcpy(x, save, sizeof(save)); c.rollbacks++; break; }
    double R[9];
    polar(x + 6, R);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) x[6 + 3 * j + i] = R[3 * i + j];
    if (floor_on && x[2] < 0.0 && x[5] < 0) { x[2] = 0; x[5] = 0; c.floor++; }
    return true;
}

// setInput: NaN -> mean, clamp; returns whether any input was clamped
bool set_input(Vehicle &q, const double rpm[4]) {
    const isdf_sim_params *p = q.p;
    bool cl = false;
    for (int i = 0; i < 4; i++) {
        double u = rpm[i];
        if (std::isnan(u)) u = (p->max_rpm + p->min_rpm) / 2;
        if (u > p->max_rpm) { u = p->max_rpm; cl = true; }
        else if (u < p->min_rpm) { u = p->min_rpm; cl = true; }
        q.input[i] = u;
    }
    return cl;
}

struct Command {   // the simulator's Command struct
    float force[3];
    float qx, qy, qz, qw;
    float kR[3], kOm[3], corrections[3];
    float current_yaw;
    int use_external_yaw;
};

void quat_to_R(double w, double x, double y, double z, double R[9]) {   // Eigen's toRotationMatrix
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.0 - (txx + tyy);
}

void R_to_quat(const double m[9], double q[4]) {   // Eigen's Quaternion(Matrix3) (w, x, y, z)
    auto M = [&](int i, int j) { return m[3 * i + j]; };
    double t = M(0, 0) + M(1, 1) + M(2, 2);
    if (t > 0) {
        t = std::sqrt(t + 1.0);
        q[0] = 0.5 * t;
        t = 0.5 / t;
        q[1] = (M(2, 1) - M(1, 2)) * t;
        q[2] = (M(0, 2) - M(2, 0)) * t;
        q[3] = (M(1, 0) - M(0, 1)) * t;
    } else {
        int i = 0;
        if (M(1, 1) > M(0, 0)) i = 1;
        if (M(2, 2) > M(i, i)) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(M(i, i) - M(j, j) - M(k, k) + 1.0);
        q[1 + i] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (M(k, j) - M(j, k)) * t;
        q[1 + j] = (M(j, i) + M(i, j)) * t;
        q[1 + k] = (M(k, i) + M(i, k)) * t;
    }
}

void qmul(const double a[4], const double b[4], double o[4]) {   // Eigen's quat_product (w, x, y, z)
    o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
    o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
    o[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
    o[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}

// getControl (quadrotor_simulator_so3.cpp); R of the state (row-major), omega
void get_control(const isdf_sim_params *p, const double Rs[9], const double om[3], const Command &cmd, double rpm[4]) {
    const double _kf = p->kf, _km = p->km;
    const double kf = _kf - cmd.corrections[0];
    const double km = _km / _kf * kf;
    const double d = p->arm;
    const float I[3][3] = {{(float)p->J[0], 0.0f, 0.0f}, {0.0f, (float)p->J[1], 0.0f}, {0.0f, 0.0f, (float)p->J[2]}};
    // R_to_ypr (uav_utils/geometry_utils.h)
    const double n0 = Rs[0], n1 = Rs[3], n2 = Rs[6], o0 = Rs[1], o1 = Rs[4], a0 = Rs[2], a1 = Rs[5];
    const double y = std::atan2(n1, n0);
    const double pt = std::atan2(-n2, n0 * std::cos(y) + n1 * std::sin(y));
    const double r = std::atan2(a0 * std::sin(y) - a1 * std::cos(y), -o0 * std::sin(y) + o1 * std::cos(y));
    const double yaw = cmd.use_external_yaw ? (double)cmd.current_yaw : y;
    const double qz[4] = {std::cos(0.5 * yaw), std::sin(0.5 * yaw) * 0.0, std::sin(0.5 * yaw) * 0.0, std::sin(0.5 * yaw) * 1.0};
    const double qy[4] = {std::cos(0.5 * pt), std::sin(0.5 * pt) * 0.0, std::sin(0.5 * pt) * 1.0, std::sin(0.5 * pt) * 0.0};
    const double qx[4] = {std::cos(0.5 * r), std::sin(0.5 * r) * 1.0, std::sin(0.5 * r) * 0.0, std::sin(0.5 * r) * 0.0};
    double qzy[4], qq[4], R[9];
    qmul(qz, qy, qzy);
    qmul(qzy, qx, qq);
    quat_to_R(qq[0], qq[1], qq[2], qq[3], R);
    const float R11 = R[0], R12 = R[1], R13 = R[2], R21 = R[3], R22 = R[4], R23 = R[5], R31 = R[6], R32 = R[7], R33 = R[8];
    const float Om1 = om[0], Om2 = om[1], Om3 = om[2];
    const float Rd11 = cmd.qw * cmd.qw + cmd.qx * cmd.qx - cmd.qy * cmd.qy - cmd.qz * cmd.qz;
    const float Rd12 = 2 * (cmd.qx * cmd.qy - cmd.qw * cmd.qz);
    const float Rd13 = 2 * (cmd.qx * cmd.qz + cmd.qw * cmd.qy);
    const float Rd21 = 2 * (cmd.qx * cmd.qy + cmd.qw * cmd.qz);
    const float Rd22 = cmd.qw * cmd.qw - cmd.qx * cmd.qx + cmd.qy * cmd.qy - cmd.qz * cmd.qz;
    const float Rd23 = 2 * (cmd.qy * cmd.qz - cmd.qw * cmd.qx);
    const float Rd31 = 2 * (cmd.qx * cmd.qz - cmd.qw * cmd.qy);
    const float Rd32 = 2 * (cmd.qy * cmd.qz + cmd.qw * cmd.qx);
    const float Rd33 = cmd.qw * cmd.qw - cmd.qx * cmd.qx - cmd.qy * cmd.qy + cmd.qz * cmd.qz;
    const float Psi = 0.5f * (3.0f - (Rd11 * R11 + Rd21 * R21 + Rd31 * R31 + Rd12 * R12 + Rd22 * R22 + Rd32 * R32 + Rd13 * R13 + Rd23 * R23 +
                                      Rd33 * R33));
    float force = 0;
    if (Psi < 1.0f) force = cmd.force[0] * R13 + cmd.force[1] * R23 + cmd.force[2] * R33;
    const float eR1 = 0.5f * (R12 * Rd13 - R13 * Rd12 + R22 * Rd23 - R23 * Rd22 + R32 * Rd33 - R33 * Rd32);
    const float eR2 = 0.5f * (R13 * Rd11 - R11 * Rd13 - R21 * Rd23 + R23 * Rd21 - R31 * Rd33 + R33 * Rd31);
    const float eR3 = 0.5f * (R11 * Rd12 - R12 * Rd11 + R21 * Rd22 - R22 * Rd21 + R31 * Rd32 - R32 * Rd31);
    const float eOm1 = Om1, eOm2 = Om2, eOm3 = Om3;
    const float in1 = Om2 * (I[2][0] * Om1 + I[2][1] * Om2 + I[2][2] * Om3) - Om3 * (I[1][0] * Om1 + I[1][1] * Om2 + I[1][2] * Om3);
    const float in2 = Om3 * (I[0][0] * Om1 + I[0][1] * Om2 + I[0][2] * Om3) - Om1 * (I[2][0] * Om1 + I[2][1] * Om2 + I[2][2] * Om3);
    const float in3 = Om1 * (I[1][0] * Om1 + I[1][1] * Om2 + I[1][2] * Om3) - Om2 * (I[0][0] * Om1 + I[0][1] * Om2 + I[0][2] * Om3);
    const float M1 = -cmd.kR[0] * eR1 - cmd.kOm[0] * eOm1 + in1;
    const float M2 = -cmd.kR[1] * eR2 - cmd.kOm[1] * eOm2 + in2;
    const float M3 = -cmd.kR[2] * eR3 - cmd.kOm[2] * eOm3 + in3;
    float w_sq[4];
    w_sq[0] = force / (4 * kf) - M2 / (2 * d * kf) + M3 / (4 * km);
    w_sq[1] = force / (4 * kf) + M2 / (2 * d * kf) + M3 / (4 * km);
    w_sq[2] = force / (4 * kf) + M1 / (2 * d * kf) - M3 / (4 * km);
    w_sq[3] = force / (4 * kf) - M1 / (2 * d * kf) - M3 / (4 * km);
    for (int i = 0; i < 4; i++) {
        if (w_sq[i] < 0) w_sq[i] = 0;
        rpm[i] = sqrtf(w_sq[i]);
    }
}

double norm3(const double v[3]) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// SO3Control::calculateControl with yaw 0 -> force, orientation (w, x, y, z)
void calculate_control(const isdf_sim_params *p, const double pos[3], const double vel[3], const double acc[3], const double dp[3],
                       const double dv[3], const double da[3], double force[3], double quat[4]) {
    const double m = p->ctrl_mass, g = p->ctrl_grav;
    const bool use_p = !(std::isnan(dp[0]) || std::isnan(dp[1]) || std::isnan(dp[2]));
    const bool use_v = !(std::isnan(dv[0]) || std::isnan(dv[1]) || std::isnan(dv[2]));
    const bool use_a = !(std::isnan(da[0]) || std::isnan(da[1]) || std::isnan(da[2]));
    double te[3] = {0, 0, 0};
    for (int i = 0; i < 3; i++) {
        if (use_p) te[i] += dp[i] - pos[i];
        if (use_v) te[i] += dv[i] - vel[i];
        if (use_a) te[i] += da[i] - acc[i];
    }
    double ka[3];
    for (int i = 0; i < 3; i++) ka[i] = std::fabs(te[i]) > 3 ? 0 : (std::fabs(te[i]) * 0.2);
    const double e3[3] = {0, 0, 1};
    for (int i = 0; i < 3; i++) force[i] = m * g * e3[i];
    for (int i = 0; i < 3; i++) {
        if (use_p) force[i] += p->kx[i] * (dp[i] - pos[i]);
        if (use_v) force[i] += p->kv[i] * (dv[i] - vel[i]);
        if (use_a) force[i] += m * ka[i] * (da[i] - acc[i]) + m * da[i];
    }
    const double theta = M_PI / 2;
    const double c = std::cos(theta);
    double f[3];
    for (int i = 0; i < 3; i++) f[i] = force[i] - m * g * e3[i];
    const double fn = norm3(force);
    if (0.0 * (force[0] / fn) + 0.0 * (force[1] / fn) + 1.0 * (force[2] / fn) < c) {
        const double nf = norm3(f);
        const double A = c * c * nf * nf - f[2] * f[2];
        const double B = 2 * (c * c - 1) * f[2] * m * g;
        const double C = (c * c - 1) * m * m * g * g;
        const double s = (-B + std::sqrt(B * B - 4 * A * C)) / (2 * A);
        for (int i = 0; i < 3; i++) force[i] = s * f[i] + m * g * e3[i];
    }
    double b3[3], b2[3], b1[3];
    const double b1d[3] = {std::cos(0.0), std::sin(0.0), 0};
    const double fn2 = norm3(force);
    if (fn2 > 1e-6) for (int i = 0; i < 3; i++) b3[i] = force[i] / fn2;
    else { b3[0] = 0; b3[1] = 0; b3[2] = 1; }
    double cr[3] = {b3[1] * b1d[2] - b3[2] * b1d[1], b3[2] * b1d[0] - b3[0] * b1d[2], b3[0] * b1d[1] - b3[1] * b1d[0]};
    double n = cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2];
    for (int i = 0; i < 3; i++) b2[i] = n > 0 ? cr[i] / std::sqrt(n) : cr[i];
    double cr2[3] = {b2[1] * b3[2] - b2[2] * b3[1], b2[2] * b3[0] - b2[0] * b3[2], b2[0] * b3[1] - b2[1] * b3[0]};
    n = cr2[0] * cr2[0] + cr2[1] * cr2[1] + cr2[2] * cr2[2];
    for (int i = 0; i < 3; i++) b1[i] = n > 0 ? cr2[i] / std::sqrt(n) : cr2[i];
    const double Rm[9] = {b1[0], b2[0], b3[0], b1[1], b2[1], b3[1], b1[2], b2[2], b3[2]};
    R_to_quat(Rm, quat);
}

// tf::getYaw(Quaterniond): Matrix3x3(q).getEulerYPR, solution 1
double tf_yaw(const double q[4]) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double dd = x * x + y * y + z * z + w * w;
    const double s = 2.0 / dd;
    const double ys = y * s, zs = z * s;
    const double wz = w * zs, wy = w * ys;
    const double xy = x * ys, xz = x * zs, yy = y * ys, zz = z * zs;
    const double m00 = 1.0 - (yy + zz), m10 = xy + wz, m20 = xz - wy;
    if (std::fabs(m20) >= 1) return 0.0;
    const double pitch = -std::asin(m20);
    return std::atan2(m10 / std::cos(pitch), m00 / std::cos(pitch));
}

void poison(isdf_sim_summary &s) {
    s.max_err = s.t_max_err = s.rms_err = s.final_err = s.max_tilt = s.max_omega = s.t_diverged = NaN;
    s.accepted = s.rejected = -1;
    s.clamped_steps = s.floor_contacts = s.nan_rollbacks = -1;
    s.diverged = 1;
}

}  // namespace

extern "C" {

// one rollout of the closed loop: log (cap_log x 21, may be NULL) and summary. n_ticks and m = sim_rate / cmd_rate come from the caller.
void sim_rollout(const isdf_sim_params *p, int N, const double *T, const double *C, const double *init, const double *dist, int n_ticks,
                 int m, int cap_log, double *log, isdf_sim_summary *out) {
    isdf_sim_summary s;
    std::memset(&s, 0, sizeof(s));
    if (log) for (long long i = 0; i < (long long)cap_log * ISDF_SIM_DOUBLES; i++) log[i] = NaN;
    if (N < 1) { poison(s); s.t_diverged = NaN; *out = s; return; }
    Traj tr = {T, C, N, 0.0};
    for (int i = 0; i < N; i++) tr.dur += T[i];
    Vehicle q;
    vehicle_init(q, p, dist);
    double x[22];
    for (int i = 0; i < 3; i++) { x[i] = init[i]; x[3 + i] = init[3 + i]; x[15 + i] = init[10 + i]; }
    double R0[9];
    quat_to_R(init[6], init[7], init[8], init[9], R0);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) x[6 + 3 * j + i] = R0[3 * i + j];
    for (int i = 0; i < 4; i++) x[18 + i] = init[13 + i];
    const double dt = 1 / p->sim_rate;
    Counters c;
    double des_p[3] = {NaN, NaN, NaN}, des_v[3] = {NaN, NaN, NaN}, des_a[3] = {NaN, NaN, NaN};
    Command cmd;
    double last_rpm[4] = {0, 0, 0, 0};
    double sum_sq = 0.0;
    s.max_err = -1.0; s.t_max_err = NaN; s.t_diverged = NaN; s.max_tilt = 0.0; s.max_omega = 0.0;
    int ticks = 0;
    for (int k = 0; k < n_ticks; k++) {
        if (k > 0) {
            bool ok = true;
            for (int st = 0; st < m && ok; st++) {
                double Rs[9];
                for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rs[3 * i + j] = x[6 + 3 * j + i];
                double rpm[4];
                get_control(p, Rs, x + 15, cmd, rpm);
                for (int i = 0; i < 4; i++) if (std::isnan(rpm[i])) rpm[i] = last_rpm[i];
                for (int i = 0; i < 4; i++) last_rpm[i] = rpm[i];
                if (set_input(q, rpm)) c.clamped++;
                ok = model_step(q, x, dt, p->floor, c);
            }
            if (!ok) { s.diverged = 1; s.t_diverged = (double)k / p->cmd_rate; break; }
        }
        const double tk = (double)k / p->cmd_rate;
        // odometry
        double Rs[9], quat[4];
        for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rs[3 * i + j] = x[6 + 3 * j + i];
        R_to_quat(Rs, quat);
        const double cur_yaw = tf_yaw(quat);
        // command
        if (tk < tr.dur) traj_pva(tr, tk, des_p, des_v, des_a);
        double force[3], oq[4];
        calculate_control(p, x, x + 3, q.acc, des_p, des_v, des_a, force, oq);
        for (int i = 0; i < 3; i++) {
            cmd.force[i] = (float)force[i]; cmd.kR[i] = (float)p->kR[i]; cmd.kOm[i] = (float)p->kOm[i];
            cmd.corrections[i] = (float)p->corrections[i];
        }
        cmd.qw = (float)oq[0]; cmd.qx = (float)oq[1]; cmd.qy = (float)oq[2]; cmd.qz = (float)oq[3];
        cmd.current_yaw = (float)cur_yaw;
        cmd.use_external_yaw = p->use_external_yaw;
        // the tick's record and statistics
        const double e[3] = {x[0] - des_p[0], x[1] - des_p[1], x[2] - des_p[2]};
        const double err = norm3(e);
        bool finite = true;
        for (int i = 0; i < 22; i++) finite = finite && std::isfinite(x[i]);
        if (log && k % p->log_every == 0 && k / p->log_every < cap_log) {
            double *r = log + (size_t)(k / p->log_every) * ISDF_SIM_DOUBLES;
            r[0] = tk;
            for (int i = 0; i < 3; i++) { r[1 + i] = x[i]; r[4 + i] = x[3 + i]; r[11 + i] = x[15 + i]; r[18 + i] = des_p[i]; }
            for (int i = 0; i < 4; i++) { r[7 + i] = quat[i]; r[14 + i] = x[18 + i]; }
        }
        ticks++;
        if (!finite || !(err <= p->diverge_dist)) { s.diverged = 1; s.t_diverged = tk; }
        if (err > s.max_err) { s.max_err = err; s.t_max_err = tk; }
        sum_sq += err * err;
        s.final_err = err;
        const double tilt = std::acos(std::fmin(1.0, std::fmax(-1.0, Rs[8])));
        if (tilt > s.max_tilt) s.max_tilt = tilt;
        const double on = norm3(x + 15);
        if (on > s.max_omega) s.max_omega = on;
        if (s.diverged) break;
    }
    if (ticks == 0) { s.max_err = s.final_err = s.rms_err = NaN; }
    else s.rms_err = std::sqrt(sum_sq / ticks);
    if (s.max_err < 0) s.max_err = NaN;
    s.accepted = c.acc; s.rejected = c.rej; s.clamped_steps = c.clamped; s.floor_contacts = c.floor; s.nan_rollbacks = c.rollbacks;
    *out = s;
}

// pieces of the model for unit tests --------------------------------------------------------------------------------------------
// the right-hand side at x with the given input and disturbance (dist may be NULL); acc (3) gets getAcc()
void sim_rhs(const isdf_sim_params *p, const double *x, const double *input, const double *dist, double *dx, double *acc) {
    Vehicle q;
    vehicle_init(q, p, dist);
    for (int i = 0; i < 4; i++) q.input[i] = input[i];
    rhs(q, x, dx);
    for (int i = 0; i < 3; i++) acc[i] = q.acc[i];
}

// n open-loop steps with a fixed commanded rpm (through setInput) from x (22, in place); counts: accepted, rejected, clamped, floor, rollbacks
int sim_open_loop(const isdf_sim_params *p, double *x, const double *rpm, const double *dist, int n, int64_t *counts) {
    Vehicle q;
    vehicle_init(q, p, dist);
    Counters c;
    const double dt = 1 / p->sim_rate;
    int ok = 1;
    for (int s = 0; s < n && ok; s++) {
        if (set_input(q, rpm)) c.clamped++;
        ok = model_step(q, x, dt, p->floor, c);
    }
    counts[0] = c.acc; counts[1] = c.rej; counts[2] = c.clamped; counts[3] = c.floor; counts[4] = c.rollbacks;
    return ok;
}

// getControl on a state's R (row-major 9) and omega; cmd_f: force[3], qw, qx, qy, qz, current_yaw (rounded to float as the simulator's
// Command); gains from p
void sim_get_control(const isdf_sim_params *p, const double *R, const double *omega, const double *cmd_f, double *rpm) {
    Command cmd;
    for (int i = 0; i < 3; i++) {
        cmd.force[i] = (float)cmd_f[i]; cmd.kR[i] = (float)p->kR[i]; cmd.kOm[i] = (float)p->kOm[i]; cmd.corrections[i] = (float)p->corrections[i];
    }
    cmd.qw = (float)cmd_f[3]; cmd.qx = (float)cmd_f[4]; cmd.qy = (float)cmd_f[5]; cmd.qz = (float)cmd_f[6];
    cmd.current_yaw = (float)cmd_f[7];
    cmd.use_external_yaw = p->use_external_yaw;
    get_control(p, R, omega, cmd, rpm);
}

// setInput of the model: the input the motors are driven to; returns whether it clamped
int sim_set_input(const isdf_sim_params *p, const double *rpm, double *input) {
    Vehicle q;
    vehicle_init(q, p, nullptr);
    const int cl = set_input(q, rpm);
    for (int i = 0; i < 4; i++) input[i] = q.input[i];
    return cl;
}

// SO3Control::calculateControl with yaw 0 -> force (3), orientation (w, x, y, z)
void sim_calculate_control(const isdf_sim_params *p, const double *pos, const double *vel, const double *acc, const double *dp, const double *dv,
                           const double *da, double *force, double *quat) {
    calculate_control(p, pos, vel, acc, dp, dv, da, force, quat);
}
}
