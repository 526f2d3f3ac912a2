// ORACLE — TEST INFRASTRUCTURE ONLY.
// C ABI over the reference's own simulator objects, compiled UNMODIFIED from where they lie (oracle/sim.mk):
//   so3_quadrotor_simulator/src/dynamics/Quadrotor.cpp   Quadrotor::operator(), step, setInput, getAcc (odeint::integrate: the vendored
//                                                          integrate_adaptive with controlled_runge_kutta<runge_kutta_dopri5>)
//   so3_control/src/SO3Control.cpp                       SO3Control::calculateControl
//   so3_quadrotor_simulator/src/quadrotor_simulator_so3.cpp  its static getControl (this file #includes it; sim.mk renames its main)
//   utils/include/utils/trajectory.hpp                   Trajectory<5>, the closed-loop driver's command source
// against the stand-ins under oracle/_shim_sim (Eigen restated, Boost and ROS declared; see their headers). Parameters arrive as the
// library's isdf_sim_params so that both sides read the same numbers.
#include "quadrotor_simulator_so3.cpp"
#include "ode/boost/numeric/odeint.hpp"
#include <so3_control/SO3Control.h>
#include <utils/trajectory.hpp>
#include <cstdint>
#include <cstring>
#include <limits>
#include "../include/isdf.h"

namespace odeint = boost::numeric::odeint;
using QuadrotorSimulator::Quadrotor;
typedef Quadrotor::InternalState IState;

namespace {
const double NaN = std::numeric_limits<double>::quiet_NaN();

void configure(Quadrotor &q, const isdf_sim_params *p, const double *dist) {
    q.setMass(p->mass);
    q.setGravity(p->grav);
    q.setInertia(Eigen::Vector3d(p->J[0], p->J[1], p->J[2]).asDiagonal());
    q.setPropellerThrustCoefficient(p->kf);
    q.setPropellerMomentCoefficient(p->km);
    q.setArmLength(p->arm);
    q.setMotorTimeConstant(p->motor_tau);
    q.setMaxRPM(p->max_rpm);
    q.setMinRPM(p->min_rpm);
    q.setExternalForce(dist ? Eigen::Vector3d(dist[0], dist[1], dist[2]) : Eigen::Vector3d::Zero());
    q.setExternalMoment(dist ? Eigen::Vector3d(dist[3], dist[4], dist[5]) : Eigen::Vector3d::Zero());
}

void set_state(Quadrotor &q, const double *x) {   // the 22-double state, R column-major as the internal state holds it
    Quadrotor::State s;
    for (int i = 0; i < 3; i++) {
        s.x(i) = x[i]; s.v(i) = x[3 + i]; s.omega(i) = x[15 + i];
        for (int j = 0; j < 3; j++) s.R(i, j) = x[6 + 3 * j + i];
    }
    for (int i = 0; i < 4; i++) s.motor_rpm(i) = x[18 + i];
    q.setState(s);
}

void get_state(const Quadrotor &q, double *x) {
    const Quadrotor::State &s = q.getState();
    for (int i = 0; i < 3; i++) {
        x[i] = s.x(i); x[3 + i] = s.v(i); x[15 + i] = s.omega(i);
        for (int j = 0; j < 3; j++) x[6 + 3 * j + i] = s.R(i, j);
    }
    for (int i = 0; i < 4; i++) x[18 + i] = s.motor_rpm(i);
}

// the same Quadrotor behind a call counter; the 1 + 6 tries calls of one integrate_adaptive give its tries. cap: calls after which the
// run is abandoned (the library's bound of 100000 tries per step, which odeint does not have)
struct Counting {
    Quadrotor *q; long long calls, cap;
    void operator()(const IState &x, IState &dx, const double t) {
        if (++calls > cap) throw std::length_error("tries");
        (*q)(x, dx, t);
    }
};
// integrate_adaptive's observer: called at the start and after every accepted try
struct Accepted {
    long long calls;
    void operator()(const IState &, double) { calls++; }
};

// Quadrotor::step(dt) on q, with the accepted and rejected dopri5 tries counted by running the vendored integrate_adaptive with the same
// stepper on a counting copy first. Returns 1, 0 when odeint throws (1000 tries in one step), -1 at the library's 100000-try bound, with
// the tries counted as the library counts them: accepted ones from the observer, the rest rejected. (When odeint throws, the observer
// cannot tell whether the 1000th try was accepted, which the library counts as accepted: every case here that reaches that rule would
// differ by one there, and none does, see tests/test_gpu_sim_reference.py.)
// rollbacks / floors count steps whose integrated state had a NaN (step() restores the state before the step) and steps whose resulting
// state (integrated or restored) was below the floor and moving down, which step() puts on the floor. same: whether the counting run's
// integration is the one step() made, bit for bit (checked when step() neither rolled back nor clamped at the floor: the state step() left
// equals the counting run's state with R re-orthonormalised as step() does).
int counted_step(Quadrotor &q, double dt, long long &acc, long long &rej, int *same, int32_t *rollbacks, int32_t *floors) {
    Quadrotor copy = q;
    Counting cnt{&copy, 0, 1 + 6LL * 100000};
    double x0[22];
    get_state(q, x0);
    IState s;
    for (int i = 0; i < 22; i++) s[i] = x0[i];
    Accepted obs{0};
    int status = 1;
    try {
        const size_t steps = odeint::integrate_adaptive(odeint::controlled_runge_kutta<odeint::runge_kutta_dopri5<IState>>(), boost::ref(cnt), s,
                                                        0.0, dt, dt, boost::ref(obs));
        if ((long long)steps != obs.calls - 1) *same = 0;
    } catch (const std::overflow_error &) {
        status = 0;
    } catch (const std::length_error &) {
        status = -1;
    }
    const long long tries = (cnt.calls - 1) / 6, accepted = obs.calls - 1;
    acc += accepted;
    rej += tries - accepted;
    if (status != 1) return status;
    q.step(dt);
    bool nan = false;
    for (int i = 0; i < 22; i++) nan = nan || std::isnan(s[i]);
    const double *base = nan ? x0 : &s[0];
    const bool floor = base[2] < 0.0 && base[5] < 0;   // step() puts the vehicle on the floor
    *rollbacks += nan;
    *floors += floor;
    {
        double x[22];
        get_state(q, x);
        if (!nan && !floor) {   // the integrated state itself
            Eigen::Matrix3d Rm;
            for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Rm(i, j) = s[6 + 3 * j + i];
            Eigen::LLT<Eigen::Matrix3d> llt(Rm.transpose() * Rm);
            Eigen::Matrix3d P = llt.matrixL();
            Eigen::Matrix3d Rn = Rm * P.inverse();
            for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) s[6 + 3 * j + i] = Rn(i, j);
            bool eq = copy.getAcc() == q.getAcc();
            for (int i = 0; i < 22; i++) eq = eq && std::memcmp(&s[i], &x[i], sizeof(double)) == 0;
            if (!eq) *same = 0;
        }
    }
    return 1;
}

Command make_command(const isdf_sim_params *p, const double *force, const double *quat, double current_yaw) {
    Command c;
    for (int i = 0; i < 3; i++) {
        c.force[i] = (float)force[i]; c.kR[i] = (float)p->kR[i]; c.kOm[i] = (float)p->kOm[i]; c.corrections[i] = (float)p->corrections[i];
    }
    c.qw = (float)quat[0]; c.qx = (float)quat[1]; c.qy = (float)quat[2]; c.qz = (float)quat[3];
    c.current_yaw = (float)current_yaw;
    c.use_external_yaw = p->use_external_yaw != 0;
    return c;
}

// tf::getYaw(q): tf::Matrix3x3(q).getEulerYPR(yaw, pitch, roll), solution 1 (ROS tf is not part of the reference tree; restated)
double tf_yaw(const Eigen::Quaterniond &q) {
    const double d = q.x() * q.x() + q.y() * q.y() + q.z() * q.z() + q.w() * q.w();
    const double s = 2.0 / d;
    const double ys = q.y() * s, zs = q.z() * s;
    const double wz = q.w() * zs, wy = q.w() * ys;
    const double xy = q.x() * ys, xz = q.x() * zs, yy = q.y() * ys, zz = q.z() * zs;
    const double m00 = 1.0 - (yy + zz), m10 = xy + wz, m20 = xz - wy;
    if (std::fabs(m20) >= 1) return 0.0;
    const double pitch = -std::asin(m20);
    return std::atan2(m10 / std::cos(pitch), m00 / std::cos(pitch));
}
}  // namespace

extern "C" {
// Quadrotor::operator() at x with input rpm (through setInput, so clamped) and disturbance dist (NULL: none); acc gets getAcc()
void ref_sim_rhs(const isdf_sim_params *p, const double *x, const double *rpm, const double *dist, double *dx, double *acc) {
    Quadrotor q;
    configure(q, p, dist);
    q.setInput(rpm[0], rpm[1], rpm[2], rpm[3]);
    IState xs, d;
    for (int i = 0; i < 22; i++) xs[i] = x[i];
    q(xs, d, 0.0);
    for (int i = 0; i < 22; i++) dx[i] = d[i];
    for (int i = 0; i < 3; i++) acc[i] = q.getAcc()(i);
}

// one Quadrotor::step(1 / sim_rate) from x (22, in place) at input rpm; counts: accepted, rejected, same, rollbacks, floor contacts
int ref_sim_step(const isdf_sim_params *p, double *x, const double *rpm, const double *dist, int64_t *counts) {
    Quadrotor q;
    configure(q, p, dist);
    set_state(q, x);
    q.setInput(rpm[0], rpm[1], rpm[2], rpm[3]);
    long long acc = 0, rej = 0;
    int same = 1;
    int32_t rollbacks = 0, floors = 0;
    const int ok = counted_step(q, 1 / p->sim_rate, acc, rej, &same, &rollbacks, &floors);
    if (ok == 1) get_state(q, x);
    counts[0] = acc; counts[1] = rej; counts[2] = same; counts[3] = rollbacks; counts[4] = floors;
    return ok;
}

// setInput: the input the motors are driven to, read back through the right-hand side at rest with motor_time_constant 1 (input_ is private;
// rpm' = (input - 0) / 1 is the input exactly)
void ref_sim_set_input(const isdf_sim_params *p, const double *rpm, double *input) {
    Quadrotor q;
    configure(q, p, nullptr);
    q.setMotorTimeConstant(1.0);
    q.setInput(rpm[0], rpm[1], rpm[2], rpm[3]);
    IState xs, d;
    for (int i = 0; i < 22; i++) xs[i] = 0.0;
    xs[6] = xs[10] = xs[14] = 1.0;
    q(xs, d, 0.0);
    for (int i = 0; i < 4; i++) input[i] = d[18 + i];
}

// getControl on a state with R (row-major 9) and omega; cmd_f: force[3], qw, qx, qy, qz, current_yaw; gains, corrections and
// use_external_yaw from p
void ref_sim_get_control(const isdf_sim_params *p, const double *R, const double *omega, const double *cmd_f, double *rpm) {
    Quadrotor q;
    configure(q, p, nullptr);
    double x[22] = {0};
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) x[6 + 3 * j + i] = R[3 * i + j];
    for (int i = 0; i < 3; i++) x[15 + i] = omega[i];
    set_state(q, x);
    const Control c = getControl(q, make_command(p, cmd_f, cmd_f + 3, cmd_f[7]));
    for (int i = 0; i < 4; i++) rpm[i] = c.rpm[i];
}

// SO3Control::calculateControl with yaw 0, yaw_dot 0 -> force (3), orientation (w, x, y, z)
void ref_sim_calculate_control(const isdf_sim_params *p, const double *pos, const double *vel, const double *acc, const double *dp,
                               const double *dv, const double *da, double *force, double *quat) {
    SO3Control c;
    c.setMass(p->ctrl_mass);
    c.setGravity(p->ctrl_grav);
    c.setPosition(Eigen::Vector3d(pos[0], pos[1], pos[2]));
    c.setVelocity(Eigen::Vector3d(vel[0], vel[1], vel[2]));
    c.setAcc(Eigen::Vector3d(acc[0], acc[1], acc[2]));
    c.calculateControl(Eigen::Vector3d(dp[0], dp[1], dp[2]), Eigen::Vector3d(dv[0], dv[1], dv[2]), Eigen::Vector3d(da[0], da[1], da[2]), 0.0, 0.0,
                       Eigen::Vector3d(p->kx[0], p->kx[1], p->kx[2]), Eigen::Vector3d(p->kv[0], p->kv[1], p->kv[2]));
    const Eigen::Vector3d &f = c.getComputedForce();
    const Eigen::Quaterniond &o = c.getComputedOrientation();
    for (int i = 0; i < 3; i++) force[i] = f(i);
    quat[0] = o.w(); quat[1] = o.x(); quat[2] = o.y(); quat[3] = o.z();
}

// The closed loop of include/isdf.h ("closed loop", the Definition's Step, Attitude loop, Position loop and Horizon paragraphs) composed from
// the objects above: the one restated part of this library. Trajectory: N pieces, durations T, coefficients C in the library's layout
// (6N x 3 column-major, ascending powers). The reference floor is always on (p->floor is the library's switch); a rollout that reaches the
// library's 100000-try bound reads as diverged, where the reference itself would not return. same: 0 if any step's counting run differed
// from Quadrotor::step.
void ref_sim_rollout(const isdf_sim_params *p, int N, const double *T, const double *C, const double *init, const double *dist, int n_ticks,
                     int m, int cap_log, double *log, isdf_sim_summary *out, int *same) {
    isdf_sim_summary s;
    std::memset(&s, 0, sizeof(s));
    *same = 1;
    for (long long i = 0; i < (long long)cap_log * ISDF_SIM_DOUBLES; i++) log[i] = NaN;
    std::vector<double> durs(T, T + N);
    std::vector<Trajectory<5>::CoefficientMat> cm(N);
    for (int i = 0; i < N; i++)
        for (int d = 0; d < 3; d++)
            for (int k = 0; k < 6; k++) cm[i](d, 5 - k) = C[6 * N * d + 6 * i + k];
    Trajectory<5> traj(durs, cm);
    double dur = 0.0;
    for (int i = 0; i < N; i++) dur += T[i];
    Quadrotor q;
    configure(q, p, dist);
    double x[22];
    for (int i = 0; i < 3; i++) { x[i] = init[i]; x[3 + i] = init[3 + i]; x[15 + i] = init[10 + i]; }
    const Eigen::Matrix3d R0 = Eigen::Quaterniond(init[6], init[7], init[8], init[9]).toRotationMatrix();
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) x[6 + 3 * j + i] = R0(i, j);
    for (int i = 0; i < 4; i++) x[18 + i] = init[13 + i];
    set_state(q, x);
    const double dt = 1 / p->sim_rate;
    Eigen::Vector3d des_p(NaN, NaN, NaN), des_v(NaN, NaN, NaN), des_a(NaN, NaN, NaN), imu_acc = Eigen::Vector3d::Zero();
    Command cmd{};
    Control control{};
    long long acc = 0, rej = 0;
    double sum_sq = 0.0;
    s.max_err = -1.0; s.t_max_err = NaN; s.t_diverged = NaN;
    int ticks = 0;
    for (int k = 0; k < n_ticks; k++) {
        if (k > 0) {   // m simulator loop iterations (quadrotor_simulator_so3.cpp main)
            int ok = 1;
            for (int st = 0; st < m && ok == 1; st++) {
                const Control last = control;
                control = getControl(q, cmd);
                for (int i = 0; i < 4; i++) if (std::isnan(control.rpm[i])) control.rpm[i] = last.rpm[i];
                bool clamped = false;
                for (int i = 0; i < 4; i++) clamped = clamped || control.rpm[i] > p->max_rpm || control.rpm[i] < p->min_rpm;
                s.clamped_steps += clamped;
                q.setInput(control.rpm[0], control.rpm[1], control.rpm[2], control.rpm[3]);
                ok = counted_step(q, dt, acc, rej, same, &s.nan_rollbacks, &s.floor_contacts);
                imu_acc = q.getAcc();
            }
            if (ok != 1) { s.diverged = 1; s.t_diverged = (double)k / p->cmd_rate; break; }
        }
        const double tk = (double)k / p->cmd_rate;
        const Quadrotor::State &st = q.getState();
        const Eigen::Quaterniond oq(st.R);
        const double cur_yaw = tf_yaw(oq);
        if (tk < dur) { des_p = traj.getPos(tk); des_v = traj.getVel(tk); des_a = traj.getAcc(tk); }
        SO3Control ctl;
        ctl.setMass(p->ctrl_mass);
        ctl.setGravity(p->ctrl_grav);
        ctl.setPosition(st.x);
        ctl.setVelocity(st.v);
        ctl.setAcc(k > 0 ? imu_acc : Eigen::Vector3d::Zero());
        ctl.calculateControl(des_p, des_v, des_a, 0.0, 0.0, Eigen::Vector3d(p->kx[0], p->kx[1], p->kx[2]), Eigen::Vector3d(p->kv[0], p->kv[1], p->kv[2]));
        const Eigen::Vector3d &f = ctl.getComputedForce();
        const Eigen::Quaterniond &o = ctl.getComputedOrientation();
        const double fa[3] = {f(0), f(1), f(2)}, qa[4] = {o.w(), o.x(), o.y(), o.z()};
        cmd = make_command(p, fa, qa, cur_yaw);
        const double err = (st.x - des_p).norm();
        bool finite = true;
        get_state(q, x);
        for (int i = 0; i < 22; i++) finite = finite && std::isfinite(x[i]);
        if (k % p->log_every == 0 && k / p->log_every < cap_log) {
            double *r = log + (size_t)(k / p->log_every) * ISDF_SIM_DOUBLES;
            const double qv[4] = {oq.w(), oq.x(), oq.y(), oq.z()};
            r[0] = tk;
            for (int i = 0; i < 3; i++) { r[1 + i] = x[i]; r[4 + i] = x[3 + i]; r[11 + i] = x[15 + i]; r[18 + i] = des_p(i); }
            for (int i = 0; i < 4; i++) { r[7 + i] = qv[i]; r[14 + i] = x[18 + i]; }
        }
        ticks++;
        if (!finite || !(err <= p->diverge_dist)) { s.diverged = 1; s.t_diverged = tk; }
        if (err > s.max_err) { s.max_err = err; s.t_max_err = tk; }
        sum_sq += err * err;
        s.final_err = err;
        const double tilt = std::acos(std::fmin(1.0, std::fmax(-1.0, st.R(2, 2))));
        if (tilt > s.max_tilt) s.max_tilt = tilt;
        if (st.omega.norm() > s.max_omega) s.max_omega = st.omega.norm();
        if (s.diverged) break;
    }
    s.rms_err = ticks ? std::sqrt(sum_sq / ticks) : NaN;
    if (s.max_err < 0) s.max_err = NaN;
    s.accepted = acc; s.rejected = rej;
    *out = s;
}
}
