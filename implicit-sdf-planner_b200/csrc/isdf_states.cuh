// Executing a trajectory: the state at a time and the robot's body posed there.
//   k_traj_states : SweptVolumeManager::process (sw_manager.hpp:948-988) at one (trajectory, local time) per thread: getPos / getVel /
//                   getAcc / getJer (trajectory.hpp:545-563 locatePieceIdx, then the piece's running powers; the same arithmetic as
//                   traj_pvaj) and FlatnessMap::forward(vel, acc, jer, psi = 0, dpsi = 0, thr, quat, omg) (flatness.hpp:150-228).
//   k_pose_points : Shape::Transform(quat, trans) (Shape.hpp:753-757, 786-793) of caller-given body points at each state.
// Both are bit-identical restatements, so they are compiled only into the -fmad=false unit (isdf_api.cu).
#pragma once
#include "isdf_swept.cuh"

namespace isdf {

constexpr int STATE_DOUBLES = 20;   // pos[3] vel[3] acc[3] jer[3] quat[4] (w, x, y, z) omg[3] thr
constexpr int STATES_THREADS = 256;
constexpr int STATES_PAD = STATE_DOUBLES + 1;   // odd stride of a staged record: a half-warp's 8-byte shared stores hit 16 distinct bank pairs

struct FlatForwardParams { double mass, grav, dh_over_m, dv, cp, veps; };

// FlatnessMap::forward (flatness.hpp:150-228) with psi = dpsi = 0, operation by operation: cos(0.5 psi) = cos(psi) = 1 and
// sin(0.5 psi) = sin(psi) = 0 stay operands, so products with them keep the reference's signs of zero and its NaN propagation.
__device__ __forceinline__ void flat_forward_yaw0(const FlatForwardParams &f, d3 vel, d3 acc, d3 jer, double quat[4], double omg[3], double &thr) {
    const double c_half_psi = 1.0, s_half_psi = 0.0, c_psi = 1.0, s_psi = 0.0, dpsi = 0.0;
    const double v0 = vel.x, v1 = vel.y, v2 = vel.z, a0 = acc.x, a1 = acc.y, a2 = acc.z;
    const double cp_term = sqrt(v0 * v0 + v1 * v1 + v2 * v2 + f.veps);
    const double w_term = 1.0 + f.cp * cp_term;
    const double w0 = w_term * v0, w1 = w_term * v1, w2 = w_term * v2;
    const double zu0 = a0 + f.dh_over_m * w0, zu1 = a1 + f.dh_over_m * w1, zu2 = a2 + f.dh_over_m * w2 + f.grav;
    const double zu_sqr0 = zu0 * zu0, zu_sqr1 = zu1 * zu1, zu_sqr2 = zu2 * zu2;
    const double zu01 = zu0 * zu1, zu12 = zu1 * zu2, zu02 = zu0 * zu2;
    const double zu_sqr_norm = zu_sqr0 + zu_sqr1 + zu_sqr2;
    const double zu_norm = sqrt(zu_sqr_norm);
    const double z0 = zu0 / zu_norm, z1 = zu1 / zu_norm, z2 = zu2 / zu_norm;
    const double ng_den = zu_sqr_norm * zu_norm;
    const double ng00 = (zu_sqr1 + zu_sqr2) / ng_den, ng01 = -zu01 / ng_den, ng02 = -zu02 / ng_den;
    const double ng11 = (zu_sqr0 + zu_sqr2) / ng_den, ng12 = -zu12 / ng_den, ng22 = (zu_sqr0 + zu_sqr1) / ng_den;
    const double v_dot_a = v0 * a0 + v1 * a1 + v2 * a2;
    const double dw_term = f.cp * v_dot_a / cp_term;
    const double dw0 = w_term * a0 + dw_term * v0, dw1 = w_term * a1 + dw_term * v1, dw2 = w_term * a2 + dw_term * v2;
    const double dz_term0 = jer.x + f.dh_over_m * dw0, dz_term1 = jer.y + f.dh_over_m * dw1, dz_term2 = jer.z + f.dh_over_m * dw2;
    const double dz0 = ng00 * dz_term0 + ng01 * dz_term1 + ng02 * dz_term2;
    const double dz1 = ng01 * dz_term0 + ng11 * dz_term1 + ng12 * dz_term2;
    const double dz2 = ng02 * dz_term0 + ng12 * dz_term1 + ng22 * dz_term2;
    const double f_term0 = f.mass * a0 + f.dv * w0, f_term1 = f.mass * a1 + f.dv * w1, f_term2 = f.mass * (a2 + f.grav) + f.dv * w2;
    thr = z0 * f_term0 + z1 * f_term1 + z2 * f_term2;
    const double tilt_den = sqrt(2.0 * (1.0 + z2));
    const double tilt0 = 0.5 * tilt_den, tilt1 = -z1 / tilt_den, tilt2 = z0 / tilt_den;
    quat[0] = tilt0 * c_half_psi;
    quat[1] = tilt1 * c_half_psi + tilt2 * s_half_psi;
    quat[2] = tilt2 * c_half_psi - tilt1 * s_half_psi;
    quat[3] = tilt0 * s_half_psi;
    const double omg_den = z2 + 1.0;
    const double omg_term = dz2 / omg_den;
    omg[0] = dz0 * s_psi - dz1 * c_psi - (z0 * s_psi - z1 * c_psi) * omg_term;
    omg[1] = dz0 * c_psi + dz1 * s_psi - (z0 * c_psi + z1 * s_psi) * omg_term;
    omg[2] = (z1 * dz0 - z0 * dz1) / omg_den + dpsi;
}

// One record per query. Trajectory b of the ragged layout has pieces [off[b], off[b+1]), durations T + off[b] and its own 6N x 3 column-major
// block at C + 18 off[b]; an index outside [0, B) or a trajectory without pieces gives an all-NaN record. Each warp stages its 32 records in
// shared memory and writes them as 20 contiguous 256-byte runs (one record per thread would store at a 160-byte stride).
__global__ void __launch_bounds__(STATES_THREADS) k_traj_states(const int *off, const double *T, const double *C, int B, long long Q,
                                                                const int *traj, const double *times, const FlatForwardParams fp, double *out) {
    __shared__ double stage[STATES_THREADS / 32][32 * STATES_PAD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *s = stage[warp];
    for (long long base = ((long long)blockIdx.x * STATES_THREADS + warp * 32); base < Q; base += (long long)gridDim.x * STATES_THREADS) {
        const long long q = base + lane;
        double r[STATE_DOUBLES];
#pragma unroll
        for (int k = 0; k < STATE_DOUBLES; k++) r[k] = __longlong_as_double(0x7ff8000000000000ll);
        if (q < Q) {
            const int b = traj[q];
            if (b >= 0 && b < B) {
                const int p0 = off[b], n = off[b + 1] - p0;
                if (n > 0) {
                    const TrajView tr = {T + p0, C + 18 * (size_t)p0, n};
                    d3 p, v, a, j;
                    traj_pvaj(tr, times[q], p, v, a, j);
                    r[0] = p.x; r[1] = p.y; r[2] = p.z; r[3] = v.x; r[4] = v.y; r[5] = v.z;
                    r[6] = a.x; r[7] = a.y; r[8] = a.z; r[9] = j.x; r[10] = j.y; r[11] = j.z;
                    flat_forward_yaw0(fp, v, a, j, r + 12, r + 16, r[19]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < STATE_DOUBLES; k++) s[lane * STATES_PAD + k] = r[k];
        __syncwarp();
        const long long nrec = Q - base < 32 ? Q - base : 32;
        double *dst = out + base * STATE_DOUBLES;
#pragma unroll 4
        for (int e = lane; e < nrec * STATE_DOUBLES; e += 32) {
            const int rec = e / STATE_DOUBLES;
            dst[e] = s[rec * STATES_PAD + (e - rec * STATE_DOUBLES)];
        }
        __syncwarp();
    }
}

// ---- the rest of a trajectory from t0 (isdf_trajectory_shift) ------------------------------------------------------------------------
// per trajectory b: the piece first[b] and local time tau[b] of t0[b] (traj_locate), and the pieces cnt[b] of the rest: 0 when t0 is not in
// [0, D) (D the left-to-right sum of T), not finite, or the trajectory has no piece; piece first[b] counts when T_i - tau > 0. out_off[0] = 0.
__global__ void k_shift_locate(int B, const int *off, const double *T, const double *t0, int *cnt, int *first, double *tau, int *out_off) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) out_off[0] = 0;
    if (b >= B) return;
    const int p0 = off[b], n = off[b + 1] - p0;
    double D = 0.0;
    for (int i = 0; i < n; i++) D += T[p0 + i];
    double t = t0[b];
    int c = 0, i = 0;
    if (n > 0 && t >= 0.0 && t < D) {   // false for NaN; t < D excludes +Inf
        const TrajView tr = {T + p0, nullptr, n};
        i = traj_locate(tr, t);
        c = (n - i - 1) + (T[p0 + i] - t > 0.0 ? 1 : 0);
    }
    cnt[b] = c; first[b] = i; tau[b] = t;
}

// one warp per trajectory: the rest's pieces at out_off[b], piece first[b] re-expanded about tau when kept, the later ones copied. Output
// piece k of N' pieces has coefficient r of axis a at out_C + 18 out_off[b] + 6 (a N' + k) + r (6N' x 3 column-major).
__global__ void k_shift_write(int B, const int *off, const double *T, const double *C, const int *cnt, const int *first, const double *tau,
                              const int *out_off, double *out_T, double *out_C) {
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= B) return;
    const int b = (int)w, n2 = cnt[b];
    if (n2 == 0) return;
    const int p0 = off[b], n = off[b + 1] - p0, i = first[b], o = out_off[b];
    const int skip = (n - i) - n2;   // 1 when piece i is dropped (t0 on its end)
    const double *Cb = C + 18 * (size_t)p0;
    double *Co = out_C + 18 * (size_t)o;
    // the copied pieces: output piece k is input piece i + skip + k, from k = 1 (k = 0 when piece i is dropped); 19 doubles per piece
    const int kfirst = skip ? 0 : 1;
    for (int e = lane; e < (n2 - kfirst) * 19; e += 32) {
        const int k = kfirst + e / 19, r = e % 19, src = i + skip + k;
        if (r == 18) out_T[o + k] = T[p0 + src];
        else {
            const int a = r / 6, m = r % 6;
            Co[6 * (a * n2 + k) + m] = Cb[6 * (a * n + src) + m];
        }
    }
    if (skip || lane >= 3) return;
    // piece i about tau, one axis per lane: d_k = sum_{j=k..5} (C(j,k) c_j) tau^(j-k), ascending j, tau^m the running product
    const double t = tau[b];
    const double binom[6][6] = {{1, 0, 0, 0, 0, 0}, {1, 1, 0, 0, 0, 0}, {1, 2, 1, 0, 0, 0}, {1, 3, 3, 1, 0, 0}, {1, 4, 6, 4, 1, 0}, {1, 5, 10, 10, 5, 1}};
    double pw[6];
    pw[0] = 1.0;
    for (int m = 1; m < 6; m++) pw[m] = pw[m - 1] * t;
    const double *c = Cb + 6 * (lane * n + i);
    for (int k = 0; k < 6; k++) {
        double d = 0.0;
        for (int j = k; j < 6; j++) d += (binom[j][k] * c[j]) * pw[j - k];
        Co[6 * (lane * n2) + k] = d;
    }
    if (lane == 0) out_T[o] = T[p0 + i] - t;
}

constexpr int POSE_THREADS = 256;
constexpr int POSE_MAX_STATES = 256;   // states per CTA
constexpr long long POSE_TARGET = 8192;   // output doubles a CTA aims for: enough stores in flight per CTA, few CTAs for small P

// out[(q P + p) 3 + k] = ((R_k0 b0 + R_k1 b1) + R_k2 b2) + pos_k, R = quat_rot(quat_q) (Eigen's toRotationMatrix): Shape::Transform.
// CTA g poses states [g S, g S + S): R and pos of each once into shared memory, then consecutive threads write consecutive output doubles of
// that contiguous S P 3 range. Each thread steps its (state, point, axis) by the block size without a division.
__global__ void __launch_bounds__(POSE_THREADS) k_pose_points(long long Q, const double *states, int P, const double *body, int S,
                                                              double *out) {
    __shared__ double rp[POSE_MAX_STATES][12];   // rows of R, then pos
    const long long L = 3ll * P;
    const long long groups = (Q + S - 1) / S;
    const int dq = (int)(POSE_THREADS / L), dr = (int)(POSE_THREADS % L), dp = dr / 3, dk = dr % 3;
    for (long long g = blockIdx.x; g < groups; g += gridDim.x) {
        const long long q0 = g * S;
        const int ns = (int)(Q - q0 < S ? Q - q0 : S);
        __syncthreads();
        for (int i = threadIdx.x; i < ns; i += POSE_THREADS) {
            const double *st = states + (q0 + i) * STATE_DOUBLES;
            quat4 qq; qq.w = st[12]; qq.x = st[13]; qq.y = st[14]; qq.z = st[15];
            const rot3 R = quat_rot(qq);
            double *d = rp[i];
            d[0] = R.r0.x; d[1] = R.r0.y; d[2] = R.r0.z; d[3] = R.r1.x; d[4] = R.r1.y; d[5] = R.r1.z;
            d[6] = R.r2.x; d[7] = R.r2.y; d[8] = R.r2.z; d[9] = st[0]; d[10] = st[1]; d[11] = st[2];
        }
        __syncthreads();
        const long long n = (long long)ns * L;
        double *dst = out + q0 * L;
        int s = (int)(threadIdx.x / L), r = (int)(threadIdx.x % L), p = r / 3, k = r % 3;
        for (long long e = threadIdx.x; e < n; e += POSE_THREADS) {
            const double *d = rp[s];
            const double *b = body + 3 * (size_t)p;
            dst[e] = ((d[3 * k] * b[0] + d[3 * k + 1] * b[1]) + d[3 * k + 2] * b[2]) + d[9 + k];
            s += dq; p += dp; k += dk;
            if (k >= 3) { k -= 3; p++; }
            if (p >= P) { p -= P; s++; }
        }
    }
}

}  // namespace isdf
