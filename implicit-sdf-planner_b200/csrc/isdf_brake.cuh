// Braking to a certified stop along the remaining trajectory (isdf_trajectory_brake, DESIGN §3.21).
//   k_brake_setup  : one thread per (trajectory, candidate): head, tail, durations and waypoints of the candidate in k_minco_forward's layout;
//   k_minco_forward: the candidates' MINCO S3 solve with the durations given (MincoArgs::T_in);
//   the clearance and dynamic-limit certificates over all candidates (N0 = M), then
//   k_brake_select : one thread per trajectory: the largest candidate that is CERTIFIED and FEASIBLE, its summary and piece count;
//   a scan of the counts into the output offsets, and
//   k_brake_write  : one warp per trajectory: the chosen candidate's pieces into the ragged output.
// The schedule is a definition restated bit for bit (tests/brake_oracle.py), so this header is compiled only into the -fmad=false unit.
#pragma once
#include "isdf_states.cuh"
#include "isdf_certify.cuh"
#include "isdf_dynlimits.cuh"

namespace isdf {

constexpr int BRAKE_NO_INPUT = -1, BRAKE_NONE = 0, BRAKED = 1;   // isdf_brake_status

struct BrakeSummary {   // isdf_brake_summary
    int status, candidate;
    double tau_stop, duration;
    int certified, feasible;
    CertSummary cert;
    DynSummary dyn;
};

// tau_max of trajectory b (include/isdf.h): min(t_stop_max, D) with D the left-to-right sum of T; NaN when there is no input
__device__ __forceinline__ double brake_tau_max(const int *off, const double *T, const double *t_stop_max, int b) {
    const int p0 = off[b], n = off[b + 1] - p0;
    double D = 0.0;
    for (int i = 0; i < n; i++) D += T[p0 + i];
    const double ts = t_stop_max[b];
    const double tm = ts < D ? ts : D;
    const bool ok = n > 0 && ts == ts && tm > 0.0 && tm < __longlong_as_double(0x7ff0000000000000ll);
    return ok ? tm : __longlong_as_double(0x7ff8000000000000ll);
}

// candidate q = b K + k: head and tail (3x3 column-major, columns p, v, a; 9 per candidate), its M durations at Tin + q M and its
// decision vector at x + q (4M - 3) ([M unused duration slots | 3 (M - 1) waypoints]). Without an input the candidate rests at `rest`
// with unit durations.
__global__ void k_brake_setup(int B, int K, int M, const int *off, const double *T, const double *C, const double *t_stop_max, double rx,
                              double ry, double rz, double *head, double *tail, double *Tin, double *x) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (long long)B * K) return;
    const int b = (int)(q / K), k = (int)(q - (long long)b * K);
    const double tm = brake_tau_max(off, T, t_stop_max, b);
    double *h = head + 9 * q, *t = tail + 9 * q, *d = Tin + (size_t)q * M, *xq = x + (size_t)q * (4 * M - 3);
    for (int i = 0; i < M; i++) xq[i] = 0.0;
    if (!(tm == tm)) {
        const double r[3] = {rx, ry, rz};
        for (int ax = 0; ax < 3; ax++) {
            h[ax] = r[ax]; t[ax] = r[ax];
            h[3 + ax] = 0.0; h[6 + ax] = 0.0; t[3 + ax] = 0.0; t[6 + ax] = 0.0;
            for (int j = 1; j < M; j++) xq[M + 3 * (j - 1) + ax] = r[ax];
        }
        for (int i = 0; i < M; i++) d[i] = 1.0;
        return;
    }
    const int p0 = off[b];
    const TrajView tr = {T + p0, C + 18 * (size_t)p0, off[b + 1] - p0};
    const double tau = tm * ((double)(k + 1) / (double)K);
    d3 p, v, a, j3;
    traj_pvaj(tr, 0.0, p, v, a, j3);
    h[0] = p.x; h[1] = p.y; h[2] = p.z; h[3] = v.x; h[4] = v.y; h[5] = v.z; h[6] = a.x; h[7] = a.y; h[8] = a.z;
    traj_pvaj(tr, tau, p, v, a, j3);
    t[0] = p.x; t[1] = p.y; t[2] = p.z;
    for (int e = 3; e < 9; e++) t[e] = 0.0;
    const double dur = (tau + tau) / (double)M;
    for (int i = 0; i < M; i++) d[i] = dur;
    for (int j = 1; j < M; j++) {
        const double u = (double)(M - j) / (double)M;
        const double f = 1.0 - u * u;
        traj_pvaj(tr, tau * f, p, v, a, j3);
        double *w = xq + M + 3 * (j - 1);
        w[0] = p.x; w[1] = p.y; w[2] = p.z;
    }
}

// per trajectory: the largest k whose candidate is CERTIFIED (cs[q].verdict == 1) and FEASIBLE (ds[q].verdict == 1); summary, piece count
// cnt[b] (M or 0) and chosen candidate pick[b]; out_off[0] = 0
__global__ void k_brake_select(int B, int K, int M, const int *off, const double *T, const double *t_stop_max, const double *Tc,
                               const CertSummary *cs, const DynSummary *ds, const CertSummary cbad, const DynSummary dbad, BrakeSummary *sum,
                               int *cnt, int *pick, int *out_off) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b == 0) out_off[0] = 0;
    if (b >= B) return;
    const double tm = brake_tau_max(off, T, t_stop_max, b);
    BrakeSummary s;
    s.status = BRAKE_NO_INPUT; s.candidate = -1;
    s.tau_stop = s.duration = __longlong_as_double(0x7ff8000000000000ll);
    s.certified = s.feasible = 0;
    s.cert = cbad; s.dyn = dbad;
    if (tm == tm) {
        s.status = BRAKE_NONE;
        for (int k = 0; k < K; k++) {
            const long long q = (long long)b * K + k;
            const bool ck = cs[q].verdict == 1, dk = ds[q].verdict == 1;
            s.certified += ck; s.feasible += dk;
            if (ck && dk) s.candidate = k;
        }
        if (s.candidate >= 0) {
            const long long q = (long long)b * K + s.candidate;
            s.status = BRAKED;
            s.tau_stop = tm * ((double)(s.candidate + 1) / (double)K);
            double D = 0.0;
            for (int i = 0; i < M; i++) D += Tc[(size_t)q * M + i];
            s.duration = D;
            s.cert = cs[q]; s.dyn = ds[q];
        }
    }
    sum[b] = s;
    cnt[b] = s.status == BRAKED ? M : 0;
    pick[b] = s.candidate;
}

// one warp per braked trajectory: candidate q's M pieces from the concatenated block (piece q M + i of a 6 P x 3 column-major block,
// P = B K M) into out_T / out_C at out_off[b] (its own 6M x 3 column-major block)
__global__ void k_brake_write(int B, int K, int M, const int *pick, const double *Tc, const double *Cc, const int *out_off, double *out_T,
                              double *out_C) {
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= B) return;
    const int b = (int)w, k = pick[b];
    if (k < 0) return;
    const size_t q = (size_t)b * K + k, rows = (size_t)6 * B * K * M;
    const int o = out_off[b];
    for (int e = lane; e < 19 * M; e += 32) {
        const int i = e / 19, r = e - 19 * i;
        if (r == 18) out_T[o + i] = Tc[q * M + i];
        else {
            const int a = r / 6, m = r - 6 * a;
            out_C[18 * (size_t)o + 6 * (a * M + i) + m] = Cc[(size_t)a * rows + 6 * (q * M + i) + m];
        }
    }
}

}  // namespace isdf
