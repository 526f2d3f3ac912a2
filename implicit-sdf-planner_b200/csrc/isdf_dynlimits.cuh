// Dynamic-limit certificate (isdf_trajectory_dynamics, include/isdf.h): proven bounds of speed, acceleration, body rate, tilt and thrust
// over every time of a trajectory, from the clearance check's samples and interval refinement.
//
// Six channels, every one a maximum: 0 |v|, 1 |a|, 2 |omega|, 3 tilt, 4 thrust, 5 -thrust (its maximum is minus the thrust minimum).
//   Interval [ta, tb] of piece i: the polynomial re-expanded about te = ta + 0.5 (tb - ta) (Taylor coefficients d_k as enclosures),
//   v = d_1 + [-1, 1] sum_{k>=2} k |d_k| h^(k-1), a and j likewise, h = sup |t - te|; then every quantity in outward-rounded interval
//   arithmetic (dyn_channels). The same evaluation at h = 0, te = t encloses the exact value at a sample: its lower end is proven attained.
//   Division by an enclosure reaching 0 (|zu|, 1 + z_z, and s when speed_eps = 0) makes the affected channels [0, +inf] (tilt: [0, pi],
//   thrust: [-|F|, |F|]).
//
// Rounds (host loop in isdf_api.cu): k_dyn_decide, k_dyn_emit, one 4-byte read of the number of splits.
//   * k_dyn_decide — one CTA per trajectory over its contiguous, time-ordered segment of active intervals: first the samples made in the
//     previous round fold into the running maxima (value, then earliest time), then every interval is bounded, classified against the
//     updated maxima and ranked (the first intervals in order that want to split get the remaining samples). The last CTA to finish
//     (ticket) turns the per-trajectory split counts into offsets.
//   * k_dyn_emit — one thread per active interval: children and the midpoint sample, whose point enclosure is evaluated there.
// A trajectory's result depends only on its own intervals and samples: the same bits alone or inside a batch.
#pragma once
#include "isdf_types.cuh"
#include "isdf_interval.cuh"
#include "isdf_certify.cuh"

namespace isdf {

constexpr int DYN_THREADS = 256;
constexpr int DYN_CH = 6;
constexpr double DYN_ACOS_PAD = 0x1p-49;   // relative pad of acos: 8 ulp, CUDA documents at most 2

struct DynSample { double t, q[DYN_CH]; int piece, pad; };   // t: local time; q: lower ends of the point enclosure, NaN: not finite
static_assert(sizeof(DynSample) == 64, "sample record");
struct DynTraj {
    double up[DYN_CH], att[DYN_CH], tatt[DYN_CH];
    int bad, used, undecided, depth, seg_off, seg_cnt, split_pref, nsplit;
};
// one per trajectory; layout of isdf_dynamics_summary
struct DynSummary {
    double upper[5], attained[5], t_attained[5];
    double thrust_lower, thrust_attained_min, t_thrust_attained_min;
    int verdict, violated, undecided, samples, undecided_intervals, depth;
};
static_assert(sizeof(DynSummary) == 168, "isdf_dynamics_summary layout");

struct DynArgs {
    FlatParams fp;
    double mass, dv;                       // vehicle_mass, vert_drag: the thrust's FlatnessMap::forward terms
    double lim[DYN_CH], tol[DYN_CH];       // +inf: reported, not checked
    int N, K, N0, B, max_depth, max_samples;
    const double *T, *C;
    double *toff;                          // N: trajectory time at which each piece starts
    DynSample *smp;
    CertInterval *cur, *next;              // active intervals of the round / of the next round
    int *dec;                              // per active interval: split rank in its trajectory, -1 for a leaf
    DynTraj *traj;                         // B
    DynSummary *summary;                   // B
    int S_cur, nact;
    int *tot;                              // {splits of the round, ticket}
};

// enclosures of v, a, j of piece i over |t - te| <= h (C: 6N x 3 column-major); h = 0 encloses the exact values at te
__device__ __forceinline__ void dyn_vaj(const double *C, int N, int i, double te, double h, ivl v[3], ivl a[3], ivl j[3]) {
    double hp[5];   // h^0 .. h^4
    hp[0] = 1.0;
#pragma unroll
    for (int k = 1; k < 5; k++) hp[k] = __dmul_ru(hp[k - 1], h);
    ivl tp[6];
    tp[0] = iv(1.0);
#pragma unroll
    for (int k = 1; k < 6; k++) tp[k] = imul(tp[k - 1], iv(te));
#pragma unroll 1
    for (int ax = 0; ax < 3; ax++) {
        double c[6];
#pragma unroll
        for (int k = 0; k < 6; k++) c[k] = __ldg(C + 6 * N * ax + 6 * i + k);
        ivl d[6];
#pragma unroll
        for (int k = 1; k < 6; k++) d[k] = taylor_coeff(c, tp, k);
        double vr = 0.0, ar = 0.0, jr = 0.0;
#pragma unroll
        for (int k = 2; k < 6; k++) {
            const double m = imag(d[k]);
            vr = __dadd_ru(vr, __dmul_ru(__dmul_ru((double)k, m), hp[k - 1]));
            if (k >= 3) ar = __dadd_ru(ar, __dmul_ru(__dmul_ru((double)(k * (k - 1)), m), hp[k - 2]));
            if (k >= 4) jr = __dadd_ru(jr, __dmul_ru(__dmul_ru((double)(k * (k - 1) * (k - 2)), m), hp[k - 3]));
        }
        v[ax] = iwiden(d[1], vr);
        a[ax] = iwiden(imul(iv(2.0), d[2]), ar);
        j[ax] = iwiden(imul(iv(6.0), d[3]), jr);
    }
}

__device__ __forceinline__ ivl inorm(const ivl w[3]) { return isqrt(iadd(iadd(isqr(w[0]), isqr(w[1])), isqr(w[2]))); }

// the six channels (lo, hi) over the boxes v, a, j: |v|, |a|, |omega|, tilt, thrust, -thrust
__device__ __forceinline__ void dyn_channels(const DynArgs &A, const ivl v[3], const ivl a[3], const ivl j[3], double lo[DYN_CH], double hi[DYN_CH]) {
    const FlatParams &fp = A.fp;
    const ivl sv = iadd(iadd(isqr(v[0]), isqr(v[1])), isqr(v[2]));
    const ivl spd = isqrt(sv), acc = inorm(a);
    lo[0] = spd.lo; hi[0] = spd.hi; lo[1] = acc.lo; hi[1] = acc.hi;
    const ivl s = isqrt(iadd(sv, iv(fp.veps)));
    const ivl kap = iadd(iv(1.0), imul(iv(fp.cp), s));
    ivl zu[3], F[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const ivl w = imul(kap, v[k]);
        zu[k] = iadd(a[k], imul(iv(fp.dh_over_m), w));
        F[k] = iadd(imul(iv(A.mass), a[k]), imul(iv(A.dv), w));
    }
    zu[2] = iadd(zu[2], iv(fp.grav));
    F[2] = iadd(F[2], imul(iv(A.mass), iv(fp.grav)));
    const ivl n = inorm(zu);
    const double Fm = inorm(F).hi;   // |thrust| <= |F| since |z| = 1
    double th_lo = -Fm, th_hi = Fm, ti_lo = 0.0, ti_hi = __dmul_ru(3.141592653589793, 1.0 + DYN_ACOS_PAD), om_lo = 0.0, om_hi = INFINITY;
    if (n.lo > 0.0) {
        ivl z[3];
#pragma unroll
        for (int k = 0; k < 3; k++) z[k] = idivp(zu[k], n);
        const ivl th = iadd(iadd(imul(z[0], F[0]), imul(z[1], F[1])), imul(z[2], F[2]));
        th_lo = fmax(th_lo, th.lo); th_hi = fmin(th_hi, th.hi);
        const double zl = fmin(fmax(z[2].lo, -1.0), 1.0), zh = fmin(fmax(z[2].hi, -1.0), 1.0);   // z_z lies in [-1, 1]
        ti_lo = __dmul_rd(acos(zh), 1.0 - DYN_ACOS_PAD);
        ti_hi = __dmul_ru(acos(zl), 1.0 + DYN_ACOS_PAD);
        const ivl od = iadd(iv(1.0), z[2]);
        if (od.lo > 0.0 && (fp.cp == 0.0 || s.lo > 0.0)) {
            const ivl vda = iadd(iadd(imul(v[0], a[0]), imul(v[1], a[1])), imul(v[2], a[2]));
            const ivl lam = fp.cp == 0.0 ? iv(0.0) : idivp(imul(iv(fp.cp), vda), s);
            ivl xi[3];
#pragma unroll
            for (int k = 0; k < 3; k++) xi[k] = iadd(j[k], imul(iv(fp.dh_over_m), iadd(imul(kap, a[k]), imul(lam, v[k]))));
            const ivl zxi = iadd(iadd(imul(z[0], xi[0]), imul(z[1], xi[1])), imul(z[2], xi[2]));
            ivl dz[3];
#pragma unroll
            for (int k = 0; k < 3; k++) dz[k] = idivp(isub(xi[k], imul(z[k], zxi)), n);
            const ivl ot = idivp(dz[2], od);
            ivl om[3];
            om[0] = iadd(ineg(dz[1]), imul(z[1], ot));
            om[1] = isub(dz[0], imul(z[0], ot));
            om[2] = idivp(isub(imul(z[1], dz[0]), imul(z[0], dz[1])), od);
            const ivl o = inorm(om);
            om_lo = o.lo; om_hi = o.hi;
        }
    }
    lo[2] = om_lo; hi[2] = om_hi; lo[3] = ti_lo; hi[3] = ti_hi;
    lo[4] = th_lo; hi[4] = th_hi; lo[5] = -th_hi; hi[5] = -th_lo;
}

// point enclosure at local time t of piece i: lower ends into q; all NaN when v, a or j is not finite there
__device__ __forceinline__ void dyn_point(const DynArgs &A, int i, double t, double q[DYN_CH]) {
    ivl v[3], a[3], j[3];
    dyn_vaj(A.C, A.N, i, t, 0.0, v, a, j);
    bool fin = true;
#pragma unroll
    for (int k = 0; k < 3; k++) fin = fin && isfinite(v[k].lo + v[k].hi + a[k].lo + a[k].hi + j[k].lo + j[k].hi);
    double hi[DYN_CH];
    dyn_channels(A, v, a, j, q, hi);
    if (!fin)
#pragma unroll
        for (int c = 0; c < DYN_CH; c++) q[c] = nan("");
}

// upper ends of the interval enclosure over [ta, tb] of piece i; NaN reads +inf
__device__ __forceinline__ void dyn_bound(const DynArgs &A, int i, double ta, double tb, double hi[DYN_CH]) {
    const double te = ta + 0.5 * (tb - ta);
    const double h = fmax(fmax(__dadd_ru(tb, -te), __dadd_ru(te, -ta)), 0.0);
    ivl v[3], a[3], j[3];
    dyn_vaj(A.C, A.N, i, te, h, v, a, j);
    double lo[DYN_CH];
    dyn_channels(A, v, a, j, lo, hi);
#pragma unroll
    for (int c = 0; c < DYN_CH; c++) if (hi[c] != hi[c]) hi[c] = INFINITY;
}

#ifdef ISDF_CLEARANCE_TU
// initial samples (the clearance check's, piece-major) with their point enclosures and intervals; per-trajectory state, piece start times
__global__ void __launch_bounds__(DYN_THREADS) k_dyn_init(const __grid_constant__ DynArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x, K = A.K;
    if (k < A.N * (K + 1)) {
        const int i = k / (K + 1), j = k - i * (K + 1);
        const double step = A.T[i] * (1.0 / K);
        DynSample s;
        s.t = j * step; s.piece = i; s.pad = 0;
        dyn_point(A, i, s.t, s.q);
        A.smp[k] = s;
        if (j < K) {
            CertInterval I;
            I.ta = j * step; I.tb = (j + 1 == K) ? A.T[i] : (j + 1) * step;
            I.sa = k; I.sb = k + 1; I.piece = i; I.depth = 0; I.pad = 0;
            I.flags = CERT_FOLD_A | (j + 1 == K ? CERT_FOLD_B : 0);
            A.cur[i * K + j] = I;
        }
    }
    if (k < A.B) {
        double t = 0.0;
        for (int q = 0; q < A.N0; q++) { A.toff[k * A.N0 + q] = t; t += A.T[k * A.N0 + q]; }
        DynTraj s;
        for (int c = 0; c < DYN_CH; c++) { s.up[c] = -INFINITY; s.att[c] = -INFINITY; s.tatt[c] = INFINITY; }
        s.bad = s.used = s.undecided = s.depth = 0;
        s.seg_off = k * A.N0 * K; s.seg_cnt = A.N0 * K;
        s.split_pref = s.nsplit = 0;
        A.traj[k] = s;
    }
    if (k == 0) { A.tot[0] = 0; A.tot[1] = 0; }
}

// (value, time) maximum: larger value, ties to the earlier time
__device__ __forceinline__ bool dyn_key_more(double v, double t, double bv, double bt) { return v > bv || (v == bv && t < bt); }

__global__ void __launch_bounds__(DYN_THREADS) k_dyn_decide(const __grid_constant__ DynArgs A) {
    __shared__ int s_w[DYN_THREADS / 32];
    __shared__ double s_v[DYN_THREADS], s_t[DYN_THREADS];
    __shared__ int s_i[2][DYN_THREADS];
    __shared__ int s_bad, s_last;
    const int b = blockIdx.x, tid = threadIdx.x;
    const DynTraj Tr = A.traj[b];
    const int off = Tr.seg_off, cnt = Tr.seg_cnt;
    // 1. the samples of the previous round (each folded by exactly one interval: its flags)
    double kv[DYN_CH], kt[DYN_CH];
    int bad = 0;
#pragma unroll
    for (int c = 0; c < DYN_CH; c++) { kv[c] = -INFINITY; kt[c] = INFINITY; }
    auto fold = [&](int si) {
        const DynSample &S = A.smp[si];
        const double t = A.toff[S.piece] + S.t;
#pragma unroll
        for (int c = 0; c < DYN_CH; c++) {
            const double v = S.q[c];
            if (v != v) bad = 1;
            else if (dyn_key_more(v, t, kv[c], kt[c])) { kv[c] = v; kt[c] = t; }
        }
    };
    for (int k = tid; k < cnt; k += DYN_THREADS) {
        const CertInterval &I = A.cur[off + k];
        if (I.flags & CERT_FOLD_A) fold(I.sa);
        if (I.flags & CERT_FOLD_B) fold(I.sb);
    }
    if (tid == 0) s_bad = Tr.bad;
    __syncthreads();
    if (bad) s_bad = 1;
    double att[DYN_CH], tatt[DYN_CH];
#pragma unroll 1
    for (int c = 0; c < DYN_CH; c++) {
        s_v[tid] = kv[c]; s_t[tid] = kt[c];
        __syncthreads();
        for (int o = DYN_THREADS / 2; o > 0; o >>= 1) {
            if (tid < o && dyn_key_more(s_v[tid + o], s_t[tid + o], s_v[tid], s_t[tid])) { s_v[tid] = s_v[tid + o]; s_t[tid] = s_t[tid + o]; }
            __syncthreads();
        }
        att[c] = Tr.att[c]; tatt[c] = Tr.tatt[c];
        if (dyn_key_more(s_v[0], s_t[0], att[c], tatt[c])) { att[c] = s_v[0]; tatt[c] = s_t[0]; }
        __syncthreads();
    }
    const int tbad = s_bad;
    // 2. bounds, classification and ranks of the intervals
    int used = Tr.used, nsplit = 0, und = 0, dep = 0;
    double up[DYN_CH];
#pragma unroll
    for (int c = 0; c < DYN_CH; c++) up[c] = -INFINITY;
    for (int base = 0; base < cnt; base += DYN_THREADS) {
        const int k = base + tid;
        const bool valid = k < cnt;
        bool wants = false, open = false;
        double hi[DYN_CH];
        CertInterval I;
        if (valid) {
            I = A.cur[off + k];
            dyn_bound(A, I.piece, I.ta, I.tb, hi);
            bool need = false;
#pragma unroll
            for (int c = 0; c < DYN_CH; c++) {
                const bool over = hi[c] > A.lim[c];
                open = open || over;
                need = need || (over && att[c] <= A.lim[c]) || hi[c] > att[c] + A.tol[c];
            }
            const double m = I.ta + 0.5 * (I.tb - I.ta);
            wants = need && !tbad && I.depth < A.max_depth && I.ta < m && m < I.tb;
        }
        int total;
        const int rank = cert_block_scan(wants ? 1 : 0, total, s_w);
        const int allowed = max(A.max_samples - used, 0);
        const bool split = wants && rank < allowed;
        if (valid) {
            A.dec[off + k] = split ? nsplit + rank : -1;
            if (!split) {
#pragma unroll
                for (int c = 0; c < DYN_CH; c++) up[c] = fmax(up[c], hi[c]);
                und += open;
                dep = max(dep, I.depth);
            }
        }
        const int took = min(total, allowed);
        nsplit += took; used += took;
    }
    // block reductions: maxima, integer sums and maxima — independent of the thread schedule
    DynTraj s = Tr;
#pragma unroll 1
    for (int c = 0; c < DYN_CH; c++) {
        s_v[tid] = up[c];
        if (c == 0) { s_i[0][tid] = und; s_i[1][tid] = dep; }
        __syncthreads();
        for (int o = DYN_THREADS / 2; o > 0; o >>= 1) {
            if (tid < o) {
                s_v[tid] = fmax(s_v[tid], s_v[tid + o]);
                if (c == 0) { s_i[0][tid] += s_i[0][tid + o]; s_i[1][tid] = max(s_i[1][tid], s_i[1][tid + o]); }
            }
            __syncthreads();
        }
        s.up[c] = fmax(s.up[c], s_v[0]);
        s.att[c] = att[c]; s.tatt[c] = tatt[c];
        __syncthreads();
    }
    if (tid == 0) {
        s.bad = tbad;
        s.undecided += s_i[0][0];
        if (cnt > 0) s.depth = max(s.depth, s_i[1][0]);
        s.used = used; s.nsplit = nsplit;
        A.traj[b] = s;
        __threadfence();
        s_last = atomicAdd(A.tot + 1, 1) == A.B - 1;
    }
    __syncthreads();
    if (!s_last) return;
    // last CTA: split offsets of every trajectory (trajectory order) and the next round's segments
    __threadfence();
    int sp = 0;
    for (int base = 0; base < A.B; base += DYN_THREADS) {
        const int q = base + tid;
        const int ns = q < A.B ? __ldcg(&A.traj[q].nsplit) : 0;
        int ts;
        const int es = cert_block_scan(ns, ts, s_w);
        if (q < A.B) { A.traj[q].split_pref = sp + es; A.traj[q].seg_off = 2 * (sp + es); A.traj[q].seg_cnt = 2 * ns; }
        sp += ts;
    }
    if (tid == 0) { A.tot[0] = sp; A.tot[1] = 0; }
}

__global__ void __launch_bounds__(DYN_THREADS) k_dyn_emit(const __grid_constant__ DynArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.nact) return;
    const int d = A.dec[k];
    if (d < 0) return;
    const CertInterval I = A.cur[k];
    const int r = A.traj[I.piece / A.N0].split_pref + d, si = A.S_cur + r;
    const double m = I.ta + 0.5 * (I.tb - I.ta);
    DynSample s;
    s.t = m; s.piece = I.piece; s.pad = 0;
    dyn_point(A, I.piece, m, s.q);
    A.smp[si] = s;
    CertInterval L = I, R = I;
    L.tb = m; L.sb = si; L.depth = I.depth + 1; L.flags = 0;
    R.ta = m; R.sa = si; R.depth = I.depth + 1; R.flags = CERT_FOLD_A;
    A.next[2 * r] = L; A.next[2 * r + 1] = R;
}

__global__ void __launch_bounds__(DYN_THREADS) k_dyn_finish(const __grid_constant__ DynArgs A) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= A.B) return;
    const DynTraj s = A.traj[b];
    DynSummary o;
    int viol = 0, und = 0;
    for (int c = 0; c < DYN_CH; c++) {
        if (s.att[c] > A.lim[c]) viol |= 1 << c;
        else if (!(s.up[c] <= A.lim[c])) und |= 1 << c;
    }
    for (int c = 0; c < 5; c++) { o.upper[c] = s.up[c]; o.attained[c] = s.att[c]; o.t_attained[c] = s.tatt[c]; }
    o.thrust_lower = -s.up[5]; o.thrust_attained_min = -s.att[5]; o.t_thrust_attained_min = s.tatt[5];
    if (s.bad) {   // a sample that is not finite: no bound holds
        for (int c = 0; c < 5; c++) o.upper[c] = o.attained[c] = nan("");
        o.thrust_lower = o.thrust_attained_min = nan("");
    }
    o.verdict = (s.bad || viol) ? -1 : (und == 0 ? 1 : 0);
    o.violated = viol; o.undecided = s.bad ? 0 : und;
    o.samples = A.N0 * (A.K + 1) + s.used;
    o.undecided_intervals = s.undecided;
    o.depth = s.depth;
    A.summary[b] = o;
}
#endif  // ISDF_CLEARANCE_TU

// ---- launch interface (isdf_clearance_tu.cu) --------------------------------------------------------------------------------------
cudaError_t dyn_init_launch(const DynArgs &A, cudaStream_t st);
cudaError_t dyn_round_launch(const DynArgs &A, cudaStream_t st);    // k_dyn_decide + k_dyn_emit over A.nact intervals
cudaError_t dyn_finish_launch(const DynArgs &A, cudaStream_t st);

}  // namespace isdf
