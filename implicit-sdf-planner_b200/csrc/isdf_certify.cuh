// Continuous clearance certificate (isdf_trajectory_certify, include/isdf.h): the clearance check's samples, then interval refinement
// with a sound motion bound until every interval between two samples is proven clear, a sample collides, or the budget runs out.
//
// Per interval [ta, tb] of piece i with endpoint samples (clearances c_a, c_b from k_clearance_scan):
//   D_e = P_e + r Q_e + eps_e bounds how far any body point moves over the interval from where it was at the endpoint's time t_e, so
//   lb = max(c_a - D_a, c_b - D_b) bounds the clearance at every t of the interval (DESIGN §3.11 has the derivation).
//   P_e   translation: the piece polynomial re-expanded about t_e (Taylor coefficients d_1..d_5 per axis), sum |d_k| h^k per axis,
//         Euclidean norm of the three; h = sup |t - t_e| over the interval (tb - ta except where a piece's last sample is not at T_i).
//   Q_e   rotation: v and a enclosed over the interval in Taylor form, the flatness map zu -> z -> R(z) in interval arithmetic, R(z) in
//         the closed form of the zero-yaw attitude; Q_e = Frobenius norm of the enclosure of R(z(t)) - R(z(t_e)). +inf when the
//         enclosure of |zu| or of 1 + z_z reaches 0.
//   eps_e the pose pad: 1e-10 (1 + A_e + 2H + (r + 2H) kappa_e / delta_e), A_e = sum |c_k| |t_e|^k, kappa_e the relative condition of
//         zu at t_e, delta_e = 1 + z_z at t_e; it covers the rounding of the scan's own pose and SDF (round-to-nearest, FMA).
//   Every operation of the bound is rounded outward (__dadd_rd/_ru, __dmul_rd/_ru, __ddiv_rd/_ru, __dsqrt_rd/_ru).
//
// Rounds (host loop in isdf_api.cu): k_clearance_scan over the round's new samples (sample-list mode; it also sets the trajectory's hit
// flag), k_certify_decide, k_certify_emit, one 4-byte read of the number of splits.
//   * k_certify_decide — one CTA per trajectory over its contiguous, time-ordered segment of active intervals: bounds, classification,
//     the per-trajectory budget (the first intervals in order that want to split get the remaining samples), ranks from a block scan,
//     and the trajectory's running minima and counts. Only that CTA touches the trajectory's state, so no atomics order anything; the
//     last CTA to finish (ticket) turns the per-trajectory split and leaf counts into offsets.
//   * k_certify_emit — one thread per active interval: children and midpoint samples at their compacted positions (trajectory order,
//     then interval order), finished intervals to the leaf list.
// A trajectory's result depends only on its own intervals and samples: the same bits alone or inside a batch.
#pragma once
#include "isdf_types.cuh"
#include "isdf_clearance.cuh"
#include "isdf_interval.cuh"

namespace isdf {

constexpr int CERT_THREADS = 256;
constexpr double CERT_EPS_REL = 1e-10;
enum { CERT_FOLD_A = 1, CERT_FOLD_B = 2 };             // the interval is the first to see its sample a / b: fold it into the minima
enum { LEAF_DROPPED = -1, LEAF_UNDECIDED = 0, LEAF_SAFE = 1 };

struct CertInterval { double ta, tb; int sa, sb, piece, depth, flags, pad; };
struct CertScratch { double Da, Db; int dec, state; };   // dec >= 0: split rank in the trajectory; < 0: ~leaf rank
// record of isdf_dbg_certify_leaves
struct CertLeaf { double ta, tb, ca, cb, Da, Db; int piece, state; };
static_assert(sizeof(CertLeaf) == 56, "leaf record");
struct CertTraj {
    double lb, min_clear, t_min, first_hit;
    long long voxel_min;
    int used, undecided, depth, seg_off, seg_cnt, split_pref, leaf_pref, nsplit, nleaf, pad;
};
// one per trajectory; layout of isdf_certify_summary
struct CertSummary {
    double lower_bound, min_clearance, t_min, first_hit;
    long long voxel_min;
    int verdict, samples, undecided, depth;
};
static_assert(sizeof(CertSummary) == 56, "isdf_certify_summary layout");

struct CertArgs {
    FlatParams fp;
    double r, H, margin;
    int N, K, N0, B, max_depth, max_samples;
    const double *T, *C;
    double *toff;                  // N: trajectory time at which each piece starts
    int *sp; double *st, *sc;      // samples: piece, local time, clearance
    long long *sv;                 // witness
    int *hit;                      // B
    CertInterval *cur, *next;   // active intervals of the round / of the next round
    CertScratch *scr;
    CertLeaf *leaves;
    CertTraj *traj;                // B
    CertSummary *summary;          // B
    int S_cur, L_cur, nact;
    int *tot;                      // {splits of the round, ticket}
};

// enclosure of the zero-yaw attitude R(z(v, a)) over boxes v, a (rows of R, 9 entries); false when |zu| or 1 + z_z may vanish.
// kappa (upper bound of (|a| + dh kap |v| + g) / |zu|) and delta (lower bound of 1 + z_z) feed the pose pad.
__device__ __forceinline__ bool cert_rot(const FlatParams &fp, const ivl v[3], const ivl a[3], ivl R[9], double &kappa, double &delta) {
    const ivl s = isqrt(iadd(iadd(iadd(isqr(v[0]), isqr(v[1])), isqr(v[2])), iv(fp.veps)));
    const ivl kap = iadd(iv(1.0), imul(iv(fp.cp), s));
    ivl zu[3];
#pragma unroll
    for (int k = 0; k < 3; k++) zu[k] = iadd(a[k], imul(iv(fp.dh_over_m), imul(kap, v[k])));
    zu[2] = iadd(zu[2], iv(fp.grav));
    const ivl n = isqrt(iadd(iadd(isqr(zu[0]), isqr(zu[1])), isqr(zu[2])));
    if (!(n.lo > 0.0)) return false;
    const ivl zx = idivp(zu[0], n), zy = idivp(zu[1], n), zz = idivp(zu[2], n);
    const ivl op = iadd(iv(1.0), zz);
    if (!(op.lo > 0.0)) return false;
    const ivl xx = idivp(isqr(zx), op), yy = idivp(isqr(zy), op), xy = idivp(imul(zx, zy), op);
    R[0] = isub(iv(1.0), xx); R[1] = ineg(xy); R[2] = zx;
    R[3] = ineg(xy); R[4] = isub(iv(1.0), yy); R[5] = zy;
    R[6] = ineg(zx); R[7] = ineg(zy); R[8] = zz;
    auto nrm = [](const ivl w[3]) { return __dsqrt_ru(__dadd_ru(__dadd_ru(__dmul_ru(imag(w[0]), imag(w[0])), __dmul_ru(imag(w[1]), imag(w[1]))),
                                                                __dmul_ru(imag(w[2]), imag(w[2])))); };
    const double num = __dadd_ru(__dadd_ru(nrm(a), __dmul_ru(__dmul_ru(fp.dh_over_m, kap.hi), nrm(v))), fabs(fp.grav));
    kappa = __ddiv_ru(num, n.lo);
    delta = op.lo;
    return true;
}

// D_e of include/isdf.h for piece i over [ta, tb], measured from the pose at t_e. C: 6N x 3 column-major.
__device__ __forceinline__ double cert_bound(const FlatParams &fp, double r, double H, const double *C, int N, int i, double ta, double tb, double te) {
    const double h = fmax(fmax(__dadd_ru(tb, -te), __dadd_ru(te, -ta)), 0.0);
    double hp[6];
    hp[0] = 1.0;
#pragma unroll
    for (int k = 1; k < 6; k++) hp[k] = __dmul_ru(hp[k - 1], h);
    ivl tp[6];
    tp[0] = iv(1.0);
#pragma unroll
    for (int k = 1; k < 6; k++) tp[k] = imul(tp[k - 1], iv(te));
    double P2 = 0.0, A = 0.0;
    ivl ve[3], vi[3], ae[3], ai[3];
#pragma unroll
    for (int ax = 0; ax < 3; ax++) {
        double c[6];
#pragma unroll
        for (int k = 0; k < 6; k++) c[k] = __ldg(C + 6 * N * ax + 6 * i + k);
        double m[6];   // |d_k|
        ivl d1 = iv(0.0), d2 = iv(0.0);
#pragma unroll
        for (int k = 1; k < 6; k++) {
            const ivl d = taylor_coeff(c, tp, k);
            m[k] = imag(d);
            if (k == 1) d1 = d;
            if (k == 2) d2 = d;
        }
        double disp = 0.0, vr = 0.0, ar = 0.0, a0 = fabs(c[0]);
#pragma unroll
        for (int k = 1; k < 6; k++) {
            disp = __dadd_ru(disp, __dmul_ru(m[k], hp[k]));
            if (k >= 2) vr = __dadd_ru(vr, __dmul_ru(__dmul_ru((double)k, m[k]), hp[k - 1]));
            if (k >= 3) ar = __dadd_ru(ar, __dmul_ru(__dmul_ru((double)(k * (k - 1)), m[k]), hp[k - 2]));
            a0 = __dadd_ru(a0, __dmul_ru(fabs(c[k]), fmax(fabs(tp[k].lo), fabs(tp[k].hi))));
        }
        P2 = __dadd_ru(P2, __dmul_ru(disp, disp));
        A = __dadd_ru(A, a0);
        ve[ax] = d1; vi[ax] = iwiden(d1, vr);
        ae[ax] = imul(iv(2.0), d2); ai[ax] = iwiden(ae[ax], ar);
    }
    const double P = __dsqrt_ru(P2);
    ivl Ri[9], Re[9];
    double ki, di, ke, de;
    if (!cert_rot(fp, vi, ai, Ri, ki, di) || !cert_rot(fp, ve, ae, Re, ke, de)) return INFINITY;
    double Q2 = 0.0;
#pragma unroll
    for (int k = 0; k < 9; k++) { const double w = imag(isub(Ri[k], Re[k])); Q2 = __dadd_ru(Q2, __dmul_ru(w, w)); }
    const double Q = __dsqrt_ru(Q2);
    const double H2 = __dmul_ru(2.0, H);
    const double eps = __dmul_ru(CERT_EPS_REL, __dadd_ru(__dadd_ru(__dadd_ru(1.0, A), H2), __dmul_ru(__dadd_ru(r, H2), __ddiv_ru(ke, de))));
    const double D = __dadd_ru(__dadd_ru(P, __dmul_ru(r, Q)), eps);
    return D <= 1.7976931348623157e308 ? D : INFINITY;   // NaN and overflow: no bound
}

// lb of an interval: c NaN (non-finite pose) counts as -inf
__device__ __forceinline__ double cert_lb(double ca, double cb, double Da, double Db) {
    const double a = ca != ca ? -INFINITY : __dadd_rd(ca, -Da), b = cb != cb ? -INFINITY : __dadd_rd(cb, -Db);
    return fmax(a, b);
}

#ifdef ISDF_CLEARANCE_TU
// initial samples (the clearance check's, piece-major) and intervals; per-trajectory state and piece start times
__global__ void __launch_bounds__(CERT_THREADS) k_certify_init(const __grid_constant__ CertArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x, K = A.K;
    if (k < A.N * (K + 1)) {
        const int i = k / (K + 1), j = k - i * (K + 1);
        const double step = A.T[i] * (1.0 / K);
        A.sp[k] = i;
        A.st[k] = j * step;
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
        CertTraj s;
        s.lb = s.min_clear = s.t_min = s.first_hit = INFINITY;
        s.voxel_min = -1;
        s.used = s.undecided = s.depth = 0;
        s.seg_off = k * A.N0 * K; s.seg_cnt = A.N0 * K;
        s.split_pref = s.leaf_pref = s.nsplit = s.nleaf = s.pad = 0;
        A.traj[k] = s;
        A.hit[k] = 0;
    }
    if (k == 0) { A.tot[0] = 0; A.tot[1] = 0; }
}

// exclusive block scan of v over CERT_THREADS threads; every thread gets the block total
__device__ __forceinline__ int cert_block_scan(int v, int &total, int *s_w) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) s_w[w] = x;
    __syncthreads();
    int base = 0;
    total = 0;
    for (int q = 0; q < CERT_THREADS / 32; q++) { if (q < w) base += s_w[q]; total += s_w[q]; }
    __syncthreads();
    return base + x - v;
}

// sample minimum key: (clearance, NaN as -inf; trajectory time; witness as unsigned, so -1 sorts last)
__device__ __forceinline__ bool cert_key_less(double v, double t, long long x, double bv, double bt, long long bx) {
    return v < bv || (v == bv && (t < bt || (t == bt && (unsigned long long)x < (unsigned long long)bx)));
}

__global__ void __launch_bounds__(CERT_THREADS) k_certify_decide(const __grid_constant__ CertArgs A) {
    __shared__ int s_w[CERT_THREADS / 32];
    __shared__ double s_d[4][CERT_THREADS];
    __shared__ long long s_x[CERT_THREADS];
    __shared__ int s_i[2][CERT_THREADS];
    __shared__ int s_last;
    const int b = blockIdx.x, tid = threadIdx.x;
    const CertTraj Tr = A.traj[b];
    const int off = Tr.seg_off, cnt = Tr.seg_cnt, hit = A.hit[b];
    int used = Tr.used, nsplit = 0, nleaf = 0;
    double lbm = INFINITY, kv = INFINITY, kt = INFINITY, fh = INFINITY;
    long long kx = -1;
    int und = 0, dep = 0;
    auto fold = [&](int s) {
        double v = A.sc[s];
        if (v != v) v = -INFINITY;
        const double t = A.toff[A.sp[s]] + A.st[s];
        const long long x = A.sv[s];
        if (cert_key_less(v, t, x, kv, kt, kx)) { kv = v; kt = t; kx = x; }
        if (!(v >= A.margin)) fh = fmin(fh, t);
    };
    for (int base = 0; base < cnt; base += CERT_THREADS) {
        const int k = base + tid;
        const bool valid = k < cnt;
        bool wants = false, safe = false;
        CertInterval I;
        double Da = 0, Db = 0, lb = 0;
        if (valid) {
            I = A.cur[off + k];
            const double ca = A.sc[I.sa], cb = A.sc[I.sb];
#pragma unroll 1
            for (int e = 0; e < 2; e++) {   // one endpoint at a time: the bound's interval state is not doubled in registers
                const double D = cert_bound(A.fp, A.r, A.H, A.C, A.N, I.piece, I.ta, I.tb, A.st[e ? I.sb : I.sa]);
                if (e) Db = D; else Da = D;
            }
            lb = cert_lb(ca, cb, Da, Db);
            if (I.flags & CERT_FOLD_A) fold(I.sa);
            if (I.flags & CERT_FOLD_B) fold(I.sb);
            safe = lb >= A.margin;
            const double m = I.ta + 0.5 * (I.tb - I.ta);
            wants = !safe && !hit && I.depth < A.max_depth && I.ta < m && m < I.tb;
        }
        int total;
        const int rank = cert_block_scan(wants ? 1 : 0, total, s_w);
        const int allowed = max(A.max_samples - used, 0);
        const bool split = wants && rank < allowed;
        const int srank = min(rank, allowed);
        if (valid) {
            const int state = safe ? LEAF_SAFE : (hit ? LEAF_DROPPED : LEAF_UNDECIDED);
            CertScratch sc;
            sc.Da = Da; sc.Db = Db; sc.state = state;
            sc.dec = split ? nsplit + srank : ~(nleaf + (tid - srank));
            A.scr[off + k] = sc;
            if (!split) {
                lbm = fmin(lbm, lb != lb ? -INFINITY : lb);
                und += state == LEAF_UNDECIDED;
                dep = max(dep, I.depth);
            }
        }
        const int took = min(total, allowed), nvalid = min(cnt - base, CERT_THREADS);
        nsplit += took; nleaf += nvalid - took; used += took;
    }
    // block reductions: minima with their keys, integer sums and maxima — independent of the thread schedule
    s_d[0][tid] = lbm; s_d[1][tid] = kv; s_d[2][tid] = kt; s_d[3][tid] = fh; s_x[tid] = kx; s_i[0][tid] = und; s_i[1][tid] = dep;
    __syncthreads();
    for (int o = CERT_THREADS / 2; o > 0; o >>= 1) {
        if (tid < o) {
            s_d[0][tid] = fmin(s_d[0][tid], s_d[0][tid + o]);
            if (cert_key_less(s_d[1][tid + o], s_d[2][tid + o], s_x[tid + o], s_d[1][tid], s_d[2][tid], s_x[tid])) {
                s_d[1][tid] = s_d[1][tid + o]; s_d[2][tid] = s_d[2][tid + o]; s_x[tid] = s_x[tid + o];
            }
            s_d[3][tid] = fmin(s_d[3][tid], s_d[3][tid + o]);
            s_i[0][tid] += s_i[0][tid + o];
            s_i[1][tid] = max(s_i[1][tid], s_i[1][tid + o]);
        }
        __syncthreads();
    }
    if (tid == 0) {
        CertTraj s = Tr;
        s.lb = fmin(s.lb, s_d[0][0]);
        if (cert_key_less(s_d[1][0], s_d[2][0], s_x[0], s.min_clear, s.t_min, s.voxel_min)) { s.min_clear = s_d[1][0]; s.t_min = s_d[2][0]; s.voxel_min = s_x[0]; }
        s.first_hit = fmin(s.first_hit, s_d[3][0]);
        s.undecided += s_i[0][0];
        if (cnt > 0) s.depth = max(s.depth, s_i[1][0]);
        s.used = used; s.nsplit = nsplit; s.nleaf = nleaf;
        A.traj[b] = s;
        __threadfence();
        s_last = atomicAdd(A.tot + 1, 1) == A.B - 1;
    }
    __syncthreads();
    if (!s_last) return;
    // last CTA: split / leaf offsets of every trajectory (trajectory order) and the next round's segments
    __threadfence();
    int sp = 0, lp = 0;
    for (int base = 0; base < A.B; base += CERT_THREADS) {
        const int q = base + tid;
        const int ns = q < A.B ? __ldcg(&A.traj[q].nsplit) : 0, nl = q < A.B ? __ldcg(&A.traj[q].nleaf) : 0;
        int ts, tl;
        const int es = cert_block_scan(ns, ts, s_w), el = cert_block_scan(nl, tl, s_w);
        if (q < A.B) {
            A.traj[q].split_pref = sp + es; A.traj[q].leaf_pref = lp + el;
            A.traj[q].seg_off = 2 * (sp + es); A.traj[q].seg_cnt = 2 * ns;
        }
        sp += ts; lp += tl;
    }
    if (tid == 0) { A.tot[0] = sp; A.tot[1] = 0; }
}

__global__ void __launch_bounds__(CERT_THREADS) k_certify_emit(const __grid_constant__ CertArgs A) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= A.nact) return;
    const CertInterval I = A.cur[k];
    const CertScratch sc = A.scr[k];
    const CertTraj &Tr = A.traj[I.piece / A.N0];
    if (sc.dec >= 0) {
        const int r = Tr.split_pref + sc.dec, s = A.S_cur + r;
        const double m = I.ta + 0.5 * (I.tb - I.ta);
        A.sp[s] = I.piece; A.st[s] = m;
        CertInterval L = I, R = I;
        L.tb = m; L.sb = s; L.depth = I.depth + 1; L.flags = 0;
        R.ta = m; R.sa = s; R.depth = I.depth + 1; R.flags = CERT_FOLD_A;
        A.next[2 * r] = L; A.next[2 * r + 1] = R;
    } else {
        CertLeaf l;
        l.ta = I.ta; l.tb = I.tb; l.ca = A.sc[I.sa]; l.cb = A.sc[I.sb]; l.Da = sc.Da; l.Db = sc.Db; l.piece = I.piece; l.state = sc.state;
        A.leaves[A.L_cur + Tr.leaf_pref + ~sc.dec] = l;
    }
}

__global__ void __launch_bounds__(CERT_THREADS) k_certify_finish(const __grid_constant__ CertArgs A) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= A.B) return;
    const CertTraj s = A.traj[b];
    CertSummary o;
    o.verdict = A.hit[b] ? -1 : (s.undecided == 0 ? 1 : 0);
    o.lower_bound = s.lb;
    o.min_clearance = s.min_clear == -INFINITY ? nan("") : s.min_clear;
    o.t_min = s.t_min;
    o.voxel_min = s.voxel_min;
    o.first_hit = s.first_hit == INFINITY ? -1.0 : s.first_hit;
    o.samples = A.N0 * (A.K + 1) + s.used;
    o.undecided = s.undecided;
    o.depth = s.depth;
    A.summary[b] = o;
}

// isdf_dbg_certify_bound: (D_a, D_b) of caller-given intervals
__global__ void k_certify_bound(const __grid_constant__ CertArgs A, int n, const int *piece, const double *ta, const double *tb, double *out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    out[2 * k] = cert_bound(A.fp, A.r, A.H, A.C, A.N, piece[k], ta[k], tb[k], ta[k]);
    out[2 * k + 1] = cert_bound(A.fp, A.r, A.H, A.C, A.N, piece[k], ta[k], tb[k], tb[k]);
}
#endif  // ISDF_CLEARANCE_TU

// ---- launch interface (isdf_clearance_tu.cu) --------------------------------------------------------------------------------------
cudaError_t certify_init_launch(const CertArgs &A, cudaStream_t st);
cudaError_t certify_round_launch(const CertArgs &A, cudaStream_t st);    // k_certify_decide + k_certify_emit over A.nact intervals
cudaError_t certify_finish_launch(const CertArgs &A, cudaStream_t st);
cudaError_t certify_bound_launch(const CertArgs &A, int n, const int *piece, const double *ta, const double *tb, double *out, cudaStream_t st);

}  // namespace isdf
