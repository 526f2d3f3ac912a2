// Runs the certificates' interval primitives on the device, record by record (TEST INFRASTRUCTURE for test_gpu_interval_exact.py).
// The headers are included unchanged, so what runs here is what the clearance, swept-volume and dynamic-limit kernels run.
//
//   interval_probe <op> <in> <out> <n>     in: n records of PROBE_IN doubles, out: n records of PROBE_OUT doubles (unused slots NaN)
//
// op  inputs                                                   outputs
//  0  iadd   a.lo a.hi b.lo b.hi                               lo hi
//  1  isub   a.lo a.hi b.lo b.hi                               lo hi
//  2  ineg   a.lo a.hi                                         lo hi
//  3  imul   a.lo a.hi b.lo b.hi                               lo hi
//  4  isqr   a.lo a.hi                                         lo hi
//  5  idivp  a.lo a.hi b.lo b.hi                               lo hi
//  6  isqrt  a.lo a.hi                                         lo hi
//  7  iwiden a.lo a.hi rad                                     lo hi
//  8  inorm  w0.lo w0.hi w1.lo w1.hi w2.lo w2.hi               lo hi
//  9  taylor c0..c5 te h                                       d1..d5 (lo hi each), disp, v, a, j (lo hi each); tp and hp as
//                                                              cert_bound and dyn_vaj build them
// 10  flat_enclose  fp[5] v[6] a[6]                            ok, kap (2), zu (6), n (2)
// 11  cert_rot      fp[5] v[6] a[6]                            ok, R (18, row-major), kappa, delta
// 12  dyn_channels  fp[5] mass dv v[6] a[6] j[6]               lo[6] hi[6]
// 13  cert_bound    fp[5] r H C[18] ta tb te                   D
// 14  dyn_bound     fp[5] mass dv C[18] ta tb                  hi[6]
// 15  dyn_point     fp[5] mass dv C[18] t                      q[6]
// fp = {mass, grav, dh_over_m, cp, veps}; boxes are (lo, hi) per axis; C is one piece, 6 x 3 column-major (axis-major t^k).
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "../include/isdf.h"
#include "../implicit-sdf-planner_b200/csrc/isdf_types.cuh"
#include "../implicit-sdf-planner_b200/csrc/isdf_interval.cuh"
#include "../implicit-sdf-planner_b200/csrc/isdf_certify.cuh"
#include "../implicit-sdf-planner_b200/csrc/isdf_dynlimits.cuh"

constexpr int PROBE_IN = 32, PROBE_OUT = 48;

using namespace isdf;

__device__ ivl ld(const double *p) { ivl r; r.lo = p[0]; r.hi = p[1]; return r; }
__device__ void st(double *p, ivl a) { p[0] = a.lo; p[1] = a.hi; }
__device__ FlatParams ldfp(const double *p) { FlatParams f; f.mass = p[0]; f.grav = p[1]; f.dh_over_m = p[2]; f.cp = p[3]; f.veps = p[4]; return f; }
__device__ void ld3(const double *p, ivl w[3]) { for (int k = 0; k < 3; k++) w[k] = ld(p + 2 * k); }

__global__ void k_probe(int op, int n, const double *in, double *out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const double *x = in + (size_t)r * PROBE_IN;
    double *y = out + (size_t)r * PROBE_OUT;
    for (int k = 0; k < PROBE_OUT; k++) y[k] = nan("");
    switch (op) {
    case 0: st(y, iadd(ld(x), ld(x + 2))); break;
    case 1: st(y, isub(ld(x), ld(x + 2))); break;
    case 2: st(y, ineg(ld(x))); break;
    case 3: st(y, imul(ld(x), ld(x + 2))); break;
    case 4: st(y, isqr(ld(x))); break;
    case 5: st(y, idivp(ld(x), ld(x + 2))); break;
    case 6: st(y, isqrt(ld(x))); break;
    case 7: st(y, iwiden(ld(x), x[2])); break;
    case 8: { ivl w[3]; ld3(x, w); st(y, inorm(w)); break; }
    case 9: {
        double c[6];
        for (int k = 0; k < 6; k++) c[k] = x[k];
        const double te = x[6], h = x[7];
        double hp[6];
        hp[0] = 1.0;
        for (int k = 1; k < 6; k++) hp[k] = __dmul_ru(hp[k - 1], h);
        ivl tp[6];
        tp[0] = iv(1.0);
        for (int k = 1; k < 6; k++) tp[k] = imul(tp[k - 1], iv(te));
        ivl d[6], v, a, j;
        double disp;
        taylor_axis(c, tp, hp, d, disp, v, a, j);
        for (int k = 1; k < 6; k++) st(y + 2 * (k - 1), d[k]);
        y[10] = disp;
        st(y + 11, v); st(y + 13, a); st(y + 15, j);
        // taylor_coeff on its own, as cert_bound's callers see it through taylor_axis
        for (int k = 1; k < 6; k++) st(y + 17 + 2 * (k - 1), taylor_coeff(c, tp, k));
        break;
    }
    case 10: {
        const FlatParams fp = ldfp(x);
        ivl v[3], a[3], kap, zu[3], nn;
        ld3(x + 5, v); ld3(x + 11, a);
        y[0] = flat_enclose(fp, v, a, kap, zu, nn) ? 1.0 : 0.0;
        st(y + 1, kap);
        for (int k = 0; k < 3; k++) st(y + 3 + 2 * k, zu[k]);
        st(y + 9, nn);
        break;
    }
    case 11: {
        const FlatParams fp = ldfp(x);
        ivl v[3], a[3], R[9];
        ld3(x + 5, v); ld3(x + 11, a);
        double kappa = nan(""), delta = nan("");
        const bool ok = cert_rot(fp, v, a, R, kappa, delta);
        y[0] = ok ? 1.0 : 0.0;
        if (ok) {
            for (int k = 0; k < 9; k++) st(y + 1 + 2 * k, R[k]);
            y[19] = kappa; y[20] = delta;
        }
        break;
    }
    case 12: {
        DynArgs A;
        A.fp = ldfp(x); A.mass = x[5]; A.dv = x[6];
        ivl v[3], a[3], j[3];
        ld3(x + 7, v); ld3(x + 13, a); ld3(x + 19, j);
        double lo[DYN_CH], hi[DYN_CH];
        dyn_channels(A, v, a, j, lo, hi);
        for (int c = 0; c < DYN_CH; c++) { y[c] = lo[c]; y[DYN_CH + c] = hi[c]; }
        break;
    }
    case 13: y[0] = cert_bound(ldfp(x), x[5], x[6], x + 7, 1, 0, x[25], x[26], x[27]); break;
    case 14: {
        DynArgs A;
        A.fp = ldfp(x); A.mass = x[5]; A.dv = x[6]; A.C = x + 7; A.N = 1;
        double hi[DYN_CH];
        dyn_bound(A, 0, x[25], x[26], hi);
        for (int c = 0; c < DYN_CH; c++) y[c] = hi[c];
        break;
    }
    case 15: {
        DynArgs A;
        A.fp = ldfp(x); A.mass = x[5]; A.dv = x[6]; A.C = x + 7; A.N = 1;
        dyn_point(A, 0, x[25], y);
        break;
    }
    default: break;
    }
}

static void check(cudaError_t e, const char *what) {
    if (e != cudaSuccess) { std::fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e)); std::exit(2); }
}

int main(int argc, char **argv) {
    if (argc != 5) { std::fprintf(stderr, "usage: interval_probe <op> <in> <out> <n>\n"); return 1; }
    const int op = std::atoi(argv[1]), n = std::atoi(argv[4]);
    std::vector<double> hin((size_t)n * PROBE_IN), hout((size_t)n * PROBE_OUT);
    FILE *f = std::fopen(argv[2], "rb");
    if (!f || std::fread(hin.data(), sizeof(double), hin.size(), f) != hin.size()) { std::fprintf(stderr, "cannot read %s\n", argv[2]); return 1; }
    std::fclose(f);
    double *din = nullptr, *dout = nullptr;
    check(cudaMalloc(&din, hin.size() * sizeof(double)), "cudaMalloc");
    check(cudaMalloc(&dout, hout.size() * sizeof(double)), "cudaMalloc");
    check(cudaMemcpy(din, hin.data(), hin.size() * sizeof(double), cudaMemcpyHostToDevice), "copy in");
    if (n > 0) k_probe<<<(n + 127) / 128, 128>>>(op, n, din, dout);
    check(cudaGetLastError(), "launch");
    check(cudaMemcpy(hout.data(), dout, hout.size() * sizeof(double), cudaMemcpyDeviceToHost), "copy out");
    cudaFree(din); cudaFree(dout);
    f = std::fopen(argv[3], "wb");
    if (!f || std::fwrite(hout.data(), sizeof(double), hout.size(), f) != hout.size()) { std::fprintf(stderr, "cannot write %s\n", argv[3]); return 1; }
    std::fclose(f);
    std::printf("INTERVAL PROBE OK %d %d\n", op, n);
    return 0;
}
