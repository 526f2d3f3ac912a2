// Outward-rounded interval arithmetic and the Taylor re-expansion of a piece polynomial, shared by the continuous clearance certificate
// (isdf_certify.cuh) and the dynamic-limit certificate (isdf_dynlimits.cuh). Every operation rounds its lower end down and its upper
// end up (__dadd_rd/_ru, __dmul_rd/_ru, __ddiv_rd/_ru, __dsqrt_rd/_ru), so an interval result contains the exact real result.
#pragma once
#include "isdf_math.cuh"

namespace isdf {

struct ivl { double lo, hi; };
__device__ __forceinline__ ivl iv(double x) { ivl r; r.lo = x; r.hi = x; return r; }
__device__ __forceinline__ ivl iadd(ivl a, ivl b) { ivl r; r.lo = __dadd_rd(a.lo, b.lo); r.hi = __dadd_ru(a.hi, b.hi); return r; }
__device__ __forceinline__ ivl isub(ivl a, ivl b) { ivl r; r.lo = __dadd_rd(a.lo, -b.hi); r.hi = __dadd_ru(a.hi, -b.lo); return r; }
__device__ __forceinline__ ivl ineg(ivl a) { ivl r; r.lo = -a.hi; r.hi = -a.lo; return r; }
__device__ __forceinline__ ivl imul(ivl a, ivl b) {
    ivl r;
    r.lo = fmin(fmin(__dmul_rd(a.lo, b.lo), __dmul_rd(a.lo, b.hi)), fmin(__dmul_rd(a.hi, b.lo), __dmul_rd(a.hi, b.hi)));
    r.hi = fmax(fmax(__dmul_ru(a.lo, b.lo), __dmul_ru(a.lo, b.hi)), fmax(__dmul_ru(a.hi, b.lo), __dmul_ru(a.hi, b.hi)));
    return r;
}
__device__ __forceinline__ ivl isqr(ivl a) {
    const double m = fmax(fabs(a.lo), fabs(a.hi)), n = (a.lo > 0.0) ? a.lo : (a.hi < 0.0 ? -a.hi : 0.0);
    ivl r; r.lo = __dmul_rd(n, n); r.hi = __dmul_ru(m, m); return r;
}
// a / b for b.lo > 0
__device__ __forceinline__ ivl idivp(ivl a, ivl b) {
    ivl r;
    r.lo = a.lo >= 0.0 ? __ddiv_rd(a.lo, b.hi) : __ddiv_rd(a.lo, b.lo);
    r.hi = a.hi >= 0.0 ? __ddiv_ru(a.hi, b.lo) : __ddiv_ru(a.hi, b.hi);
    return r;
}
__device__ __forceinline__ ivl isqrt(ivl a) { ivl r; r.lo = __dsqrt_rd(fmax(a.lo, 0.0)); r.hi = __dsqrt_ru(a.hi); return r; }
__device__ __forceinline__ double imag(ivl a) { return fmax(fabs(a.lo), fabs(a.hi)); }
__device__ __forceinline__ ivl iwiden(ivl a, double rad) { ivl r; r.lo = __dadd_rd(a.lo, -rad); r.hi = __dadd_ru(a.hi, rad); return r; }

// Taylor coefficient d_k (k >= 1) of the quintic sum_q c_q t^q re-expanded about t_e: sum_{q >= k} binom(q, k) c_q t_e^(q-k), with
// tp[m] an enclosure of t_e^m
__device__ __forceinline__ ivl taylor_coeff(const double c[6], const ivl tp[6], int k) {
    const double binom[6][6] = {{1, 0, 0, 0, 0, 0}, {1, 1, 0, 0, 0, 0}, {1, 2, 1, 0, 0, 0}, {1, 3, 3, 1, 0, 0}, {1, 4, 6, 4, 1, 0}, {1, 5, 10, 10, 5, 1}};
    ivl d = iv(0.0);
#pragma unroll
    for (int q = k; q < 6; q++) d = iadd(d, imul(imul(iv(binom[q][k]), iv(c[q])), tp[q - k]));
    return d;
}

}  // namespace isdf
