// Translation unit of the trajectory clearance kernels (isdf_clearance.cuh): k_clearance_scan<0|1|2>, k_clearance_summary, and of the
// continuous certificate built on them (isdf_certify.cuh).
// Compiled WITH FMA contraction and the division-free closest-point test, like the discrete path; a third unit of its own so that the
// objects of the other two stay exactly what they are.
#define ISDF_CLEARANCE_TU 1
#define ISDF_FAST_TRI 1
#include "../../include/isdf.h"
#include "isdf_types.cuh"
#include "isdf_clearance.cuh"
#include "isdf_certify.cuh"

namespace isdf {

cudaError_t clearance_scan_launch(const ClrArgs &A, int mode, unsigned grid, cudaStream_t st) {
    if (mode == 2) k_clearance_scan<2><<<grid, CLR_THREADS, 0, st>>>(A);
    else if (mode == 1) k_clearance_scan<1><<<grid, CLR_THREADS, 0, st>>>(A);
    else k_clearance_scan<0><<<grid, CLR_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t clearance_launch(const ClrArgs &A, int mode, unsigned grid, cudaStream_t st) {
    cudaError_t e = clearance_scan_launch(A, mode, grid, st);
    if (e != cudaSuccess) return e;
    k_clearance_summary<<<(unsigned)(A.N / A.N0), CLR_SUM_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t certify_init_launch(const CertArgs &A, cudaStream_t st) {
    const int n = max(A.N * (A.K + 1), A.B);
    k_certify_init<<<(n + CERT_THREADS - 1) / CERT_THREADS, CERT_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t certify_round_launch(const CertArgs &A, cudaStream_t st) {
    k_certify_decide<<<A.B, CERT_THREADS, 0, st>>>(A);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || A.nact == 0) return e;
    k_certify_emit<<<(A.nact + CERT_THREADS - 1) / CERT_THREADS, CERT_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t certify_finish_launch(const CertArgs &A, cudaStream_t st) {
    k_certify_finish<<<(A.B + CERT_THREADS - 1) / CERT_THREADS, CERT_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t certify_bound_launch(const CertArgs &A, int n, const int *piece, const double *ta, const double *tb, double *out, cudaStream_t st) {
    k_certify_bound<<<(n + 127) / 128, 128, 0, st>>>(A, n, piece, ta, tb, out);
    return cudaGetLastError();
}

cudaError_t clearance_resident_blocks(int *blocks) {
    int b0 = 0, b1 = 0, b2 = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b0, k_clearance_scan<0>, CLR_THREADS, 0);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b1, k_clearance_scan<1>, CLR_THREADS, 0);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b2, k_clearance_scan<2>, CLR_THREADS, 0);
    *blocks = min(b0, min(b1, b2));
    return e;
}

}  // namespace isdf
