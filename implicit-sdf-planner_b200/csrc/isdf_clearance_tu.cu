// Translation unit of the trajectory clearance kernels (isdf_clearance.cuh): k_clearance_scan<0|1|2>, k_clearance_summary, of the
// continuous certificate built on them (isdf_certify.cuh), of the certified swept volume that shares the certificate's pose and
// motion bound (isdf_sweptvol.cuh) and of the dynamic-limit certificate that shares its rounds (isdf_dynlimits.cuh).
// Compiled WITH FMA contraction and the division-free closest-point test, like the discrete path; a third unit of its own so that the
// objects of the other two stay exactly what they are.
#define ISDF_CLEARANCE_TU 1
#define ISDF_FAST_TRI 1
#include "../../include/isdf.h"
#include "isdf_types.cuh"
#include "isdf_clearance.cuh"
#include "isdf_certify.cuh"
#include "isdf_sweptvol.cuh"
#include "isdf_dynlimits.cuh"

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

cudaError_t dyn_init_launch(const DynArgs &A, cudaStream_t st) {
    const int n = max(A.N * (A.K + 1), A.B);
    k_dyn_init<<<(n + DYN_THREADS - 1) / DYN_THREADS, DYN_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t dyn_round_launch(const DynArgs &A, cudaStream_t st) {
    k_dyn_decide<<<A.B, DYN_THREADS, 0, st>>>(A);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || A.nact == 0) return e;
    k_dyn_emit<<<(A.nact + DYN_THREADS - 1) / DYN_THREADS, DYN_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t dyn_finish_launch(const DynArgs &A, cudaStream_t st) {
    k_dyn_finish<<<(A.B + DYN_THREADS - 1) / DYN_THREADS, DYN_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t sv_prep_launch(const SvolArgs &A, cudaStream_t st) {
    const int n = max(A.N * (A.K + 1), 1);
    k_sv_prep<<<(n + CERT_THREADS - 1) / CERT_THREADS, CERT_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t sv_bricks_launch(const SvolArgs &A, int nbricks, bool fill, cudaStream_t st) {
    const unsigned grid = (unsigned)((nbricks + SV_WARPS - 1) / SV_WARPS);
    if (fill) k_sv_bricks<true><<<grid, SV_THREADS, 0, st>>>(A, nbricks);
    else k_sv_bricks<false><<<grid, SV_THREADS, 0, st>>>(A, nbricks);
    return cudaGetLastError();
}

cudaError_t sv_refine_launch(const SvolArgs &A, int mode, int nitems, unsigned grid, cudaStream_t st) {
    if (mode == 1) k_sv_refine<1><<<grid, SV_THREADS, 0, st>>>(A, nitems);
    else k_sv_refine<0><<<grid, SV_THREADS, 0, st>>>(A, nitems);
    return cudaGetLastError();
}

cudaError_t sv_scan_launch(long long *a, long long n, long long *bsum, cudaStream_t st) {
    const long long nb = (n + SV_SCAN_THREADS - 1) / SV_SCAN_THREADS;
    if (nb > 0) k_sv_scan_blocks<<<(unsigned)nb, SV_SCAN_THREADS, 0, st>>>(a, n, bsum);
    k_sv_scan_top<<<1, SV_SCAN_THREADS, 0, st>>>(bsum, nb, a, n);
    if (nb > 0) k_sv_scan_add<<<(unsigned)nb, SV_SCAN_THREADS, 0, st>>>(a, n, bsum);
    return cudaGetLastError();
}

cudaError_t sv_mesh_count_launch(const SvolMeshArgs &M, cudaStream_t st) {
    const long long n = (long long)M.X * M.Y * M.Z;
    k_sv_mt_count<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(M);
    return cudaGetLastError();
}

cudaError_t sv_mesh_emit_launch(const SvolMeshArgs &M, cudaStream_t st) {
    const long long n = (long long)M.X * M.Y * M.Z;
    k_sv_mt_emit<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(M);
    return cudaGetLastError();
}

cudaError_t sv_refine_resident_blocks(int *blocks) {
    int b0 = 0, b1 = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b0, k_sv_refine<0>, SV_THREADS, 0);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b1, k_sv_refine<1>, SV_THREADS, 0);
    *blocks = min(b0, b1);
    return e;
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
