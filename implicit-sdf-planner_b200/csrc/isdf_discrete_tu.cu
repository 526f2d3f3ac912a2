// Translation unit of the discrete-path kernels (isdf_discrete.cuh): k_discrete_mesh, k_discrete_analytic, k_discrete_epilogue,
// k_build_items. Compiled WITH FMA contraction (nvcc default): nothing on this path replays a sequential decision of the
// reference, its parity bar is the north star's 1e-6 (observed ~1e-15), and un-fused FP64 costs the mesh kernel
// time. The swept-volume search, whose accept/reject sequence must replay the reference's bit for bit, stays in
// isdf_api.cu under -fmad=false. ISDF_FAST_TRI selects the division-free closest-point test (isdf_mesh.cuh) for this TU only.
#define ISDF_DISCRETE_TU 1
#define ISDF_FAST_TRI 1
#include "../../include/isdf.h"
#include "isdf_types.cuh"
#include "isdf_discrete.cuh"

namespace isdf {

cudaError_t discrete_launch_scan(const DiscArgs &A, bool mesh, unsigned grid, cudaStream_t st) {
    if (mesh && A.shape.mesh.sign_mode == MESH_SIGN_WINDING) k_discrete_mesh<true><<<grid, DISC_THREADS, 0, st>>>(A);
    else if (mesh) k_discrete_mesh<false><<<grid, DISC_THREADS, 0, st>>>(A);
    else k_discrete_analytic<<<grid, DISC_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t discrete_launch_prologue(const DiscArgs &A, int M, cudaStream_t st) {
    k_discrete_prologue<<<(unsigned)((M + PRO_SAMPLES - 1) / PRO_SAMPLES), PRO_SAMPLES, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t discrete_launch_epilogue(const DiscArgs &A, cudaStream_t st) {
    k_discrete_epilogue<<<(unsigned)A.N, EPI_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t discrete_launch_build_items(const unsigned *work, int rank, int world, int M, int max_split, int warp_slots, int *items,
                                        int *item_count, cudaStream_t st) {
    if (items_cached(M)) k_build_items<true><<<1, 1024, 0, st>>>(work, rank, world, M, max_split, warp_slots, items, item_count);
    else k_build_items<false><<<1, 1024, 0, st>>>(work, rank, world, M, max_split, warp_slots, items, item_count);
    return cudaGetLastError();
}

cudaError_t discrete_resident_blocks(int *mesh_blocks, int *analytic_blocks) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, (const void *)k_discrete_analytic);   // fails loudly if the sm_90a image cannot run here
    if (e != cudaSuccess) return e;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(mesh_blocks, k_discrete_mesh<false>, DISC_THREADS, 0);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(analytic_blocks, k_discrete_analytic, DISC_THREADS, 0);
}

// vaj: n x 9 (vel, acc, jer); grads: n x 10 (quat_grad 4, omg_grad 3, vel_grad 3); out: n x 16 (quat 4, omg 3, gV 3, gA 3, gJ 3)
__global__ void k_dbg_flatness(const FlatParams fp, int n, const double *vaj, const double *grads, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *x = vaj + 9 * (size_t)i, *gr = grads + 10 * (size_t)i;
    const d3 v = mk3(x[0], x[1], x[2]), a = mk3(x[3], x[4], x[5]), j = mk3(x[6], x[7], x[8]);
    FlatState fs;
    flat_state(fp, v, a, j, fs);
    const quat4 q = flat_quat(fs);
    const quat4 q2 = flat_quat_only(fp, v, a);
    const d3 om = flat_omega(fs);
    const double qb[4] = {gr[0], gr[1], gr[2], gr[3]};
    d3 gV, gA, gJ;
    flat_adjoint(fp, fs, v, a, qb, mk3(gr[4], gr[5], gr[6]), mk3(gr[7], gr[8], gr[9]), gV, gA, gJ);
    double *o = out + 16 * (size_t)i;
    const bool same = (q.w == q2.w && q.x == q2.x && q.y == q2.y && q.z == q2.z);   // the scan kernels' quaternion-only forward
    o[0] = same ? q.w : nan(""); o[1] = q.x; o[2] = q.y; o[3] = q.z; o[4] = om.x; o[5] = om.y; o[6] = om.z;
    o[7] = gV.x; o[8] = gV.y; o[9] = gV.z; o[10] = gA.x; o[11] = gA.y; o[12] = gA.z; o[13] = gJ.x; o[14] = gJ.y; o[15] = gJ.z;
}

cudaError_t discrete_launch_dbg_flatness(const FlatParams &fp, int n, const double *vaj, const double *grads, double *out, cudaStream_t st) {
    k_dbg_flatness<<<(n + 127) / 128, 128, 0, st>>>(fp, n, vaj, grads, out);
    return cudaGetLastError();
}

}  // namespace isdf
