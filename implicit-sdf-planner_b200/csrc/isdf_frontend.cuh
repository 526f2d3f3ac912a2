// Front end: attitude-kernel collision checks for the whole map at once (SURVEY §8f row 4).
//
// Reference (per A* node expansion, serial): the robot is rasterised into one kernel_size^3 occupancy kernel per
// (roll, pitch) attitude (Shape.hpp:405-461); kernelConv<true> (sw_manager.hpp:821-846) ANDs the kernel's byte rows with the
// inflated, byte-packed map (PCSmap_manager.h:46-78) at the voxel; visit_kernels_by_distance (sw_manager.hpp:852-913) tries the
// level attitude and then a BFS over the attitude grid until a kernel fits; checkKernelValue (:914-941) maps that back to angles.
//
// GPU mapping: the question "which attitudes fit at voxel v" is answered for EVERY voxel in one pass, as a 128-bit mask per
// voxel, so the graph search itself does O(1) lookups. The convolution is turned inside out: instead of testing up to 121 kernels
// x 169 rows per voxel, each kernel offset (a,b,c) carries the SET OF ATTITUDES whose kernel occupies it (a 128-bit mask,
// kernel_size^3 x 16 B = 35 KB in shared memory); a voxel ORs the masks of the OCCUPIED voxels of its window — found with the same
// bit-row reads as the discrete collision kernel — and the attitudes left unset are collision-free. Work per voxel is
// proportional to the obstacles near it, not to the number of attitudes; integer/bit arithmetic only, so parity with the
// reference's byte AND is exact (cells outside the map are free, like the reference's inflation margin).
//   k_frontend_kernels      one thread per (attitude, a, b, c): SDF at the rotated body point <= margin
//   k_frontend_offset_masks one thread per (a, b, c): the 128-bit attitude set of that offset
//   k_frontend_feasibility  one thread per run of 4 voxels along z: window scan + mask OR -> collision-free attitude masks
//   k_frontend_core / k_frontend_survivors  the same masks in two passes: core rows settle most voxels, the full accumulation runs on the rest
//   k_frontend_check        one thread per query: same mask, then the reference's visiting order (level pose, BFS from the father)
#pragma once
#include "isdf_types.cuh"

namespace isdf {

constexpr int FE_MAX_ATT = 128;

struct FrontArgs {
    DevGrid grid;
    DevShape shape;          // analytic shapes: rot = I, trans = 0 (the pre-transform is applied explicitly, see k_frontend_kernels)
    double rot[9], trans[3]; // the shape's real pre-transform
    int ks, natt, xk, yk;
    double res, margin;
    const double *att_rot;   // natt x 9 row-major: Rx(roll) * Ry(pitch), built on the host exactly like Eigen does
    uint8_t *kernels;        // natt x ks^3 booleans, address a*ks*ks + b*ks + c
    uint32_t *offset_masks;  // ks^3 x 4
    uint32_t *out;           // X*Y*Z x 4 (feasibility) — or n x 4 for the batched check
    uint32_t *trav;          // non-null: traversability output instead of masks (isdf_frontpath.cuh), one bit per voxel in the layout of
                             // grid.bits, zero-filled beforehand: bit set = some attitude fits and the voxel itself is free
    // two-pass feasibility: rows of the kernel CORE (offsets occupied in EVERY attitude's kernel), the survivor list and its counter
    const uint2 *core_rows;  // ncore x {a | b << 8, bits over c}
    int ncore;
    // pattern tables (pass 2, table-driven): every union row is cut into chunks of <= FE_CHUNK_BITS offsets along c; tab[off + pattern] =
    // OR of the offset masks of the pattern's set bits. chunks: {a | b << 8 | c0 << 16 | len << 24, off}
    const uint2 *chunks; int nchunk; const uint4 *tab; int ntab;
    const uint2 *urows;      // nurow x {a | b << 8, bits over c}: the kernel rows ANY attitude occupies (every other offset's mask is zero)
    int nurow;
    uint2 *surv;             // runs with at least one voxel that no core offset settles: {run index, bit j = voxel j of the run is open}
    unsigned *surv_count;
    // batched check
    int nq;
    const int *q_ind;        // nq x 3
    const double *q_father;  // nq x 2 (roll, pitch) degrees
    double *q_child;         // nq x 2
    uint8_t *q_ok;           // nq
    const uint8_t *order;    // natt x natt: visiting order of visit_kernels_by_distance for every start attitude (0xff = end)
    double max_roll, max_pitch, ang_res;
};

__global__ void k_frontend_kernels(const __grid_constant__ FrontArgs A) {
    const int n3 = A.ks * A.ks * A.ks;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)A.natt * n3) return;
    const int att = (int)(t / n3), v = (int)(t - (long long)att * n3);
    const int a = v / (A.ks * A.ks), b = (v / A.ks) % A.ks, c = v % A.ks;
    const int side = (int)(0.5 * (A.ks - 1));
    const d3 pos = mk3(A.res * a - side * A.res, A.res * b - side * A.res, A.res * c - side * A.res);
    const double *R = A.att_rot + 9 * att;
    double sdf;
    if (A.shape.kind == ISDF_SHAPE_BALL || A.shape.kind == ISDF_SHAPE_POINT) sdf = shape_sdf_analytic(A.shape, pos);     // ignore R_obj
    else if (A.shape.kind == ISDF_SHAPE_MESH) {
        const d3 q = mk3(pos.x * R[0] + pos.y * R[3] + pos.z * R[6], pos.x * R[1] + pos.y * R[4] + pos.z * R[7], pos.x * R[2] + pos.y * R[5] + pos.z * R[8]);
        d3 g;
        sdf = mesh_sdf_grad(A.shape.mesh, q, 1e300, g);                                                               // pos * R_obj
    } else {
        const double x = pos.x - A.trans[0], y = pos.y - A.trans[1], z = pos.z - A.trans[2];                           // ((pos - trans) * Rotate) * R_obj
        const d3 p1 = mk3(x * A.rot[0] + y * A.rot[3] + z * A.rot[6], x * A.rot[1] + y * A.rot[4] + z * A.rot[7], x * A.rot[2] + y * A.rot[5] + z * A.rot[8]);
        const d3 q = mk3(p1.x * R[0] + p1.y * R[3] + p1.z * R[6], p1.x * R[1] + p1.y * R[4] + p1.z * R[7], p1.x * R[2] + p1.y * R[5] + p1.z * R[8]);
        sdf = shape_sdf_analytic(A.shape, q);   // A.shape carries identity rot / zero trans: only the body is evaluated
    }
    A.kernels[t] = (sdf <= A.margin) ? 1 : 0;
}

__global__ void k_frontend_offset_masks(const __grid_constant__ FrontArgs A) {
    const int n3 = A.ks * A.ks * A.ks;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n3) return;
    uint32_t m[4] = {0, 0, 0, 0};
    for (int att = 0; att < A.natt; att++)
        if (A.kernels[(size_t)att * n3 + v]) m[att >> 5] |= 1u << (att & 31);
    for (int k = 0; k < 4; k++) A.offset_masks[4 * v + k] = m[k];
}

// attitudes whose kernel collides with the map when centred on voxel (ix, iy, iz); sm = offset masks in shared memory
__device__ __forceinline__ void frontend_colliding(const FrontArgs &A, const uint32_t *sm, int ix, int iy, int iz, uint32_t m[4]) {
    const DevGrid &G = A.grid;
    const int ks = A.ks, side = (ks - 1) / 2;
    const uint32_t full[4] = {A.natt >= 32 ? 0xffffffffu : ((1u << A.natt) - 1u),
                              A.natt >= 64 ? 0xffffffffu : (A.natt > 32 ? ((1u << (A.natt - 32)) - 1u) : 0u),
                              A.natt >= 96 ? 0xffffffffu : (A.natt > 64 ? ((1u << (A.natt - 64)) - 1u) : 0u),
                              A.natt >= 128 ? 0xffffffffu : (A.natt > 96 ? ((1u << (A.natt - 96)) - 1u) : 0u)};
    m[0] = m[1] = m[2] = m[3] = 0u;
    const int z0 = iz - side;                            // window z range [z0, z0 + ks)
    const int w0 = (z0 >= 0) ? (z0 >> 5) : -1;           // word holding z0 (floor division for z0 >= -32)
    const int sh = z0 - 32 * w0;                         // 0..31
    const unsigned long long wmask = (ks >= 64) ? ~0ull : ((1ull << ks) - 1ull);
    for (int a = 0; a < ks; a++) {
        const int x = ix + a - side;
        if (x < 0 || x >= G.X) continue;
        for (int b = 0; b < ks; b++) {
            const int y = iy + b - side;
            if (y < 0 || y >= G.Y) continue;
            const uint32_t *row = G.bits + ((size_t)x * G.Y + y) * G.Zw;
            const uint32_t lo = (w0 >= 0 && w0 < G.Zw) ? __ldg(row + w0) : 0u;
            const uint32_t hi = (w0 + 1 >= 0 && w0 + 1 < G.Zw) ? __ldg(row + w0 + 1) : 0u;
            unsigned long long bits = ((((unsigned long long)hi << 32) | lo) >> sh) & wmask;   // bit c = voxel z0 + c (words past Z are zero)
            const uint32_t *mrow = sm + 4 * (size_t)((a * ks + b) * ks);
            while (bits) {
                const int c = __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                m[0] |= mrow[4 * c]; m[1] |= mrow[4 * c + 1]; m[2] |= mrow[4 * c + 2]; m[3] |= mrow[4 * c + 3];
            }
        }
        if (m[0] == full[0] && m[1] == full[1] && m[2] == full[2] && m[3] == full[3]) return;   // nothing fits any more
    }
}

__device__ __forceinline__ void frontend_stage_masks(const FrontArgs &A, uint32_t *sm) {
    const int n = 4 * A.ks * A.ks * A.ks;
    for (int k = threadIdx.x; k < n; k += blockDim.x) sm[k] = A.offset_masks[k];
    __syncthreads();
}

// traversability output: fit bit j = some attitude fits at voxel iz0 + j of a z-run (runs never straddle a 32-voxel word); the run's
// free voxels among them are ORed into A.trav
__device__ __forceinline__ void frontend_mark_run(const FrontArgs &A, int ix, int iy, int iz0, unsigned fit) {
    if (!fit) return;
    const size_t w = ((size_t)ix * A.grid.Y + iy) * A.grid.Zw + (iz0 >> 5);
    const unsigned bits = (fit << (iz0 & 31)) & ~__ldg(A.grid.bits + w);
    if (bits) atomicOr(A.trav + w, bits);
}
__device__ __forceinline__ bool any4(uint4 v) { return (v.x | v.y | v.z | v.w) != 0u; }

// One thread per run of FE_ZRUN voxels along z: the run's window rows are read once (ks + FE_ZRUN - 1 bits), every occupied map
// voxel found in a row is applied to each of the run's voxels it overlaps (offset c = bit - j), one 128-bit shared-memory load
// and four ORs per (occupied voxel, run voxel) pair.
constexpr int FE_ZRUN = 4;
__global__ void __launch_bounds__(256) k_frontend_feasibility(const __grid_constant__ FrontArgs A) {
    extern __shared__ __align__(16) uint32_t fe_sm[];
    frontend_stage_masks(A, fe_sm);
    const uint4 *sm4 = reinterpret_cast<const uint4 *>(fe_sm);
    const DevGrid &G = A.grid;
    const int ks = A.ks, side = (ks - 1) / 2;
    const int zruns = (G.Z + FE_ZRUN - 1) / FE_ZRUN;
    const long long nrun = (long long)G.X * G.Y * zruns;
    const uint4 valid = make_uint4(A.natt >= 32 ? 0xffffffffu : ((1u << A.natt) - 1u),
                                   A.natt >= 64 ? 0xffffffffu : (A.natt > 32 ? ((1u << (A.natt - 32)) - 1u) : 0u),
                                   A.natt >= 96 ? 0xffffffffu : (A.natt > 64 ? ((1u << (A.natt - 64)) - 1u) : 0u),
                                   A.natt >= 128 ? 0xffffffffu : (A.natt > 96 ? ((1u << (A.natt - 96)) - 1u) : 0u));
    const int wbits = ks + FE_ZRUN - 1;                                  // <= 32 (ks <= 29)
    const unsigned long long wmask = (1ull << wbits) - 1ull;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < nrun; r += (long long)gridDim.x * blockDim.x) {
        const int zr = (int)(r % zruns), iy = (int)((r / zruns) % G.Y), ix = (int)(r / ((long long)zruns * G.Y));
        const int iz0 = zr * FE_ZRUN;
        uint4 m[FE_ZRUN];
#pragma unroll
        for (int j = 0; j < FE_ZRUN; j++) m[j] = make_uint4(0u, 0u, 0u, 0u);
        const int z0 = iz0 - side;                                       // bit p of a row window = voxel z0 + p
        const int w0 = (z0 >= 0) ? (z0 >> 5) : -1;
        const int sh = z0 - 32 * w0;
        // only the kernel rows some attitude occupies can contribute (the masks of all other offsets are zero)
        for (int k = 0; k < A.nurow; k++) {
            const uint2 ur = __ldg(A.urows + k);
            const int a = (int)(ur.x & 0xffu), b = (int)(ur.x >> 8);
            const int x = ix + a - side, y = iy + b - side;
            if (x < 0 || x >= G.X || y < 0 || y >= G.Y) continue;
            const uint32_t *row = G.bits + ((size_t)x * G.Y + y) * G.Zw;
            const uint32_t lo = (w0 >= 0 && w0 < G.Zw) ? __ldg(row + w0) : 0u;
            const uint32_t hi = (sh + wbits > 32 && w0 + 1 >= 0 && w0 + 1 < G.Zw) ? __ldg(row + w0 + 1) : 0u;
            unsigned span = 0u;
#pragma unroll
            for (int j = 0; j < FE_ZRUN; j++) span |= ur.y << j;
            unsigned bits = (unsigned)(((((unsigned long long)hi << 32) | lo) >> sh) & wmask) & span;
            const uint4 *mrow = sm4 + (size_t)((a * ks + b) * ks);
            while (bits) {
                const int p = __ffs((int)bits) - 1;
                bits &= bits - 1;
#pragma unroll
                for (int j = 0; j < FE_ZRUN; j++) {
                    const int c = p - j;
                    if (c >= 0 && c < ks) { const uint4 t = mrow[c]; m[j].x |= t.x; m[j].y |= t.y; m[j].z |= t.z; m[j].w |= t.w; }
                }
            }
        }
        if (A.trav) {
            unsigned fit = 0u;
#pragma unroll
            for (int j = 0; j < FE_ZRUN; j++)
                if (iz0 + j < G.Z && any4(make_uint4(~m[j].x & valid.x, ~m[j].y & valid.y, ~m[j].z & valid.z, ~m[j].w & valid.w))) fit |= 1u << j;
            frontend_mark_run(A, ix, iy, iz0, fit);
            continue;
        }
        uint4 *o = reinterpret_cast<uint4 *>(A.out) + ((size_t)ix * G.Y + iy) * G.Z + iz0;
#pragma unroll
        for (int j = 0; j < FE_ZRUN; j++)
            if (iz0 + j < G.Z) o[j] = make_uint4(~m[j].x & valid.x, ~m[j].y & valid.y, ~m[j].z & valid.z, ~m[j].w & valid.w);
    }
}

// ---- two-pass feasibility ---------------------------------------------------------------------------------------------------------
// Most voxels of a cluttered map admit NO attitude, and most of those for one cheap reason: an occupied voxel sits on a kernel offset that
// every attitude's kernel occupies (the core of the robot: offset mask == all attitudes). Pass 1 tests only the core rows — a few dozen
// row reads and ANDs per run of voxels, no mask traffic — writes the all-colliding answer for the voxels it settles and appends the
// others' runs to a list; pass 2 runs the full mask accumulation on the listed runs' open voxels alone. Same masks as the one-pass kernel, bit for bit.
__global__ void __launch_bounds__(256) k_frontend_core(const __grid_constant__ FrontArgs A) {
    const DevGrid &G = A.grid;
    const int ks = A.ks, side = (ks - 1) / 2;
    const int zruns = (G.Z + FE_ZRUN - 1) / FE_ZRUN;
    const long long nrun = (long long)G.X * G.Y * zruns;
    const int wbits = ks + FE_ZRUN - 1;
    const unsigned long long wmask = (1ull << wbits) - 1ull;
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long rounds = (nrun + stride - 1) / stride;
    for (long long it = 0; it < rounds; it++) {                           // whole warps stay in the loop (the append is warp-wide)
        const long long r = it * stride + (long long)blockIdx.x * blockDim.x + threadIdx.x;
        unsigned alive = 0u;                                              // bit j: voxel iz0 + j exists and no core offset is occupied
        int ix = 0, iy = 0, iz0 = 0;
        if (r < nrun) {
            const int zr = (int)(r % zruns);
            iy = (int)((r / zruns) % G.Y); ix = (int)(r / ((long long)zruns * G.Y));
            iz0 = zr * FE_ZRUN;
            alive = (iz0 + FE_ZRUN <= G.Z) ? ((1u << FE_ZRUN) - 1u) : ((1u << (G.Z - iz0)) - 1u);
            const int z0 = iz0 - side;
            const int w0 = (z0 >= 0) ? (z0 >> 5) : -1;
            const int sh = z0 - 32 * w0;
            for (int k = 0; k < A.ncore && alive; k++) {
                const uint2 cr = __ldg(A.core_rows + k);
                const int x = ix + (int)(cr.x & 0xffu) - side, y = iy + (int)(cr.x >> 8) - side;
                if (x < 0 || x >= G.X || y < 0 || y >= G.Y) continue;
                const uint32_t *row = G.bits + ((size_t)x * G.Y + y) * G.Zw;
                const uint32_t lo = (w0 >= 0 && w0 < G.Zw) ? __ldg(row + w0) : 0u;
                const uint32_t hi = (sh + wbits > 32 && w0 + 1 >= 0 && w0 + 1 < G.Zw) ? __ldg(row + w0 + 1) : 0u;
                const unsigned bits = (unsigned)(((((unsigned long long)hi << 32) | lo) >> sh) & wmask);
#pragma unroll
                for (int j = 0; j < FE_ZRUN; j++)
                    if ((bits >> j) & cr.y) alive &= ~(1u << j);
            }
            const unsigned exist = (iz0 + FE_ZRUN <= G.Z) ? ((1u << FE_ZRUN) - 1u) : ((1u << (G.Z - iz0)) - 1u);
            uint4 *o = reinterpret_cast<uint4 *>(A.out) + ((size_t)ix * G.Y + iy) * G.Z + iz0;
            if (!A.trav) {                                                // a settled voxel is not traversable: nothing to mark
#pragma unroll
                for (int j = 0; j < FE_ZRUN; j++)
                    if (((exist & ~alive) >> j) & 1u) o[j] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        // warp-wide append of the runs that still have an open voxel
        const unsigned open = __ballot_sync(0xffffffffu, alive != 0u);
        if (open == 0u) continue;
        unsigned base = 0;
        if (lane == 0) base = atomicAdd(A.surv_count, (unsigned)__popc(open));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (alive) A.surv[base + __popc(open & ((1u << lane) - 1u))] = make_uint2((unsigned)r, alive);
    }
}

// pass 2: one thread per surviving run — the one-pass kernel's window scan, masks accumulated for the open voxels only
__global__ void __launch_bounds__(256) k_frontend_survivors(const __grid_constant__ FrontArgs A) {
    extern __shared__ __align__(16) uint32_t fe_sm[];
    frontend_stage_masks(A, fe_sm);
    const uint4 *sm4 = reinterpret_cast<const uint4 *>(fe_sm);
    const DevGrid &G = A.grid;
    const int ks = A.ks, side = (ks - 1) / 2;
    const int zruns = (G.Z + FE_ZRUN - 1) / FE_ZRUN;
    const unsigned n = *A.surv_count;
    const uint4 valid = make_uint4(A.natt >= 32 ? 0xffffffffu : ((1u << A.natt) - 1u),
                                   A.natt >= 64 ? 0xffffffffu : (A.natt > 32 ? ((1u << (A.natt - 32)) - 1u) : 0u),
                                   A.natt >= 96 ? 0xffffffffu : (A.natt > 64 ? ((1u << (A.natt - 64)) - 1u) : 0u),
                                   A.natt >= 128 ? 0xffffffffu : (A.natt > 96 ? ((1u << (A.natt - 96)) - 1u) : 0u));
    const int wbits = ks + FE_ZRUN - 1;
    const unsigned long long wmask = (1ull << wbits) - 1ull;
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 sv = A.surv[i];
        const unsigned r = sv.x, alive = sv.y;
        const int zr = (int)(r % (unsigned)zruns), iy = (int)((r / (unsigned)zruns) % (unsigned)G.Y), ix = (int)(r / ((unsigned)zruns * (unsigned)G.Y));
        const int iz0 = zr * FE_ZRUN;
        uint4 m[FE_ZRUN];
#pragma unroll
        for (int j = 0; j < FE_ZRUN; j++) m[j] = ((alive >> j) & 1u) ? make_uint4(0u, 0u, 0u, 0u) : valid;   // settled voxels never hold the run back
        const int z0 = iz0 - side;
        const int w0 = (z0 >= 0) ? (z0 >> 5) : -1;
        const int sh = z0 - 32 * w0;
        for (int k = 0; k < A.nurow; k++) {
            const uint2 ur = __ldg(A.urows + k);
            const int a = (int)(ur.x & 0xffu), b = (int)(ur.x >> 8);
            const int x = ix + a - side, y = iy + b - side;
            if (x < 0 || x >= G.X || y < 0 || y >= G.Y) continue;
            const uint32_t *row = G.bits + ((size_t)x * G.Y + y) * G.Zw;
            const uint32_t lo = (w0 >= 0 && w0 < G.Zw) ? __ldg(row + w0) : 0u;
            const uint32_t hi = (sh + wbits > 32 && w0 + 1 >= 0 && w0 + 1 < G.Zw) ? __ldg(row + w0 + 1) : 0u;
            unsigned span = 0u;                                  // the bits of this row that can touch an open voxel
#pragma unroll
            for (int j = 0; j < FE_ZRUN; j++) if ((alive >> j) & 1u) span |= ur.y << j;
            unsigned bits = (unsigned)(((((unsigned long long)hi << 32) | lo) >> sh) & wmask) & span;
            const uint4 *mrow = sm4 + (size_t)((a * ks + b) * ks);
            while (bits) {
                const int p = __ffs((int)bits) - 1;
                bits &= bits - 1;
#pragma unroll
                for (int j = 0; j < FE_ZRUN; j++) {
                    const int c = p - j;
                    if (c >= 0 && c < ks && ((alive >> j) & 1u)) { const uint4 t = mrow[c]; m[j].x |= t.x; m[j].y |= t.y; m[j].z |= t.z; m[j].w |= t.w; }
                }
            }
        }
        if (A.trav) {
            unsigned fit = 0u;
#pragma unroll
            for (int j = 0; j < FE_ZRUN; j++)
                if (((alive >> j) & 1u) && any4(make_uint4(~m[j].x & valid.x, ~m[j].y & valid.y, ~m[j].z & valid.z, ~m[j].w & valid.w))) fit |= 1u << j;
            frontend_mark_run(A, ix, iy, iz0, fit);
            continue;
        }
        uint4 *o = reinterpret_cast<uint4 *>(A.out) + ((size_t)ix * G.Y + iy) * G.Z + iz0;
#pragma unroll
        for (int j = 0; j < FE_ZRUN; j++)
            if ((alive >> j) & 1u) o[j] = make_uint4(~m[j].x & valid.x, ~m[j].y & valid.y, ~m[j].z & valid.z, ~m[j].w & valid.w);
    }
}

// ---- the same two passes, restated for throughput ---------------------------------------------------------------------------------
// Pass 1, bit-parallel along z: a thread owns one 32-voxel word of a z row and ORs, for every core offset, the occupancy row shifted by
// that offset — two instructions settle 32 voxels against one offset. The output buffer is zero-filled beforehand (a settled voxel's
// answer IS the zero mask), so pass 1 writes nothing but the list of runs that still have an open voxel.
constexpr int FE_RUNS_PER_WORD = 32 / FE_ZRUN;
static_assert(32 % FE_ZRUN == 0, "a z-run must not straddle a 32-voxel word");
__global__ void __launch_bounds__(256) k_frontend_core_words(const __grid_constant__ FrontArgs A) {
    const DevGrid &G = A.grid;
    const int side = (A.ks - 1) / 2;
    const int zruns = (G.Z + FE_ZRUN - 1) / FE_ZRUN;
    const long long nword = (long long)G.X * G.Y * G.Zw;
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long rounds = (nword + stride - 1) / stride;
    for (long long it = 0; it < rounds; it++) {
        const long long wi = it * stride + (long long)blockIdx.x * blockDim.x + threadIdx.x;
        unsigned open = 0u;                                               // bit z: voxel 32 zw + z exists and no core offset is occupied
        int ix = 0, iy = 0, zw = 0;
        if (wi < nword) {
            zw = (int)(wi % G.Zw); iy = (int)((wi / G.Zw) % G.Y); ix = (int)(wi / ((long long)G.Zw * G.Y));
            unsigned hit = 0u;
            for (int k = 0; k < A.ncore; k++) {
                const uint2 cr = __ldg(A.core_rows + k);
                const int x = ix + (int)(cr.x & 0xffu) - side, y = iy + (int)(cr.x >> 8) - side;
                if (x < 0 || x >= G.X || y < 0 || y >= G.Y) continue;
                const uint32_t *row = G.bits + ((size_t)x * G.Y + y) * G.Zw;
                const uint32_t w0 = (zw > 0) ? __ldg(row + zw - 1) : 0u, w1 = __ldg(row + zw), w2 = (zw + 1 < G.Zw) ? __ldg(row + zw + 1) : 0u;
                unsigned cb = cr.y;
                while (cb) {                                              // uniform across the grid: the core is a constant
                    const int d = (__ffs((int)cb) - 1) - side;            // offset along z: voxel z looks at z + d
                    cb &= cb - 1;
                    hit |= (d >= 0) ? __funnelshift_r(w1, w2, d) : __funnelshift_r(w0, w1, 32 + d);
                }
            }
            const int zleft = G.Z - 32 * zw;
            const unsigned exist = (zleft >= 32) ? 0xffffffffu : ((1u << zleft) - 1u);
            open = ~hit & exist;
        }
        // runs of this word with an open voxel -> list
        unsigned runs = 0u;                                               // bit q: run q of the word has an open voxel
#pragma unroll
        for (int q = 0; q < FE_RUNS_PER_WORD; q++) if ((open >> (q * FE_ZRUN)) & ((1u << FE_ZRUN) - 1u)) runs |= 1u << q;
        const int n = __popc(runs);
        int incl = n;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total == 0) continue;
        unsigned base = 0;
        if (lane == 31) base = atomicAdd(A.surv_count, (unsigned)total);
        base = __shfl_sync(0xffffffffu, base, 31);
        unsigned pos = base + (unsigned)(incl - n);
        const unsigned r0 = (unsigned)(((long long)ix * G.Y + iy) * zruns + (long long)zw * FE_RUNS_PER_WORD);
        while (runs) {
            const int q = __ffs((int)runs) - 1;
            runs &= runs - 1;
            A.surv[pos++] = make_uint2(r0 + (unsigned)q, (open >> (q * FE_ZRUN)) & ((1u << FE_ZRUN) - 1u));
        }
    }
}

// Pass 2, table-driven: for a chunk of <= FE_CHUNK_BITS consecutive offsets of a kernel row, the occupancy pattern under the chunk
// indexes a table whose entry is the OR of the pattern's offset masks — one shared-memory load and four ORs per (chunk, open voxel)
// whatever the pattern (the empty pattern reads the table's zero entry). No data-dependent loop, no branch.
constexpr int FE_CHUNK_BITS = 8;
__global__ void __launch_bounds__(1024) k_frontend_survivors_tab(const __grid_constant__ FrontArgs A) {
    extern __shared__ __align__(16) uint32_t fe_sm[];
    uint4 *tab = reinterpret_cast<uint4 *>(fe_sm);
    // per chunk: {row offset in words relative to the window's first row, c0 | first chunk of its row << 8 | a << 16 | b << 24, pattern mask, table offset}
    uint4 *chk = tab + A.ntab;
    const DevGrid &G = A.grid;
    for (int k = threadIdx.x; k < A.ntab; k += blockDim.x) tab[k] = A.tab[k];
    for (int k = threadIdx.x; k < A.nchunk; k += blockDim.x) {
        const uint2 c = A.chunks[k];
        const unsigned a = c.x & 0xffu, b = (c.x >> 8) & 0xffu;
        const unsigned first = (k == 0 || (A.chunks[k - 1].x & 0xffffu) != (c.x & 0xffffu)) ? 1u : 0u;
        chk[k] = make_uint4((a * (unsigned)G.Y + b) * (unsigned)G.Zw, ((c.x >> 16) & 0xffu) | (first << 8) | (a << 16) | (b << 24), (1u << (c.x >> 24)) - 1u, c.y);
    }
    __syncthreads();
    const int ks = A.ks, side = (ks - 1) / 2;
    const int zruns = (G.Z + FE_ZRUN - 1) / FE_ZRUN;
    const unsigned n = *A.surv_count;
    const uint4 valid = make_uint4(A.natt >= 32 ? 0xffffffffu : ((1u << A.natt) - 1u),
                                   A.natt >= 64 ? 0xffffffffu : (A.natt > 32 ? ((1u << (A.natt - 32)) - 1u) : 0u),
                                   A.natt >= 96 ? 0xffffffffu : (A.natt > 64 ? ((1u << (A.natt - 64)) - 1u) : 0u),
                                   A.natt >= 128 ? 0xffffffffu : (A.natt > 96 ? ((1u << (A.natt - 96)) - 1u) : 0u));
    const int wbits = ks + FE_ZRUN - 1;
    const unsigned wmask = (wbits >= 32) ? 0xffffffffu : ((1u << wbits) - 1u);
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 sv = A.surv[i];
        const unsigned r = sv.x, alive = sv.y;
        const int zr = (int)(r % (unsigned)zruns), iy = (int)((r / (unsigned)zruns) % (unsigned)G.Y), ix = (int)(r / ((unsigned)zruns * (unsigned)G.Y));
        const int iz0 = zr * FE_ZRUN;
        uint4 m[FE_ZRUN];
        unsigned am[FE_ZRUN];                                             // all ones for an open voxel: a settled voxel always reads entry 0
#pragma unroll
        for (int j = 0; j < FE_ZRUN; j++) { m[j] = make_uint4(0u, 0u, 0u, 0u); am[j] = 0u - ((alive >> j) & 1u); }
        const int z0 = iz0 - side;
        const int w0 = (z0 >= 0) ? (z0 >> 5) : -1;
        const int sh = z0 - 32 * w0;
        // interior runs (the whole window inside the map, both words of every row present): no bounds test per row
        const bool interior = ix >= side && ix + side < G.X && iy >= side && iy + side < G.Y && w0 >= 0 && w0 + 1 < G.Zw;
        const uint32_t *base = G.bits + ((long long)(ix - side) * G.Y + (long long)(iy - side)) * G.Zw + w0;   // dereferenced only when interior
        asm volatile("" : "+l"(base));                                    // keep the pointer in registers: do not recompute it per row
        unsigned bits = 0u;
        for (int k = 0; k < A.nchunk; k++) {
            const uint4 ck = chk[k];
            if (ck.y & 0x100u) {                                          // first chunk of a kernel row: read the row's window
                if (interior) {
                    const uint32_t *rp = base + ck.x;
                    bits = __funnelshift_r(__ldg(rp), __ldg(rp + 1), sh) & wmask;
                } else {
                    const int x = ix + (int)((ck.y >> 16) & 0xffu) - side, y = iy + (int)(ck.y >> 24) - side;
                    bits = 0u;
                    if (x >= 0 && x < G.X && y >= 0 && y < G.Y) {
                        const uint32_t *row = G.bits + ((size_t)x * G.Y + y) * G.Zw;
                        const uint32_t lo = (w0 >= 0 && w0 < G.Zw) ? __ldg(row + w0) : 0u;
                        const uint32_t hi = (w0 + 1 >= 0 && w0 + 1 < G.Zw) ? __ldg(row + w0 + 1) : 0u;
                        bits = (unsigned)((((unsigned long long)hi << 32) | lo) >> sh) & wmask;
                    }
                }
            }
            const unsigned bc = bits >> (ck.y & 0xffu);
            const uint4 *t = tab + ck.w;
            // no branch: pattern 0 (and every pattern of a settled voxel) reads entry 0, the zero mask
#pragma unroll
            for (int j = 0; j < FE_ZRUN; j++) {
                const uint4 v = t[(bc >> j) & ck.z & am[j]];
                m[j].x |= v.x; m[j].y |= v.y; m[j].z |= v.z; m[j].w |= v.w;
            }
        }
        if (A.trav) {
            unsigned fit = 0u;
#pragma unroll
            for (int j = 0; j < FE_ZRUN; j++)
                if (((alive >> j) & 1u) && any4(make_uint4(~m[j].x & valid.x, ~m[j].y & valid.y, ~m[j].z & valid.z, ~m[j].w & valid.w))) fit |= 1u << j;
            frontend_mark_run(A, ix, iy, iz0, fit);
            continue;
        }
        uint4 *o = reinterpret_cast<uint4 *>(A.out) + ((size_t)ix * G.Y + iy) * G.Z + iz0;
#pragma unroll
        for (int j = 0; j < FE_ZRUN; j++)
            if ((alive >> j) & 1u) o[j] = make_uint4(~m[j].x & valid.x, ~m[j].y & valid.y, ~m[j].z & valid.z, ~m[j].w & valid.w);
    }
}

// checkKernelValue's choice given the colliding set m of the child voxel: the first attitude in visit_kernels_by_distance's order that
// fits; returns 0 (child = father) when none does
__device__ __forceinline__ uint8_t frontend_visit(const FrontArgs &A, const uint32_t m[4], double fr, double fp, double &cr_out, double &cp_out) {
    const int fi = (int)((fr + A.max_roll) / A.ang_res), fj = (int)((fp + A.max_pitch) / A.ang_res);   // checkKernelValue (swm:917-918)
    double cr = fr, cp = fp;
    uint8_t ok = 0;
    if (fi >= 0 && fi < A.xk && fj >= 0 && fj < A.yk) {
        const uint8_t *ord = A.order + (size_t)(fi * A.yk + fj) * A.natt;
        for (int k = 0; k < A.natt; k++) {
            const int att = ord[k];
            if (att == 0xff) break;
            if (!((m[att >> 5] >> (att & 31)) & 1u)) {
                const int ri = att / A.yk, rj = att - ri * A.yk;
                cr = fr + (ri - fi) * A.ang_res; cp = fp + (rj - fj) * A.ang_res;
                ok = 1;
                break;
            }
        }
    }
    cr_out = cr; cp_out = cp;
    return ok;
}

__global__ void __launch_bounds__(256) k_frontend_check(const __grid_constant__ FrontArgs A) {
    extern __shared__ __align__(16) uint32_t fe_sm[];
    frontend_stage_masks(A, fe_sm);
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= A.nq) return;
    const int ix = A.q_ind[3 * q], iy = A.q_ind[3 * q + 1], iz = A.q_ind[3 * q + 2];
    const double fr = A.q_father[2 * q], fp = A.q_father[2 * q + 1];
    uint32_t m[4];
    frontend_colliding(A, fe_sm, ix, iy, iz, m);
    for (int k = 0; k < 4; k++) A.out[4 * (size_t)q + k] = ~m[k];
    double cr, cp;
    const uint8_t ok = frontend_visit(A, m, fr, fp, cr, cp);
    A.q_child[2 * q] = cr; A.q_child[2 * q + 1] = cp; A.q_ok[q] = ok;
}

}  // namespace isdf
