// Sum of the sharded evaluation's 19N+1 doubles over the ranks, through NVLink / NVSwitch PEER MEMORY instead of a library
// collective. The vector is 10 KB: an NCCL all-reduce of that size is pure latency (~45 us measured at 8 GPUs, against a
// ~100 us sharded evaluation); here the LAST CTA of the evaluation's epilogue kernel — the one that has just produced the
// rank's vector — stores it straight into every peer's receive slot (plain st.global over NVLink, 8 x 10 KB), raises a flag
// on every peer, waits for the peers' flags on its own buffer and adds the `world` slots in RANK ORDER. One kernel does the
// compute tail and the exchange; the result is bit-identical on every rank and independent of arrival order.
//
// Buffer of one rank (one cudaMalloc, exported with cudaIpcGetMemHandle, opened by the peers with cudaIpcOpenMemHandle):
//   flags[2][PEER_MAX]  unsigned long long   epoch written by rank r into flags[epoch & 1][r] after its slot is complete
//   slots[2][world][cap] double              slot of rank r for epochs of that parity
// Two parities suffice: a rank can start epoch e+1 (other parity) while a peer still reads epoch e, but it cannot finish e+1
// — and hence cannot touch parity e again — before every peer has raised its e+1 flag, which a peer does only after its
// epoch-e kernel has completed (stream order).
#pragma once
#include <cstdint>

namespace isdf {

constexpr int PEER_MAX = 16;

struct PeerArgs {
    int world, rank, cap;
    unsigned long long epoch;                 // > 0, incremented per exchange (same sequence on every rank)
    unsigned long long *flags[PEER_MAX];      // peer p's flag array (own buffer for p == rank)
    double *slots[PEER_MAX];                  // peer p's slot array
    int *status;                              // own device word: set to 1 on time-out
};

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// Executed by ALL threads of one CTA. vec[0..n) holds this rank's contribution on entry and the rank-ordered sum on exit.
__device__ __forceinline__ void peer_allreduce_block(const PeerArgs &P, double *vec, int n) {
    const int par = (int)(P.epoch & 1ull);
    const size_t slot_off = ((size_t)par * P.world + P.rank) * P.cap;
    for (int p = 0; p < P.world; p++) {
        double *dst = P.slots[p] + slot_off;
        for (int k = threadIdx.x; k < n; k += blockDim.x) dst[k] = __ldcg(vec + k);
    }
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < P.world) st_release_sys(P.flags[threadIdx.x] + par * PEER_MAX + P.rank, P.epoch);
    int timed_out = 0;
    if ((int)threadIdx.x < P.world) {
        const unsigned long long *f = P.flags[P.rank] + par * PEER_MAX + threadIdx.x;
        const long long t0 = clock64();
        while (ld_acquire_sys(f) != P.epoch) {
            if (clock64() - t0 > 4000000000ll) { *P.status = 1; timed_out = 1; break; }   // ~2 s: a peer never arrived — fail loudly, do not hang
            __nanosleep(64);
        }
    }
    // a time-out must never hand partial sums to the optimiser: the whole vector (cost first) becomes NaN, which is the header's
    // contract for a failed evaluation; the host entry points additionally read *P.status and return ISDF_ERR_CUDA
    const bool failed = __syncthreads_or(timed_out) != 0;
    const double *mine = P.slots[P.rank] + (size_t)par * P.world * P.cap;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        double s = 0.0;
        for (int p = 0; p < P.world; p++) s += __ldcv(mine + (size_t)p * P.cap + k);
        vec[k] = failed ? __longlong_as_double(0x7ff8000000000000ll) : s;
    }
}

#if !defined(ISDF_DISCRETE_TU) && !defined(ISDF_CLEARANCE_TU)   // instantiated once, in isdf_api.cu
__global__ void __launch_bounds__(512) k_peer_allreduce(const __grid_constant__ PeerArgs P, double *vec, int n) {
    peer_allreduce_block(P, vec, n);
}
#endif

}  // namespace isdf
