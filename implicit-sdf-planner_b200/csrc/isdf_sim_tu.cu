// Translation unit of the closed-loop simulation (isdf_sim.cuh): k_simulate and k_sim_poison. Compiled with -fmad=false, so the model's
// FP64 and the attitude loop's FP32 arithmetic round operation by operation like the reference's g++ -O3 build; a unit of its own so
// that the objects of the others stay exactly what they are.
#define ISDF_SIM_TU 1
#include "isdf_sim.cuh"

namespace isdf {

cudaError_t simulate_launch(const SimArgs &A, cudaStream_t st) {
    k_simulate<<<(A.R + SIM_THREADS - 1) / SIM_THREADS, SIM_THREADS, 0, st>>>(A);
    return cudaGetLastError();
}

cudaError_t sim_poison_launch(isdf_sim_summary *s, int R, cudaStream_t st) {
    k_sim_poison<<<(R + 255) / 256, 256, 0, st>>>(s, R);
    return cudaGetLastError();
}

}  // namespace isdf
