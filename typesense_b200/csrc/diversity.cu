// The diversity re-ranking kernels (diversity.cuh) in a translation unit of their own, so that the kernels of tsgpu.cu keep
// their code generation. Reached only through the launchers below; the host side is tsgpu_diversify_batch (diversity_host.inc).
#define TSDIV_KERNELS
#include <algorithm>
#include "diversity.cuh"

extern "C" __attribute__((visibility("hidden")))
cudaError_t tsgpu_launch_div_count_(const tsdiv::Params* P, unsigned nq, cudaStream_t st) {
    tsdiv::div_count_kernel<<<nq, tsdiv::kThreads, 0, st>>>(*P);
    return cudaGetLastError();
}

extern "C" __attribute__((visibility("hidden")))
cudaError_t tsgpu_launch_div_mmr_(const tsdiv::Params* P, unsigned nq, size_t smem, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(tsdiv::div_mmr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
    if(e != cudaSuccess) return e;
    tsdiv::div_mmr_kernel<<<nq, tsdiv::kThreads, smem, st>>>(*P);
    return cudaGetLastError();
}
