// kw_search_kernel<REGSCORE = true, .., DEEP = true>: the unit kernel of deep queries (TSGPU_QFLAG_DEEP_TOPSTER,
// deep_topster.cuh). Built like kw_regscore.cu — the register-resident scorer at 5 CTAs per SM — in a translation unit of its
// own with its own renamed copies of the device functions, so the kernels that existed before keep their code generation.
// Reached only through the launcher below.
#define TSGPU_KW_SEARCH_ONLY
#define TSGPU_KW_MIN_CTAS 5
#define tsdev tsdev_dp
#define tsk tsk_dp
#include <algorithm>
#include <cstring>
#include "kw_kernels.cuh"

// smem carries no top-K buffer (KP = 0); P.pool_* address the deep buffer and P.q_thr the per-query cursors
extern "C" __attribute__((visibility("hidden")))
cudaError_t tsgpu_launch_kw_search_deep(const void* index_dev, const void* kw_params, unsigned n_units, size_t smem, cudaStream_t st) {
    tsk::IndexDev ix;                     // same layouts as tsgpu.cu's tsk::IndexDev / tsk::KwParams (same header)
    tsk::KwParams P;
    std::memcpy(&ix, index_dev, sizeof ix);
    std::memcpy(&P, kw_params, sizeof P);
    auto kern = P.F == 1 ? tsk::kw_search_kernel<true, true, true> : tsk::kw_search_kernel<true, false, true>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
    if(e != cudaSuccess) return e;
    kern<<<n_units, tsk::kThreads, smem, st>>>(ix, P);
    return cudaGetLastError();
}
