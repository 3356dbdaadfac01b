// The deep vector assembly and deep hybrid fusion kernels (deep_fuse.cuh) in a translation unit of their own, so that the
// kernels of tsgpu.cu keep their code generation. The shared headers are compiled here under renamed namespaces (their
// kernels would otherwise be defined twice in the library); the parameter blocks have the same layout as tsgpu.cu's and are
// copied across. Reached only through the launchers below; the host side is deep_fuse_host.inc.
#define TSDF_KERNELS
#define tsdev tsdev_df
#define tsk tsk_df
#define tsf tsf_df
#define tsdf tsdf_k
#include <algorithm>
#include <cstring>
#include "deep_fuse.cuh"

extern "C" __attribute__((visibility("hidden")))
cudaError_t tsgpu_launch_vec_deep_pack_(const void* params, unsigned n_deep, unsigned tiles, cudaStream_t st) {
    tsdf::VecDeepParams P;
    std::memcpy(&P, params, sizeof P);
    tsdf::vec_deep_pack_kernel<<<dim3(tiles, n_deep), 256, 0, st>>>(P);
    return cudaGetLastError();
}

extern "C" __attribute__((visibility("hidden")))
cudaError_t tsgpu_launch_vec_deep_write_(const void* in, uint32_t n_out, unsigned long long found, const void* qds, uint32_t q, void* out_kv,
                                         uint32_t kv_stride, uint32_t* out_count, uint32_t* out_found, unsigned grid, cudaStream_t st) {
    tsdf::vec_deep_write_kernel<<<grid, 256, 0, st>>>(static_cast<const tsk::DeepEntry*>(in), n_out, found, static_cast<const tsk::QDesc*>(qds), q,
                                                      static_cast<tsk::KVOut*>(out_kv), kv_stride, out_count, out_found);
    return cudaGetLastError();
}

extern "C" __attribute__((visibility("hidden")))
cudaError_t tsgpu_launch_hybrid_deep_(const void* params, unsigned n_deep, size_t smem, cudaStream_t st) {
    tsdf::HybridDeepParams P;
    std::memcpy(&P, params, sizeof P);
    cudaError_t e = cudaFuncSetAttribute(tsdf::hybrid_deep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(smem, 48 * 1024));
    if(e != cudaSuccess) return e;
    tsdf::hybrid_deep_kernel<<<n_deep, tsdf::kThreads, smem, st>>>(P);
    return cudaGetLastError();
}
