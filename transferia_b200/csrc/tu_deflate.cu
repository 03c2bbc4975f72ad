// translation unit of the deflate kernels
#define TF_KERNELS_DEFLATE
#include <cuda_runtime.h>
#include "kernels_deflate.cuh"
namespace tfk {
void launch_k_deflate_chunks(dim3 grid, dim3 block, size_t smem, cudaStream_t s, DeflateArgs a) { k_deflate_chunks<<<grid, block, smem, s>>>(a); }
void launch_k_deflate_finish(dim3 grid, dim3 block, size_t smem, cudaStream_t s, DeflateArgs a) { k_deflate_finish<<<grid, block, smem, s>>>(a); }
cudaError_t deflate_kernels_init() {
    return cudaFuncSetAttribute(k_deflate_chunks, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)df_smem().total);
}
}  // namespace tfk
