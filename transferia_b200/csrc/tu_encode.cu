// translation unit of the encode kernels
#define TF_KERNELS_ENCODE
#include <cuda_runtime.h>
#include "kernels_encode.cuh"
namespace tfk {
void launch_k_strictify(dim3 grid, dim3 block, size_t smem, cudaStream_t s, StrictArgs a) { k_strictify<<<grid, block, smem, s>>>(a); }
void launch_k_filter(dim3 grid, dim3 block, size_t smem, cudaStream_t s, FilterArgs a) { k_filter<<<grid, block, smem, s>>>(a); }
void launch_k_scan_blockcnt(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint32_t* blockcnt, uint32_t* blockoff, uint32_t nblocks, DState* st) { k_scan_blockcnt<<<grid, block, smem, s>>>(blockcnt, blockoff, nblocks, st); }
void launch_k_collect_errors(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* errcode, const uint16_t* errstep, uint64_t nrows, DevRowErr* out, unsigned long long* counter, unsigned long long cap) { k_collect_errors<<<grid, block, smem, s>>>(errcode, errstep, nrows, out, counter, cap); }
void launch_k_compact_sel(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* keep, const uint32_t* blockoff, uint64_t nrows, uint32_t* sel) { k_compact_sel<<<grid, block, smem, s>>>(keep, blockoff, nrows, sel); }
void launch_k_layout_scan(dim3 grid, dim3 block, size_t smem, cudaStream_t s, LayoutArgs a) { k_layout_scan<<<grid, block, smem, s>>>(a); }
void launch_k_layout_finish(dim3 grid, dim3 block, size_t smem, cudaStream_t s, LayoutArgs a) { k_layout_finish<<<grid, block, smem, s>>>(a); }
void launch_k_layout_columnar(dim3 grid, dim3 block, size_t smem, cudaStream_t s, LayoutArgs a, ColRegions* regions) { k_layout_columnar<<<grid, block, smem, s>>>(a, regions); }
void launch_k_encode_fixed(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a) { k_encode_fixed<<<grid, block, smem, s>>>(a); }
void launch_k_pack_validity(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a) { k_pack_validity<<<grid, block, smem, s>>>(a); }
void launch_k_measure(dim3 grid, dim3 block, size_t smem, cudaStream_t s, MeasureArgs a) { k_measure<<<grid, block, smem, s>>>(a); }
}  // namespace tfk
