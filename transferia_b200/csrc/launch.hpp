// Host-callable launchers: every kernel family is compiled in its own translation unit (tu_*.cu) so that the
// families build in parallel; tfgpu.cu sees the argument structs but none of the kernel bodies.
#pragma once
#include <cuda_runtime.h>
#include "kernels_encode.cuh"
#include "kernels_str.cuh"
#include "kernels_mask.cuh"
#include "kernels_lz4.cuh"
#include "kernels_csv.cuh"
#include "kernels_json_in.cuh"
#include "kernels_n2f.cuh"
#include "kernels_dbz.cuh"
#include "kernels_json_out.cuh"
#include "kernels_deflate.cuh"
namespace tfk {
void launch_k_strictify(dim3 grid, dim3 block, size_t smem, cudaStream_t s, StrictArgs a);
void launch_k_filter(dim3 grid, dim3 block, size_t smem, cudaStream_t s, FilterArgs a);
void launch_k_scan_blockcnt(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint32_t* blockcnt, uint32_t* blockoff, uint32_t nblocks, DState* st);
void launch_k_collect_errors(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* errcode, const uint8_t* errstep, uint64_t nrows, DevRowErr* out, unsigned long long* counter, unsigned long long cap);
void launch_k_compact_sel(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* keep, const uint32_t* blockoff, uint64_t nrows, uint32_t* sel);
void launch_k_layout_scan(dim3 grid, dim3 block, size_t smem, cudaStream_t s, LayoutArgs a);
void launch_k_layout_finish(dim3 grid, dim3 block, size_t smem, cudaStream_t s, LayoutArgs a);
void launch_k_layout_columnar(dim3 grid, dim3 block, size_t smem, cudaStream_t s, LayoutArgs a, ColRegions* regions);
void launch_k_encode_fixed(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a);
void launch_k_pack_validity(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a);
void launch_k_measure(dim3 grid, dim3 block, size_t smem, cudaStream_t s, MeasureArgs a);
void launch_k_str_sizes(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a);
void launch_k_encode_str_plain(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a);
void launch_k_encode_str(dim3 grid, dim3 block, size_t smem, cudaStream_t s, EncodeArgs a);
void launch_k_mask_encode(dim3 grid, dim3 block, size_t smem, cudaStream_t s, MaskArgs a);
void launch_k_shard_ids(dim3 grid, dim3 block, size_t smem, cudaStream_t s, ShardArgs a);
void launch_k_lz4_frames(dim3 grid, dim3 block, size_t smem, cudaStream_t s, Lz4Args a);
void launch_k_frame_seal(dim3 grid, dim3 block, size_t smem, cudaStream_t s, FrameArgs a);
void launch_k_csv_count_nl(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* text, uint64_t len, uint32_t* blk_cnt, const uint32_t* endbits);
void launch_k_csv_line_index(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* text, uint64_t len, const uint32_t* blk_off, uint32_t* line_end, const uint32_t* endbits);
void launch_k_widen_lens(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const LensSrc* src, uint64_t nrows, uint32_t* out);
void launch_k_csv_pass1(dim3 grid, dim3 block, size_t smem, cudaStream_t s, CsvArgs a);
void launch_k_csv_offsets(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint32_t* span_len, uint64_t nrows, uint32_t* offsets , uint64_t* col_total);
void launch_k_offsets_sum(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint32_t* span_len, uint64_t nrows, uint32_t nchunks, uint64_t* chunk_sum);
void launch_k_offsets_chunks(dim3 grid, dim3 block, size_t smem, cudaStream_t s, uint64_t* chunk_sum, uint32_t nchunks, uint64_t* col_total);
void launch_k_offsets_write(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint32_t* span_len, uint64_t nrows, uint32_t nchunks, const uint64_t* chunk_base, const uint64_t* col_total, uint32_t* offsets);
void launch_k_csv_pass2(dim3 grid, dim3 block, size_t smem, cudaStream_t s, CsvCopyArgs a);
void launch_k_json_mark_msgs(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint64_t* msg_end, uint32_t nmsgs, uint32_t* bits);
void launch_k_json_count_nonempty(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* text, const uint32_t* line_end, uint64_t nlines, uint32_t* blk_cnt);
void launch_k_json_rank(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint8_t* text, const uint32_t* line_end, uint64_t nlines, const uint32_t* blk_off, uint32_t* rank);
void launch_k_json_msg_first(dim3 grid, dim3 block, size_t smem, cudaStream_t s, const uint64_t* msg_end, uint32_t nmsgs, const uint32_t* line_end, uint64_t nlines, const uint32_t* rank, uint32_t* msg_rank0);
void launch_k_json_pass1(dim3 grid, dim3 block, size_t smem, cudaStream_t s, JsnArgs a);
void launch_k_json_pass2(dim3 grid, dim3 block, size_t smem, cudaStream_t s, JsnWriteArgs w);
void launch_k_n2f_sizes(dim3 grid, dim3 block, size_t smem, cudaStream_t s, N2fArgs a);
void launch_k_n2f_write(dim3 grid, dim3 block, size_t smem, cudaStream_t s, N2fArgs a);
void launch_k_dbz_pass1(dim3 grid, dim3 block, size_t smem, cudaStream_t s, DbzArgs a);
void launch_k_dbz_pass2(dim3 grid, dim3 block, size_t smem, cudaStream_t s, DbzWriteArgs w);
void launch_k_json_sizes(dim3 grid, dim3 block, size_t smem, cudaStream_t s, JsonArgs a);
void launch_k_json_write(dim3 grid, dim3 block, size_t smem, cudaStream_t s, JsonArgs a);
cudaError_t dbz_kernels_init();   // dynamic shared memory limit of k_dbz_pass1
void launch_k_deflate_chunks(dim3 grid, dim3 block, size_t smem, cudaStream_t s, DeflateArgs a);
void launch_k_deflate_finish(dim3 grid, dim3 block, size_t smem, cudaStream_t s, DeflateArgs a);
cudaError_t deflate_kernels_init();   // dynamic shared memory limit of k_deflate_chunks
cudaError_t lz4_kernels_init();   // dynamic shared memory limits of k_lz4_frames / k_frame_seal
}  // namespace tfk
