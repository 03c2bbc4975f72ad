// The one launcher of tfgpu.cu. Every kernel is declared in its family header (kernels_*.cuh) and defined there under the family's
// TF_KERNELS_* guard, which only that family's translation unit (tu_*.cu) sets: the families compile in parallel, and tfgpu.cu,
// which sees the declarations but none of the kernel bodies, launches them through the host stubs those units export.
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
#include "kernels_zstd.cuh"
namespace tfk {
struct CudaError { cudaError_t e; const char* what; };      // a failed CUDA call; `what` names the call, or the kernel of a launch

// Launches kernel k on stream s and counts the launch in e->launches. With profiling on, a pair of CUDA events named after the
// kernel brackets it; the first launch of a new entry-point call (e->call, stamped by on_device) starts the profile afresh, so the
// profile holds every launch of the last call that launched anything. A launch the runtime refuses throws CudaError naming the kernel.
template <typename E, typename... P, typename... A>
void launch_kernel(E* e, const char* name, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, const A&... args) {
    e->launches++;
    if (e->prof_on) {
        if (e->prof_call != e->call) { e->prof_call = e->call; e->prof_n = 0; }
        while ((int)e->prof_ev.size() < 2 * (e->prof_n + 1)) { cudaEvent_t ev; cudaEventCreate(&ev); e->prof_ev.push_back(ev); }
        if ((int)e->prof_names.size() <= e->prof_n) e->prof_names.resize(e->prof_n + 1);
        e->prof_names[e->prof_n] = name; cudaEventRecord(e->prof_ev[2 * e->prof_n], s);
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    const cudaError_t r = cudaLaunchKernelEx(&cfg, k, args...);
    if (e->prof_on) { cudaEventRecord(e->prof_ev[2 * e->prof_n + 1], s); e->prof_n++; }
    if (r != cudaSuccess) throw CudaError{r, name};
}
}  // namespace tfk
// TF_LAUNCH(e, k_x, grid, block, smem, stream, args...): the profile name is the kernel's own
#define TF_LAUNCH(e, k, ...) ::tfk::launch_kernel(e, #k, k, __VA_ARGS__)
