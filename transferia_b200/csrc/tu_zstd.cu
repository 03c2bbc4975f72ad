// translation unit of the zstd kernels
#define TF_KERNELS_ZSTD
#include "kernels_zstd.cuh"
