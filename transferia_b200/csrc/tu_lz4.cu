// translation unit of the lz4 kernels
#define TF_KERNELS_LZ4
#include "kernels_lz4.cuh"
