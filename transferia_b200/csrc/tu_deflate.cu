// translation unit of the deflate kernels
#define TF_KERNELS_DEFLATE
#include "kernels_deflate.cuh"
