// translation unit of the str kernels
#define TF_KERNELS_STR
#include "kernels_str.cuh"
