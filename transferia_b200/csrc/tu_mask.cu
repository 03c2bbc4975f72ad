// translation unit of the mask kernels
#define TF_KERNELS_MASK
#include "kernels_mask.cuh"
