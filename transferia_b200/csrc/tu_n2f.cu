// translation unit of the n2f kernels
#define TF_KERNELS_N2F
#include "kernels_n2f.cuh"
