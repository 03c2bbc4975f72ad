// translation unit of the encode kernels
#define TF_KERNELS_ENCODE
#include "kernels_encode.cuh"
