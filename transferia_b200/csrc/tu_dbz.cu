// translation unit of the dbz kernels
#define TF_KERNELS_DBZ
#include "kernels_dbz.cuh"
