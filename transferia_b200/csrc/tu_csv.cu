// translation unit of the csv kernels
#define TF_KERNELS_CSV
#include "kernels_csv.cuh"
