// translation unit of the json_out kernels
#define TF_KERNELS_JSON_OUT
#include "kernels_json_out.cuh"
