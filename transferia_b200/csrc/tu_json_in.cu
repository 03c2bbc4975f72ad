// translation unit of the json_in kernels
#define TF_KERNELS_JSON_IN
#include "kernels_json_in.cuh"
