#include "common.cuh"
S6_API const char* sam6d_version(void) { return "sam6d_b200 0.1.0 sm_90a"; }
