// The gemm_tc_kernel instantiations of 128-wide tiles (gemm_tc.cuh: GLG_GEMM_INSTANCES_BN128); one unit per tile width
// keeps each compile short and lets them build in parallel.
#define GLG_GEMM_KERNEL_UNIT
#include "gemm_tc.cuh"

namespace glg {
GLG_GEMM_INSTANCES_BN128(GLG_GEMM_INSTANTIATE)
}  // namespace glg
