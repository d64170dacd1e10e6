// gemm_f16_kernel instantiations of the ping-pong schedule (vf_gemm_f16*): plain and split-fp16 output, 4 tile widths x
// 5 activations each.
#include "gemm_kernel.cuh"

namespace vf {
template int launch_bn<1, false, true>(GEMM_LAUNCH_ARGS);
template int launch_bn<1, true, true>(GEMM_LAUNCH_ARGS);
}  // namespace vf
