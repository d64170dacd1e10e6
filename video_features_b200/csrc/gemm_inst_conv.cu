// gemm_f16_kernel instantiations of the conv mode (vf_conv_gemm_f16) with plain fp16 weights: plain and split-fp16
// output, 4 tile widths x 5 activations each.
#include "gemm_kernel.cuh"

namespace vf {
template int launch_bn<1, false, false>(GEMM_LAUNCH_ARGS);
template int launch_bn<1, true, false>(GEMM_LAUNCH_ARGS);
}  // namespace vf
