// gemm_f16_kernel instantiations of the conv mode (vf_conv_gemm_f16) with split-fp16 weights (nsplit = 2): plain and
// split-fp16 output, 4 tile widths x 5 activations each.
#include "gemm_kernel.cuh"

namespace vf {
template int launch_bn<2, false, false>(GEMM_LAUNCH_ARGS);
template int launch_bn<2, true, false>(GEMM_LAUNCH_ARGS);
}  // namespace vf
