// The uint8 Resize + CenterCrop arithmetic shared by the video-transformer patch kernels (swin3d_kernels.cu,
// mvit_kernels.cu): torchvision's F.resize of a uint8 frame (bilinear, no antialias: float interpolation of the bytes,
// torch.round half to even), evaluated at one pixel of the crop window, as IEEE fp32 ops in torch's order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vf {

// torch's CPU upsample_bilinear2d (align_corners=False, no scale factor) source index and weights for output index d,
// as r21d_kernels.cu computes them, with the output size a run-time value
__device__ __forceinline__ void bilinear_tap(int d, int in, int out, int& i0, int& i1, float& l0, float& l1) {
    const float scale = __fdiv_rn(float(in), float(out));
    const float src = fmaxf(__fmaf_rn(scale, __fadd_rn(float(d), 0.5f), -0.5f), 0.f);
    i0 = min(int(floorf(src)), in - 1);
    l1 = fminf(fmaxf(__fsub_rn(src, float(i0)), 0.f), 1.f);
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    l0 = __fsub_rn(1.f, l1);
}

// channel sc of the resized uint8 pixel between rows (h0, h1) with weights (a0, a1) and columns (w0, w1) with weights
// (b0, b1) of the W-wide interleaved 3-channel frame fr, divided by 255
__device__ __forceinline__ float resized_unit(const uint8_t* __restrict__ fr, int W, int sc, int h0, int h1, float a0,
                                              float a1, int w0, int w1, float b0, float b1) {
    auto px = [&](int hh, int ww) { return float(__ldg(fr + (int64_t(hh) * W + ww) * 3 + sc)); };
    const float t0 = __fmaf_rn(b0, px(h0, w0), __fmul_rn(b1, px(h0, w1)));
    const float t1 = __fmaf_rn(b0, px(h1, w0), __fmul_rn(b1, px(h1, w1)));
    return __fdiv_rn(rintf(__fmaf_rn(a0, t0, __fmul_rn(a1, t1))), 255.f);
}

}  // namespace vf
