// Launchers of the S3D input kernels: R(2+1)D's transform, gather and fp32 pack templates (r21d_kernels.cu) at S3D's
// geometry.  The temporal phase repack, the max pools and the (2,7,7) head are R(2+1)D's and I3D's kernels
// (r21d_kernels.h, i3d_kernels.cu), called from s3d.cu.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "r21d_kernels.h"

namespace vf {

// Stem phase rows: a frame of the 224 x 224 crop as a [115][115] volume of rows [16 hi | 16 lo]; row (hq, wq) holds
// x[2(hq-2)+ph][2(wq-2)+pw][c] at column (ph*2+pw)*4 + c (c < 3), zero outside the crop.
constexpr int S3D_Q = 115;
constexpr int S3D_CROP = 224;
constexpr int S3D_RESIZE = 256;

// nf uint8 BGR frames of H x W -> per-frame phase volume [nf][115][115][32]: BGR->RGB, torch bilinear resize to
// 256 x 256 on uint8 (float interpolation, round half to even; evaluated on the crop window (cy, cx) only), /255,
// Normalize, split-fp16
int s3d_frames_u8(const uint8_t* frames, int nf, int H, int W, int cy, int cx, __half* out, cudaStream_t s);
// per-frame phase volume -> clip phase volume [m][T+2][115][115][32] (border frames zero)
int s3d_clip_gather(const __half* frames, const R21DStarts& st, int m, int T, __half* out, cudaStream_t s);
// m x 3 x T x 224 x 224 fp32 clips (already normalised) -> clip phase volume [m][T+2][115][115][32]
int s3d_pack_f32(const float* clips, int m, int T, __half* out, cudaStream_t s);

}  // namespace vf
