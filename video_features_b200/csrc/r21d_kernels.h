// Launchers of the R(2+1)D memory-bound kernels (r21d_kernels.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vf {

// zero-bordered 3-D volume [n][Tp][Hp][Wp][C]; valid region [t0,t1) x [h0,h1) x [w0,w1).  Same leading fields as the
// Vol of i3d.cu, so it can be handed to launch_unpack_ndhwc_raw.
struct Vol3 {
    int n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1;
    __host__ __device__ int64_t rows() const { return int64_t(n) * Tp * Hp * Wp; }
    __host__ __device__ int T() const { return t1 - t0; }
    __host__ __device__ int H() const { return h1 - h0; }
    __host__ __device__ int W() const { return w1 - w0; }
};

// clip indices of one gather: clip b of the chunk starts at frame first[b] of the per-frame phase volume
constexpr int R21D_MAX_CHUNK = 256;
struct R21DStarts { int first[R21D_MAX_CHUNK]; };

// Stem phase rows: a frame of the 112 x 112 crop as a [59][59] volume of rows [16 hi | 16 lo]; row (hq, wq) holds
// x[2(hq-2)+ph][2(wq-2)+pw][c] at column (ph*2+pw)*4 + c (c < 3), zero outside the crop.
constexpr int R21D_Q = 59;

// nf uint8 BGR frames of H x W -> per-frame phase volume [nf][59][59][32]: BGR->RGB, /255, torch bilinear resize to
// 128 x 171 (evaluated on the crop window (cy, cx) only), Normalize, split-fp16
int r21d_frames_u8(const uint8_t* frames, int nf, int H, int W, int cy, int cx, __half* out, cudaStream_t s);
// per-frame phase volume -> clip phase volume [m][T+2][59][59][32] (border frames zero)
int r21d_clip_gather(const __half* frames, const R21DStarts& st, int m, int T, __half* out, cudaStream_t s);
// m x 3 x T x 112 x 112 fp32 clips (already normalised) -> clip phase volume [m][T+2][59][59][32]
int r21d_pack_f32(const float* clips, int m, int T, __half* out, cudaStream_t s);
// temporal space-to-depth for a stride-2 (3,1,1) pad-1 consumer: out[q][p*C + c] = in_valid[2(q-1)+p][c] (zero outside);
// vo has vi's spatial extents, To = (Ti-1)/2 + 1 frames, border 1
int r21d_temporal_phase(const __half* in, const Vol3& vi, int C, __half* out, const Vol3& vo, cudaStream_t s);
// (2,2,2) subsample for the 1x1x1 stride-2 downsample: out_valid[t][y][x] = in_valid[2t][2y][2x]  (rows of C elements)
int r21d_subsample(const __half* in, const Vol3& vi, int C, __half* out, const Vol3& vo, cudaStream_t s);
// AdaptiveAvgPool3d(1) + flatten of split rows of C channels: out [v.n][C] fp32, fixed summation order
int r21d_avgpool(const __half* in, const Vol3& v, int C, float* out, cudaStream_t s);

}  // namespace vf
