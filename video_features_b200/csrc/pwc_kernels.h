// Launchers of the PWC-Net memory-bound kernels (pwc_kernels.cu).  Volumes are raft_kernels.h's Vol2: channels-last
// fp16 rows of zero-bordered 2-D volumes, every activation a split-fp16 pair [hi | lo].
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "raft_kernels.h"

namespace vf {

// frames n x (Hs x Ws x 3 if !chw else 3 x Hs x Ws), uint8 or fp32 in [0,255] -> x[:, [2,1,0]] / 255 -> bilinear
// (align_corners=False) resize to the valid region of `vo` (H x W) -> rows of 16 columns [hi 8 (3 used) | lo 8]
int pwc_input_pack(const void* img, int is_u8, int chw, int n, int Hs, int Ws, __half* out, const Vol2& vo, cudaStream_t s);
// second frame's features of every pair, backward-warped: out[b][y+4][x+4][c] (fp32, border 4, C channels) =
// mask * bilinear(f2)(x + dbl*u, y + dbl*v) with zeros outside (grid_sample, align_corners=True), mask = 1 where the
// in-bounds bilinear weights sum to more than 0.999, else 0; pair b reads frame b+1 of `feat` (pitch ldf, [hi C8 | lo C8])
// and its flow (hi, lo at column uf_col, uf_col + 8 of `cat`); uf_col < 0: no warp (level 6).  mask_out (may be null):
// the mask per pair and pixel.
int pwc_warp(const __half* feat, const Vol2& vf, int ldf, int C, int C8, const __half* cat, const Vol2& vc, int ldc,
             int uf_col, float dbl, int n_pairs, float* out, float* mask_out, cudaStream_t s);
// cost volume of every pair: leaky_relu(sum_c f1(y,x) f2w(y+dy, x+dx) / C, 0.1) for the 81 displacements (c = 9(dy+4) +
// dx+4) written as split pairs at columns vol_col (hi) / vol_col + 88 (lo) of `cat`; f1_col >= 0 also copies the first
// frame's features (2*C8 columns) to column f1_col.
int pwc_correlation(const __half* feat, const Vol2& vf, int ldf, int C, int C8, const float* f2w, __half* cat,
                    const Vol2& vc, int ldc, int vol_col, int f1_col, int n_pairs, cudaStream_t s);
// ConvTranspose2d(4, 2, 1) output phases -> the next finer level: up[coarse row][(py*2+px)*2 + ch] (fp32, pitch 8) goes
// to fine position (2m+py, 2n+px) as a split pair at columns col (hi 8) / col + 8 (lo 8) of `cat`
int pwc_up_scatter(const float* up, const Vol2& vu, __half* cat, const Vol2& vc, int ldc, int col, cudaStream_t s);
// 20 * bilinear(flow + refine, (Ho, Wo), align_corners=False), x scaled by Wo/Wp and y by Ho/Hp -> out (n, 2, Ho, Wo)
int pwc_output(const __half* flow, const float* refine, const Vol2& v, int n, int Ho, int Wo, int Hp, int Wp, float* out,
               cudaStream_t s);

}  // namespace vf
