// Kernels of the DINOv2 towers (dinov2_kernels.cu), used by dinov2.cu: the 14-pixel patch transform, token assembly and
// ViT-g/14's SwiGLU.  The attention is clip_vitl_kernels.h's vitl_attention, the LayerNorms swin3d_kernels.h's.
#pragma once
#include "internal.h"

namespace vf {

constexpr int DV_CROP = 224, DV_RESIZE = 256, DV_PATCH = 14, DV_GRID = 16, DV_PATCHES = DV_GRID * DV_GRID;
constexpr int DV_PK = 592;          // patch-row columns: 3 * 14 * 14 = 588, zero-padded to a multiple of 8

// fp16 patch rows [n * 256, DV_PK], column c * 196 + ky * 14 + kx (the flattening of patch_embed.proj.weight), columns
// 588..591 zero.  u8: n x src_h x src_w x 3 BGR frames (already resized), the 224 crop window at (cy, cx), RGB channel c
// read from byte 2 - c, ToTensor + ImageNet Normalize in fp32.  f32: n x 3 x 224 x 224, already normalised.
int dinov2_patchify_u8(const uint8_t* src, int n, int src_h, int src_w, int cy, int cx, __half* patches, cudaStream_t s);
int dinov2_patchify_f32(const float* src, int n, __half* patches, cudaStream_t s);
// Token rows of the fp32 residual stream x [n * S, D] (S = 1 + n_reg + 256): row 0 cls_pos0 (cls_token + pos[0]),
// rows 1 .. n_reg reg[r], then patch i: emb[frame * 256 + i] + pos[1 + i]
int dinov2_tokens(const float* emb, const float* pos, const float* cls_pos0, const float* reg, int n_reg, float* x, int n,
                  int D, cudaStream_t s);
// out[r][j] = fp16(silu(a) * b), a = ab[r][j], b = ab[r][hidden + j], in fp32
int dinov2_swiglu(const float* ab, int rows, int hidden, __half* out, cudaStream_t s);

}  // namespace vf
