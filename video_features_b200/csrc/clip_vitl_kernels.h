// Kernels of the CLIP ViT-L/14 towers (clip_vitl_kernels.cu), used by clip_vitl.cu.
#pragma once
#include "internal.h"

namespace vf {

constexpr int VITL_W = 1024;        // width of the residual stream
constexpr int VITL_PATCH = 14;
constexpr int VITL_PK = 592;        // patch-matrix columns: 3 * 14 * 14 = 588, zero-padded to a multiple of 8
constexpr int VITL_MAX_S = 577;     // tokens of the 336-pixel tower

// fp16 patch matrix [n * G * G, VITL_PK] (G = npx / 14), column c * 196 + ky * 14 + kx, columns 588..591 zero.
// u8: n x src_h x src_w x 3 frames (already resized), the npx crop window at (cy, cx), ToTensor + Normalize in fp32.
// f32: n x 3 x npx x npx, already normalised.
int vitl_patchify_u8(const uint8_t* src, int n, int src_h, int src_w, int cy, int cx, int npx, __half* patches,
                     cudaStream_t s);
int vitl_patchify_f32(const float* src, int n, int npx, __half* patches, cudaStream_t s);
// token assembly + ln_pre over rows of 1024: row (frame, t): t == 0 -> cls_pos0, t > 0 -> emb[frame * (T - 1) + t - 1]
// + pos[t]; x = LN(row), fp32
int vitl_embed_layernorm(const float* emb, const float* pos, const float* cls_pos0, const float* gamma, const float* beta,
                         float* x, int n_frames, int tokens, cudaStream_t s);
// out = LN(x) over rows of 1024 fp32 (row pitch x_stride), fp16 out (row pitch out_stride)
int vitl_layernorm(const float* x, int64_t x_stride, const float* gamma, const float* beta, __half* out,
                   int64_t out_stride, int rows, cudaStream_t s);
// Self-attention, head dim 64, S <= 577 tokens per frame, keys streamed in blocks of 64.  qkv: [n_frames * S, 3 * heads * 64]
// fp16 (q | k | v, head h at columns h * 64 of each third) -> out: [n_frames * S, heads * 64] fp16.
int vitl_attention(const __half* qkv, __half* out, int n_frames, int S, int heads, cudaStream_t s);

}  // namespace vf
