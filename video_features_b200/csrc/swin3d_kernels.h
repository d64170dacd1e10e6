// Kernels of the Swin3D towers (swin3d.cu): the fused clip transform into patch rows, width-generic LayerNorms (patch
// embedding, norm1 / norm2, patch merging, the final norm with the clip mean) and the shifted-window attention.
#pragma once
#include "internal.h"
#include "r21d_kernels.h"

namespace vf {

constexpr int SW_CROP = 224, SW_RESIZE = 256, SW_PK = 96;     // patch rows: 3 x 2 x 4 x 4 columns
constexpr int SW_HEAD_DIM = 32, SW_TABLE = 15 * 13 * 13;     // bias table rows of the (8,7,7) window
constexpr int SW_MAX_VOL = 8 * 7 * 7;

// Patch rows of m clips of T frames: row (clip, t', h', w') of 96 columns c * 32 + kt * 16 + kh * 4 + kw (the
// flattening of patch_embed.proj.weight[C, 3, 2, 4, 4]); frame 2 t' + kt >= T is the zero frame F.pad appends.
// u8: frame t of clip b is frames[st.first[b] + t] (H x W x 3 BGR); BGR->RGB, bilinear resize to rh x rw of the
// 224 x 224 window at (cy, cx) as torch's float interpolation of the bytes, round half to even, /255, Normalize.
int swin3d_patch_u8(const uint8_t* frames, const R21DStarts& st, int m, int T, int H, int W, int rh, int rw, int cy,
                    int cx, __half* out, cudaStream_t s);
// f32: m x 3 x T x 224 x 224 clips, already transformed
int swin3d_patch_f32(const float* clips, int m, int T, __half* out, cudaStream_t s);
// LayerNorm (two-pass fp32 statistics, eps 1e-5 unless given: MViT's are 1e-6) of rows of C fp32 -> fp16 or fp32 rows
// (pitch C); out_f32 only: a non-null out2 receives a second copy
int swin3d_layernorm(const float* x, int C, const float* gamma, const float* beta, void* out, int out_f32, int64_t rows,
                     cudaStream_t s, float* out2 = nullptr, float eps = 1e-5f);
// PatchMerging: x [n][T'][H][W][C] fp32 (H, W even) -> LayerNorm of the rows [x0 | x1 | x2 | x3] (4C) -> fp16
// [n][T'][H/2][W/2][4C]
int swin3d_merge_layernorm(const float* x, int n, int Tq, int H, int W, int C, const float* gamma, const float* beta,
                           __half* out, cudaStream_t s);
// final norm: normed = LayerNorm(x) per row (fp32) and feat[b][c] = the mean of clip b's `per_clip` rows, summed in a
// fixed order
int swin3d_norm_mean(const float* x, int n, int per_clip, int C, const float* gamma, const float* beta, float* normed,
                     float* feat, cudaStream_t s);

// Shifted-window attention on natural-order rows.  qkv: [n][Tq][H][W][3C] fp16 (q | k | v, head h at columns h * 32),
// bias_qkv: the 3C fp32 qkv bias (the k / v of padded positions), table: [2535][heads] fp32 -> att [n][Tq][H][W][C] fp16.
// win / shift as torchvision's _get_window_and_shift_size leaves them.
struct SwinAttnGeom {
    int n, Tq, H, W, C;
    int win[3], shift[3];
};
int swin3d_attention(const __half* qkv, const float* bias_qkv, const float* table, __half* att, const SwinAttnGeom& g,
                     cudaStream_t s);
// the clamped window / shift of one block: size (Tq, H, W), shifted = odd block
SwinAttnGeom swin3d_attn_geom(int n, int Tq, int H, int W, int C, bool shifted);

}  // namespace vf
