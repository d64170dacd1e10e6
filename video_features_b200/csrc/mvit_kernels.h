// Kernels of the MViT towers (mvit.cu): the fused clip transform into the rows of the overlapping patch conv, the
// patch embedding's class token and position embeddings, the head pooling (depthwise 3x3x3 conv + LayerNorm per head),
// the pooling attention and the skip max-pool.  Token rows are per clip [class token | T' x H x W tokens, t-major].
#pragma once
#include "internal.h"
#include "r21d_kernels.h"

namespace vf {

constexpr int MV_CROP = 224, MV_RESIZE = 256, MV_T = 16, MV_TQ = 8, MV_HEAD_DIM = 96;
constexpr int MV_PATCH_K = 441, MV_PK = 448;            // 3 x 3 x 7 x 7 patch columns, zero-padded to a GEMM width
constexpr int MV_MAX_KEYS = 416;                         // keys per shared-memory chunk of the attention
constexpr int MV_MAX_REL = 48;                           // kv grid t + h + w extents the rel-pos bias holds

// Patch rows of m clips of 16 frames: row (clip, t', h', w') (8 x 56 x 56 per clip) of 448 columns, column
// c * 147 + kt * 49 + kh * 7 + kw the flattening of conv_proj.weight[96, 3, 3, 7, 7] for input frame 2 t' + kt - 1,
// row 4 h' + kh - 3, column 4 w' + kw - 3 (zero outside the clip: Conv3d's padding (1, 3, 3)); columns 441.. zero.
// u8: frame t of clip b is frames[st.first[b] + t] (H x W x 3 BGR); BGR->RGB, bilinear resize to rh x rw of the 224 x 224
// window at (cy, cx) as swin3d_patch_u8 does, /255, Normalize(0.45, 0.225).
int mvit_patch_u8(const uint8_t* frames, const R21DStarts& st, int m, int H, int W, int rh, int rw, int cy, int cx,
                  __half* out, cudaStream_t s);
// f32: m x 3 x 16 x 224 x 224 clips, already transformed
int mvit_patch_f32(const float* clips, int m, __half* out, cudaStream_t s);
// emb: m x 25088 conv rows of 96 fp32 (bias added) -> x (and x2): per clip row 0 = class_token (+ class_pos), row 1 + p
// = emb[p] (+ temporal_pos[t] + spatial_pos[h * 56 + w]); the position tables are null for MViT-V2
int mvit_embed(const float* emb, const float* class_token, const float* class_pos, const float* temporal_pos,
               const float* spatial_pos, int m, float* x, float* x2, cudaStream_t s);

// Head pooling of one of q / k / v: src rows [n][1 + T H W] of pitch ld_src (column h * 96 + d = head h, channel d) ->
// depthwise Conv3d(96, 96, 3, stride (1, stride, stride), pad 1, no bias; weight [96][27]) per head on the tokens, the
// class token passed through, then LayerNorm(96, eps 1e-6) on every row -> dst [n][1 + T Ho Wo][heads * 96] fp16
// (Ho = (H - 1) / stride + 1).
int mvit_head_pool(const __half* src, int ld_src, int n, int heads, int T, int H, int W, int stride,
                   const float* weight, const float* gamma, const float* beta, __half* dst, cudaStream_t s);
// Skip path of a stride block: MaxPool3d((1,3,3), (1,2,2), (0,1,1)) of x [n][1 + T H W][C] fp32 -> y
// [n][1 + T Ho Wo][C], the class token copied
int mvit_skip_pool(const float* x, int n, int C, int T, int H, int W, float* y, cudaStream_t s);

// Pooling attention: q [n][1 + Nq][heads * 96] (row pitch ldq), k / v [n][1 + Nk][heads * 96] fp16 -> out
// [n][1 + Nq][heads * 96] fp16: softmax(q k^T / sqrt(96) + bias) v per (clip, head), fp32 softmax.  rel: bias(q, k) =
// q . rel_t[dist_t] + q . rel_h[dist_h] + q . rel_w[dist_w] on token rows and columns (torchvision's _add_rel_pos with
// its ratio-scaled distances; tables of 2 max(q, k) - 1 rows of 96).  resid: + q on token rows.
struct MViTAttnGeom {
    int n, heads;
    int q_thw[3], k_thw[3];     // token grids, the class token excluded
    int ldq;
    int rel, resid;
};
int mvit_attention(const __half* q, const __half* k, const __half* v, const float* rel_h, const float* rel_w,
                   const float* rel_t, __half* out, const MViTAttnGeom& g, cudaStream_t s);

}  // namespace vf
