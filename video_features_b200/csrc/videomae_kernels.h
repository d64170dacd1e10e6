// Kernels of the VideoMAE towers (videomae.cu): the tubelet transform, the positional add, the clip mean and the
// long-sequence wgmma attention.
#pragma once
#include "internal.h"
#include "r21d_kernels.h"

namespace vf {

constexpr int VM_T = 16, VM_CROP = 224, VM_TUBE = 2, VM_PATCH = 16;
constexpr int VM_TOKENS = (VM_T / VM_TUBE) * (VM_CROP / VM_PATCH) * (VM_CROP / VM_PATCH);   // 1568
constexpr int VM_PK = 3 * VM_TUBE * VM_PATCH * VM_PATCH;                                      // 1536
constexpr int VM_MAX_S = 2048;

// the processor's Normalize constants, fp32
struct VmNorm { float mean[3], std[3]; };

// Tubelet rows of m clips: row (clip, t / 2, y, x) of 1536 columns c * 512 + dt * 256 + py * 16 + px (the flattening
// of patch_embeddings.projection.weight[D, 3, 2, 16, 16]).
// u8: frame t of clip b is frames[st.first[b] + t] (H x W x 3 BGR, already resized); the 224 x 224 window at (cy, cx),
// BGR->RGB, fp32(double(v) / 255), then (x - mean) / std in fp32, then fp16.
int videomae_tubelets_u8(const uint8_t* frames, const R21DStarts& st, int m, int H, int W, int cy, int cx,
                         const VmNorm& nm, __half* out, cudaStream_t s);
// f32: m x 16 x 3 x 224 x 224 clips (the processor's pixel_values), already transformed
int videomae_tubelets_f32(const float* clips, int m, __half* out, cudaStream_t s);
// x[clip][token] += pos[token] (fp32, rows of D)
int videomae_add_pos(float* x, const float* pos, int m, int D, cudaStream_t s);
// pooled[clip] = the mean of the clip's 1568 fp32 rows of D, summed in a fixed order
int videomae_mean(const float* x, int m, int D, float* pooled, cudaStream_t s);
// non-causal attention, head dim 64, on [n * S][3 * heads * 64] fp16 qkv rows -> [n * S][heads * 64] fp16;
// 1 <= S <= VM_MAX_S.  Rounding as vitl_attention: fp32 scores, P rounded to fp16 per 64-key block relative to the
// running max, fp32 output rescaled by 1 / l, rounded once to fp16.
int videomae_attention(const __half* qkv, __half* out, int n, int S, int heads, cudaStream_t s);

}  // namespace vf
