// Kernels of the CLIP text tower (clip_text.cu): token embedding, causal self-attention, the EOT-row gather and the
// row L2 normalisation the zero-shot head shares.
#pragma once
#include "internal.h"

namespace vf {

constexpr int CT_HEAD_DIM = 64, CT_MAX_CTX = 77;

// x[b][t] = tok_emb[tokens[b][t]] + pos[t] for t < L: n x L rows of W fp32; tokens rows of `ctx` int32 on the device
int clip_text_embed(const int32_t* tokens, int ctx, int n, int L, const float* tok_emb, const float* pos, int W, float* x,
                    cudaStream_t s);
// Causal self-attention, heads of 64: qkv n x L rows [q | k | v] of 3W fp16 (head h at columns h * 64 of each) ->
// att n x L x W fp16, row i = softmax(q_i k_j / 8, j <= i) . v_j.  Row i reads rows 0..i only and its sums run in an
// order fixed by i alone, so its result does not depend on L.  L <= 77.
int clip_text_attention(const __half* qkv, int n, int L, int heads, __half* att, cudaStream_t s);
// out[b] = x[b][eot[b]]: rows of W fp32 of n prompts of L rows
int clip_text_gather(const float* x, const int32_t* eot, int n, int L, int W, float* out, cudaStream_t s);
// out[r] = x[r] / ||x[r]||_2 over rows of C fp32 (in place allowed); the sum of squares runs in a fixed order
int l2_normalize_rows(const float* x, int n, int C, float* out, cudaStream_t s);

}  // namespace vf
