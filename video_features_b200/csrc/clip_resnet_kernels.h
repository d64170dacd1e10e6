// Launchers of the CLIP ResNet memory- and latency-bound kernels (clip_resnet_kernels.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "raft_kernels.h"

namespace vf {

// frames -> split phase volume [n][npx/2 + 2][npx/2 + 2][32] of the 3x3/2 stem conv.  is_u8: n x Hr x Wr x 3 uint8,
// already resized, cropped at (cy, cx) and normalised; else n x 3 x npx x npx fp32, already normalised.
int clip_rn_input_pack(const void* src, int is_u8, int n, int Hr, int Wr, int cy, int cx, int npx, __half* out,
                       cudaStream_t s);
// layer4 (valid region of v, E channels) -> T = HW + 1 token rows per frame [hi E | lo E]: mean, then the positions,
// each plus its positional embedding (pos: device fp32 [T][E])
int clip_rn_tokens(const __half* in, const Vol2& v, int E, const float* pos, __half* tokens, cudaStream_t s);
// one query per (frame, head) over T keys: kv [n*T][2E] fp32 (k | v), q [n][E] fp32 -> out [n][hi E | lo E]
int clip_rn_attention(const float* kv, const float* q, int n, int T, int E, __half* out, cudaStream_t s);

}  // namespace vf
