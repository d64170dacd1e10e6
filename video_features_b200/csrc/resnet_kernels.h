// Launchers of the ResNet memory-bound kernels (resnet_kernels.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "raft_kernels.h"

namespace vf {

// frames -> split phase volume [n][115][115][32] of the 7x7/2 stem.  is_u8: n x Hr x Wr x 3 BGR uint8, cropped at
// (cy, cx) and normalised; else n x 3 x 224 x 224 fp32, already normalised (Hr, Wr, cy, cx unused).
int resnet_input_pack(const void* src, int is_u8, int n, int Hr, int Wr, int cy, int cx, __half* out, cudaStream_t s);
// MaxPool2d(3, 2, 1) from the valid region of vi into the border-1 volume vo (split rows of C channels)
int resnet_maxpool(const __half* in, const Vol2& vi, int C, __half* out, const Vol2& vo, cudaStream_t s);
// global average pool of the valid region: out [v.n][C] fp32
int resnet_avgpool(const __half* in, const Vol2& v, int C, float* out, cudaStream_t s);

}  // namespace vf
