// Memory-bound kernels of the DINOv2 towers (dinov2.cu): the 14-pixel patch transform from resized BGR bytes, the token
// assembly (class, register and patch rows with the 224-px positional table) and ViT-g/14's SwiGLU.
#include "common.cuh"
#include "dinov2_kernels.h"

namespace vf {

namespace {

// the hub's eval preset: Normalize with ImageNet statistics, float32-rounded like torch does
__constant__ float kDvMean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float kDvStd[3] = {0.229f, 0.224f, 0.225f};

inline unsigned nblocks(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// One thread: 8 consecutive columns of one patch row (74 groups cover the 592 columns).  ToTensor (v / 255) then
// Normalize ((x - mean) / std) as IEEE fp32 ops in torchvision's order, then fp16.
template <bool U8>
__global__ void patchify_kernel(const void* __restrict__ src, int n, int src_h, int src_w, int cy, int cx,
                                __half* __restrict__ out) {
    constexpr int GROUPS = DV_PK / 8;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * DV_PATCHES * GROUPS) return;
    const int grp = int(idx % GROUPS);
    const int64_t row = idx / GROUPS;
    const int p = int(row % DV_PATCHES), b = int(row / DV_PATCHES);
    const int py = p / DV_GRID, px = p % DV_GRID;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int col = grp * 8 + i;
        v[i] = 0.f;
        if (col < 3 * DV_PATCH * DV_PATCH) {
            const int c = col / 196, r = col % 196;
            const int y = py * DV_PATCH + r / DV_PATCH, x = px * DV_PATCH + r % DV_PATCH;
            if (U8) {
                const uint8_t u = __ldg(static_cast<const uint8_t*>(src) +
                                        ((int64_t(b) * src_h + cy + y) * src_w + cx + x) * 3 + (2 - c));
                v[i] = __fdiv_rn(__fsub_rn(__fdiv_rn(float(u), 255.0f), kDvMean[c]), kDvStd[c]);
            } else {
                v[i] = __ldg(static_cast<const float*>(src) + ((int64_t(b) * 3 + c) * DV_CROP + y) * DV_CROP + x);
            }
        }
    }
    *reinterpret_cast<uint4*>(out + row * DV_PK + grp * 8) =
        make_uint4(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7]));
}

// One thread: 4 consecutive columns of one token row
__global__ void tokens_kernel(const float* __restrict__ emb, const float* __restrict__ pos,
                              const float* __restrict__ cls_pos0, const float* __restrict__ reg, int n_reg,
                              float* __restrict__ x, int64_t rows, int D) {
    const int q = D / 4;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= rows * q) return;
    const int col = int(idx % q) * 4;
    const int64_t row = idx / q;
    const int S = 1 + n_reg + DV_PATCHES;
    const int64_t frame = row / S;
    const int t = int(row - frame * S);
    float4 v;
    if (t == 0) {
        v = __ldg(reinterpret_cast<const float4*>(cls_pos0 + col));
    } else if (t <= n_reg) {
        v = __ldg(reinterpret_cast<const float4*>(reg + int64_t(t - 1) * D + col));
    } else {
        const int i = t - 1 - n_reg;
        const float4 a = __ldg(reinterpret_cast<const float4*>(emb + (frame * DV_PATCHES + i) * D + col));
        const float4 p = __ldg(reinterpret_cast<const float4*>(pos + int64_t(1 + i) * D + col));
        v = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
    }
    *reinterpret_cast<float4*>(x + row * D + col) = v;
}

__device__ __forceinline__ float silu_mul(float a, float b) { return __fdiv_rn(a, 1.0f + expf(-a)) * b; }

// One thread: 4 consecutive hidden columns of one row
__global__ void swiglu_kernel(const float* __restrict__ ab, int64_t rows, int hidden, __half* __restrict__ out) {
    const int q = hidden / 4;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= rows * q) return;
    const int col = int(idx % q) * 4;
    const int64_t row = idx / q;
    const float4 a = __ldg(reinterpret_cast<const float4*>(ab + row * 2 * hidden + col));
    const float4 b = __ldg(reinterpret_cast<const float4*>(ab + row * 2 * hidden + hidden + col));
    *reinterpret_cast<uint2*>(out + row * hidden + col) =
        make_uint2(pack_half2(silu_mul(a.x, b.x), silu_mul(a.y, b.y)), pack_half2(silu_mul(a.z, b.z), silu_mul(a.w, b.w)));
}

}  // namespace

int dinov2_patchify_u8(const uint8_t* src, int n, int src_h, int src_w, int cy, int cx, __half* patches, cudaStream_t s) {
    const int64_t total = int64_t(n) * DV_PATCHES * (DV_PK / 8);
    patchify_kernel<true><<<nblocks(total, 256), 256, 0, s>>>(src, n, src_h, src_w, cy, cx, patches);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int dinov2_patchify_f32(const float* src, int n, __half* patches, cudaStream_t s) {
    const int64_t total = int64_t(n) * DV_PATCHES * (DV_PK / 8);
    patchify_kernel<false><<<nblocks(total, 256), 256, 0, s>>>(src, n, DV_CROP, DV_CROP, 0, 0, patches);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int dinov2_tokens(const float* emb, const float* pos, const float* cls_pos0, const float* reg, int n_reg, float* x, int n,
                  int D, cudaStream_t s) {
    if (D % 4 || n_reg < 0) return fail(VF_ERR_INVALID, "dinov2_tokens: width %d, %d registers", D, n_reg);
    const int64_t rows = int64_t(n) * (1 + n_reg + DV_PATCHES);
    tokens_kernel<<<nblocks(rows * (D / 4), 256), 256, 0, s>>>(emb, pos, cls_pos0, reg, n_reg, x, rows, D);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int dinov2_swiglu(const float* ab, int rows, int hidden, __half* out, cudaStream_t s) {
    if (rows < 0 || hidden <= 0 || hidden % 4)
        return fail(VF_ERR_INVALID, "dinov2_swiglu: %d rows of %d hidden columns (a multiple of 4)", rows, hidden);
    if (rows == 0) return VF_OK;
    swiglu_kernel<<<nblocks(int64_t(rows) * (hidden / 4), 256), 256, 0, s>>>(ab, rows, hidden, out);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // namespace vf
