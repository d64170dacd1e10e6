// Memory-bound kernels of the ResNet path: the fused frame transform (crop + ToTensor + Normalize + stem phase pack),
// the 3x3/2 max-pool and the global average pool.  Activations are split-fp16 rows [hi C | lo C] of zero-bordered
// channels-last 2-D volumes (raft_kernels.h Vol2); see resnet.cu for the geometry.
#include "common.cuh"
#include "internal.h"
#include "raft_kernels.h"

namespace vf {

namespace {

// torchvision Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]), float32-rounded like torch does
__constant__ float kImgMean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float kImgStd[3] = {0.229f, 0.224f, 0.225f};

__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// 224x224 normalised frames -> phase volume of the 7x7 stride-2 pad-3 stem: row (b, hq, wq) of a [n][115][115] volume
// holds x[2(hq-2)+ph][2(wq-2)+pw][c] at column (ph*2+pw)*4 + c of [16 hi | 16 lo] (c < 3; zero outside the image).
// u8 source: n x Hr x Wr x 3 BGR frames (already resized); the 224 crop at (cy, cx), RGB channel c = source channel 2-c,
// ToTensor (v / 255) then Normalize ((x - mean) / std) as IEEE fp32 ops in torchvision's order.
// f32 source: n x 3 x 224 x 224, already normalised (the tensor the reference hands to the model).
template <bool U8>
__global__ void resnet_input_pack_kernel(const void* __restrict__ src, int n, int Hr, int Wr, int cy, int cx,
                                         __half* __restrict__ out) {
    constexpr int Q = 115;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * Q * Q) return;
    const int wq = int(idx % Q), hq = int((idx / Q) % Q), b = int(idx / (Q * Q));
    __align__(16) __half vals[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) vals[i] = __float2half_rn(0.f);
#pragma unroll
    for (int ph = 0; ph < 2; ++ph)
#pragma unroll
        for (int pw = 0; pw < 2; ++pw) {
            const int y = 2 * (hq - 2) + ph, x = 2 * (wq - 2) + pw;
            if (y < 0 || y >= 224 || x < 0 || x >= 224) continue;       // the stem's zero padding
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float v;
                if (U8) {
                    const uint8_t* p = static_cast<const uint8_t*>(src);
                    const uint8_t u = __ldg(p + ((int64_t(b) * Hr + cy + y) * Wr + cx + x) * 3 + (2 - c));
                    v = __fdiv_rn(__fsub_rn(__fdiv_rn(float(u), 255.0f), kImgMean[c]), kImgStd[c]);
                } else {
                    v = __ldg(static_cast<const float*>(src) + ((int64_t(b) * 3 + c) * 224 + y) * 224 + x);
                }
                split_half(v, vals[(ph * 2 + pw) * 4 + c], vals[16 + (ph * 2 + pw) * 4 + c]);
            }
        }
    uint4* o = reinterpret_cast<uint4*>(out + idx * 32);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = reinterpret_cast<const uint4*>(vals)[i];
}

// MaxPool2d(3, stride 2, padding 1) on split rows: out valid (i, j) = max over in valid rows 2i-1..2i+1, columns
// 2j-1..2j+1 (those inside the image).  The winner's (hi, lo) pair is copied, so the pool is exact.  The input is
// post-ReLU and every window holds a valid element, so skipping the padding equals -inf padding.  8 channels / thread;
// border positions of the output volume are written as zeros.
__global__ void maxpool_kernel(const __half* __restrict__ in, Vol2 vi, int C, __half* __restrict__ out, Vol2 vo) {
    const int cg = C >> 3;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(vo.n) * vo.Hp * vo.Wp * cg) return;
    const int c8 = int(idx % cg);
    const int64_t pos = idx / cg;
    const int wq = int(pos % vo.Wp), hq = int((pos / vo.Wp) % vo.Hp), b = int(pos / (int64_t(vo.Wp) * vo.Hp));
    __half* o = out + pos * (2 * C) + c8 * 8;
    if (hq < vo.h0 || hq >= vo.h1 || wq < vo.w0 || wq >= vo.w1) {
        *reinterpret_cast<uint4*>(o) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(o + C) = make_uint4(0, 0, 0, 0);
        return;
    }
    const int i = hq - vo.h0, j = wq - vo.w0, Hi = vi.h1 - vi.h0, Wi = vi.w1 - vi.w0;
    float best[8];
    __align__(16) __half bh[8], bl[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) best[k] = -INFINITY;
    for (int dy = -1; dy <= 1; ++dy) {
        const int y = 2 * i + dy;
        if (y < 0 || y >= Hi) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int x = 2 * j + dx;
            if (x < 0 || x >= Wi) continue;
            const __half* p = in + ((int64_t(b) * vi.Hp + y + vi.h0) * vi.Wp + x + vi.w0) * (2 * C) + c8 * 8;
            const uint4 h4 = __ldg(reinterpret_cast<const uint4*>(p)), l4 = __ldg(reinterpret_cast<const uint4*>(p + C));
            const __half *ph = reinterpret_cast<const __half*>(&h4), *pl = reinterpret_cast<const __half*>(&l4);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float v = __half2float(ph[k]) + __half2float(pl[k]);
                if (v > best[k]) { best[k] = v; bh[k] = ph[k]; bl[k] = pl[k]; }
            }
        }
    }
    *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(bh);
    *reinterpret_cast<uint4*>(o + C) = *reinterpret_cast<const uint4*>(bl);
}

// AdaptiveAvgPool2d(1) + flatten: out[b][c] = mean over the valid region of (hi + lo), summed in a fixed order (one
// thread per (b, c)), fp32.
__global__ void avgpool_kernel(const __half* __restrict__ in, Vol2 v, int C, float* __restrict__ out, int n) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * C) return;
    const int c = int(idx % C), b = int(idx / C);
    float s = 0.f;
    for (int y = v.h0; y < v.h1; ++y)
        for (int x = v.w0; x < v.w1; ++x) {
            const __half* p = in + ((int64_t(b) * v.Hp + y) * v.Wp + x) * (2 * C) + c;
            s += __half2float(p[0]) + __half2float(p[C]);
        }
    out[idx] = s / float((v.h1 - v.h0) * (v.w1 - v.w0));
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int resnet_input_pack(const void* src, int is_u8, int n, int Hr, int Wr, int cy, int cx, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(n) * 115 * 115;
    if (is_u8) resnet_input_pack_kernel<true><<<nb(total, 256), 256, 0, s>>>(src, n, Hr, Wr, cy, cx, out);
    else       resnet_input_pack_kernel<false><<<nb(total, 256), 256, 0, s>>>(src, n, Hr, Wr, cy, cx, out);
    LAUNCH_CHECK();
}
int resnet_maxpool(const __half* in, const Vol2& vi, int C, __half* out, const Vol2& vo, cudaStream_t s) {
    const int64_t total = vo.rows() * (C / 8);
    maxpool_kernel<<<nb(total, 256), 256, 0, s>>>(in, vi, C, out, vo);
    LAUNCH_CHECK();
}
int resnet_avgpool(const __half* in, const Vol2& v, int C, float* out, cudaStream_t s) {
    const int64_t total = int64_t(v.n) * C;
    avgpool_kernel<<<nb(total, 256), 256, 0, s>>>(in, v, C, out, v.n);
    LAUNCH_CHECK();
}

}  // namespace vf
