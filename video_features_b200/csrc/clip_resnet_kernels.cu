// Memory- and latency-bound kernels of the CLIP ResNet towers (clip_resnet.cu): the fused frame transform into the stem's
// phase volume, the attention-pool tokens and the attention-pool attention.  Activations are split-fp16 rows
// [hi C | lo C] (raft_kernels.h Vol2).
#include "clip_resnet_kernels.h"
#include "common.cuh"
#include "internal.h"

namespace vf {

namespace {

// clip.clip._transform's Normalize, float32-rounded like torch does
__constant__ float kRnMean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float kRnStd[3] = {0.26862954f, 0.26130258f, 0.27577711f};

__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// npx x npx normalised frames -> phase volume of the 3x3 stride-2 pad-1 stem conv: row (b, hq, wq) of a [n][S+2][S+2]
// volume (S = npx / 2) holds x[2(hq-1)+ph][2(wq-1)+pw][c] at column (ph*2+pw)*4 + c of [16 hi | 16 lo] (c < 3; zero
// outside the image).  u8 source: n x Hr x Wr x 3 frames, already resized; the npx crop at (cy, cx), channel c = source
// channel c (the decoder's order goes in unswapped, as in the reference), ToTensor (v / 255) then Normalize
// ((x - mean) / std) as IEEE fp32 ops in torchvision's order.  f32 source: n x 3 x npx x npx, already normalised.
template <bool U8>
__global__ void input_pack_kernel(const void* __restrict__ src, int n, int Hr, int Wr, int cy, int cx, int npx,
                                  __half* __restrict__ out) {
    const int Q = npx / 2 + 2;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * Q * Q) return;
    const int wq = int(idx % Q), hq = int((idx / Q) % Q), b = int(idx / (int64_t(Q) * Q));
    __align__(16) __half vals[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) vals[i] = __float2half_rn(0.f);
#pragma unroll
    for (int ph = 0; ph < 2; ++ph)
#pragma unroll
        for (int pw = 0; pw < 2; ++pw) {
            const int y = 2 * (hq - 1) + ph, x = 2 * (wq - 1) + pw;
            if (y < 0 || y >= npx || x < 0 || x >= npx) continue;       // the stem's zero padding
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float v;
                if (U8) {
                    const uint8_t* p = static_cast<const uint8_t*>(src);
                    const uint8_t u = __ldg(p + ((int64_t(b) * Hr + cy + y) * Wr + cx + x) * 3 + c);
                    v = __fdiv_rn(__fsub_rn(__fdiv_rn(float(u), 255.0f), kRnMean[c]), kRnStd[c]);
                } else {
                    v = __ldg(static_cast<const float*>(src) + ((int64_t(b) * 3 + c) * npx + y) * npx + x);
                }
                split_half(v, vals[(ph * 2 + pw) * 4 + c], vals[16 + (ph * 2 + pw) * 4 + c]);
            }
        }
    uint4* o = reinterpret_cast<uint4*>(out + idx * 32);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = reinterpret_cast<const uint4*>(vals)[i];
}

// AttentionPool2d's tokens, one thread per (frame, channel): token 0 = mean over the valid region of (hi + lo), summed
// in row-major order in fp32, token t = position t - 1 (row-major over (h, w)); each plus positional_embedding[t], in
// fp32, written as a split pair into row b * T + t of [hi E | lo E].
__global__ void tokens_kernel(const __half* __restrict__ in, Vol2 v, int E, const float* __restrict__ pos,
                              __half* __restrict__ tokens) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(v.n) * E) return;
    const int c = int(idx % E), b = int(idx / E);
    const int W = v.w1 - v.w0, T = (v.h1 - v.h0) * W + 1;
    __half* o = tokens + int64_t(b) * T * 2 * E + c;
    float s = 0.f;
    for (int y = v.h0; y < v.h1; ++y)
        for (int x = v.w0; x < v.w1; ++x) {
            const __half* p = in + ((int64_t(b) * v.Hp + y) * v.Wp + x) * (2 * E) + c;
            const float xv = __half2float(p[0]) + __half2float(p[E]);
            s += xv;
            const int t = (y - v.h0) * W + (x - v.w0) + 1;
            split_half(xv + pos[int64_t(t) * E + c], o[int64_t(t) * 2 * E], o[int64_t(t) * 2 * E + E]);
        }
    split_half(s / float(T - 1) + pos[c], o[0], o[E]);
}

// One query (token 0) per (frame, head) over T keys, head dim 64: scores (q / 8) . k, softmax, sum p v, all fp32.
// kv: rows b * T + t of [k E | v E] fp32, q: rows b of [E] fp32 (both with their biases); out: split rows [hi E | lo E].
// 128 threads: scores t = tid, tid + 128, ...; the weighted sum splits the keys over two halves of 64 threads.
__global__ void __launch_bounds__(128) attention_kernel(const float* __restrict__ kv, const float* __restrict__ q,
                                                        int T, int E, __half* __restrict__ out) {
    extern __shared__ float p[];          // T scores / weights
    __shared__ float qs[64], red[4], part[64];
    const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 64) qs[tid] = q[int64_t(b) * E + h * 64 + tid] * 0.125f;
    __syncthreads();
    const float* kb = kv + int64_t(b) * T * 2 * E + h * 64;
    float m = -INFINITY;
    for (int t = tid; t < T; t += 128) {
        const float4* k4 = reinterpret_cast<const float4*>(kb + int64_t(t) * 2 * E);
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < 16; ++d) {
            const float4 k = __ldg(k4 + d);
            s = fmaf(qs[4 * d], k.x, s); s = fmaf(qs[4 * d + 1], k.y, s);
            s = fmaf(qs[4 * d + 2], k.z, s); s = fmaf(qs[4 * d + 3], k.w, s);
        }
        p[t] = s;
        m = fmaxf(m, s);
    }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) red[warp] = m;
    __syncthreads();
    m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    __syncthreads();
    float l = 0.f;
    for (int t = tid; t < T; t += 128) {
        const float e = expf(p[t] - m);
        p[t] = e;
        l += e;
    }
    for (int o = 16; o; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    if (lane == 0) red[warp] = l;
    __syncthreads();
    l = (red[0] + red[1]) + (red[2] + red[3]);
    const int d = tid & 63, half = tid >> 6;
    const float* vb = kb + E + d;
    float acc = 0.f;
    for (int t = half; t < T; t += 2) acc = fmaf(p[t], __ldg(vb + int64_t(t) * 2 * E), acc);
    if (half) part[d] = acc;
    __syncthreads();
    if (!half) {
        __half* o = out + int64_t(b) * 2 * E + h * 64 + d;
        split_half((acc + part[d]) / l, o[0], o[E]);
    }
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int clip_rn_input_pack(const void* src, int is_u8, int n, int Hr, int Wr, int cy, int cx, int npx, __half* out,
                       cudaStream_t s) {
    const int Q = npx / 2 + 2;
    const int64_t total = int64_t(n) * Q * Q;
    if (is_u8) input_pack_kernel<true><<<nb(total, 256), 256, 0, s>>>(src, n, Hr, Wr, cy, cx, npx, out);
    else       input_pack_kernel<false><<<nb(total, 256), 256, 0, s>>>(src, n, Hr, Wr, cy, cx, npx, out);
    LAUNCH_CHECK();
}
int clip_rn_tokens(const __half* in, const Vol2& v, int E, const float* pos, __half* tokens, cudaStream_t s) {
    const int64_t total = int64_t(v.n) * E;
    tokens_kernel<<<nb(total, 256), 256, 0, s>>>(in, v, E, pos, tokens);
    LAUNCH_CHECK();
}
int clip_rn_attention(const float* kv, const float* q, int n, int T, int E, __half* out, cudaStream_t s) {
    // the T scores sit in dynamic shared memory beside the kernel's static arrays, within the 48 KB a launch gets
    // without opting in
    static size_t static_bytes = 0;
    if (!static_bytes) {
        cudaFuncAttributes fa;
        VF_CUDA(cudaFuncGetAttributes(&fa, attention_kernel));
        static_bytes = fa.sharedSizeBytes;
    }
    if (T < 1 || static_bytes + size_t(T) * sizeof(float) > 48 * 1024)
        return fail(VF_ERR_INVALID, "clip_rn_attention: %d tokens; the scores fit %zu", T,
                    (48 * 1024 - static_bytes) / sizeof(float));
    attention_kernel<<<dim3(E / 64, n), 128, size_t(T) * sizeof(float), s>>>(kv, q, T, E, out);
    LAUNCH_CHECK();
}

}  // namespace vf
