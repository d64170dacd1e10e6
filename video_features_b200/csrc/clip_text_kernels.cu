// Kernels of the CLIP text tower (clip_text_kernels.h).
#include <math.h>

#include "clip_text_kernels.h"
#include "common.cuh"

namespace vf {

namespace {

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

__global__ void embed_kernel(const int32_t* __restrict__ tokens, int ctx, int n, int L, const float* __restrict__ tok_emb,
                             const float* __restrict__ pos, int W, float* __restrict__ x) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * L * W) return;
    const int c = int(idx % W);
    const int64_t row = idx / W;
    const int t = int(row % L), b = int(row / L);
    x[idx] = tok_emb[int64_t(tokens[int64_t(b) * ctx + t]) * W + c] + pos[int64_t(t) * W + c];
}

constexpr int AT_WARPS = 4;
constexpr int AT_KPITCH = CT_HEAD_DIM + 1;      // K rows padded: lanes reading 32 different keys hit 32 banks

// One CTA per (head, prompt): the prompt's K / V of this head in shared memory as fp32; warp w computes rows w, w + 4,
// ...  Lane l owns keys l, l + 32, l + 64 for the scores and output channels l, l + 32 for P.V.  Every loop over keys
// stops at the row's own index, and the warp reductions are fixed butterflies, so row i's bits depend on rows 0..i only.
__global__ void __launch_bounds__(AT_WARPS * 32) attention_kernel(const __half* __restrict__ qkv, int L, int heads,
                                                                  __half* __restrict__ att) {
    __shared__ float ks[CT_MAX_CTX * AT_KPITCH];
    __shared__ float vs[CT_MAX_CTX * CT_HEAD_DIM];
    __shared__ float qs[AT_WARPS][CT_HEAD_DIM];
    __shared__ float ps[AT_WARPS][96];
    const int h = blockIdx.x, b = blockIdx.y, W = heads * CT_HEAD_DIM;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const __half* base = qkv + int64_t(b) * L * 3 * W + h * CT_HEAD_DIM;
    for (int idx = threadIdx.x; idx < L * CT_HEAD_DIM; idx += blockDim.x) {
        const int t = idx / CT_HEAD_DIM, d = idx % CT_HEAD_DIM;
        const __half* r = base + int64_t(t) * 3 * W;
        ks[t * AT_KPITCH + d] = __half2float(r[W + d]);
        vs[t * CT_HEAD_DIM + d] = __half2float(r[2 * W + d]);
    }
    __syncthreads();
    for (int i = warp; i < L; i += AT_WARPS) {
        const __half* qr = base + int64_t(i) * 3 * W;
        qs[warp][lane] = __half2float(qr[lane]);
        qs[warp][lane + 32] = __half2float(qr[lane + 32]);
        __syncwarp();
        float sc[3], mx = -INFINITY;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            const int j = lane + 32 * t;
            sc[t] = -INFINITY;
            if (j <= i) {
                float acc = 0.f;
#pragma unroll 16
                for (int d = 0; d < CT_HEAD_DIM; ++d) acc = fmaf(qs[warp][d], ks[j * AT_KPITCH + d], acc);
                sc[t] = acc * 0.125f;                    // 1 / sqrt(64), exact
                mx = fmaxf(mx, sc[t]);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            const int j = lane + 32 * t;
            if (j <= i) {
                const float e = expf(sc[t] - mx);
                ps[warp][j] = e;
                sum += e;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        __syncwarp();
        float a0 = 0.f, a1 = 0.f;
        for (int j = 0; j <= i; ++j) {
            const float p = ps[warp][j];
            a0 = fmaf(p, vs[j * CT_HEAD_DIM + lane], a0);
            a1 = fmaf(p, vs[j * CT_HEAD_DIM + lane + 32], a1);
        }
        __half* o = att + (int64_t(b) * L + i) * W + h * CT_HEAD_DIM;
        o[lane] = __float2half_rn(a0 / sum);
        o[lane + 32] = __float2half_rn(a1 / sum);
        __syncwarp();                                    // qs / ps are rewritten by the warp's next row
    }
}

__global__ void gather_kernel(const float* __restrict__ x, const int32_t* __restrict__ eot, int n, int L, int W,
                              float* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * W) return;
    const int b = int(idx / W), c = int(idx % W);
    out[idx] = x[(int64_t(b) * L + eot[b]) * W + c];
}

constexpr int NORM_THREADS = 256;

// one CTA per row: per-thread strided sums, then a fixed shared-memory tree
__global__ void __launch_bounds__(NORM_THREADS) l2_normalize_kernel(const float* __restrict__ x, int C,
                                                                    float* __restrict__ out) {
    __shared__ float red[NORM_THREADS];
    const float* r = x + int64_t(blockIdx.x) * C;
    float ss = 0.f;
    for (int c = threadIdx.x; c < C; c += NORM_THREADS) ss = fmaf(r[c], r[c], ss);
    red[threadIdx.x] = ss;
    __syncthreads();
    for (int o = NORM_THREADS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    const float norm = sqrtf(red[0]);
    float* w = out + int64_t(blockIdx.x) * C;
    for (int c = threadIdx.x; c < C; c += NORM_THREADS) w[c] = r[c] / norm;
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int clip_text_embed(const int32_t* tokens, int ctx, int n, int L, const float* tok_emb, const float* pos, int W, float* x,
                    cudaStream_t s) {
    if (n <= 0) return VF_OK;
    embed_kernel<<<nb(int64_t(n) * L * W, 256), 256, 0, s>>>(tokens, ctx, n, L, tok_emb, pos, W, x);
    LAUNCH_CHECK();
}

int clip_text_attention(const __half* qkv, int n, int L, int heads, __half* att, cudaStream_t s) {
    if (n < 0 || L < 1 || L > CT_MAX_CTX || heads < 1 || heads > 64)
        return fail(VF_ERR_INVALID, "clip_text_attention: %d prompts of %d rows, %d heads (rows must be 1..%d)", n, L,
                    heads, CT_MAX_CTX);
    if (n == 0) return VF_OK;
    attention_kernel<<<dim3(heads, n), AT_WARPS * 32, 0, s>>>(qkv, L, heads, att);
    LAUNCH_CHECK();
}

int clip_text_gather(const float* x, const int32_t* eot, int n, int L, int W, float* out, cudaStream_t s) {
    if (n <= 0) return VF_OK;
    gather_kernel<<<nb(int64_t(n) * W, 256), 256, 0, s>>>(x, eot, n, L, W, out);
    LAUNCH_CHECK();
}

int l2_normalize_rows(const float* x, int n, int C, float* out, cudaStream_t s) {
    if (n < 0 || C < 1) return fail(VF_ERR_INVALID, "l2_normalize_rows: %d rows of %d", n, C);
    if (n == 0) return VF_OK;
    l2_normalize_kernel<<<n, NORM_THREADS, 0, s>>>(x, C, out);
    LAUNCH_CHECK();
}

}  // namespace vf
