// Classifier head for --show_pred: logits = features . W^T + b, softmax and top-k, all in fp32 on the CUDA cores.
// Replaces the reference's `model.fc(feats)` (ResNet, R(2+1)D) and I3D's conv3d_0c_1x1 + mean over time
// (models/i3d/i3d_src/i3d_net.py:266-274), followed by utils/utils.py:19-47's softmax + sort.
//
// Two launches per call:
//   head_logits_kernel: a 16-row x 64-class tile per block; 32-wide K slices of the features and of W are staged
//     through shared memory; each logit is ONE sequential fp32 FMA chain over k = 0 .. K-1 starting from 0, then + b.
//     The head is < 0.3 GFLOP per call, so there is nothing to gain from the split-fp16 wgmma GEMM, and fp32 FMA keeps
//     the logits at the reference's arithmetic.
//   head_softmax_topk_kernel: one block per row: max, sum of expf(l - max), p = expf(l - max) / sum (torch's
//     max-subtracted softmax), then k rounds of a block argmax over p.  Order: p descending; equal p by the lower
//     class index; NaN (a row with a NaN or infinite logit has an all-NaN softmax, as in torch) above every number.
#include <float.h>
#include <math.h>

#include "internal.h"

struct vf_head : vf::EngineCore {
    int C = 0, K = 0;
    float* w = nullptr;       // [C][K]
    float* b = nullptr;       // [C]
};

namespace vf {

constexpr int HB_M = 16, HB_N = 64, HB_K = 32, HB_THREADS = 256, HEAD_MAX_K = 8;
constexpr int HEAD_MAX_ROWS = 65535 * HB_M;

__global__ void __launch_bounds__(HB_THREADS) head_logits_kernel(const float* __restrict__ X, int n, int K,
                                                                 const float* __restrict__ W,
                                                                 const float* __restrict__ bias, int C,
                                                                 float* __restrict__ L) {
    __shared__ float ws[HB_N][HB_K + 1];
    __shared__ float xs[HB_M][HB_K];
    const int t = threadIdx.x, tx = t % HB_N, ty = t / HB_N;      // class tx of the tile, rows ty, ty + 4, ...
    const int c0 = blockIdx.x * HB_N, r0 = blockIdx.y * HB_M;
    float acc[HB_M / 4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 < K; k0 += HB_K) {
#pragma unroll
        for (int q = 0; q < HB_N * HB_K / HB_THREADS; ++q) {
            const int i = (t + q * HB_THREADS) / HB_K, j = (t + q * HB_THREADS) % HB_K;
            const int c = c0 + i, k = k0 + j;
            ws[i][j] = (c < C && k < K) ? W[size_t(c) * K + k] : 0.f;
        }
#pragma unroll
        for (int q = 0; q < HB_M * HB_K / HB_THREADS; ++q) {
            const int i = (t + q * HB_THREADS) / HB_K, j = (t + q * HB_THREADS) % HB_K;
            const int r = r0 + i, k = k0 + j;
            xs[i][j] = (r < n && k < K) ? X[size_t(r) * K + k] : 0.f;
        }
        __syncthreads();
        const int kn = min(HB_K, K - k0);          // zero-filled columns past K are not added: the chain stays exact
#pragma unroll 8
        for (int kk = 0; kk < kn; ++kk) {
            const float w = ws[tx][kk];
#pragma unroll
            for (int a = 0; a < HB_M / 4; ++a) acc[a] = fmaf(xs[ty + 4 * a][kk], w, acc[a]);
        }
        __syncthreads();
    }
    const int c = c0 + tx;
    if (c >= C) return;
    const float bc = bias[c];
#pragma unroll
    for (int a = 0; a < HB_M / 4; ++a) {
        const int r = r0 + ty + 4 * a;
        if (r < n) L[size_t(r) * C + c] = acc[a] + bc;
    }
}

// The top-k's total order, torch.sort(descending=True, stable=True)'s: NaN above every number, larger values first,
// equal values (and NaNs among themselves) by the lower index.  bi < 0 is "no candidate yet", below everything.
__device__ __forceinline__ bool head_better(float v, int i, float bv, int bi) {
    if (i < 0) return false;
    if (bi < 0) return true;
    const bool vn = isnan(v), bn = isnan(bv);
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

__global__ void __launch_bounds__(HB_THREADS) head_softmax_topk_kernel(const float* __restrict__ L, int C,
                                                                       float* __restrict__ P, int k,
                                                                       int* __restrict__ top_idx,
                                                                       float* __restrict__ top_logit,
                                                                       float* __restrict__ top_prob) {
    __shared__ float red_v[HB_THREADS / 32];
    __shared__ int red_i[HB_THREADS / 32];
    __shared__ int chosen[HEAD_MAX_K];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nw = HB_THREADS / 32;
    const size_t row = blockIdx.x;
    const float* l = L + row * C;
    float* p = P + row * C;

    float m = -INFINITY;
    for (int c = t; c < C; c += HB_THREADS) m = fmaxf(m, l[c]);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) red_v[warp] = m;
    __syncthreads();
    m = red_v[0];
    for (int w = 1; w < nw; ++w) m = fmaxf(m, red_v[w]);
    __syncthreads();

    float s = 0.f;
    for (int c = t; c < C; c += HB_THREADS) s += expf(l[c] - m);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red_v[warp] = s;
    __syncthreads();
    s = 0.f;
    for (int w = 0; w < nw; ++w) s += red_v[w];
    __syncthreads();
    for (int c = t; c < C; c += HB_THREADS) p[c] = expf(l[c] - m) / s;
    __syncthreads();                               // p[] written by other threads is read below (same block)

    for (int j = 0; j < k; ++j) {
        float bv = 0.f;
        int bi = -1;                               // k <= C: some class is always left, so the block's winner is valid
        for (int c = t; c < C; c += HB_THREADS) {
            bool taken = false;
            for (int q = 0; q < j; ++q) taken |= chosen[q] == c;
            const float v = p[c];
            if (!taken && head_better(v, c, bv, bi)) { bv = v; bi = c; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (head_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
        __syncthreads();
        if (t == 0) {
            for (int w = 1; w < nw; ++w)
                if (head_better(red_v[w], red_i[w], bv, bi)) { bv = red_v[w]; bi = red_i[w]; }
            chosen[j] = bi;
            top_idx[row * k + j] = bi;
            top_logit[row * k + j] = l[bi];
            top_prob[row * k + j] = bv;
        }
        __syncthreads();
    }
}

}  // namespace vf

using namespace vf;

extern "C" {

int vf_head_destroy(vf_head_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_head_create(vf_head_t** out, const float* weight, const float* bias, int n_classes, int n_features, int device) {
    if (!out || !weight || !bias) return fail(VF_ERR_INVALID, "head_create: null argument");
    *out = nullptr;
    if (n_classes < 1 || n_features < 1)
        return fail(VF_ERR_INVALID, "head_create: %d classes x %d features", n_classes, n_features);
    VF_TRY(check_device(device));
    vf_head* h = new vf_head();
    h->who = "head_create";
    h->device = device; h->C = n_classes; h->K = n_features;
    const size_t wn = size_t(n_classes) * n_features;
    auto body = [&]() -> int {
        VF_TRY(ralloc(h, &h->w, wn));
        VF_TRY(ralloc(h, &h->b, size_t(n_classes)));
        VF_CUDA(cudaMemcpy(h->w, weight, wn * sizeof(float), cudaMemcpyHostToDevice));
        VF_CUDA(cudaMemcpy(h->b, bias, size_t(n_classes) * sizeof(float), cudaMemcpyHostToDevice));
        return VF_OK;
    };
    const int st = body();
    if (st != VF_OK) { vf_head_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_head_info(const vf_head_t* h, int* n_classes, int* n_features) {
    if (!h || !n_classes || !n_features) return fail(VF_ERR_INVALID, "head_info: null argument");
    *n_classes = h->C;
    *n_features = h->K;
    return VF_OK;
}

int vf_head_forward(vf_head_t* h, const float* feats, int n, int n_features, float* logits, float* probs, int k,
                    int32_t* top_idx, float* top_logit, float* top_prob, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "head_forward: null handle");
    if (n < 0 || n > HEAD_MAX_ROWS) return fail(VF_ERR_INVALID, "head_forward: %d rows (1 .. %d)", n, HEAD_MAX_ROWS);
    if (n_features != h->K)
        return fail(VF_ERR_INVALID, "head_forward: rows of %d features, the head takes %d", n_features, h->K);
    if (k < 1 || k > HEAD_MAX_K || k > h->C)
        return fail(VF_ERR_INVALID, "head_forward: k = %d (1 .. %d, at most the %d classes)", k, HEAD_MAX_K, h->C);
    if (n == 0) return VF_OK;
    if (!feats || !logits || !probs || !top_idx || !top_logit || !top_prob)
        return fail(VF_ERR_INVALID, "head_forward: null argument");
    VF_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid((h->C + HB_N - 1) / HB_N, (n + HB_M - 1) / HB_M);
    head_logits_kernel<<<grid, HB_THREADS, 0, s>>>(feats, n, h->K, h->w, h->b, h->C, logits);
    VF_CUDA(cudaGetLastError());
    head_softmax_topk_kernel<<<n, HB_THREADS, 0, s>>>(logits, h->C, probs, k, top_idx, top_logit, top_prob);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // extern "C"
