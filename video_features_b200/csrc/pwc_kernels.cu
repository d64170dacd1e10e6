// Memory-bound kernels of the PWC-Net path (pwc.cu has the geometry).  The convolutions run on the conv-GEMM; what is
// left is the input pack, the backward warp, the 81-channel cost volume, the transposed-conv scatter and the output
// upsample.  Arithmetic is fp32 throughout; values read from split-fp16 pairs are hi + lo.
#include "common.cuh"
#include "internal.h"
#include "pwc_kernels.h"

namespace vf {

namespace {

__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// torch's bilinear source index for align_corners=False (area_pixel_compute_source_index): clamped below at 0
__device__ __forceinline__ void src_index(int dst, int in, int out, int& i0, int& i1, float& l0, float& l1) {
    const float scale = float(in) / float(out);
    float src = __fsub_rn(__fmul_rn(scale, float(dst) + 0.5f), 0.5f);
    if (src < 0.f) src = 0.f;
    i0 = int(src);
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    l1 = __fsub_rn(src, float(i0));
    l0 = __fsub_rn(1.f, l1);
}

// pwc_net.py:230-245: BGR <-> RGB swap, /255, F.interpolate(bilinear, align_corners=False) to the /64 size
template <typename TIn>
__global__ void input_pack_kernel(const TIn* __restrict__ img, int n, int Hs, int Ws, int chw, __half* __restrict__ out,
                                  Vol2 vo) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(vo.n) * vo.Hp * vo.Wp) return;
    const int q = int(idx % vo.Wp), p = int((idx / vo.Wp) % vo.Hp), b = int(idx / (int64_t(vo.Wp) * vo.Hp));
    __align__(16) __half vals[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) vals[i] = __float2half_rn(0.f);
    if (p >= vo.h0 && p < vo.h1 && q >= vo.w0 && q < vo.w1) {
        int y0, y1, x0, x1;
        float ly0, ly1, lx0, lx1;
        src_index(p - vo.h0, Hs, (vo.h1 - vo.h0), y0, y1, ly0, ly1);
        src_index(q - vo.w0, Ws, (vo.w1 - vo.w0), x0, x1, lx0, lx1);
        auto px = [&](int y, int x, int c) -> float {
            const float v = chw ? float(img[((int64_t(b) * 3 + c) * Hs + y) * Ws + x])
                                : float(img[((int64_t(b) * Hs + y) * Ws + x) * 3 + c]);
            return __fdiv_rn(v, 255.0f);
        };
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int cs = 2 - c;                                         // x[:, [2, 1, 0]]
            const float t0 = __fadd_rn(__fmul_rn(px(y0, x0, cs), lx0), __fmul_rn(px(y0, x1, cs), lx1));
            const float t1 = __fadd_rn(__fmul_rn(px(y1, x0, cs), lx0), __fmul_rn(px(y1, x1, cs), lx1));
            split_half(__fadd_rn(__fmul_rn(t0, ly0), __fmul_rn(t1, ly1)), vals[c], vals[8 + c]);
        }
    }
    uint4* o = reinterpret_cast<uint4*>(out + idx * 16);
    o[0] = reinterpret_cast<const uint4*>(vals)[0];
    o[1] = reinterpret_cast<const uint4*>(vals)[1];
}

// pwc_net.py:23-41 with grid_sample's align_corners=True (torch 1.2, which the reference pins): pixel (x + u, y + v)
__global__ void warp_kernel(const __half* __restrict__ feat, Vol2 vf, int ldf, int C, int C8, const __half* __restrict__ cat,
                            Vol2 vc, int ldc, int uf_col, float dbl, int n_pairs, float* __restrict__ out,
                            float* __restrict__ mask_out) {
    const int H = (vf.h1 - vf.h0), W = (vf.w1 - vf.w0);
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n_pairs) * H * W * C) return;
    const int c = int(idx % C);
    const int64_t pix = idx / C;
    const int x = int(pix % W), y = int((pix / W) % H), b = int(pix / (int64_t(W) * H));
    const __half* f2 = feat + int64_t(b + 1) * vf.Hp * vf.Wp * ldf;          // frame b + 1
    auto at = [&](int yy, int xx) -> float {
        const __half* s = f2 + ((int64_t(yy + vf.h0)) * vf.Wp + xx + vf.w0) * ldf + c;
        return __half2float(s[0]) + __half2float(s[C8]);
    };
    float val;
    if (uf_col < 0) {
        val = at(y, x);
    } else {
        const __half* r = cat + ((int64_t(b) * vc.Hp + y + vc.h0) * vc.Wp + x + vc.w0) * ldc + uf_col;
        const float u = __half2float(r[0]) + __half2float(r[8]), v = __half2float(r[1]) + __half2float(r[9]);
        const float ix = __fadd_rn(float(x), __fmul_rn(u, dbl)), iy = __fadd_rn(float(y), __fmul_rn(v, dbl));
        const float fx0 = floorf(ix), fy0 = floorf(iy);
        const int x0 = int(fx0), y0 = int(fy0);
        const float ax = __fsub_rn(ix, fx0), ay = __fsub_rn(iy, fy0);
        const float wts[4] = {__fmul_rn(1.f - ax, 1.f - ay), __fmul_rn(ax, 1.f - ay), __fmul_rn(1.f - ax, ay), __fmul_rn(ax, ay)};
        float acc = 0.f, msum = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int xx = x0 + (k & 1), yy = y0 + (k >> 1);
            if (xx < 0 || xx >= W || yy < 0 || yy >= H) continue;
            acc = __fadd_rn(acc, __fmul_rn(wts[k], at(yy, xx)));
            msum = __fadd_rn(msum, wts[k]);
        }
        const float m = msum > 0.999f ? 1.f : 0.f;
        val = acc * m;
        if (mask_out && c == 0) mask_out[pix] = m;
    }
    out[((int64_t(b) * (H + 8) + y + 4) * (W + 8) + x + 4) * C + c] = val;
}

// correlation.py:44-112: one block per pixel of a pair; threads 0..80 are the displacements
__global__ void correlation_kernel(const __half* __restrict__ feat, Vol2 vf, int ldf, int C, int C8,
                                   const float* __restrict__ f2w, __half* __restrict__ cat, Vol2 vc, int ldc, int vol_col,
                                   int f1_col) {
    extern __shared__ float f1s[];
    const int H = (vf.h1 - vf.h0), W = (vf.w1 - vf.w0);
    const int64_t pix = blockIdx.x;
    const int x = int(pix % W), y = int((pix / W) % H), b = int(pix / (int64_t(W) * H));
    const __half* f1 = feat + ((int64_t(b) * vf.Hp + y + vf.h0) * vf.Wp + x + vf.w0) * ldf;     // frame b
    __half* row = cat + ((int64_t(b) * vc.Hp + y + vc.h0) * vc.Wp + x + vc.w0) * ldc;
    for (int c = threadIdx.x; c < C; c += blockDim.x) f1s[c] = __half2float(f1[c]) + __half2float(f1[C8 + c]);
    if (f1_col >= 0)
        for (int j = threadIdx.x; j < 2 * C8; j += blockDim.x) row[f1_col + j] = f1[j];
    __syncthreads();
    const int d = threadIdx.x;
    if (d >= 81) return;
    const int dy = d / 9 - 4, dx = d % 9 - 4;
    const float* s2 = f2w + ((int64_t(b) * (H + 8) + y + 4 + dy) * (W + 8) + x + 4 + dx) * C;
    float sum = 0.f;
    for (int c = 0; c < C; ++c) sum = fmaf(f1s[c], s2[c], sum);
    float v = __fdiv_rn(sum, float(C));
    v = v > 0.f ? v : __fmul_rn(v, 0.1f);
    split_half(v, row[vol_col + d], row[vol_col + 88 + d]);
}

__global__ void up_scatter_kernel(const float* __restrict__ up, Vol2 vu, __half* __restrict__ cat, Vol2 vc, int ldc, int col) {
    const int H = (vc.h1 - vc.h0), W = (vc.w1 - vc.w0);
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(vc.n) * H * W) return;
    const int X = int(idx % W), Y = int((idx / W) % H), b = int(idx / (int64_t(W) * H));
    const int ph = ((Y & 1) << 1) | (X & 1);
    const float* s = up + ((int64_t(b) * vu.Hp + (Y >> 1) + vu.h0) * vu.Wp + (X >> 1) + vu.w0) * 8 + 2 * ph;
    __align__(16) __half vals[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) vals[i] = __float2half_rn(0.f);
    split_half(s[0], vals[0], vals[8]);
    split_half(s[1], vals[1], vals[9]);
    uint4* o = reinterpret_cast<uint4*>(cat + ((int64_t(b) * vc.Hp + Y + vc.h0) * vc.Wp + X + vc.w0) * ldc + col);
    o[0] = reinterpret_cast<const uint4*>(vals)[0];
    o[1] = reinterpret_cast<const uint4*>(vals)[1];
}

// pwc_net.py:256-261
__global__ void output_kernel(const __half* __restrict__ flow, const float* __restrict__ refine, Vol2 v, int n, int Ho,
                              int Wo, float sx, float sy, float* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * Ho * Wo) return;
    const int X = int(idx % Wo), Y = int((idx / Wo) % Ho), b = int(idx / (int64_t(Wo) * Ho));
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    src_index(Y, (v.h1 - v.h0), Ho, y0, y1, ly0, ly1);
    src_index(X, (v.w1 - v.w0), Wo, x0, x1, lx0, lx1);
    auto at = [&](int yy, int xx, int c) -> float {
        const int64_t r = (int64_t(b) * v.Hp + yy + v.h0) * v.Wp + xx + v.w0;
        const __half* f = flow + r * 16;
        return __fadd_rn(__half2float(f[c]) + __half2float(f[8 + c]), refine[r * 8 + c]);
    };
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const float t0 = __fadd_rn(__fmul_rn(at(y0, x0, c), lx0), __fmul_rn(at(y0, x1, c), lx1));
        const float t1 = __fadd_rn(__fmul_rn(at(y1, x0, c), lx0), __fmul_rn(at(y1, x1, c), lx1));
        const float val = __fmul_rn(20.f, __fadd_rn(__fmul_rn(t0, ly0), __fmul_rn(t1, ly1)));
        out[((int64_t(b) * 2 + c) * Ho + Y) * Wo + X] = __fmul_rn(val, c == 0 ? sx : sy);
    }
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int pwc_input_pack(const void* img, int is_u8, int chw, int n, int Hs, int Ws, __half* out, const Vol2& vo, cudaStream_t s) {
    const int64_t total = vo.rows();
    if (is_u8) input_pack_kernel<uint8_t><<<nb(total, 256), 256, 0, s>>>(static_cast<const uint8_t*>(img), n, Hs, Ws, chw, out, vo);
    else       input_pack_kernel<float><<<nb(total, 256), 256, 0, s>>>(static_cast<const float*>(img), n, Hs, Ws, chw, out, vo);
    LAUNCH_CHECK();
}
int pwc_warp(const __half* feat, const Vol2& vf, int ldf, int C, int C8, const __half* cat, const Vol2& vc, int ldc,
             int uf_col, float dbl, int n_pairs, float* out, float* mask_out, cudaStream_t s) {
    const int64_t total = int64_t(n_pairs) * vf.H() * vf.W() * C;
    warp_kernel<<<nb(total, 256), 256, 0, s>>>(feat, vf, ldf, C, C8, cat, vc, ldc, uf_col, dbl, n_pairs, out, mask_out);
    LAUNCH_CHECK();
}
int pwc_correlation(const __half* feat, const Vol2& vf, int ldf, int C, int C8, const float* f2w, __half* cat,
                    const Vol2& vc, int ldc, int vol_col, int f1_col, int n_pairs, cudaStream_t s) {
    const int64_t blocks = int64_t(n_pairs) * vf.H() * vf.W();
    correlation_kernel<<<unsigned(blocks), 96, C * sizeof(float), s>>>(feat, vf, ldf, C, C8, f2w, cat, vc, ldc, vol_col, f1_col);
    LAUNCH_CHECK();
}
int pwc_up_scatter(const float* up, const Vol2& vu, __half* cat, const Vol2& vc, int ldc, int col, cudaStream_t s) {
    const int64_t total = int64_t(vc.n) * vc.H() * vc.W();
    up_scatter_kernel<<<nb(total, 256), 256, 0, s>>>(up, vu, cat, vc, ldc, col);
    LAUNCH_CHECK();
}
int pwc_output(const __half* flow, const float* refine, const Vol2& v, int n, int Ho, int Wo, int Hp, int Wp, float* out,
               cudaStream_t s) {
    const int64_t total = int64_t(n) * Ho * Wo;
    const float sx = float(double(Wo) / double(Wp)), sy = float(double(Ho) / double(Hp));
    output_kernel<<<nb(total, 256), 256, 0, s>>>(flow, refine, v, n, Ho, Wo, sx, sy, out);
    LAUNCH_CHECK();
}

}  // namespace vf
