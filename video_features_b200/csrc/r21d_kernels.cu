// Memory-bound kernels of the R(2+1)D path: the fused clip transform (BGR->RGB, /255, torch-exact bilinear resize of
// the crop window, Normalize, stem phase pack), the clip gather, the temporal phase repack and (2,2,2) subsample of the
// stride-2 blocks, and the global average pool.  The transform, gather and fp32 pack are templates on the geometry and
// also serve S3D (s3d_kernels.h), whose stem has the same phase layout at 224 x 224.  Activations are split-fp16 rows [hi C | lo C] of zero-bordered
// channels-last 3-D volumes (r21d_kernels.h Vol3); see r21d.cu for the geometry.
#include "common.cuh"
#include "internal.h"
#include "r21d_kernels.h"
#include "s3d_kernels.h"

namespace vf {

namespace {

// reference KINETICS_MEAN / KINETICS_STD (also torchvision's video presets), float32-rounded like torch.as_tensor does
__constant__ float kKinMean[3] = {0.43216f, 0.394666f, 0.37645f};
__constant__ float kKinStd[3] = {0.22803f, 0.22145f, 0.216989f};

__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// torch's CPU upsample_bilinear2d (align_corners=False, no scale factor) source index and weights for output index d:
// scale = float(in) / out, src = max(fma(scale, d + 0.5, -0.5), 0) (the compiler contracts torch's
// scale * (d + 0.5) - 0.5), i0 = min(floor(src), in - 1), l1 = clamp(src - i0, 0, 1), l0 = 1 - l1.
__device__ __forceinline__ void bilinear_tap(int d, int in, int out, int& i0, int& i1, float& l0, float& l1) {
    const float scale = __fdiv_rn(float(in), float(out));
    const float src = fmaxf(__fmaf_rn(scale, __fadd_rn(float(d), 0.5f), -0.5f), 0.f);
    i0 = min(int(floorf(src)), in - 1);
    l1 = fminf(fmaxf(__fsub_rn(src, float(i0)), 0.f), 1.f);
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    l0 = __fsub_rn(1.f, l1);
}

// One thread per phase row (frame f, hq, wq) of the per-frame stem phase volume [nf][Q][Q][32] of a CROP x CROP crop
// of the frame resized to RH x RW.  The ops of the clip transform in its order, as IEEE fp32, the crop only selecting
// resized positions:
//   R(2+1)D (U8_RESIZE false): x = u8 / 255; resized = fma(l0h, t0, l1h * t1) with t = fma(l0w, x_0, l1w * x_1)
//     (torch's `t0 * w0 + t1 * w1`, contracted); Normalize (resized - mean) / std.
//   S3D (U8_RESIZE true): F.resize of the uint8 frame is the same float interpolation of the bytes, stored as uint8
//     after torch.round (half to even); then /255 and Normalize.
template <int Q, int CROP, int RH, int RW, bool U8_RESIZE>
__global__ void frames_u8_kernel(const uint8_t* __restrict__ src, int nf, int H, int W, int cy, int cx,
                                 __half* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(nf) * Q * Q) return;
    const int wq = int(idx % Q), hq = int((idx / Q) % Q), f = int(idx / (Q * Q));
    const uint8_t* fr = src + int64_t(f) * H * W * 3;
    __align__(16) __half vals[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) vals[i] = __float2half_rn(0.f);
#pragma unroll
    for (int ph = 0; ph < 2; ++ph) {
        const int y = 2 * (hq - 2) + ph;
        if (y < 0 || y >= CROP) continue;           // the stem's zero padding
        int h0, h1;
        float a0, a1;
        bilinear_tap(y + cy, H, RH, h0, h1, a0, a1);
#pragma unroll
        for (int pw = 0; pw < 2; ++pw) {
            const int x = 2 * (wq - 2) + pw;
            if (x < 0 || x >= CROP) continue;
            int w0, w1;
            float b0, b1;
            bilinear_tap(x + cx, W, RW, w0, w1, b0, b1);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int sc = 2 - c;                // RGB channel c = BGR channel 2 - c
                auto px = [&](int hh, int ww) {
                    const float b = float(__ldg(fr + (int64_t(hh) * W + ww) * 3 + sc));
                    return U8_RESIZE ? b : __fdiv_rn(b, 255.f);
                };
                const float x00 = px(h0, w0), x01 = px(h0, w1), x10 = px(h1, w0), x11 = px(h1, w1);
                const float t0 = __fmaf_rn(b0, x00, __fmul_rn(b1, x01));
                const float t1 = __fmaf_rn(b0, x10, __fmul_rn(b1, x11));
                float r = __fmaf_rn(a0, t0, __fmul_rn(a1, t1));
                if (U8_RESIZE) r = __fdiv_rn(rintf(r), 255.f);
                const float v = __fdiv_rn(__fsub_rn(r, kKinMean[c]), kKinStd[c]);
                split_half(v, vals[(ph * 2 + pw) * 4 + c], vals[16 + (ph * 2 + pw) * 4 + c]);
            }
        }
    }
    uint4* o = reinterpret_cast<uint4*>(out + idx * 32);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = reinterpret_cast<const uint4*>(vals)[i];
}

// one thread per 16-byte quarter of a clip phase row
template <int Q>
__global__ void clip_gather_kernel(const __half* __restrict__ frames, R21DStarts st, int m, int T,
                                   __half* __restrict__ out) {
    constexpr int QQ = Q * Q;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(m) * (T + 2) * QQ * 4) return;
    const int part = int(idx % 4);
    const int64_t row = idx / 4;
    const int pos = int(row % QQ), tq = int((row / QQ) % (T + 2)), b = int(row / (int64_t(QQ) * (T + 2)));
    uint4 v = make_uint4(0, 0, 0, 0);
    if (tq >= 1 && tq <= T)
        v = __ldg(reinterpret_cast<const uint4*>(frames + ((int64_t(st.first[b]) + tq - 1) * QQ + pos) * 32) + part);
    reinterpret_cast<uint4*>(out + row * 32)[part] = v;
}

// one thread per clip phase row; clips are (m, 3, T, CROP, CROP)
template <int Q, int CROP>
__global__ void pack_f32_kernel(const float* __restrict__ x, int m, int T, __half* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(m) * (T + 2) * Q * Q) return;
    const int wq = int(idx % Q), hq = int((idx / Q) % Q), tq = int((idx / (Q * Q)) % (T + 2));
    const int b = int(idx / (int64_t(Q) * Q * (T + 2)));
    __align__(16) __half vals[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) vals[i] = __float2half_rn(0.f);
    if (tq >= 1 && tq <= T) {
#pragma unroll
        for (int ph = 0; ph < 2; ++ph)
#pragma unroll
            for (int pw = 0; pw < 2; ++pw) {
                const int y = 2 * (hq - 2) + ph, xx = 2 * (wq - 2) + pw;
                if (y < 0 || y >= CROP || xx < 0 || xx >= CROP) continue;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float v = __ldg(x + (((int64_t(b) * 3 + c) * T + tq - 1) * CROP + y) * CROP + xx);
                    split_half(v, vals[(ph * 2 + pw) * 4 + c], vals[16 + (ph * 2 + pw) * 4 + c]);
                }
            }
    }
    uint4* o = reinterpret_cast<uint4*>(out + idx * 32);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = reinterpret_cast<const uint4*>(vals)[i];
}

// 8 elements per thread; every position of vo is written
__global__ void temporal_phase_kernel(const __half* __restrict__ in, Vol3 vi, int C, __half* __restrict__ out, Vol3 vo) {
    const int cg = C >> 3;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= vo.rows() * 2 * cg) return;
    const int c8 = int(idx % cg), p = int((idx / cg) % 2);
    const int64_t pos = idx / (2 * cg);
    const int64_t hw = int64_t(vo.Hp) * vo.Wp;
    const int64_t sp = pos % hw;
    const int q = int((pos / hw) % vo.Tp), b = int(pos / (hw * vo.Tp));
    const int t = 2 * (q - vo.t0) + p;              // valid-region frame of the input
    uint4 v = make_uint4(0, 0, 0, 0);
    if (q >= vo.t0 && q < vo.t1 && t < vi.t1 - vi.t0)
        v = __ldg(reinterpret_cast<const uint4*>(in + ((int64_t(b) * vi.Tp + t + vi.t0) * hw + sp) * C + c8 * 8));
    *reinterpret_cast<uint4*>(out + pos * (2 * C) + p * C + c8 * 8) = v;
}

__global__ void subsample_kernel(const __half* __restrict__ in, Vol3 vi, int C, __half* __restrict__ out, Vol3 vo) {
    const int cg = C >> 3;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= vo.rows() * cg) return;
    const int c8 = int(idx % cg);
    const int64_t pos = idx / cg;
    const int wq = int(pos % vo.Wp), hq = int((pos / vo.Wp) % vo.Hp), tq = int((pos / (int64_t(vo.Wp) * vo.Hp)) % vo.Tp);
    const int b = int(pos / (int64_t(vo.Wp) * vo.Hp * vo.Tp));
    uint4 v = make_uint4(0, 0, 0, 0);
    if (tq >= vo.t0 && tq < vo.t1 && hq >= vo.h0 && hq < vo.h1 && wq >= vo.w0 && wq < vo.w1) {
        const int t = 2 * (tq - vo.t0) + vi.t0, y = 2 * (hq - vo.h0) + vi.h0, x = 2 * (wq - vo.w0) + vi.w0;
        v = __ldg(reinterpret_cast<const uint4*>(in + (((int64_t(b) * vi.Tp + t) * vi.Hp + y) * vi.Wp + x) * C + c8 * 8));
    }
    *reinterpret_cast<uint4*>(out + pos * C + c8 * 8) = v;
}

// out[b][c] = mean over the valid region of (hi + lo), one thread per (b, c), summed in a fixed order
__global__ void avgpool_kernel(const __half* __restrict__ in, Vol3 v, int C, float* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(v.n) * C) return;
    const int c = int(idx % C), b = int(idx / C);
    float s = 0.f;
    for (int t = v.t0; t < v.t1; ++t) {
        float plane = 0.f;
        for (int y = v.h0; y < v.h1; ++y)
            for (int x = v.w0; x < v.w1; ++x) {
                const __half* p = in + (((int64_t(b) * v.Tp + t) * v.Hp + y) * v.Wp + x) * (2 * C) + c;
                plane += __half2float(p[0]) + __half2float(p[C]);
            }
        s += plane;
    }
    out[idx] = s / float(v.T() * v.H() * v.W());
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

// R(2+1)D: 112 crop of Resize((128, 171)) on [59][59]; S3D: 224 crop of Resize((256, 256)) on uint8, [115][115]
int r21d_frames_u8(const uint8_t* frames, int nf, int H, int W, int cy, int cx, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(nf) * R21D_Q * R21D_Q;
    frames_u8_kernel<R21D_Q, 112, 128, 171, false><<<nb(total, 256), 256, 0, s>>>(frames, nf, H, W, cy, cx, out);
    LAUNCH_CHECK();
}
int s3d_frames_u8(const uint8_t* frames, int nf, int H, int W, int cy, int cx, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(nf) * S3D_Q * S3D_Q;
    frames_u8_kernel<S3D_Q, S3D_CROP, S3D_RESIZE, S3D_RESIZE, true><<<nb(total, 256), 256, 0, s>>>(frames, nf, H, W,
                                                                                                   cy, cx, out);
    LAUNCH_CHECK();
}
int r21d_clip_gather(const __half* frames, const R21DStarts& st, int m, int T, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * (T + 2) * R21D_Q * R21D_Q * 4;
    clip_gather_kernel<R21D_Q><<<nb(total, 256), 256, 0, s>>>(frames, st, m, T, out);
    LAUNCH_CHECK();
}
int s3d_clip_gather(const __half* frames, const R21DStarts& st, int m, int T, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * (T + 2) * S3D_Q * S3D_Q * 4;
    clip_gather_kernel<S3D_Q><<<nb(total, 256), 256, 0, s>>>(frames, st, m, T, out);
    LAUNCH_CHECK();
}
int r21d_pack_f32(const float* clips, int m, int T, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * (T + 2) * R21D_Q * R21D_Q;
    pack_f32_kernel<R21D_Q, 112><<<nb(total, 256), 256, 0, s>>>(clips, m, T, out);
    LAUNCH_CHECK();
}
int s3d_pack_f32(const float* clips, int m, int T, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * (T + 2) * S3D_Q * S3D_Q;
    pack_f32_kernel<S3D_Q, S3D_CROP><<<nb(total, 256), 256, 0, s>>>(clips, m, T, out);
    LAUNCH_CHECK();
}
int r21d_temporal_phase(const __half* in, const Vol3& vi, int C, __half* out, const Vol3& vo, cudaStream_t s) {
    if (C % 8) return fail(VF_ERR_INVALID, "r21d_temporal_phase: C=%d must be a multiple of 8", C);
    temporal_phase_kernel<<<nb(vo.rows() * 2 * (C / 8), 256), 256, 0, s>>>(in, vi, C, out, vo);
    LAUNCH_CHECK();
}
int r21d_subsample(const __half* in, const Vol3& vi, int C, __half* out, const Vol3& vo, cudaStream_t s) {
    if (C % 8) return fail(VF_ERR_INVALID, "r21d_subsample: C=%d must be a multiple of 8", C);
    subsample_kernel<<<nb(vo.rows() * (C / 8), 256), 256, 0, s>>>(in, vi, C, out, vo);
    LAUNCH_CHECK();
}
int r21d_avgpool(const __half* in, const Vol3& v, int C, float* out, cudaStream_t s) {
    avgpool_kernel<<<nb(int64_t(v.n) * C, 256), 256, 0, s>>>(in, v, C, out);
    LAUNCH_CHECK();
}

}  // namespace vf
