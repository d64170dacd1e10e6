// Memory-bound kernels of the I3D path: stem phase packing, zero-padding max pools, the (2,7,7) average pool +
// temporal mean head, and a diagnostic unpack.  All operate on channels-last fp16 rows of zero-bordered volumes.
#include "common.cuh"
#include "internal.h"

namespace vf {

struct DVol {   // device-side view of a zero-bordered volume (same leading fields as Vol in i3d.cu)
    int n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1;
};

namespace {

inline unsigned nblocks(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// Stem operand layout ("phase volume", all three pack kernels): the stride-2 7x7x7 stem is a stride-1 4x4x4 conv over the
// 8 space-time phases.  Row (tq, hq, wq) of the volume [n][Tq][115][115] holds FOUR phase vectors, those of the source
// rows hq-1 .. hq+2 (slot sb = source row hq + sb - 1), each 8*C channels:
//   out[tq][hq][wq][sb*8C + ((pt*2+ph)*2+pw)*C + c] = x[c][2(tq-1)+pt][2(hq+sb-2)+ph][2(wq-1)+pw]   (zero outside the clip)
// i.e. the 4 h-taps are pre-gathered into the row, so the GEMM needs only the 4 t-taps (each a run of 4 w-positions x
// 32*C channels): 3 KB of A operand per output row instead of 16 unaligned 192-byte runs.
//
// x: [n][C][T][224][224] fp32 (already cropped + scaled to [-1,1], what the reference feeds I3D)
__global__ void i3d_phase_pack_f32_kernel(const float* __restrict__ x, int n, int C, int T, __half* __restrict__ out,
                                          int Tq) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = int64_t(n) * Tq * 115 * 115;
    if (idx >= total) return;
    const int wq = int(idx % 115);
    const int hq = int((idx / 115) % 115);
    const int tq = int((idx / (115 * 115)) % Tq);
    const int b = int(idx / (int64_t(115) * 115 * Tq));
    const int w0 = 2 * (wq - 1);
    for (int sb = 0; sb < 4; ++sb) {
        __half* o = out + idx * (32 * C) + sb * (8 * C);
        const int hs = hq + sb - 1;
        for (int pt = 0; pt < 2; ++pt) {
            const int t = 2 * (tq - 1) + pt;
            for (int ph = 0; ph < 2; ++ph) {
                const int hh = 2 * (hs - 1) + ph;
                const bool ok = (t >= 0) && (t < T) && (hh >= 0) && (hh < 224) && (w0 >= 0) && (w0 < 224);
                for (int c = 0; c < C; ++c) {
                    float2 v = make_float2(0.f, 0.f);
                    if (ok) v = __ldg(reinterpret_cast<const float2*>(
                                x + (((int64_t(b) * C + c) * T + t) * 224 + hh) * 224 + w0));
                    o[((pt * 2 + ph) * 2 + 0) * C + c] = __float2half_rn(v.x);
                    o[((pt * 2 + ph) * 2 + 1) * C + c] = __float2half_rn(v.y);
                }
            }
        }
    }
}

// Fused T2 transform + phase packing straight from the resized uint8 frames (extract_i3d.py:62-66 rgb stream):
// frames [n][T][Hr][Wr][3] uint8 -> TensorCenterCrop(224) at (cy,cx) -> 2*x/255 - 1 (fp32, the reference's operation
// order) -> fp16 phase volume.  Channel order is the decoder's (the reference never swaps BGR, SURVEY quirk 1).
// stack b starts at frame b * stack_stride (>= T: a stack may be a window of a longer frame buffer).
// Stores: a thread owns one 192-byte row, so direct 16-byte stores of a warp would land 192 bytes apart (half-used
// sectors).  The rows of a block are contiguous in the output, so they are staged in shared memory (row pitch 13 x 16 B:
// conflict-free) and written out as one contiguous, fully coalesced run.
constexpr int PACK_THREADS = 128;
__device__ __forceinline__ void pack_flush(const uint4* stage, int row_u4, int pitch_u4, __half* out, int64_t row0, int rows) {
    __syncthreads();
    uint4* g = reinterpret_cast<uint4*>(out) + row0 * row_u4;
    const int total = rows * row_u4;
    for (int i = threadIdx.x; i < total; i += PACK_THREADS) {
        const int r = i / row_u4, j = i - r * row_u4;
        g[i] = stage[r * pitch_u4 + j];
    }
}

__global__ void __launch_bounds__(PACK_THREADS) i3d_phase_pack_u8_kernel(const uint8_t* __restrict__ frames, int n, int T,
                                         int64_t stack_stride, int Hr, int Wr, int cy, int cx, __half* __restrict__ out, int Tq) {
    // the transform of a byte, in the reference's fp32 operation order, has 256 possible results: one table per block
    // instead of 96 IEEE divisions per thread
    __shared__ __half lut[256];
    __shared__ __align__(16) uint4 stage[PACK_THREADS * 13];
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        lut[i] = __float2half_rn(__fsub_rn(__fdiv_rn(__fmul_rn(2.0f, float(i)), 255.0f), 1.0f));
    __syncthreads();
    const int64_t row0 = int64_t(blockIdx.x) * PACK_THREADS;
    const int64_t idx = row0 + threadIdx.x;
    const int64_t total = int64_t(n) * Tq * 115 * 115;
    if (idx < total) {
        const int wq = int(idx % 115);
        const int hq = int((idx / 115) % 115);
        const int tq = int((idx / (115 * 115)) % Tq);
        const int b = int(idx / (int64_t(115) * 115 * Tq));
        const int w0 = 2 * (wq - 1);
        const __half zero = __float2half_rn(0.f);
#pragma unroll 1
        for (int sb = 0; sb < 4; ++sb) {
            __align__(16) __half vals[24];
            const int hs = hq + sb - 1;
#pragma unroll
            for (int pt = 0; pt < 2; ++pt) {
                const int t = 2 * (tq - 1) + pt;
#pragma unroll
                for (int ph = 0; ph < 2; ++ph) {
                    const int hh = 2 * (hs - 1) + ph;
                    const bool ok = (t >= 0) && (t < T) && (hh >= 0) && (hh < 224) && (w0 >= 0) && (w0 < 224);
                    const uint8_t* p = frames + (((int64_t(b) * stack_stride + (ok ? t : 0)) * Hr + cy + (ok ? hh : 0)) * Wr + cx + (ok ? w0 : 0)) * 3;
#pragma unroll
                    for (int pw = 0; pw < 2; ++pw)
#pragma unroll
                        for (int c = 0; c < 3; ++c)
                            vals[((pt * 2 + ph) * 2 + pw) * 3 + c] = ok ? lut[__ldg(p + pw * 3 + c)] : zero;
                }
            }
            uint4* o = stage + threadIdx.x * 13 + sb * 3;
            const uint4* v4 = reinterpret_cast<const uint4*>(vals);
            o[0] = v4[0]; o[1] = v4[1]; o[2] = v4[2];
        }
    }
    const int rows = int(min(int64_t(PACK_THREADS), total - row0));
    pack_flush(stage, 12, 13, out, row0, rows);
}

// Fused T3 transform + phase packing for the flow stream (extract_i3d.py:67-73): flow [n][T][2][H][W] fp32 (the RAFT
// output, still padded) -> crop 224 at (cy,cx) -> clamp(+-20) -> 128 + 255/40*f -> round half-to-even (+20 -> 256, not
// clipped, as the reference) -> 2*x/255 - 1 -> fp16 phase volume with 16 channels.
__global__ void __launch_bounds__(PACK_THREADS) i3d_phase_pack_flow_kernel(const float* __restrict__ flow, int n, int T, int H,
                                           int W, int cy, int cx, __half* __restrict__ out, int Tq) {
    __shared__ __align__(16) uint4 stage[PACK_THREADS * 9];      // 128-byte rows at a 144-byte pitch
    const int64_t row0 = int64_t(blockIdx.x) * PACK_THREADS;
    const int64_t idx = row0 + threadIdx.x;
    const int64_t total = int64_t(n) * Tq * 115 * 115;
    if (idx < total) {
    const int wq = int(idx % 115);
    const int hq = int((idx / 115) % 115);
    const int tq = int((idx / (115 * 115)) % Tq);
    const int b = int(idx / (int64_t(115) * 115 * Tq));
    const int w0 = 2 * (wq - 1);
#pragma unroll 1
    for (int sb = 0; sb < 4; ++sb) {
        __align__(16) __half vals[16];
        const int hs = hq + sb - 1;
#pragma unroll
        for (int pt = 0; pt < 2; ++pt) {
            const int t = 2 * (tq - 1) + pt;
#pragma unroll
            for (int ph = 0; ph < 2; ++ph) {
                const int hh = 2 * (hs - 1) + ph;
                const bool ok = (t >= 0) && (t < T) && (hh >= 0) && (hh < 224) && (w0 >= 0) && (w0 < 224);
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float2 f = make_float2(0.f, 0.f);
                    if (ok) {
                        const float* p = flow + (((int64_t(b) * T + t) * 2 + c) * H + cy + hh) * W + cx + w0;
                        f.x = __ldg(p); f.y = __ldg(p + 1);
                    }
#pragma unroll
                    for (int pw = 0; pw < 2; ++pw) {
                        float v = pw ? f.y : f.x;
                        if (ok) {
                            v = fminf(fmaxf(v, -20.0f), 20.0f);
                            v = rintf(__fadd_rn(128.0f, __fmul_rn(6.375f, v)));
                            v = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, v), 255.0f), 1.0f);
                        }
                        vals[((pt * 2 + ph) * 2 + pw) * 2 + c] = __float2half_rn(v);
                    }
                }
            }
        }
        uint4* o = stage + threadIdx.x * 9 + sb * 2;
        const uint4* v4 = reinterpret_cast<const uint4*>(vals);
        o[0] = v4[0]; o[1] = v4[1];
    }
    }
    const int rows = int(min(int64_t(PACK_THREADS), total - row0));
    pack_flush(stage, 8, 9, out, row0, rows);
}

// ---- split-fp16 pair tensors.  Every tensor that a 1x1x1 conv or a pool reads is stored as a pair x = hi + lo (two fp16
// numbers, ~22 mantissa bits), row = [hi C | lo C]: a CPU emulation of the trained rgb net puts 6.8e-4 of the 8.1e-4 output
// error on the fp16 rounding of exactly these tensors (the stem pool output alone: 4.1e-4), and only 2.7e-4 on the inputs of
// the 3x3x3 convs, which carry the FLOPs and stay single fp16.  A pair is the canonical split of its fp32 value, so
// hi + lo is exact in fp32 and max() picks one of the input pairs.
__device__ __forceinline__ void pair_split8(const float* v, uint4& hi4, uint4& lo4) {
    __align__(16) __half hi[8], lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        hi[j] = __float2half_rn(v[j]);
        lo[j] = __float2half_rn(v[j] - __half2float(hi[j]));
    }
    hi4 = *reinterpret_cast<const uint4*>(hi);
    lo4 = *reinterpret_cast<const uint4*>(lo);
}
__device__ __forceinline__ void pair_load_max8(const __half* p, int C, float* m) {
    const uint4 h4 = __ldg(reinterpret_cast<const uint4*>(p)), l4 = __ldg(reinterpret_cast<const uint4*>(p + C));
    const __half2* hh = reinterpret_cast<const __half2*>(&h4);
    const __half2* ll = reinterpret_cast<const __half2*>(&l4);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = __half22float2(hh[j]), b = __half22float2(ll[j]);
        m[2 * j] = fmaxf(m[2 * j], a.x + b.x);
        m[2 * j + 1] = fmaxf(m[2 * j + 1], a.y + b.y);
    }
}

// Max pool over the VALID region of the input volume with ZERO padding semantics (MaxPool3dTFPadding: ConstantPad3d(0)
// then ceil-mode MaxPool3d; inputs are post-ReLU so 0 never wins wrongly).  Input and output are pair tensors (rows of
// 2C).  One thread = one output position x 8 channels; border positions of the output volume are written as zeros.
__global__ void maxpool3d_kernel(const __half* __restrict__ in, DVol vi, __half* __restrict__ out, DVol vo, int C,
                                 int kt, int kh, int kw, int st, int sh, int sw, int pt, int ph, int pw) {
    const int cg = C >> 3;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = int64_t(vo.n) * vo.Tp * vo.Hp * vo.Wp * cg;
    if (idx >= total) return;
    const int c8 = int(idx % cg);
    const int64_t pos = idx / cg;
    const int w = int(pos % vo.Wp);
    const int hh = int((pos / vo.Wp) % vo.Hp);
    const int t = int((pos / (int64_t(vo.Wp) * vo.Hp)) % vo.Tp);
    const int b = int(pos / (int64_t(vo.Wp) * vo.Hp * vo.Tp));
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = 0.f;
    const bool valid = (t >= vo.t0) && (t < vo.t1) && (hh >= vo.h0) && (hh < vo.h1) && (w >= vo.w0) && (w < vo.w1);
    if (valid) {
        const int ot = t - vo.t0, oh = hh - vo.h0, ow = w - vo.w0;     // output coordinates
        const int Ti = vi.t1 - vi.t0, Hi = vi.h1 - vi.h0, Wi = vi.w1 - vi.w0;
        for (int a = 0; a < kt; ++a) {
            const int it = ot * st - pt + a;
            if (it < 0 || it >= Ti) continue;
            for (int bq = 0; bq < kh; ++bq) {
                const int ih = oh * sh - ph + bq;
                if (ih < 0 || ih >= Hi) continue;
                for (int cc = 0; cc < kw; ++cc) {
                    const int iw = ow * sw - pw + cc;
                    if (iw < 0 || iw >= Wi) continue;
                    const int64_t r = ((int64_t(b) * vi.Tp + it + vi.t0) * vi.Hp + ih + vi.h0) * vi.Wp + iw + vi.w0;
                    pair_load_max8(in + r * (2 * C) + c8 * 8, C, m);
                }
            }
        }
    }
    uint4 hi4, lo4;
    pair_split8(m, hi4, lo4);
    *reinterpret_cast<uint4*>(out + pos * (2 * C) + c8 * 8) = hi4;
    *reinterpret_cast<uint4*>(out + pos * (2 * C) + C + c8 * 8) = lo4;
}

// Same pool without bounds checks for the strided pools between stages (window / stride compile-time, padding 0 before):
// the window may run past the valid region only into the zero border, which is the zero padding (host-checked).  All
// KT*KH*KW pair loads of a thread are independent and unrolled.
template <int KT, int KH, int KW, int ST, int SH, int SW>
__global__ void maxpool3d_fast_kernel(const __half* __restrict__ in, DVol vi, __half* __restrict__ out, DVol vo, int C) {
    const int cg = C >> 3;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = int64_t(vo.n) * vo.Tp * vo.Hp * vo.Wp * cg;
    if (idx >= total) return;
    const int c8 = int(idx % cg);
    const int64_t pos = idx / cg;
    const int w = int(pos % vo.Wp);
    const int hh = int((pos / vo.Wp) % vo.Hp);
    const int t = int((pos / (int64_t(vo.Wp) * vo.Hp)) % vo.Tp);
    const int b = int(pos / (int64_t(vo.Wp) * vo.Hp * vo.Tp));
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = 0.f;
    const bool valid = (t >= vo.t0) && (t < vo.t1) && (hh >= vo.h0) && (hh < vo.h1) && (w >= vo.w0) && (w < vo.w1);
    if (valid) {
        const int it0 = (t - vo.t0) * ST + vi.t0, ih0 = (hh - vo.h0) * SH + vi.h0, iw0 = (w - vo.w0) * SW + vi.w0;
        const __half* p0 = in + (((int64_t(b) * vi.Tp + it0) * vi.Hp + ih0) * vi.Wp + iw0) * (2 * C) + c8 * 8;
        const int64_t sh = int64_t(vi.Wp) * 2 * C, st = sh * vi.Hp;
#pragma unroll
        for (int a = 0; a < KT; ++a)
#pragma unroll
            for (int bq = 0; bq < KH; ++bq)
#pragma unroll
                for (int cc = 0; cc < KW; ++cc) pair_load_max8(p0 + a * st + bq * sh + cc * 2 * C, C, m);
    }
    uint4 hi4, lo4;
    pair_split8(m, hi4, lo4);
    *reinterpret_cast<uint4*>(out + pos * (2 * C) + c8 * 8) = hi4;
    *reinterpret_cast<uint4*>(out + pos * (2 * C) + C + c8 * 8) = lo4;
}

// The Mixed blocks' branch-3 pool: 3x3x3, stride 1, zero padding 1, same volume geometry in and out (border >= 1 of
// zeros all around, which IS the padding: no bounds checks), pair tensors in and out.  One thread = (clip, t, w, 8
// channels) marching down h: per step it folds the 3 (t) x 3 (w) neighbours of one input row into a row maximum (9
// coalesced pair loads) and emits the maximum of the last three row maxima -- 9 positions per output instead of 27.
// Border positions are written as zeros.
__global__ void maxpool3d_same3_kernel(const __half* __restrict__ in, DVol v, __half* __restrict__ out, int C) {
    const int cg = C >> 3, ld = 2 * C;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = int64_t(v.n) * v.Tp * v.Wp * cg;
    if (idx >= total) return;
    const int c8 = int(idx % cg);
    const int w = int((idx / cg) % v.Wp);
    const int t = int((idx / (int64_t(cg) * v.Wp)) % v.Tp);
    const int b = int(idx / (int64_t(cg) * v.Wp * v.Tp));
    const int64_t plane = int64_t(v.Hp) * v.Wp * ld, rowp = int64_t(v.Wp) * ld;
    const int64_t base = (int64_t(b) * v.Tp + t) * plane + int64_t(w) * ld + c8 * 8;     // (b, t, h = 0, w), hi half
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    auto store_zero = [&](int hh) {
        *reinterpret_cast<uint4*>(out + base + hh * rowp) = z4;
        *reinterpret_cast<uint4*>(out + base + hh * rowp + C) = z4;
    };
    if (t < v.t0 || t >= v.t1 || w < v.w0 || w >= v.w1) {
        for (int hh = 0; hh < v.Hp; ++hh) store_zero(hh);
        return;
    }
    auto row_max = [&](int hh, float* m) {          // max over (t-1..t+1, w-1..w+1) of input row hh
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = 0.f;
#pragma unroll
        for (int dt = -1; dt <= 1; ++dt)
#pragma unroll
            for (int dw = -1; dw <= 1; ++dw) pair_load_max8(in + base + dt * plane + hh * rowp + dw * ld, C, m);
    };
    float r0[8], r1[8], r2[8];
    for (int hh = 0; hh < v.h0; ++hh) store_zero(hh);
    row_max(v.h0 - 1, r0);
    row_max(v.h0, r1);
    for (int hh = v.h0; hh < v.h1; ++hh) {
        row_max(hh + 1, r2);
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[j] = fmaxf(fmaxf(r0[j], r1[j]), r2[j]); r0[j] = r1[j]; r1[j] = r2[j]; }
        uint4 hi4, lo4;
        pair_split8(o, hi4, lo4);
        *reinterpret_cast<uint4*>(out + base + hh * rowp) = hi4;
        *reinterpret_cast<uint4*>(out + base + hh * rowp + C) = lo4;
    }
    for (int hh = v.h1; hh < v.Hp; ++hh) store_zero(hh);
}

// AvgPool3d((2,7,7), stride 1) on a T3 x 7 x 7 map -> (T3-1) x 1 x 1, squeeze, mean over time (i3d_net.py:258-264):
// feature[c] = 1/(T3-1) * sum_{t'} 1/98 * sum_{dt<2,h,w} x[t'+dt][h][w][c].   One block per clip, thread = channel.
// The input is a pair tensor (rows of 2C).
__global__ void i3d_head_kernel(const __half* __restrict__ in, DVol v, int C, float* __restrict__ out) {
    const int b = blockIdx.y;
    const int T3 = v.t1 - v.t0;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
        float acc = 0.f;
        for (int t = 0; t < T3; ++t) {
            float plane = 0.f;
            for (int hh = 0; hh < 7; ++hh)
                for (int w = 0; w < 7; ++w) {
                    const int64_t r = ((int64_t(b) * v.Tp + t + v.t0) * v.Hp + hh + v.h0) * v.Wp + w + v.w0;
                    plane += __half2float(in[r * (2 * C) + c]) + __half2float(in[r * (2 * C) + C + c]);
                }
            const float wgt = (t == 0 || t == T3 - 1) ? 1.f : 2.f;    // interior planes sit in two (2,7,7) windows
            acc += wgt * plane;
        }
        out[int64_t(b) * C + c] = acc / (98.f * float(T3 - 1));
    }
}

// diagnostic: valid region of a bordered channels-last volume -> fp32 NCTHW
// (lo_off > 0: the columns are hi halves of a pair tensor, lo halves lo_off columns to the right)
__global__ void unpack_ndhwc_kernel(const __half* __restrict__ in, DVol v, int ld, int c_off, int c_cnt, int lo_off,
                                    float* __restrict__ out) {
    const int T = v.t1 - v.t0, H = v.h1 - v.h0, W = v.w1 - v.w0;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t total = int64_t(v.n) * c_cnt * T * H * W;
    if (idx >= total) return;
    const int w = int(idx % W);
    const int hh = int((idx / W) % H);
    const int t = int((idx / (int64_t(W) * H)) % T);
    const int c = int((idx / (int64_t(W) * H * T)) % c_cnt);
    const int b = int(idx / (int64_t(W) * H * T * c_cnt));
    const int64_t r = ((int64_t(b) * v.Tp + t + v.t0) * v.Hp + hh + v.h0) * v.Wp + w + v.w0;
    out[idx] = __half2float(in[r * ld + c_off + c]) + (lo_off > 0 ? __half2float(in[r * ld + c_off + c + lo_off]) : 0.f);
}

}  // namespace

// the host-side Vol in i3d.cu has the same leading fields; these launchers take it by const reference there
struct VolHost {
    int n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1;
};
static DVol to_dev(const void* p) {
    const VolHost* v = static_cast<const VolHost*>(p);
    return DVol{v->n, v->Tp, v->Hp, v->Wp, v->t0, v->t1, v->h0, v->h1, v->w0, v->w1};
}

int launch_i3d_phase_pack_f32(const float* x, int n, int C, int T, __half* out, int Tq, cudaStream_t s) {
    const int64_t total = int64_t(n) * Tq * 115 * 115;
    i3d_phase_pack_f32_kernel<<<nblocks(total, 256), 256, 0, s>>>(x, n, C, T, out, Tq);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}
int launch_i3d_phase_pack_u8(const uint8_t* frames, int n, int T, int64_t stack_stride, int Hr, int Wr, int cy, int cx,
                             __half* out, int Tq, cudaStream_t s) {
    const int64_t total = int64_t(n) * Tq * 115 * 115;
    i3d_phase_pack_u8_kernel<<<nblocks(total, PACK_THREADS), PACK_THREADS, 0, s>>>(frames, n, T, stack_stride, Hr, Wr, cy, cx, out, Tq);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}
int launch_i3d_phase_pack_flow(const float* flow, int n, int T, int H, int W, int cy, int cx, __half* out, int Tq,
                               cudaStream_t s) {
    const int64_t total = int64_t(n) * Tq * 115 * 115;
    i3d_phase_pack_flow_kernel<<<nblocks(total, PACK_THREADS), PACK_THREADS, 0, s>>>(flow, n, T, H, W, cy, cx, out, Tq);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}
// Which kernel launch_maxpool3d_raw runs (VF_POOL_*):
//   same3: a 3x3x3 / 1 pad 1 pool onto the input's own geometry with a border of at least 1 on every side;
//   fast:  padding 0 before, the last window of every axis ends inside the input's zero border, and the window / stride
//          is one the fast kernel is instantiated for;
//   general: everything else.
int maxpool3d_path_raw(const void* vi, const void* vo, int kt, int kh, int kw, int st, int sh, int sw, int pt, int ph,
                       int pw) {
    const DVol a = to_dev(vi), b = to_dev(vo);
    const bool same_geom = a.n == b.n && a.Tp == b.Tp && a.Hp == b.Hp && a.Wp == b.Wp && a.t0 == b.t0 && a.t1 == b.t1 &&
                           a.h0 == b.h0 && a.h1 == b.h1 && a.w0 == b.w0 && a.w1 == b.w1;
    if (same_geom && kt == 3 && kh == 3 && kw == 3 && st == 1 && sh == 1 && sw == 1 && pt == 1 && ph == 1 && pw == 1 &&
        a.t0 >= 1 && a.h0 >= 1 && a.w0 >= 1 && a.t1 < a.Tp && a.h1 < a.Hp && a.w1 < a.Wp)
        return VF_POOL_SAME3;
    const int To = b.t1 - b.t0, Ho = b.h1 - b.h0, Wo = b.w1 - b.w0;
    const bool fits = pt == 0 && ph == 0 && pw == 0 && To > 0 && Ho > 0 && Wo > 0 &&
                      a.t0 + (To - 1) * st + kt <= a.Tp && a.h0 + (Ho - 1) * sh + kh <= a.Hp &&
                      a.w0 + (Wo - 1) * sw + kw <= a.Wp;
    const bool window = (kt == 1 && kh == 3 && kw == 3 && st == 1 && sh == 2 && sw == 2) ||
                        (kt == 3 && kh == 3 && kw == 3 && st == 2 && sh == 2 && sw == 2) ||
                        (kt == 2 && kh == 2 && kw == 2 && st == 2 && sh == 2 && sw == 2);
    return fits && window ? VF_POOL_FAST : VF_POOL_GENERAL;
}

int launch_maxpool3d_raw(const __half* in, const void* vi, __half* out, const void* vo, int C, int kt, int kh, int kw,
                         int st, int sh, int sw, int pt, int ph, int pw, cudaStream_t s) {
    if (C % 8) return fail(VF_ERR_INVALID, "maxpool3d: C=%d must be a multiple of 8", C);
    const DVol a = to_dev(vi), b = to_dev(vo);
    const int path = maxpool3d_path_raw(vi, vo, kt, kh, kw, st, sh, sw, pt, ph, pw);
    if (path == VF_POOL_SAME3) {
        const int64_t threads = int64_t(a.n) * a.Tp * a.Wp * (C / 8);
        maxpool3d_same3_kernel<<<nblocks(threads, 128), 128, 0, s>>>(in, a, out, C);
        VF_CUDA(cudaGetLastError());
        return VF_OK;
    }
    const int64_t total = int64_t(b.n) * b.Tp * b.Hp * b.Wp * (C / 8);
    if (path == VF_POOL_FAST) {
#define VF_POOL_CASE(KT, KH, KW, ST, SH, SW)                                                                      \
        if (kt == KT && kh == KH && kw == KW && st == ST && sh == SH && sw == SW) {                               \
            maxpool3d_fast_kernel<KT, KH, KW, ST, SH, SW><<<nblocks(total, 256), 256, 0, s>>>(in, a, out, b, C);   \
            VF_CUDA(cudaGetLastError());                                                                          \
            return VF_OK;                                                                                         \
        }
        VF_POOL_CASE(1, 3, 3, 1, 2, 2)
        VF_POOL_CASE(3, 3, 3, 2, 2, 2)
        VF_POOL_CASE(2, 2, 2, 2, 2, 2)
#undef VF_POOL_CASE
        return fail(VF_ERR_INVALID, "maxpool3d: no fast kernel for window %dx%dx%d / %dx%dx%d", kt, kh, kw, st, sh, sw);
    }
    maxpool3d_kernel<<<nblocks(total, 256), 256, 0, s>>>(in, a, out, b, C, kt, kh, kw, st, sh, sw, pt, ph, pw);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}
int launch_i3d_head_raw(const __half* in, const void* vi, int C, float* out, cudaStream_t s) {
    const DVol a = to_dev(vi);
    i3d_head_kernel<<<dim3((C + 63) / 64, a.n), 64, 0, s>>>(in, a, C, out);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}
int launch_unpack_ndhwc_raw(const __half* in, const void* vi, int C, int c_off, int c_cnt, int ld, int lo_off, float* out,
                            cudaStream_t s) {
    const DVol a = to_dev(vi);
    const int64_t total = int64_t(a.n) * c_cnt * (a.t1 - a.t0) * (a.h1 - a.h0) * (a.w1 - a.w0);
    (void)C;
    unpack_ndhwc_kernel<<<nblocks(total, 256), 256, 0, s>>>(in, a, ld, c_off, c_cnt, lo_off, out);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // namespace vf

namespace {

// a volume the pool / head kernels can index: positive extents, the valid region inside the padded one
bool vol_ok(const int* v) {
    return v[0] > 0 && v[1] > 0 && v[2] > 0 && v[3] > 0 && 0 <= v[4] && v[4] < v[5] && v[5] <= v[1] && 0 <= v[6] &&
           v[6] < v[7] && v[7] <= v[2] && 0 <= v[8] && v[8] < v[9] && v[9] <= v[3];
}

}  // namespace

extern "C" {

int vf_debug_maxpool3d(const void* in, const int* vol_in, void* out, const int* vol_out, int C, const int* k,
                       const int* s, const int* p, int* path, void* stream) {
    if (!in || !vol_in || !out || !vol_out || !k || !s || !p || !path)
        return vf::fail(VF_ERR_INVALID, "debug_maxpool3d: null argument");
    if (!vol_ok(vol_in) || !vol_ok(vol_out) || vol_in[0] != vol_out[0] || C <= 0)
        return vf::fail(VF_ERR_INVALID, "debug_maxpool3d: bad volume or C=%d", C);
    for (int j = 0; j < 3; ++j)
        if (k[j] < 1 || s[j] < 1 || p[j] < 0) return vf::fail(VF_ERR_INVALID, "debug_maxpool3d: bad window");
    *path = vf::maxpool3d_path_raw(vol_in, vol_out, k[0], k[1], k[2], s[0], s[1], s[2], p[0], p[1], p[2]);
    return vf::launch_maxpool3d_raw(static_cast<const __half*>(in), vol_in, static_cast<__half*>(out), vol_out, C, k[0],
                                    k[1], k[2], s[0], s[1], s[2], p[0], p[1], p[2], static_cast<cudaStream_t>(stream));
}

int vf_debug_i3d_head(const void* in, const int* vol, int C, float* out, void* stream) {
    if (!in || !vol || !out) return vf::fail(VF_ERR_INVALID, "debug_i3d_head: null argument");
    if (!vol_ok(vol) || C <= 0 || vol[5] - vol[4] < 2 || vol[7] - vol[6] != 7 || vol[9] - vol[8] != 7)
        return vf::fail(VF_ERR_INVALID, "debug_i3d_head: the valid region must be T3 >= 2 x 7 x 7 (C=%d)", C);
    return vf::launch_i3d_head_raw(static_cast<const __half*>(in), vol, C, out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
