// Kernels of the Swin3D towers (swin3d.cu): the fused clip transform into patch rows, width-generic LayerNorms and the
// shifted-window attention.  Rows are always in natural (clip, t', h', w') order: the attention kernel owns the
// windowing (padding, cyclic shift, partition and its reverse) through an index map, so no other pass moves rows.
#include <atomic>

#include "common.cuh"
#include "mma_sync.cuh"
#include "resize_u8.cuh"
#include "swin3d_kernels.h"

namespace vf {

namespace {

// the Swin3D_*_Weights.KINETICS400_V1 presets' Normalize (ImageNet statistics), float32-rounded like torch does
__constant__ float kSwMean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float kSwStd[3] = {0.229f, 0.224f, 0.225f};

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// One thread per (patch row, channel c, temporal tap kt): the 16 columns c * 32 + kt * 16 + kh * 4 + kw.
// U8: F.resize of the uint8 frame (float interpolation of the bytes, torch.round half to even, uint8), /255, Normalize,
// as IEEE fp32 ops in torchvision's order, evaluated on the crop window only.
template <bool U8>
__global__ void patch_kernel(const void* __restrict__ src, R21DStarts st, int m, int T, int H, int W, int rh, int rw,
                             int cy, int cx, __half* __restrict__ out) {
    const int Tq = (T + 1) / 2;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(m) * Tq * 56 * 56 * 6) return;
    const int sub = int(idx % 6), c = sub >> 1, kt = sub & 1;
    const int64_t row = idx / 6;
    const int wq = int(row % 56), hq = int((row / 56) % 56), tq = int((row / 3136) % Tq), b = int(row / (3136 * int64_t(Tq)));
    const int t = 2 * tq + kt;
    __align__(16) __half v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = __float2half_rn(0.f);
    if (t < T) {
        if (U8) {
            const uint8_t* fr = static_cast<const uint8_t*>(src) + (int64_t(st.first[b]) + t) * H * W * 3;
            const int sc = 2 - c;                   // RGB channel c = BGR channel 2 - c
#pragma unroll
            for (int kh = 0; kh < 4; ++kh) {
                int h0, h1;
                float a0, a1;
                bilinear_tap(hq * 4 + kh + cy, H, rh, h0, h1, a0, a1);
#pragma unroll
                for (int kw = 0; kw < 4; ++kw) {
                    int w0, w1;
                    float b0, b1;
                    bilinear_tap(wq * 4 + kw + cx, W, rw, w0, w1, b0, b1);
                    const float r = resized_unit(fr, W, sc, h0, h1, a0, a1, w0, w1, b0, b1);
                    v[kh * 4 + kw] = __float2half_rn(__fdiv_rn(__fsub_rn(r, kSwMean[c]), kSwStd[c]));
                }
            }
        } else {
            const float* x = static_cast<const float*>(src) + ((int64_t(b) * 3 + c) * T + t) * SW_CROP * SW_CROP;
#pragma unroll
            for (int kh = 0; kh < 4; ++kh)
#pragma unroll
                for (int kw = 0; kw < 4; ++kw)
                    v[kh * 4 + kw] = __float2half_rn(__ldg(x + (hq * 4 + kh) * SW_CROP + wq * 4 + kw));
        }
    }
    uint4* o = reinterpret_cast<uint4*>(out + row * SW_PK + c * 32 + kt * 16);
    o[0] = reinterpret_cast<const uint4*>(v)[0];
    o[1] = reinterpret_cast<const uint4*>(v)[1];
}

// LayerNorm statistics of one row of C fp32 (one warp; lane-strided partial sums, then the butterfly): two passes
__device__ __forceinline__ void ln_stats(const float* __restrict__ xr, int C, int lane, float& mean, float& rstd,
                                         float eps = 1e-5f) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += xr[c];
    mean = warp_sum(s) / float(C);
    float q = 0.f;
    for (int c = lane; c < C; c += 32) {
        const float d = xr[c] - mean;
        q += d * d;
    }
    rstd = rsqrtf(warp_sum(q) / float(C) + eps);
}

__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, int C, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, void* __restrict__ out,
                                                        int out_f32, float* __restrict__ out2, int64_t rows,
                                                        float eps) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t row = int64_t(blockIdx.x) * 8 + warp;
    if (row >= rows) return;
    const float* xr = x + row * C;
    float mean, rstd;
    ln_stats(xr, C, lane, mean, rstd, eps);
    for (int c = lane; c < C; c += 32) {
        const float y = (xr[c] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c);
        if (out_f32) {
            static_cast<float*>(out)[row * C + c] = y;
            if (out2) out2[row * C + c] = y;
        } else {
            static_cast<__half*>(out)[row * C + c] = __float2half_rn(y);
        }
    }
}

// PatchMerging: the merged row is [x0 | x1 | x2 | x3] (x0 [0::2, 0::2], x1 [1::2, 0::2], x2 [0::2, 1::2],
// x3 [1::2, 1::2]: H-odd before W-odd), part p at columns p * C ..; each pass walks the four parts in turn
__global__ void __launch_bounds__(256) merge_layernorm_kernel(const float* __restrict__ x, int n, int Tq, int H, int W,
                                                              int C, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, __half* __restrict__ out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int H2 = H / 2, W2 = W / 2;
    const int64_t row = int64_t(blockIdx.x) * 8 + warp;
    if (row >= int64_t(n) * Tq * H2 * W2) return;
    const int w2 = int(row % W2), h2 = int((row / W2) % H2);
    const int64_t bt = row / (int64_t(W2) * H2);
    const float* x00 = x + ((bt * H + 2 * h2) * W + 2 * w2) * C;
    const int64_t dy = int64_t(W) * C;                 // one row down (H odd); one column right (W odd) is C
    const int K = 4 * C;
    float s = 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const float* src = x00 + (p & 1) * dy + (p >> 1) * C;
        for (int c = lane; c < C; c += 32) s += src[c];
    }
    const float mean = warp_sum(s) / float(K);
    float q = 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const float* src = x00 + (p & 1) * dy + (p >> 1) * C;
        for (int c = lane; c < C; c += 32) {
            const float d = src[c] - mean;
            q += d * d;
        }
    }
    const float rstd = rsqrtf(warp_sum(q) / float(K) + 1e-5f);
    __half* o = out + row * K;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const float* src = x00 + (p & 1) * dy + (p >> 1) * C;
        for (int c = lane; c < C; c += 32)
            o[p * C + c] = __float2half_rn((src[c] - mean) * rstd * __ldg(gamma + p * C + c) + __ldg(beta + p * C + c));
    }
}

// One CTA of 8 warps per clip: warp w normalises rows w, w + 8, ... and sums each of its lane's C / 32 columns; the 8
// warp partials are then added in warp order.  C is a multiple of 32, at most 1024.
__global__ void __launch_bounds__(256) norm_mean_kernel(const float* __restrict__ x, int per_clip, int C,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        float* __restrict__ normed, float* __restrict__ feat) {
    __shared__ float part[8][1024];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.x;
    const int per_lane = C / 32;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int r = warp; r < per_clip; r += 8) {
        const int64_t row = int64_t(b) * per_clip + r;
        const float* xr = x + row * C;
        float mean, rstd;
        ln_stats(xr, C, lane, mean, rstd);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            if (i < per_lane) {
                const int c = lane + 32 * i;
                const float y = (xr[c] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c);
                normed[row * C + c] = y;
                acc[i] += y;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 32; ++i)
        if (i < per_lane) part[warp][lane + 32 * i] = acc[i];
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += 256) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += part[w][c];
        feat[int64_t(b) * C + c] = s / float(per_clip);
    }
}

// ---- shifted-window attention
// One CTA of 8 warps per (clip, window, head).  Setup maps each of the window's vol tokens (t-major in-window
// coordinates) to its natural row: shifted padded position p' = window origin + local, natural padded position
// p = (p' + shift) mod padded size, and a row only when p lies inside (Tq, H, W); a padded position is a zero row after
// norm1, so its k and v are the qkv bias.  The whole window's K and V for the head stay in shared memory (at most
// 448 x 32 each, rows padded to 40 halves for conflict-free ldmatrix) with the head's column of the bias table.
// Each warp walks 16-query tiles: scores by mma.sync m16n8k16 over 64-key blocks, s = q.k * 32^-0.5 +
// table[(dt + 7) * 169 + (dh + 6) * 13 + (dw + 6)] (+ -100 where the two tokens' shift regions differ), fp32 online
// softmax, P rounded to fp16, P.V accumulated in fp32, 1 / sum applied to the fp32 output, fp16 out.  Keys past vol
// score -inf; padded queries are computed and not stored.
constexpr int WA_LD = 40, WA_KB = 64, WA_MAXN = 448;
constexpr int WA_SMEM = 2 * WA_MAXN * WA_LD * 2 + SW_TABLE * 4 + 3 * WA_MAXN * 4;

__global__ void __launch_bounds__(256, 2) window_attention_kernel(const __half* __restrict__ qkv,
                                                                  const float* __restrict__ bias_qkv,
                                                                  const float* __restrict__ table,
                                                                  __half* __restrict__ att, SwinAttnGeom g) {
    extern __shared__ __align__(16) uint8_t wa_smem[];
    __half (*Ks)[WA_LD] = reinterpret_cast<__half (*)[WA_LD]>(wa_smem);
    __half (*Vs)[WA_LD] = reinterpret_cast<__half (*)[WA_LD]>(wa_smem + WA_MAXN * WA_LD * 2);
    float* tab = reinterpret_cast<float*>(wa_smem + 2 * WA_MAXN * WA_LD * 2);
    int* rowof = reinterpret_cast<int*>(tab + SW_TABLE);
    int* basep = rowof + WA_MAXN;
    int* regp = basep + WA_MAXN;

    const int heads = gridDim.y, head = blockIdx.y;
    const int wt = g.win[0], wh = g.win[1], ww = g.win[2], vol = wt * wh * ww;
    const int Tp = (g.Tq + wt - 1) / wt * wt, Hp = (g.H + wh - 1) / wh * wh, Wp = (g.W + ww - 1) / ww * ww;
    const int nwt = Tp / wt, nwh = Hp / wh, nww = Wp / ww;
    const int win_id = blockIdx.x % (nwt * nwh * nww), b = blockIdx.x / (nwt * nwh * nww);
    const int oa = win_id / (nwh * nww) * wt, ob = win_id / nww % nwh * wh, oc = win_id % nww * ww;
    const bool masked = g.shift[0] + g.shift[1] + g.shift[2] > 0;
    const int C = g.C, ld = 3 * C;
    const int nkeys = (vol + WA_KB - 1) / WA_KB * WA_KB;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    for (int j = tid; j < nkeys; j += 256) {
        int r = -1, base = 0, reg = -1;
        if (j < vol) {
            const int lt = j / (wh * ww), lh = j / ww % wh, lw = j % ww;
            const int st = oa + lt, sh = ob + lh, sw = oc + lw;           // shifted padded position
            const int pt = (st + g.shift[0]) % Tp, ph = (sh + g.shift[1]) % Hp, pw = (sw + g.shift[2]) % Wp;
            if (pt < g.Tq && ph < g.H && pw < g.W) r = ((b * g.Tq + pt) * g.H + ph) * g.W + pw;
            base = lt * 169 + lh * 13 + lw;
            reg = 0;
            if (masked) {
                auto region = [](int p, int P, int w, int s) { return p < P - w ? 0 : (p < P - s ? 1 : 2); };
                reg = region(st, Tp, wt, g.shift[0]) * 9 + region(sh, Hp, wh, g.shift[1]) * 3 + region(sw, Wp, ww, g.shift[2]);
            }
        }
        rowof[j] = r; basep[j] = base; regp[j] = reg;
    }
    for (int i = tid; i < SW_TABLE; i += 256) tab[i] = __ldg(table + int64_t(i) * heads + head);
    __syncthreads();
    for (int i = tid; i < nkeys * 8; i += 256) {       // K and V rows, 4 x 16 B each
        const int j = i >> 3, m = (i >> 2) & 1, seg = i & 3;
        __half* dst = m == 0 ? &Ks[j][seg * 8] : &Vs[j][seg * 8];
        const int col = (1 + m) * C + head * SW_HEAD_DIM + seg * 8;
        const int r = rowof[j];
        if (r >= 0) {
            cp_async16(dst, qkv + int64_t(r) * ld + col);
        } else {
            __align__(16) __half v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = __float2half_rn(j < vol ? __ldg(bias_qkv + col + e) : 0.f);
            *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(v);
        }
    }
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    __syncthreads();

    const int gq = lane >> 2, tq = lane & 3;
    const float sc = 0.17677669529663687f;            // 32^-0.5
    const float L2E = 1.4426950408889634f;
    const int ntiles = (vol + 15) / 16, nblk = nkeys / WA_KB;
    for (int qt = warp; qt < ntiles; qt += 8) {
        const int q_lo = qt * 16 + gq, q_hi = q_lo + 8;
        const int r_lo = q_lo < vol ? rowof[q_lo] : -1, r_hi = q_hi < vol ? rowof[q_hi] : -1;
        uint32_t aq[2][4];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const int col = head * SW_HEAD_DIM + ks * 16 + 2 * tq;
            auto ld2 = [&](int r, int cc) {
                return r >= 0 ? __ldg(reinterpret_cast<const unsigned int*>(qkv + int64_t(r) * ld + cc)) : 0u;
            };
            aq[ks][0] = ld2(r_lo, col);
            aq[ks][1] = ld2(r_hi, col);
            aq[ks][2] = ld2(r_lo, col + 8);
            aq[ks][3] = ld2(r_hi, col + 8);
        }
        const int base_lo = q_lo < vol ? basep[q_lo] : 0, base_hi = q_hi < vol ? basep[q_hi] : 0;
        const int reg_lo = q_lo < vol ? regp[q_lo] : 0, reg_hi = q_hi < vol ? regp[q_hi] : 0;
        float o[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
        float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
        for (int kb = 0; kb < nblk; ++kb) {
            float s[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
                uint32_t bk[4];
                ldsm_x4(bk, &Ks[kb * WA_KB + nt * 8 + (lane & 7)][(lane >> 3) * 8]);
                mma16816(s[nt], aq[0], bk[0], bk[1]);
                mma16816(s[nt], aq[1], bk[2], bk[3]);
            }
            float n_lo = m_lo, n_hi = m_hi;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int key = kb * WA_KB + nt * 8 + 2 * tq + j;
                    if (key < vol) {
                        const int kbase = 1267 - basep[key], kreg = regp[key];
                        float a = s[nt][j] * sc + tab[base_lo + kbase];
                        float c = s[nt][2 + j] * sc + tab[base_hi + kbase];
                        if (kreg != reg_lo) a += -100.0f;
                        if (kreg != reg_hi) c += -100.0f;
                        s[nt][j] = a * L2E;
                        s[nt][2 + j] = c * L2E;
                    } else {
                        s[nt][j] = s[nt][2 + j] = -INFINITY;
                    }
                    n_lo = fmaxf(n_lo, s[nt][j]);
                    n_hi = fmaxf(n_hi, s[nt][2 + j]);
                }
            }
            n_lo = fmaxf(n_lo, __shfl_xor_sync(0xffffffffu, n_lo, 1));
            n_lo = fmaxf(n_lo, __shfl_xor_sync(0xffffffffu, n_lo, 2));
            n_hi = fmaxf(n_hi, __shfl_xor_sync(0xffffffffu, n_hi, 1));
            n_hi = fmaxf(n_hi, __shfl_xor_sync(0xffffffffu, n_hi, 2));
            const float r0 = exp2f(m_lo - n_lo), r1 = exp2f(m_hi - n_hi);   // exp2f(-inf) == 0 on the first block
            m_lo = n_lo; m_hi = n_hi;
            l_lo *= r0; l_hi *= r1;
#pragma unroll
            for (int i = 0; i < 4; ++i) { o[i][0] *= r0; o[i][1] *= r0; o[i][2] *= r1; o[i][3] *= r1; }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    s[nt][j] = exp2f(s[nt][j] - m_lo);
                    s[nt][2 + j] = exp2f(s[nt][2 + j] - m_hi);
                    l_lo += s[nt][j];
                    l_hi += s[nt][2 + j];
                }
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {        // 16 keys per step: P fragments straight from the score fragments
                uint32_t pa[4];
                pa[0] = pack_half2(s[2 * kk][0], s[2 * kk][1]);
                pa[1] = pack_half2(s[2 * kk][2], s[2 * kk][3]);
                pa[2] = pack_half2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
                pa[3] = pack_half2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
                for (int np = 0; np < 2; ++np) {
                    uint32_t bv[4];
                    ldsm_x4_trans(bv, &Vs[kb * WA_KB + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][np * 16 + (lane >> 4) * 8]);
                    mma16816(o[2 * np], pa, bv[0], bv[1]);
                    mma16816(o[2 * np + 1], pa, bv[2], bv[3]);
                }
            }
        }
        l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
        l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
        l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
        l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
        const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int col = head * SW_HEAD_DIM + nt * 8 + 2 * tq;
            if (r_lo >= 0)
                *reinterpret_cast<uint32_t*>(att + int64_t(r_lo) * C + col) = pack_half2(o[nt][0] * inv_lo, o[nt][1] * inv_lo);
            if (r_hi >= 0)
                *reinterpret_cast<uint32_t*>(att + int64_t(r_hi) * C + col) = pack_half2(o[nt][2] * inv_hi, o[nt][3] * inv_hi);
        }
    }
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int swin3d_patch_u8(const uint8_t* frames, const R21DStarts& st, int m, int T, int H, int W, int rh, int rw, int cy,
                    int cx, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * ((T + 1) / 2) * 3136 * 6;
    patch_kernel<true><<<nb(total, 256), 256, 0, s>>>(frames, st, m, T, H, W, rh, rw, cy, cx, out);
    LAUNCH_CHECK();
}

int swin3d_patch_f32(const float* clips, int m, int T, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * ((T + 1) / 2) * 3136 * 6;
    R21DStarts st;
    st.first[0] = 0;
    patch_kernel<false><<<nb(total, 256), 256, 0, s>>>(clips, st, m, T, 0, 0, 0, 0, 0, 0, out);
    LAUNCH_CHECK();
}

int swin3d_layernorm(const float* x, int C, const float* gamma, const float* beta, void* out, int out_f32, int64_t rows,
                     cudaStream_t s, float* out2, float eps) {
    if (out2 && !out_f32) return fail(VF_ERR_INVALID, "swin3d_layernorm: a second copy needs fp32 output");
    layernorm_kernel<<<nb(rows, 8), 256, 0, s>>>(x, C, gamma, beta, out, out_f32, out2, rows, eps);
    LAUNCH_CHECK();
}

int swin3d_merge_layernorm(const float* x, int n, int Tq, int H, int W, int C, const float* gamma, const float* beta,
                           __half* out, cudaStream_t s) {
    if ((H | W) & 1) return fail(VF_ERR_INVALID, "swin3d_merge_layernorm: odd extent %dx%d", H, W);
    const int64_t rows = int64_t(n) * Tq * (H / 2) * (W / 2);
    merge_layernorm_kernel<<<nb(rows, 8), 256, 0, s>>>(x, n, Tq, H, W, C, gamma, beta, out);
    LAUNCH_CHECK();
}

int swin3d_norm_mean(const float* x, int n, int per_clip, int C, const float* gamma, const float* beta, float* normed,
                     float* feat, cudaStream_t s) {
    if (C % 32 || C > 1024) return fail(VF_ERR_INVALID, "swin3d_norm_mean: width %d", C);
    norm_mean_kernel<<<n, 256, 0, s>>>(x, per_clip, C, gamma, beta, normed, feat);
    LAUNCH_CHECK();
}

SwinAttnGeom swin3d_attn_geom(int n, int Tq, int H, int W, int C, bool shifted) {
    SwinAttnGeom g;
    g.n = n; g.Tq = Tq; g.H = H; g.W = W; g.C = C;
    const int size[3] = {Tq, H, W}, win[3] = {8, 7, 7};
    for (int i = 0; i < 3; ++i) {
        g.win[i] = win[i];
        g.shift[i] = shifted ? win[i] / 2 : 0;
        if (size[i] <= win[i]) { g.win[i] = size[i]; g.shift[i] = 0; }
    }
    return g;
}

int swin3d_attention(const __half* qkv, const float* bias_qkv, const float* table, __half* att, const SwinAttnGeom& g,
                     cudaStream_t s) {
    const int vol = g.win[0] * g.win[1] * g.win[2];
    if (g.n < 1 || g.Tq < 1 || g.H < 1 || g.W < 1 || g.C < SW_HEAD_DIM || g.C % SW_HEAD_DIM || vol < 1 ||
        vol > SW_MAX_VOL || g.win[0] > 8 || g.win[1] > 7 || g.win[2] > 7)
        return fail(VF_ERR_INVALID, "swin3d_attention: %d clips of %dx%dx%d x %d, window %dx%dx%d", g.n, g.Tq, g.H, g.W,
                    g.C, g.win[0], g.win[1], g.win[2]);
    for (int i = 0; i < 3; ++i)
        if (g.win[i] < 1 || g.shift[i] < 0 || g.shift[i] >= g.win[i])
            return fail(VF_ERR_INVALID, "swin3d_attention: window %d shift %d along dim %d", g.win[i], g.shift[i], i);
    static std::atomic<bool> attr_set[64];       // per device, as gemm_kernel.cuh's launch_gemm
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        VF_CUDA(cudaFuncSetAttribute(window_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WA_SMEM));
        if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    const int nw = (g.Tq + g.win[0] - 1) / g.win[0] * ((g.H + g.win[1] - 1) / g.win[1]) * ((g.W + g.win[2] - 1) / g.win[2]);
    const dim3 grid(unsigned(g.n) * unsigned(nw), unsigned(g.C / SW_HEAD_DIM));
    window_attention_kernel<<<grid, 256, WA_SMEM, s>>>(qkv, bias_qkv, table, att, g);
    LAUNCH_CHECK();
}

}  // namespace vf
