// Kernels of the MViT towers (mvit.cu): fused clip transform into patch rows, class token and position embeddings,
// head pooling, pooling attention and the skip max-pool.
#include <atomic>

#include "common.cuh"
#include "mma_sync.cuh"
#include "mvit_kernels.h"
#include "resize_u8.cuh"

namespace vf {

namespace {

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

constexpr int MV_TOKENS = MV_TQ * 56 * 56;       // 25088 patch rows per clip

// One thread per (patch row, channel c, temporal tap kt): the 49 columns c * 147 + kt * 49 + ..; sub 9 zeroes the pad
// columns 441..447.  U8: swin3d_patch_u8's transform with the MViT presets' Normalize(0.45, 0.225).
template <bool U8>
__global__ void patch_kernel(const void* __restrict__ src, R21DStarts st, int m, int H, int W, int rh, int rw, int cy,
                             int cx, __half* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(m) * MV_TOKENS * 10) return;
    const int sub = int(idx % 10);
    const int64_t row = idx / 10;
    __half* o = out + row * MV_PK;
    if (sub == 9) {
        for (int i = MV_PATCH_K; i < MV_PK; ++i) o[i] = __float2half_rn(0.f);
        return;
    }
    const int c = sub / 3, kt = sub % 3;
    const int wq = int(row % 56), hq = int((row / 56) % 56), tq = int((row / 3136) % MV_TQ), b = int(row / MV_TOKENS);
    const int t = 2 * tq + kt - 1;
    o += c * 147 + kt * 49;
    if (t < 0 || t >= MV_T) {
        for (int i = 0; i < 49; ++i) o[i] = __float2half_rn(0.f);
        return;
    }
    for (int kh = 0; kh < 7; ++kh) {
        const int y = hq * 4 + kh - 3;
        const bool yin = y >= 0 && y < MV_CROP;
        int h0 = 0, h1 = 0;
        float a0 = 0.f, a1 = 0.f;
        if (U8 && yin) bilinear_tap(y + cy, H, rh, h0, h1, a0, a1);
        for (int kw = 0; kw < 7; ++kw) {
            const int x = wq * 4 + kw - 3;
            float v = 0.f;
            if (yin && x >= 0 && x < MV_CROP) {
                if (U8) {
                    const uint8_t* fr = static_cast<const uint8_t*>(src) + (int64_t(st.first[b]) + t) * H * W * 3;
                    int w0, w1;
                    float b0, b1;
                    bilinear_tap(x + cx, W, rw, w0, w1, b0, b1);
                    const float r = resized_unit(fr, W, 2 - c, h0, h1, a0, a1, w0, w1, b0, b1);   // RGB c = BGR 2 - c
                    v = __fdiv_rn(__fsub_rn(r, 0.45f), 0.225f);
                } else {
                    const float* xs = static_cast<const float*>(src) + ((int64_t(b) * 3 + c) * MV_T + t) * MV_CROP * MV_CROP;
                    v = __ldg(xs + y * MV_CROP + x);
                }
            }
            o[kh * 7 + kw] = __float2half_rn(v);
        }
    }
}

__global__ void embed_kernel(const float* __restrict__ emb, const float* __restrict__ cls, const float* __restrict__ cls_pos,
                             const float* __restrict__ tpos, const float* __restrict__ spos, int m, float* __restrict__ x,
                             float* __restrict__ x2) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const int64_t per_clip = int64_t(1 + MV_TOKENS) * 96;
    if (idx >= m * per_clip) return;
    const int c = int(idx % 96);
    const int64_t r = (idx / 96) % (1 + MV_TOKENS), b = idx / per_clip;
    float v;
    if (r == 0) {
        v = __ldg(cls + c);
        if (cls_pos) v = __fadd_rn(v, __ldg(cls_pos + c));
    } else {
        const int64_t p = r - 1;
        v = emb[(b * MV_TOKENS + p) * 96 + c];
        if (tpos) v = __fadd_rn(v, __fadd_rn(__ldg(tpos + (p / 3136) * 96 + c), __ldg(spos + (p % 3136) * 96 + c)));
    }
    x[idx] = v;
    x2[idx] = v;
}

// One warp per (clip, output row, head); lane holds channels lane, lane + 32, lane + 64.
__global__ void __launch_bounds__(256) head_pool_kernel(const __half* __restrict__ src, int ld_src, int n, int heads,
                                                        int T, int H, int W, int stride, const float* __restrict__ wt,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        __half* __restrict__ dst) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
    const int64_t n_in = 1 + int64_t(T) * H * W, n_out = 1 + int64_t(T) * Ho * Wo;
    const int64_t job = int64_t(blockIdx.x) * 8 + warp;
    if (job >= n * n_out * heads) return;
    const int head = int(job % heads);
    const int64_t r = (job / heads) % n_out, b = job / (heads * n_out);
    const __half* base = src + b * n_in * ld_src + head * MV_HEAD_DIM;
    float acc[3] = {0.f, 0.f, 0.f};
    if (r == 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) acc[i] = __half2float(base[lane + 32 * i]);
    } else {
        const int64_t p = r - 1;
        const int to = int(p / (int64_t(Ho) * Wo)), ho = int(p / Wo % Ho), wo = int(p % Wo);
        for (int dt = 0; dt < 3; ++dt) {
            const int t = to + dt - 1;
            if (t < 0 || t >= T) continue;
            for (int dh = 0; dh < 3; ++dh) {
                const int h = ho * stride + dh - 1;
                if (h < 0 || h >= H) continue;
                for (int dw = 0; dw < 3; ++dw) {
                    const int w = wo * stride + dw - 1;
                    if (w < 0 || w >= W) continue;
                    const __half* xr = base + (1 + (int64_t(t) * H + h) * W + w) * ld_src;
                    const int tap = dt * 9 + dh * 3 + dw;
#pragma unroll
                    for (int i = 0; i < 3; ++i)
                        acc[i] = __fmaf_rn(__ldg(wt + (lane + 32 * i) * 27 + tap), __half2float(xr[lane + 32 * i]), acc[i]);
                }
            }
        }
    }
    const float mean = warp_sum(acc[0] + acc[1] + acc[2]) / 96.f;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) q += (acc[i] - mean) * (acc[i] - mean);
    const float rstd = rsqrtf(warp_sum(q) / 96.f + 1e-6f);
    __half* o = dst + (b * n_out + r) * int64_t(heads) * MV_HEAD_DIM + head * MV_HEAD_DIM;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const int c = lane + 32 * i;
        o[c] = __float2half_rn((acc[i] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c));
    }
}

__global__ void skip_pool_kernel(const float* __restrict__ x, int n, int C, int T, int H, int W, float* __restrict__ y) {
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    const int64_t n_in = 1 + int64_t(T) * H * W, n_out = 1 + int64_t(T) * Ho * Wo;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= n * n_out * C) return;
    const int c = int(idx % C);
    const int64_t r = (idx / C) % n_out, b = idx / (int64_t(C) * n_out);
    const float* xb = x + b * n_in * C + c;
    if (r == 0) { y[idx] = xb[0]; return; }
    const int64_t p = r - 1;
    const int t = int(p / (int64_t(Ho) * Wo)), ho = int(p / Wo % Ho), wo = int(p % Wo);
    float v = -INFINITY;
    for (int dh = 0; dh < 3; ++dh) {
        const int h = 2 * ho + dh - 1;
        if (h < 0 || h >= H) continue;
        for (int dw = 0; dw < 3; ++dw) {
            const int w = 2 * wo + dw - 1;
            if (w < 0 || w >= W) continue;
            v = fmaxf(v, xb[(1 + (int64_t(t) * H + h) * W + w) * C]);
        }
    }
    y[idx] = v;
}

// ---- pooling attention
// One CTA of 8 warps per (query-tile group, head, clip); the (clip, head)'s K and V (rows of 96, padded to 104 halves
// for conflict-free ldmatrix) stay in shared memory when they fit in one chunk of 416 keys (the 393 keys of the
// non-transition blocks) and are streamed through it chunk by chunk otherwise (the 1569 of the q-stride blocks).  Each warp walks 16-query tiles: scores by
// mma.sync m16n8k16 over 32-key blocks, s = q.k / sqrt(96) (+ the rel-pos bias), fp32 online softmax, P rounded to
// fp16, P.V accumulated in fp32, 1 / sum applied to the fp32 output (+ q), fp16 out.  Keys past the last score -inf;
// query rows past the last are computed and not stored.  The rel-pos terms of a tile (16 rows x (kt + kh + kw) dot
// products of the unscaled q with the table rows its distances select) go to the warp's shared scratch first.
constexpr int MA_LD = 104, MA_KB = 32;
constexpr int MA_SMEM = 2 * MV_MAX_KEYS * MA_LD * 2 + MV_MAX_KEYS * 4 + 8 * 16 * MV_MAX_REL * 4;

struct RelArgs {
    const float *h, *w, *t;
    float qr[3], kr[3];        // torchvision's q / k distance ratios (t, h, w) as float32
};

// _add_rel_pos's distance: int(qi * q_ratio - (ki + (1 - K)) * k_ratio) in float32
__device__ __forceinline__ int rel_dist(int qi, int ki, int K, float qr, float kr) {
    return int(__fsub_rn(__fmul_rn(float(qi), qr), __fmul_rn(__fadd_rn(float(ki), float(1 - K)), kr)));
}

__global__ void __launch_bounds__(256, 1) pool_attention_kernel(const __half* __restrict__ q, const __half* __restrict__ k,
                                                                const __half* __restrict__ v, RelArgs ra,
                                                                __half* __restrict__ out, MViTAttnGeom g) {
    extern __shared__ __align__(16) uint8_t ma_smem[];
    __half (*Ks)[MA_LD] = reinterpret_cast<__half (*)[MA_LD]>(ma_smem);
    __half (*Vs)[MA_LD] = reinterpret_cast<__half (*)[MA_LD]>(ma_smem + MV_MAX_KEYS * MA_LD * 2);
    int* keyoff = reinterpret_cast<int*>(ma_smem + 2 * MV_MAX_KEYS * MA_LD * 2);
    float* rb_all = reinterpret_cast<float*>(keyoff + MV_MAX_KEYS);

    const int head = blockIdx.y, b = blockIdx.z, heads = g.heads, C = heads * MV_HEAD_DIM;
    const int QT = g.q_thw[0], QH = g.q_thw[1], QW = g.q_thw[2], KT = g.k_thw[0], KH = g.k_thw[1], KW = g.k_thw[2];
    const int nq = 1 + QT * QH * QW, nk = 1 + KT * KH * KW, NB = KT + KH + KW;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const __half* kb0 = k + int64_t(b) * nk * C + head * MV_HEAD_DIM;
    const __half* vb0 = v + int64_t(b) * nk * C + head * MV_HEAD_DIM;
    const __half* qb0 = q + int64_t(b) * nq * g.ldq + head * MV_HEAD_DIM;

    // one chunk of up to MV_MAX_KEYS keys from key c0 into shared memory, rows padded to a 32-key block with zeros
    auto load_chunk = [&](int c0) {
        const int rows = min(MV_MAX_KEYS, nk - c0), padded = (rows + MA_KB - 1) / MA_KB * MA_KB;
        for (int i = tid; i < padded * 24; i += 256) {         // K and V rows, 12 x 16 B each
            const int j = i / 24, m = (i / 12) & 1, seg = i % 12;
            __half* dst = m == 0 ? &Ks[j][seg * 8] : &Vs[j][seg * 8];
            if (j < rows) {
                cp_async16(dst, (m == 0 ? kb0 : vb0) + int64_t(c0 + j) * C + seg * 8);
            } else {
                *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
            }
        }
        for (int j = tid; j < padded; j += 256) {
            const int key = c0 + j;
            int off = -1;
            if (key >= 1 && key < nk) {
                const int p = key - 1, a = p / (KH * KW), hh = p / KW % KH, ww = p % KW;
                off = a | ((KT + hh) << 8) | ((KT + KH + ww) << 16);
            }
            keyoff[j] = off;
        }
        asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
    };
    const int nchunk = (nk + MV_MAX_KEYS - 1) / MV_MAX_KEYS;
    if (nchunk == 1) {                 // every tile of the CTA reuses the one chunk
        load_chunk(0);
        __syncthreads();
    }

    float* rb = rb_all + warp * 16 * MV_MAX_REL;
    const int gq = lane >> 2, tq = lane & 3;
    const float sc = 0.10206207261596575f;            // 96^-0.5
    const float L2E = 1.4426950408889634f;
    const int ntiles = (nq + 15) / 16;
    // the CTA's warps take 8 consecutive tiles per round (a warp past the last tile computes nothing it stores), so
    // that streamed chunks are shared by all of them
    for (int base = blockIdx.x * 8; base < ntiles; base += gridDim.x * 8) {
        const int qt = base + warp;
        const int q_lo = qt * 16 + gq, q_hi = q_lo + 8;
        const __half* r_lo = q_lo < nq ? qb0 + int64_t(q_lo) * g.ldq : nullptr;
        const __half* r_hi = q_hi < nq ? qb0 + int64_t(q_hi) * g.ldq : nullptr;
        uint32_t aq[6][4];
#pragma unroll
        for (int ks = 0; ks < 6; ++ks) {
            const int col = ks * 16 + 2 * tq;
            auto ld2 = [&](const __half* r, int cc) {
                return r ? __ldg(reinterpret_cast<const unsigned int*>(r + cc)) : 0u;
            };
            aq[ks][0] = ld2(r_lo, col);
            aq[ks][1] = ld2(r_hi, col);
            aq[ks][2] = ld2(r_lo, col + 8);
            aq[ks][3] = ld2(r_hi, col + 8);
        }
        if (g.rel) {
            __syncwarp();
            for (int pr = lane; pr < 16 * NB; pr += 32) {
                const int i = pr / NB, j = pr % NB, qi = qt * 16 + i;
                float acc = 0.f;
                if (qi >= 1 && qi < nq) {
                    const int p = qi - 1, t = p / (QH * QW), hh = p / QW % QH, ww = p % QW;
                    const float* tab;
                    if (j < KT) tab = ra.t + rel_dist(t, j, KT, ra.qr[0], ra.kr[0]) * MV_HEAD_DIM;
                    else if (j < KT + KH) tab = ra.h + rel_dist(hh, j - KT, KH, ra.qr[1], ra.kr[1]) * MV_HEAD_DIM;
                    else tab = ra.w + rel_dist(ww, j - KT - KH, KW, ra.qr[2], ra.kr[2]) * MV_HEAD_DIM;
                    const __half2* qr = reinterpret_cast<const __half2*>(qb0 + int64_t(qi) * g.ldq);
                    for (int d = 0; d < MV_HEAD_DIM / 2; ++d) {
                        const float2 qf = __half22float2(qr[d]);
                        acc = __fmaf_rn(qf.x, __ldg(tab + 2 * d), acc);
                        acc = __fmaf_rn(qf.y, __ldg(tab + 2 * d + 1), acc);
                    }
                }
                rb[i * MV_MAX_REL + j] = acc;
            }
            __syncwarp();
        }
        const bool rel_lo = g.rel && q_lo >= 1 && q_lo < nq, rel_hi = g.rel && q_hi >= 1 && q_hi < nq;
        const float* rb_lo = rb + gq * MV_MAX_REL;
        const float* rb_hi = rb + (gq + 8) * MV_MAX_REL;
        float o[12][4];
#pragma unroll
        for (int i = 0; i < 12; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
        float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
        for (int ch = 0; ch < nchunk; ++ch) {
        if (nchunk > 1) {
            __syncthreads();           // every warp is done with the previous chunk
            load_chunk(ch * MV_MAX_KEYS);
            __syncthreads();
        }
        const int rows = min(MV_MAX_KEYS, nk - ch * MV_MAX_KEYS), nblk = (rows + MA_KB - 1) / MA_KB;
        for (int kb = 0; kb < nblk; ++kb) {
            float s[4][4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
                for (int kc = 0; kc < 3; ++kc) {
                    uint32_t bk[4];
                    ldsm_x4(bk, &Ks[kb * MA_KB + nt * 8 + (lane & 7)][kc * 32 + (lane >> 3) * 8]);
                    mma16816(s[nt], aq[2 * kc], bk[0], bk[1]);
                    mma16816(s[nt], aq[2 * kc + 1], bk[2], bk[3]);
                }
            }
            float n_lo = m_lo, n_hi = m_hi;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int key = kb * MA_KB + nt * 8 + 2 * tq + j;
                    if (key < rows) {
                        float a = s[nt][j] * sc, c = s[nt][2 + j] * sc;
                        const int off = keyoff[key];
                        if (off >= 0) {
                            const int o0 = off & 255, o1 = (off >> 8) & 255, o2 = off >> 16;
                            if (rel_lo) a += rb_lo[o0] + rb_lo[o1] + rb_lo[o2];
                            if (rel_hi) c += rb_hi[o0] + rb_hi[o1] + rb_hi[o2];
                        }
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
            for (int i = 0; i < 12; ++i) { o[i][0] *= r0; o[i][1] *= r0; o[i][2] *= r1; o[i][3] *= r1; }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    s[nt][j] = exp2f(s[nt][j] - m_lo);
                    s[nt][2 + j] = exp2f(s[nt][2 + j] - m_hi);
                    l_lo += s[nt][j];
                    l_hi += s[nt][2 + j];
                }
            }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {        // 16 keys per step: P fragments straight from the score fragments
                uint32_t pa[4];
                pa[0] = pack_half2(s[2 * kk][0], s[2 * kk][1]);
                pa[1] = pack_half2(s[2 * kk][2], s[2 * kk][3]);
                pa[2] = pack_half2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
                pa[3] = pack_half2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
                for (int np = 0; np < 6; ++np) {
                    uint32_t bv[4];
                    ldsm_x4_trans(bv, &Vs[kb * MA_KB + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][np * 16 + (lane >> 4) * 8]);
                    mma16816(o[2 * np], pa, bv[0], bv[1]);
                    mma16816(o[2 * np + 1], pa, bv[2], bv[3]);
                }
            }
        }
        }
        l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
        l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
        l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
        l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
        const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
        const bool res_lo = g.resid && q_lo >= 1, res_hi = g.resid && q_hi >= 1;
#pragma unroll
        for (int nt = 0; nt < 12; ++nt) {
            const int col = nt * 8 + 2 * tq;
            if (r_lo) {
                float a = o[nt][0] * inv_lo, c = o[nt][1] * inv_lo;
                if (res_lo) {
                    const float2 qf = __half22float2(*reinterpret_cast<const __half2*>(r_lo + col));
                    a += qf.x; c += qf.y;
                }
                *reinterpret_cast<uint32_t*>(out + (int64_t(b) * nq + q_lo) * C + head * MV_HEAD_DIM + col) = pack_half2(a, c);
            }
            if (r_hi) {
                float a = o[nt][2] * inv_hi, c = o[nt][3] * inv_hi;
                if (res_hi) {
                    const float2 qf = __half22float2(*reinterpret_cast<const __half2*>(r_hi + col));
                    a += qf.x; c += qf.y;
                }
                *reinterpret_cast<uint32_t*>(out + (int64_t(b) * nq + q_hi) * C + head * MV_HEAD_DIM + col) = pack_half2(a, c);
            }
        }
    }
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int mvit_patch_u8(const uint8_t* frames, const R21DStarts& st, int m, int H, int W, int rh, int rw, int cy, int cx,
                  __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * MV_TOKENS * 10;
    patch_kernel<true><<<nb(total, 256), 256, 0, s>>>(frames, st, m, H, W, rh, rw, cy, cx, out);
    LAUNCH_CHECK();
}

int mvit_patch_f32(const float* clips, int m, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * MV_TOKENS * 10;
    R21DStarts st;
    st.first[0] = 0;
    patch_kernel<false><<<nb(total, 256), 256, 0, s>>>(clips, st, m, 0, 0, 0, 0, 0, 0, out);
    LAUNCH_CHECK();
}

int mvit_embed(const float* emb, const float* class_token, const float* class_pos, const float* temporal_pos,
               const float* spatial_pos, int m, float* x, float* x2, cudaStream_t s) {
    const int64_t total = int64_t(m) * (1 + MV_TOKENS) * 96;
    embed_kernel<<<nb(total, 256), 256, 0, s>>>(emb, class_token, class_pos, temporal_pos, spatial_pos, m, x, x2);
    LAUNCH_CHECK();
}

int mvit_head_pool(const __half* src, int ld_src, int n, int heads, int T, int H, int W, int stride,
                   const float* weight, const float* gamma, const float* beta, __half* dst, cudaStream_t s) {
    if (n < 1 || heads < 1 || T < 1 || H < 1 || W < 1 || stride < 1 || ld_src < heads * MV_HEAD_DIM || ld_src % 2)
        return fail(VF_ERR_INVALID, "mvit_head_pool: %d clips of %dx%dx%d, %d heads, stride %d, pitch %d", n, T, H, W,
                    heads, stride, ld_src);
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
    const int64_t jobs = int64_t(n) * (1 + int64_t(T) * Ho * Wo) * heads;
    head_pool_kernel<<<nb(jobs, 8), 256, 0, s>>>(src, ld_src, n, heads, T, H, W, stride, weight, gamma, beta, dst);
    LAUNCH_CHECK();
}

int mvit_skip_pool(const float* x, int n, int C, int T, int H, int W, float* y, cudaStream_t s) {
    if (n < 1 || C < 1 || T < 1 || H < 1 || W < 1)
        return fail(VF_ERR_INVALID, "mvit_skip_pool: %d clips of %dx%dx%d x %d", n, T, H, W, C);
    const int64_t total = int64_t(n) * (1 + int64_t(T) * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1)) * C;
    skip_pool_kernel<<<nb(total, 256), 256, 0, s>>>(x, n, C, T, H, W, y);
    LAUNCH_CHECK();
}

int mvit_attention(const __half* q, const __half* k, const __half* v, const float* rel_h, const float* rel_w,
                   const float* rel_t, __half* out, const MViTAttnGeom& g, cudaStream_t s) {
    const int64_t nq = 1 + int64_t(g.q_thw[0]) * g.q_thw[1] * g.q_thw[2];
    bool ok = g.n >= 1 && g.heads >= 1 && g.heads <= 65535 && g.ldq >= g.heads * MV_HEAD_DIM && g.ldq % 8 == 0 &&
              nq < (int64_t(1) << 30);
    for (int i = 0; i < 3; ++i) ok = ok && g.q_thw[i] >= 1 && g.k_thw[i] >= 1 && g.k_thw[i] < 256;
    ok = ok && g.k_thw[0] + g.k_thw[1] + g.k_thw[2] <= MV_MAX_REL;
    if (!ok || (g.rel && (!rel_h || !rel_w || !rel_t)))
        return fail(VF_ERR_INVALID, "mvit_attention: %d clips, %d heads, q %dx%dx%d (pitch %d), kv %dx%dx%d", g.n,
                    g.heads, g.q_thw[0], g.q_thw[1], g.q_thw[2], g.ldq, g.k_thw[0], g.k_thw[1], g.k_thw[2]);
    RelArgs ra;
    ra.h = rel_h; ra.w = rel_w; ra.t = rel_t;
    for (int i = 0; i < 3; ++i) {
        const double Q = g.q_thw[i], K = g.k_thw[i];
        ra.qr[i] = float(K / Q > 1.0 ? K / Q : 1.0);
        ra.kr[i] = float(Q / K > 1.0 ? Q / K : 1.0);
    }
    static std::atomic<bool> attr_set[64];       // per device, as gemm_kernel.cuh's launch_gemm
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        VF_CUDA(cudaFuncSetAttribute(pool_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MA_SMEM));
        if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    // two 16-query tiles per warp when that still fills two waves of CTAs, else one
    const int64_t ntiles = (nq + 15) / 16;
    int64_t groups = (ntiles + 7) / 8;
    if ((groups / 2) * g.heads * g.n >= 2 * int64_t(device_sm_count())) groups = (ntiles + 15) / 16;
    const dim3 grid(unsigned(groups), unsigned(g.heads), unsigned(g.n));
    pool_attention_kernel<<<grid, 256, MA_SMEM, s>>>(q, k, v, ra, out, g);
    LAUNCH_CHECK();
}

}  // namespace vf
