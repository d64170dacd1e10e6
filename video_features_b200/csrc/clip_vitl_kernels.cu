// Memory-bound kernels and the key-streaming attention of the CLIP ViT-L/14 towers (clip_vitl.cu): patch-14 transform,
// LayerNorm over rows of 1024, and self-attention for 257 / 577-token frames whose shared memory does not grow with
// the token count.
#include "clip_vitl_kernels.h"
#include "common.cuh"

namespace vf {

namespace {

// clip.clip._transform Normalize constants, float32-rounded like torch does
__constant__ float kVitlMean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float kVitlStd[3] = {0.26862954f, 0.26130258f, 0.27577711f};

inline unsigned nblocks(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// One thread: 8 consecutive columns of one patch row (74 groups cover the 592 columns).  Column col < 588 is
// channel col / 196, kernel row (col % 196) / 14, kernel column col % 14 -- the flattening of conv1.weight[1024, 3, 14, 14].
// ToTensor (v / 255) then Normalize ((x - mean) / std) as IEEE fp32 ops in torchvision's order, then fp16.
template <bool U8>
__global__ void patchify14_kernel(const void* __restrict__ src, int n, int src_h, int src_w, int cy, int cx, int npx,
                                  __half* __restrict__ out) {
    constexpr int GROUPS = VITL_PK / 8;
    const int G = npx / VITL_PATCH;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * G * G * GROUPS) return;
    const int grp = int(idx % GROUPS);
    const int64_t row = idx / GROUPS;
    const int p = int(row % (G * G)), b = int(row / (G * G));
    const int py = p / G, px = p % G;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int col = grp * 8 + i;
        v[i] = 0.f;
        if (col < 3 * VITL_PATCH * VITL_PATCH) {
            const int c = col / 196, r = col % 196;
            const int y = py * VITL_PATCH + r / VITL_PATCH, x = px * VITL_PATCH + r % VITL_PATCH;
            if (U8) {
                const uint8_t u = __ldg(static_cast<const uint8_t*>(src) + ((int64_t(b) * src_h + cy + y) * src_w + cx + x) * 3 + c);
                v[i] = __fdiv_rn(__fsub_rn(__fdiv_rn(float(u), 255.0f), kVitlMean[c]), kVitlStd[c]);
            } else {
                v[i] = __ldg(static_cast<const float*>(src) + ((int64_t(b) * 3 + c) * npx + y) * npx + x);
            }
        }
    }
    *reinterpret_cast<uint4*>(out + row * VITL_PK + grp * 8) =
        make_uint4(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7]));
}

// LayerNorm over rows of 1024 fp32 (eps 1e-5, biased variance): one warp per row held in registers (8 float4 per lane),
// two-pass mean / variance by warp shuffles -- the semantics of the 768-wide kernels in kernels.cu.
struct Row1024 {
    float4 v[8];
};
__device__ __forceinline__ void ln1024_write(const Row1024& r, int lane, const float* __restrict__ gamma,
                                             const float* __restrict__ beta, void* out_row, bool out_f32) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += (r.v[i].x + r.v[i].y) + (r.v[i].z + r.v[i].w);
    const float mean = warp_sum(s) * (1.0f / 1024.0f);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float a = r.v[i].x - mean, b = r.v[i].y - mean, c = r.v[i].z - mean, d = r.v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / 1024.0f) + 1e-5f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int col = (lane + 32 * i) * 4;
        const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + col));
        const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + col));
        float4 y;
        y.x = (r.v[i].x - mean) * rstd * g.x + bb.x;
        y.y = (r.v[i].y - mean) * rstd * g.y + bb.y;
        y.z = (r.v[i].z - mean) * rstd * g.z + bb.z;
        y.w = (r.v[i].w - mean) * rstd * g.w + bb.w;
        if (out_f32) *reinterpret_cast<float4*>(reinterpret_cast<float*>(out_row) + col) = y;
        else *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out_row) + col) =
                 make_uint2(pack_half2(y.x, y.y), pack_half2(y.z, y.w));
    }
}

__global__ void __launch_bounds__(256) layernorm1024_kernel(const float* __restrict__ x, int64_t x_stride,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            __half* __restrict__ out, int64_t out_stride, int rows) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= rows) return;
    const float* xr = x + int64_t(row) * x_stride;
    Row1024 r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = *reinterpret_cast<const float4*>(xr + (lane + 32 * i) * 4);
    ln1024_write(r, lane, gamma, beta, out + int64_t(row) * out_stride, false);
}

__global__ void __launch_bounds__(256) embed_layernorm1024_kernel(const float* __restrict__ emb, const float* __restrict__ pos,
                                                                  const float* __restrict__ cls_pos0,
                                                                  const float* __restrict__ gamma,
                                                                  const float* __restrict__ beta, float* __restrict__ x,
                                                                  int rows, int tokens) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + warp;
    if (row >= rows) return;
    const int frame = row / tokens, t = row - frame * tokens;
    Row1024 r;
    if (t == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) r.v[i] = __ldg(reinterpret_cast<const float4*>(cls_pos0 + (lane + 32 * i) * 4));
    } else {
        const float* er = emb + (int64_t(frame) * (tokens - 1) + (t - 1)) * VITL_W;
        const float* pr = pos + int64_t(t) * VITL_W;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(er + (lane + 32 * i) * 4));
            const float4 p = __ldg(reinterpret_cast<const float4*>(pr + (lane + 32 * i) * 4));
            r.v[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
        }
    }
    ln1024_write(r, lane, gamma, beta, x + int64_t(row) * VITL_W, true);
}

// ---- key-streaming attention
// A CTA of 4 warps owns 64 query rows (4 tiles of 16, one per warp) of one (frame, head).  The head's keys and values
// arrive in blocks of 64 rows through a two-stage cp.async ring, so shared memory is 9 KB of Q plus 2 x 2 x 9 KB of K/V
// (45 KB) whatever the token count; with the registers three CTAs fit an SM.  Per block a warp computes its 16 x 64 scores with mma.sync
// m16n8k16 (fragments by ldmatrix, row pitch 144 B), folds them into an fp32 running max and sum (online softmax),
// rounds P = exp(s - running max) to fp16 and adds P.V into fp32 accumulators rescaled by exp(old max - new max).
// The 1 / sum factor is applied to the fp32 output, which is then rounded to fp16.  Keys at or past S score -inf and
// their V rows are zero; query rows past S are zero (finite scores) and are not stored.
constexpr int AL_LD = 72, AL_KB = 64, AL_QROWS = 64;

__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t* r, const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}

__global__ void __launch_bounds__(128, 3) vitl_attention_kernel(const __half* __restrict__ qkv, __half* __restrict__ out,
                                                                int heads, int S) {
    __shared__ __align__(16) __half Qs[AL_QROWS][AL_LD];      // [query][dim]; each warp's 16 rows are reused for its O
    __shared__ __align__(16) __half Ks[2][AL_KB][AL_LD];      // [stage][key][dim]
    __shared__ __align__(16) __half Vs[2][AL_KB][AL_LD];
    const int frame = blockIdx.x / heads, head = blockIdx.x % heads;
    const int qbase = blockIdx.y * AL_QROWS;
    const int width = heads * 64, ld = 3 * width;
    const int64_t row0 = int64_t(frame) * S;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const uint4 zero = make_uint4(0, 0, 0, 0);

    for (int i = tid; i < AL_QROWS * 8; i += 128) {
        const int r = i >> 3, seg = i & 7, q = qbase + r;
        if (q < S) cp_async16(&Qs[r][seg * 8], qkv + (row0 + q) * ld + head * 64 + seg * 8);
        else *reinterpret_cast<uint4*>(&Qs[r][seg * 8]) = zero;
    }
    auto load_kv = [&](int blk, int buf) {
        for (int i = tid; i < 2 * AL_KB * 8; i += 128) {
            const int m = i / (AL_KB * 8), rem = i % (AL_KB * 8);
            const int r = rem >> 3, seg = rem & 7, key = blk * AL_KB + r;
            __half* dst = m == 0 ? &Ks[buf][r][seg * 8] : &Vs[buf][r][seg * 8];
            if (key < S) cp_async16(dst, qkv + (row0 + key) * ld + (m + 1) * width + head * 64 + seg * 8);
            else *reinterpret_cast<uint4*>(dst) = zero;
        }
    };
    const int nblk = (S + AL_KB - 1) / AL_KB;
    load_kv(0, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");

    const int q0 = warp * 16;
    const bool active = qbase + q0 < S;
    const float sc = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) * log2(e)
    uint32_t aq[4][4];
    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;

    for (int b = 0; b < nblk; ++b) {
        if (b + 1 < nblk) {
            load_kv(b + 1, (b + 1) & 1);
            asm volatile("cp.async.commit_group;\ncp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        if (active) {
            const __half (*K)[AL_LD] = Ks[b & 1];
            const __half (*V)[AL_LD] = Vs[b & 1];
            if (b == 0) {
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) ldsm_x4(aq[ks], &Qs[q0 + (lane & 15)][ks * 16 + (lane >> 4) * 8]);
            }
            float s[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
                for (int kp = 0; kp < 2; ++kp) {
                    uint32_t bk[4];
                    ldsm_x4(bk, &K[nt * 8 + (lane & 7)][kp * 32 + (lane >> 3) * 8]);
                    mma16816(s[nt], aq[2 * kp], bk[0], bk[1]);
                    mma16816(s[nt], aq[2 * kp + 1], bk[2], bk[3]);
                }
            }
            float n_lo = m_lo, n_hi = m_hi;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const bool valid = b * AL_KB + nt * 8 + 2 * t + j < S;
                    s[nt][j] = valid ? s[nt][j] * sc : -INFINITY;
                    s[nt][2 + j] = valid ? s[nt][2 + j] * sc : -INFINITY;
                    n_lo = fmaxf(n_lo, s[nt][j]);
                    n_hi = fmaxf(n_hi, s[nt][2 + j]);
                }
            }
            n_lo = fmaxf(n_lo, __shfl_xor_sync(0xffffffffu, n_lo, 1));
            n_lo = fmaxf(n_lo, __shfl_xor_sync(0xffffffffu, n_lo, 2));
            n_hi = fmaxf(n_hi, __shfl_xor_sync(0xffffffffu, n_hi, 1));
            n_hi = fmaxf(n_hi, __shfl_xor_sync(0xffffffffu, n_hi, 2));
            // rescale what was accumulated under the old maximum (exp2f(-inf) == 0 on the first block)
            const float r_lo = exp2f(m_lo - n_lo), r_hi = exp2f(m_hi - n_hi);
            m_lo = n_lo; m_hi = n_hi;
            l_lo *= r_lo; l_hi *= r_hi;
#pragma unroll
            for (int i = 0; i < 8; ++i) { o[i][0] *= r_lo; o[i][1] *= r_lo; o[i][2] *= r_hi; o[i][3] *= r_hi; }
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
                for (int np = 0; np < 4; ++np) {
                    uint32_t bv[4];
                    ldsm_x4_trans(bv, &V[kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][np * 16 + (lane >> 4) * 8]);
                    mma16816(o[2 * np], pa, bv[0], bv[1]);
                    mma16816(o[2 * np + 1], pa, bv[2], bv[3]);
                }
            }
        }
        __syncthreads();        // every warp is done with stage b & 1 before block b + 2 is loaded into it
    }
    if (!active) return;
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
#pragma unroll
    for (int np = 0; np < 4; ++np) {       // this warp's own Q rows (read into aq at block 0) stage its O rows
        *reinterpret_cast<uint32_t*>(&Qs[q0 + g][np * 16 + 2 * t]) = pack_half2(o[2 * np][0] * inv_lo, o[2 * np][1] * inv_lo);
        *reinterpret_cast<uint32_t*>(&Qs[q0 + g + 8][np * 16 + 2 * t]) = pack_half2(o[2 * np][2] * inv_hi, o[2 * np][3] * inv_hi);
        *reinterpret_cast<uint32_t*>(&Qs[q0 + g][np * 16 + 8 + 2 * t]) = pack_half2(o[2 * np + 1][0] * inv_lo, o[2 * np + 1][1] * inv_lo);
        *reinterpret_cast<uint32_t*>(&Qs[q0 + g + 8][np * 16 + 8 + 2 * t]) = pack_half2(o[2 * np + 1][2] * inv_hi, o[2 * np + 1][3] * inv_hi);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) {          // 16 rows of 128 B as 16-byte stores, 8 lanes per row
        const int r = q0 + i * 4 + (lane >> 3), seg = lane & 7, q = qbase + r;
        if (q < S)
            *reinterpret_cast<uint4*>(out + (row0 + q) * width + head * 64 + seg * 8) = *reinterpret_cast<const uint4*>(&Qs[r][seg * 8]);
    }
}

}  // namespace

int vitl_patchify_u8(const uint8_t* src, int n, int src_h, int src_w, int cy, int cx, int npx, __half* patches,
                     cudaStream_t s) {
    const int G = npx / VITL_PATCH;
    const int64_t total = int64_t(n) * G * G * (VITL_PK / 8);
    patchify14_kernel<true><<<nblocks(total, 256), 256, 0, s>>>(src, n, src_h, src_w, cy, cx, npx, patches);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int vitl_patchify_f32(const float* src, int n, int npx, __half* patches, cudaStream_t s) {
    const int G = npx / VITL_PATCH;
    const int64_t total = int64_t(n) * G * G * (VITL_PK / 8);
    patchify14_kernel<false><<<nblocks(total, 256), 256, 0, s>>>(src, n, npx, npx, 0, 0, npx, patches);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int vitl_embed_layernorm(const float* emb, const float* pos, const float* cls_pos0, const float* gamma, const float* beta,
                         float* x, int n_frames, int tokens, cudaStream_t s) {
    const int rows = n_frames * tokens;
    embed_layernorm1024_kernel<<<nblocks(rows, 8), 256, 0, s>>>(emb, pos, cls_pos0, gamma, beta, x, rows, tokens);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int vitl_layernorm(const float* x, int64_t x_stride, const float* gamma, const float* beta, __half* out,
                   int64_t out_stride, int rows, cudaStream_t s) {
    layernorm1024_kernel<<<nblocks(rows, 8), 256, 0, s>>>(x, x_stride, gamma, beta, out, out_stride, rows);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int vitl_attention(const __half* qkv, __half* out, int n_frames, int S, int heads, cudaStream_t s) {
    if (S < 1 || S > VITL_MAX_S || n_frames < 1 || heads < 1)
        return fail(VF_ERR_INVALID, "vitl_attention: %d frames x %d tokens x %d heads (1 .. %d tokens)", n_frames, S,
                    heads, VITL_MAX_S);
    const dim3 grid(unsigned(n_frames) * unsigned(heads), unsigned((S + AL_QROWS - 1) / AL_QROWS));
    vitl_attention_kernel<<<grid, 128, 0, s>>>(qkv, out, heads, S);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // namespace vf
