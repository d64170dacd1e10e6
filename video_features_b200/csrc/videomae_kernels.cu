// Kernels of the VideoMAE towers (videomae.cu): the tubelet transform, the positional add, the clip mean and the
// attention over the 1568 tokens of a clip on wgmma.
#include "common.cuh"
#include "videomae_kernels.h"
#include "wgmma.cuh"

namespace vf {

namespace {

inline unsigned nblocks(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

// One thread: 8 consecutive columns (8 pixels of one patch row) of one tubelet row; 192 groups cover the 1536 columns.
template <bool U8>
__global__ void tubelet_kernel(const void* __restrict__ src, R21DStarts st, int m, int H, int W, int cy, int cx,
                               VmNorm nm, __half* __restrict__ out) {
    constexpr int GROUPS = VM_PK / 8, G = VM_CROP / VM_PATCH;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(m) * VM_TOKENS * GROUPS) return;
    const int grp = int(idx % GROUPS);
    const int64_t row = idx / GROUPS;
    const int p = int(row % VM_TOKENS), b = int(row / VM_TOKENS);
    const int tt = p / (G * G), y = (p / G) % G, x = p % G;
    const int col0 = grp * 8;
    const int c = col0 / 512, dt = (col0 / 256) & 1, py = (col0 / 16) & 15, px0 = col0 & 15;
    const int t = tt * VM_TUBE + dt, Y = y * VM_PATCH + py, X0 = x * VM_PATCH + px0;
    float v[8];
    if (U8) {
        const uint8_t* pix = static_cast<const uint8_t*>(src) +
                             ((int64_t(st.first[b] + t) * H + cy + Y) * W + cx + X0) * 3 + (2 - c);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            // rescale in float64 then fp32 (the processor's rescale), Normalize in fp32
            const float r = __double2float_rn(__dmul_rn(double(__ldg(pix + 3 * i)), 1.0 / 255.0));
            v[i] = __fdiv_rn(__fsub_rn(r, nm.mean[c]), nm.std[c]);
        }
    } else {
        const float* f = static_cast<const float*>(src) +
                         ((int64_t(b * VM_T + t) * 3 + c) * VM_CROP + Y) * VM_CROP + X0;
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = __ldg(f + i);
    }
    *reinterpret_cast<uint4*>(out + row * VM_PK + col0) =
        make_uint4(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7]));
}

__global__ void add_pos_kernel(float4* __restrict__ x, const float4* __restrict__ pos, int64_t total4, int D4) {
    const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total4) return;
    const int64_t row = i / D4;
    const float4 p = __ldg(pos + int64_t(row % VM_TOKENS) * D4 + i % D4);
    float4 v = x[i];
    v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
    x[i] = v;
}

// (clip, 64-column slab): 4 row phases of 64 columns each sum every 4th row in order; the phases are added in order
__global__ void __launch_bounds__(256) mean_kernel(const float* __restrict__ x, int D, float* __restrict__ pooled) {
    __shared__ float part[4][64];
    const int b = blockIdx.x, col = blockIdx.y * 64 + (threadIdx.x & 63), ph = threadIdx.x >> 6;
    const float* xb = x + int64_t(b) * VM_TOKENS * D + col;
    float s = 0.f;
    for (int r = ph; r < VM_TOKENS; r += 4) s += xb[int64_t(r) * D];
    part[ph][threadIdx.x & 63] = s;
    __syncthreads();
    if (ph == 0) {
        const int c = threadIdx.x;
        pooled[int64_t(b) * D + col] = (((part[0][c] + part[1][c]) + part[2][c]) + part[3][c]) / float(VM_TOKENS);
    }
}

// ---- attention
// A CTA of two warpgroups owns 128 query rows (64 per warpgroup) of one (clip, head).  Thread 0 loads the Q tiles once
// and the head's K / V in blocks of 64 keys by TMA (128-byte swizzled 64 x 64 tiles) into a 3-stage mbarrier ring; a
// stage is refilled once all 8 warps have released it.  Per block each warpgroup computes its 64 x 64 scores with
// wgmma (Q and K both K-major in shared memory), folds them into an fp32 running max and sum per row (exp2, online
// softmax), rounds P = exp(s - running max) to fp16 in registers and adds P.V with the register-A wgmma, V read
// MN-major (transposed B) from its [key][dim] tile; the fp32 output is rescaled by exp(old max - new max) before.  The
// output times the fp32 1 / sum is rounded to fp16 once and leaves through shared memory as 16-byte stores.
// The QKV rows are one 2-D tensor of n * S rows: keys at or past S score -inf (rows of the next clip, or TMA's zero
// fill past the last row, meet P = 0); query rows past S are computed and not stored.
constexpr int VA_KB = 64, VA_STAGES = 3, VA_TILE = 64 * 128;
constexpr size_t VA_SMEM = 1024 + size_t(2 + 2 * VA_STAGES) * VA_TILE + 128;

__global__ void __launch_bounds__(256, 2) attention_kernel(const __grid_constant__ CUtensorMap tm,
                                                           __half* __restrict__ out, int heads, int S) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* Qs = base;
    uint8_t* Ks = base + 2 * VA_TILE;
    uint8_t* Vs = Ks + VA_STAGES * VA_TILE;
    uint64_t* full = reinterpret_cast<uint64_t*>(Vs + VA_STAGES * VA_TILE);
    uint64_t* empty = full + VA_STAGES;
    uint64_t* qbar = empty + VA_STAGES;
    const int head = blockIdx.y, width = heads * 64;
    const int row0 = blockIdx.z * S, qbase = blockIdx.x * 128;
    const int tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int nblk = (S + VA_KB - 1) / VA_KB;

    auto load_kv = [&](int b, int st) {
        mbar_expect_tx(&full[st], 2 * VA_TILE);
        tma_load_2d(Ks + st * VA_TILE, &tm, &full[st], width + head * 64, row0 + b * VA_KB);
        tma_load_2d(Vs + st * VA_TILE, &tm, &full[st], 2 * width + head * 64, row0 + b * VA_KB);
    };
    if (tid == 0) {
        for (int i = 0; i < VA_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
        mbar_init(qbar, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0) {
        tma_prefetch_desc(&tm);
        mbar_expect_tx(qbar, 2 * VA_TILE);
        tma_load_2d(Qs, &tm, qbar, head * 64, row0 + qbase);
        tma_load_2d(Qs + VA_TILE, &tm, qbar, head * 64, row0 + qbase + 64);
        for (int b = 0; b < VA_STAGES && b < nblk; ++b) load_kv(b, b);
    }

    const uint64_t dq = wgmma_desc_sw128(Qs + wg * VA_TILE);
    const float sc = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) * log2(e)
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
    mbar_wait(qbar, 0);

    for (int b = 0; b < nblk; ++b) {
        const int st = b % VA_STAGES;
        const uint32_t ph = uint32_t(b / VA_STAGES) & 1u;
        mbar_wait(&full[st], ph);
        const uint64_t dk = wgmma_desc_sw128(Ks + st * VA_TILE), dv = wgmma_desc_sw128(Vs + st * VA_TILE);
        float s[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) Wgmma<64>::mma(s, dq + 2 * ks, dk + 2 * ks, ks > 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<32>(s);

        float n_lo = m_lo, n_hi = m_hi;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const bool valid = b * VA_KB + 8 * j + 2 * t + e < S;
                s[4 * j + e] = valid ? s[4 * j + e] * sc : -INFINITY;
                s[4 * j + 2 + e] = valid ? s[4 * j + 2 + e] * sc : -INFINITY;
                n_lo = fmaxf(n_lo, s[4 * j + e]);
                n_hi = fmaxf(n_hi, s[4 * j + 2 + e]);
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
        for (int j = 0; j < 8; ++j) { o[4 * j] *= r_lo; o[4 * j + 1] *= r_lo; o[4 * j + 2] *= r_hi; o[4 * j + 3] *= r_hi; }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                s[4 * j + e] = exp2f(s[4 * j + e] - m_lo);
                s[4 * j + 2 + e] = exp2f(s[4 * j + 2 + e] - m_hi);
                l_lo += s[4 * j + e];
                l_hi += s[4 * j + 2 + e];
            }
        }
        // P as the A fragments of 16 keys each: the score accumulator's n8 chunks 2kk and 2kk + 1
        uint32_t pa[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            pa[kk][0] = pack_half2(s[8 * kk + 0], s[8 * kk + 1]);
            pa[kk][1] = pack_half2(s[8 * kk + 2], s[8 * kk + 3]);
            pa[kk][2] = pack_half2(s[8 * kk + 4], s[8 * kk + 5]);
            pa[kk][3] = pack_half2(s[8 * kk + 6], s[8 * kk + 7]);
        }
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) WgmmaRegAT<64>::mma(o, pa[kk], dv + kk * ((16 * 128) >> 4), 1);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<32>(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);
        if (tid == 0 && b + VA_STAGES < nblk) {
            mbar_wait(&empty[st], ph);
            load_kv(b + VA_STAGES, st);
        }
        __syncwarp();
    }

    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = 1.0f / l_lo, inv_hi = 1.0f / l_hi;
    // this warpgroup's Q tile (no longer read) stages its 64 output rows, [row][64] with 16-byte segments XOR-swizzled
    __half* O = reinterpret_cast<__half*>(Qs + wg * VA_TILE);
    const int r_lo = (warp & 3) * 16 + g, r_hi = r_lo + 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        *reinterpret_cast<uint32_t*>(O + r_lo * 64 + ((j ^ (r_lo & 7)) * 8) + 2 * t) =
            pack_half2(o[4 * j] * inv_lo, o[4 * j + 1] * inv_lo);
        *reinterpret_cast<uint32_t*>(O + r_hi * 64 + ((j ^ (r_hi & 7)) * 8) + 2 * t) =
            pack_half2(o[4 * j + 2] * inv_hi, o[4 * j + 3] * inv_hi);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) {          // the warp's 16 rows of 128 B as 16-byte stores, 8 lanes per row
        const int r = (warp & 3) * 16 + i * 4 + (lane >> 3), seg = lane & 7, q = qbase + wg * 64 + r;
        if (q < S)
            *reinterpret_cast<uint4*>(out + (int64_t(row0) + q) * width + head * 64 + seg * 8) =
                *reinterpret_cast<const uint4*>(O + r * 64 + ((seg ^ (r & 7)) * 8));
    }
}

}  // namespace

int videomae_tubelets_u8(const uint8_t* frames, const R21DStarts& st, int m, int H, int W, int cy, int cx,
                         const VmNorm& nm, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * VM_TOKENS * (VM_PK / 8);
    tubelet_kernel<true><<<nblocks(total, 256), 256, 0, s>>>(frames, st, m, H, W, cy, cx, nm, out);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int videomae_tubelets_f32(const float* clips, int m, __half* out, cudaStream_t s) {
    const int64_t total = int64_t(m) * VM_TOKENS * (VM_PK / 8);
    tubelet_kernel<false><<<nblocks(total, 256), 256, 0, s>>>(clips, R21DStarts{}, m, VM_CROP, VM_CROP, 0, 0, VmNorm{},
                                                              out);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int videomae_add_pos(float* x, const float* pos, int m, int D, cudaStream_t s) {
    const int64_t total4 = int64_t(m) * VM_TOKENS * D / 4;
    add_pos_kernel<<<nblocks(total4, 256), 256, 0, s>>>(reinterpret_cast<float4*>(x),
                                                        reinterpret_cast<const float4*>(pos), total4, D / 4);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int videomae_mean(const float* x, int m, int D, float* pooled, cudaStream_t s) {
    if (D % 64) return fail(VF_ERR_INVALID, "videomae_mean: width %d is not a multiple of 64", D);
    mean_kernel<<<dim3(unsigned(m), unsigned(D / 64)), 256, 0, s>>>(x, D, pooled);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

int videomae_attention(const __half* qkv, __half* out, int n, int S, int heads, cudaStream_t s) {
    if (S < 1 || S > VM_MAX_S || n < 1 || heads < 1 || heads > 64 || int64_t(n) * S > INT32_MAX)
        return fail(VF_ERR_INVALID, "videomae_attention: %d clips x %d tokens x %d heads (1 .. %d tokens)", n, S, heads,
                    VM_MAX_S);
    CUtensorMap tm;
    VF_TRY(make_tmap_2d(&tm, qkv, 2, uint64_t(n) * S, uint64_t(3) * heads * 64, uint64_t(3) * heads * 64 * 2, 64, 64));
    VF_CUDA(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(VA_SMEM)));
    const dim3 grid(unsigned((S + 127) / 128), unsigned(heads), unsigned(n));
    attention_kernel<<<grid, 256, VA_SMEM, s>>>(tm, out, heads, S);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // namespace vf
