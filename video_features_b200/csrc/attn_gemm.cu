// QKV projection fused with the 50-token self-attention of the ViT blocks, for sm_90a.
//
//   att[frame, token, head*64 .. +64] = softmax(q k^T / 8) v      with  [q | k | v] = h . W_qkv^T + b   (per head)
//
// Replaces, per block, the QKV GEMM + `attention50_kernel` pair (reference: third-party clip `ResidualAttentionBlock
// .attention` = nn.MultiheadAttention, called from models/CLIP/extract_clip.py:128).  Why fuse: the QKV GEMM would write
// 3 x 768 columns only for the attention kernel to read them back and emit 768: here q, k, v never leave the SM -- the
// epilogue stages them in shared memory, runs the attention of the tile's frames on mma.sync and writes the 768-wide
// result.
//
// Tiling: the weight rows are permuted so that the 192 rows [q_h | k_h | v_h] of head h are contiguous; an output tile
// is (2 frames = 100 token rows) x (one head = 192 columns), computed as a 128-row wgmma tile (the 28 rows behind the
// two frames belong to the next tile: they are computed and ignored).  Three warpgroups per CTA:
//   warpgroup 0      TMA producer (one lane), a ring of STAGES stages; it runs ahead into the next tile
//   warpgroups 1, 2  rows 0..63 / 64..127: wgmma m64n192k16 main loop, then accumulator + bias -> fp16 -> staging
//                    rows; after a named barrier each of the 8 warps runs one attention unit (16 queries of one frame:
//                    S = Q K^T on mma.sync m16n8k16, softmax in the accumulator fragments (fp32), O = P V) and stores its
//                    rows with 16-byte global stores.
// Numerics are those of attention50_kernel (fp16 q / k / v / P, fp32 scores and accumulation).
#include <string.h>

#include <atomic>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace vf {

namespace {

constexpr int BM = 128, BK = 64, BN = 192, STAGES = 4;
constexpr int FRAMES_PER_TILE = 2, TOK = 50, TILE_ROWS = FRAMES_PER_TILE * TOK;   // 100
constexpr int THREADS = 384, CONSUMER_THREADS = 256, CONSUMER_WARPS = 8;
constexpr uint32_t A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int PITCH = 200;                        // halfs per staging row: 192 + 8 (16-byte shift per row: conflict-free ldmatrix)
constexpr uint32_t STG_BYTES = BM * PITCH * 2;
constexpr uint32_t ZERO_BYTES = 128;
constexpr uint32_t BAR_BYTES = 2 * STAGES * 8;
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + STG_BYTES + ZERO_BYTES + BAR_BYTES + 1024;
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");

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
// one attention unit: 16 query rows (staging rows qrow0..qrow0+15) against the 50 keys at staging rows krow0..krow0+49
// S: [row][q 0..63 | k 64..127 | v 128..191] fp16.  The result replaces the q columns of the unit's first `nvalid` rows (the
// rows behind them belong to the next frame: they are read, their results discarded, and they are never written).
// `zero`: 128 bytes of zeros: key / value rows past the frame's 50 tokens are read from there (their scores are masked and
// their probabilities 0, but 0 x an arbitrary bit pattern must stay 0).
__device__ __forceinline__ void attention_unit(__half* S, const __half* zero, int qrow0, int krow0, int nvalid, int lane) {
    const int g = lane >> 2, t = lane & 3;
    uint32_t aq[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) ldsm_x4(aq[ks], S + (qrow0 + (lane & 15)) * PITCH + ks * 16 + (lane >> 4) * 8);
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 7; ++nt) {           // 7 key tiles of 8 cover the 50 keys
        s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {
            uint32_t bk[4];
            const int kr = nt * 8 + (lane & 7);
            ldsm_x4(bk, kr < TOK ? S + (krow0 + kr) * PITCH + 64 + kp * 32 + (lane >> 3) * 8 : zero);
            mma16816(s[nt], aq[2 * kp], bk[0], bk[1]);
            mma16816(s[nt], aq[2 * kp + 1], bk[2], bk[3]);
        }
    }
    const float sc = 0.125f * 1.4426950408889634f;   // 1/sqrt(64) * log2(e)
    float m_lo = -INFINITY, m_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 7; ++nt) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const bool valid = nt * 8 + 2 * t + j < TOK;
            s[nt][j] = valid ? s[nt][j] * sc : -INFINITY;
            s[nt][2 + j] = valid ? s[nt][2 + j] * sc : -INFINITY;
            m_lo = fmaxf(m_lo, s[nt][j]);
            m_hi = fmaxf(m_hi, s[nt][2 + j]);
        }
    }
    m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 1));
    m_lo = fmaxf(m_lo, __shfl_xor_sync(0xffffffffu, m_lo, 2));
    m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 1));
    m_hi = fmaxf(m_hi, __shfl_xor_sync(0xffffffffu, m_hi, 2));
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int nt = 0; nt < 7; ++nt) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            s[nt][j] = exp2f(s[nt][j] - m_lo);          // exp2f(-inf) == 0 for the keys past 50
            s[nt][2 + j] = exp2f(s[nt][2 + j] - m_hi);
            sum_lo += s[nt][j];
            sum_hi += s[nt][2 + j];
        }
    }
    s[7][0] = s[7][1] = s[7][2] = s[7][3] = 0.f;        // keys 56..63 of the last 16-key step: probability 0
    sum_lo += __shfl_xor_sync(0xffffffffu, sum_lo, 1);
    sum_lo += __shfl_xor_sync(0xffffffffu, sum_lo, 2);
    sum_hi += __shfl_xor_sync(0xffffffffu, sum_hi, 1);
    sum_hi += __shfl_xor_sync(0xffffffffu, sum_hi, 2);
    const float inv_lo = 1.0f / sum_lo, inv_hi = 1.0f / sum_hi;
    uint32_t pa[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        pa[kk][0] = pack_half2(s[2 * kk][0] * inv_lo, s[2 * kk][1] * inv_lo);
        pa[kk][1] = pack_half2(s[2 * kk][2] * inv_hi, s[2 * kk][3] * inv_hi);
        pa[kk][2] = pack_half2(s[2 * kk + 1][0] * inv_lo, s[2 * kk + 1][1] * inv_lo);
        pa[kk][3] = pack_half2(s[2 * kk + 1][2] * inv_hi, s[2 * kk + 1][3] * inv_hi);
    }
    __syncwarp();   // every lane's ldmatrix reads of the q rows are done before they are overwritten with O
#pragma unroll
    for (int np = 0; np < 4; ++np) {        // two dim tiles per ldmatrix.x4.trans
        float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {     // keys 50..63 carry probability 0; their v rows hold finite values (see header)
            uint32_t bv[4];
            const int vr = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
            ldsm_x4_trans(bv, vr < TOK ? S + (krow0 + vr) * PITCH + 128 + np * 16 + (lane >> 4) * 8 : zero);
            mma16816(o0, pa[kk], bv[0], bv[1]);
            mma16816(o1, pa[kk], bv[2], bv[3]);
        }
        if (g < nvalid) {
            *reinterpret_cast<uint32_t*>(S + (qrow0 + g) * PITCH + np * 16 + 2 * t) = pack_half2(o0[0], o0[1]);
            *reinterpret_cast<uint32_t*>(S + (qrow0 + g) * PITCH + np * 16 + 8 + 2 * t) = pack_half2(o1[0], o1[1]);
        }
        if (g + 8 < nvalid) {
            *reinterpret_cast<uint32_t*>(S + (qrow0 + g + 8) * PITCH + np * 16 + 2 * t) = pack_half2(o0[2], o0[3]);
            *reinterpret_cast<uint32_t*>(S + (qrow0 + g + 8) * PITCH + np * 16 + 8 + 2 * t) = pack_half2(o1[2], o1[3]);
        }
    }
    __syncwarp();
}

__global__ void __launch_bounds__(THREADS, 1)
qkv_attention_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const float* __restrict__ bias, __half* __restrict__ att, const int n_frames, const int heads) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;
    __half* S = reinterpret_cast<__half*>(smem + STAGES * STAGE_BYTES);        // staging rows [128][PITCH]
    __half* zero = reinterpret_cast<__half*>(smem + STAGES * STAGE_BYTES + STG_BYTES);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + STG_BYTES + ZERO_BYTES);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_m = (n_frames + FRAMES_PER_TILE - 1) / FRAMES_PER_TILE;
    const int num_tiles = num_m * heads;
    const int width = heads * 64;
    constexpr int num_k = 768 / BK;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], CONSUMER_WARPS);
        }
        fence_mbar_init();
    }
    if (threadIdx.x < ZERO_BYTES / 16) reinterpret_cast<uint4*>(zero)[threadIdx.x] = make_uint4(0, 0, 0, 0);
    __syncthreads();

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int m0 = (tile % num_m) * TILE_ROWS;      // rows past the matrix are zero-filled by TMA
                const int n0 = (tile / num_m) * BN;
                for (int kk = 0; kk < num_k; ++kk) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], STAGE_BYTES);
                    tma_load_2d(sA + stage * A_BYTES, &tmA, &full[stage], kk * BK, m0);
                    tma_load_2d(sB + stage * B_BYTES, &tmB, &full[stage], kk * BK, n0);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    const int wg = (warp >> 2) - 1, wq = warp & 3;
    const int e = warp - 4;                              // attention unit 0..7: frame e / 4, queries 16 (e % 4) ..
    const int f = e >> 2, tok0 = (e & 3) * 16;
    const int krow0 = TOK * f, qrow0 = krow0 + tok0;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile % num_m, head = tile / num_m;
        int prev = -1;
        for (int kb = 0; kb < num_k; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint64_t adesc = wgmma_desc_sw128(sA + stage * A_BYTES + wg * (64 * 128));
            const uint64_t bdesc = wgmma_desc_sw128(sB + stage * B_BYTES);
            wgmma_fence_regs<BN / 2>(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) Wgmma<BN>::mma(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();
            wgmma_fence_regs<BN / 2>(acc);
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs<BN / 2>(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);

        // every unit is done with the previous tile's staging rows before they are overwritten
        named_bar_sync(1, CONSUMER_THREADS);
        // accumulator register 4j + 2h + c: row (lane / 4) + 8h of this warp's 16, column 8j + 2 (lane % 4) + c
        const float* hb = bias + head * BN;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            const float2 b = __ldg(reinterpret_cast<const float2*>(hb + c));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
                *reinterpret_cast<uint32_t*>(S + r * PITCH + c) = pack_half2(acc[4 * j + 2 * h] + b.x, acc[4 * j + 2 * h + 1] + b.y);
            }
        }
        named_bar_sync(1, CONSUMER_THREADS);
        attention_unit(S, zero, qrow0, krow0, tok0 + 16 <= TOK ? 16 : TOK - tok0, lane);
        const int frame = m_blk * FRAMES_PER_TILE + f;
        if (frame < n_frames) {
            __half* orow = att + (int64_t(frame) * TOK) * width + head * 64;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = i * 4 + (lane >> 3), seg = lane & 7;
                const int tok = tok0 + r;
                if (tok < TOK)
                    *reinterpret_cast<uint4*>(orow + int64_t(tok) * width + seg * 8) =
                        *reinterpret_cast<const uint4*>(S + (qrow0 + r) * PITCH + seg * 8);
            }
        }
    }
}

}  // namespace

// h: [n_frames*50, 768] fp16 (row pitch lda); w_perm: [heads*192, 768] fp16, row h*192 + part*64 + d = in_proj row
// part*768 + h*64 + d; bias_perm likewise (fp32); att: [n_frames*50, heads*64] fp16
int qkv_attention(const __half* h, int lda, const __half* w_perm, const float* bias_perm, __half* att, int n_frames, int heads,
                  cudaStream_t stream) {
    if (n_frames <= 0) return VF_OK;
    if (heads * 64 != 768) return fail(VF_ERR_UNSUPPORTED, "qkv_attention: built for width 768 (heads * 64)");
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        VF_CUDA(cudaFuncSetAttribute(qkv_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    const int M = n_frames * TOK;
    CUtensorMap tmA, tmB;
    VF_TRY(make_tmap_2d(&tmA, h, 2, uint64_t(M), 768, uint64_t(lda) * 2, BM, BK));
    VF_TRY(make_tmap_2d(&tmB, w_perm, 2, uint64_t(heads) * BN, 768, 768 * 2, BN, BK));
    const int tiles = ((n_frames + FRAMES_PER_TILE - 1) / FRAMES_PER_TILE) * heads;
    const int sms = device_sm_count();
    const int grid = tiles < sms ? tiles : sms;
    qkv_attention_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(tmA, tmB, bias_perm, att, n_frames, heads);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // namespace vf
