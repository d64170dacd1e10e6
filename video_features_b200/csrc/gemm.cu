// Persistent warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = act( A[M,K] . B[N,K]^T * scale[n] + bias[n] )     A, B fp16 K-major; fp32 accumulate in registers;
//                                                              D fp16 or fp32
//
// Tiles are 64 x BN, walked row-major (n fastest) and strided over a grid of at most one CTA per SM.  Three warpgroups
// in a "ping-pong" schedule:
//   warpgroup 0    TMA producer (one lane, 40 registers): A and B tiles of the CTA's tiles, in order, through a
//                  128B-swizzled ring of STAGES stages, one mbarrier pair (full / empty) per stage.
//   warpgroups 1,2 consumers (232 registers each), one whole tile at a time: warpgroup 1 the CTA's even tiles, 2 its odd
//                  ones.  Per 64-wide K block, four wgmma m64nBNk16 (eight with split weights), one commit group; the
//                  stage is released as soon as the group behind it has retired.  A named-barrier pair makes the two
//                  main loops take turns, so one warpgroup's epilogue runs while the other's MMAs keep the tensor cores
//                  busy.  Epilogue: scale / bias / activation and row mask in registers, then 64-row x 128-byte subtiles
//                  through two swizzled shared-memory buffers per warpgroup, each handed to a TMA store (TMA reduce-add
//                  for `accumulate`) that TMA clips at N and M.
// The shifted-row conv mode keeps the cooperative schedule instead (template parameter PP = false): 128 x BN tiles walked
// m-fastest, warpgroups 1 and 2 on rows 0..63 and 64..127 of the same tile, with the same main loop and epilogue.
//
// Used for every dense contraction of the hot path: ViT patch-embed / QKV / out-proj / FFN GEMMs (reference:
// third-party clip `VisionTransformer.forward`, called at models/CLIP/extract_clip.py:128) and the I3D / RAFT
// convolutions in the shifted-row mode below.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <vector>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace vf {

namespace {

constexpr int BK = 64;           // 64 fp16 = one 128-byte swizzle row
constexpr int THREADS = 384;     // producer warpgroup + two consumer warpgroups
// 40 x 128 + 232 x 256 <= 64 K registers; a CTA of 384 threads starts at 168 each
constexpr uint32_t PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int EPI_ROWS = 64;                   // output rows per consumer warpgroup = rows of one TMA store box
constexpr uint32_t STG_BYTES = EPI_ROWS * 128; // one staging subtile: 64 rows x 128 bytes (64 fp16 / 32 fp32 columns)
constexpr uint32_t STAGING_BYTES = 2 * 2 * STG_BYTES;   // two warpgroups x two buffers
constexpr uint32_t SMEM_LIMIT = 227 * 1024;    // opt-in dynamic shared memory per block on sm_90
constexpr uint32_t MAX_STAGES = 8;
// operand ring = what is left after the staging buffers, the barriers of MAX_STAGES stages and the alignment slack:
// 194 KB, i.e. stages (plain / split weights) 4 / 2 at BN = 256, 6 / 3 at 192, 8 / 4 at 128, 8 / 8 at 64.
constexpr uint32_t RING_BUDGET = SMEM_LIMIT - STAGING_BYTES - 2 * MAX_STAGES * 8 - 1024;

// NSPLIT = 2: the B stage holds the hi and the lo tile of a split-fp16 weight matrix and every K step issues two
// MMAs against the same A tile.
// PP: ping-pong schedule, 64-row tiles each owned by one consumer warpgroup (plain GEMMs); otherwise the cooperative
// schedule, 128-row tiles whose rows 0..63 / 64..127 the two warpgroups share (conv mode, see run_gemm).
template <int BN, int NSPLIT, bool PP>
struct GemmCfg {
    static constexpr int BM = PP ? 64 : 128;
    static constexpr uint32_t A_BYTES = BM * BK * 2;
    static constexpr uint32_t B_TILE = BN * BK * 2;           // one of hi / lo
    static constexpr uint32_t B_BYTES = NSPLIT * B_TILE;
    static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = RING_BUDGET / STAGE_BYTES > MAX_STAGES ? MAX_STAGES : int(RING_BUDGET / STAGE_BYTES);
    static constexpr uint32_t BAR_BYTES = 2 * STAGES * 8;
    // ring | staging | barriers, + align slack
    static constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + BAR_BYTES + 1024;
    static_assert(STAGES >= 2, "at least two pipeline stages");
    static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget");
    static_assert(A_BYTES % 1024 == 0 && B_TILE % 1024 == 0, "swizzle-128B tiles must stay 1024-byte aligned");
};

// Schedule by entry point, from measurements on an H100 (DESIGN.md 4.1): plain GEMMs (the CLIP tower, RAFT's
// correlation) run ping-pong; the conv mode (I3D, RAFT, ResNet, R(2+1)D) keeps the cooperative 128-row tile, whose
// weight tile serves twice the rows -- ping-pong made those networks 13-31 % slower.
constexpr int tile_rows(bool pp) { return pp ? GemmCfg<64, 1, true>::BM : GemmCfg<64, 1, false>::BM; }

__device__ __forceinline__ float apply_act(float v, int act) {
    if (act == VF_ACT_QUICKGELU) {
        return __fdividef(v, 1.0f + __expf(-1.702f * v));   // x * sigmoid(1.702 x)
    } else if (act == VF_ACT_RELU) {
        return fmaxf(v, 0.0f);
    } else if (act == VF_ACT_SIGMOID) {
        return __fdividef(1.0f, 1.0f + __expf(-v));
    } else if (act == VF_ACT_TANH) {
        return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * v));   // saturates cleanly to +-1
    }
    return v;
}

// SPLIT: split-fp16 output (GemmEpi::split_off) -- every fp16 pair is written twice, hi at column n (tmD) and lo at
// split_off + n (tmD2).  A compile-time switch keeps the plain epilogue free of it.
// tmD / tmD2: the output as dims (N, M), row pitch ldo, 64-row x 128-byte boxes; TMA clips every store at N and M.
template <int BN, int NSPLIT, bool SPLIT, bool PP>
__global__ void __launch_bounds__(THREADS, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmD2, const GemmEpi ep,
                const int M, const int N, const __grid_constant__ ConvGeom cg) {
    using Cfg = GemmCfg<BN, NSPLIT, PP>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int BM = Cfg::BM;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
    uint8_t* sD = smem + STAGES * Cfg::STAGE_BYTES;      // staging: [warpgroup][buffer] subtiles, 1024-byte aligned
    uint64_t* full = reinterpret_cast<uint64_t*>(sD + STAGING_BYTES);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_m = (M + BM - 1) / BM;
    const int num_n = (N + BN - 1) / BN;
    const int num_tiles = num_m * num_n;
    // ping-pong: row-major (the column tiles of one A row block run together); cooperative: m fastest
    auto tile_m0 = [&](int tile) { return (PP ? tile / num_n : tile % num_m) * BM; };
    auto tile_n0 = [&](int tile) { return (PP ? tile % num_n : tile / num_m) * BN; };
    // this CTA's tiles: blockIdx.x + i * gridDim.x for i < cta_tiles (the grid is at most num_tiles, so cta_tiles >= 1)
    const int cta_tiles = (num_tiles - 1 - int(blockIdx.x)) / int(gridDim.x) + 1;
    const int kpt = (cg.k_per_tap + BK - 1) / BK;    // K blocks per filter tap (a plain GEMM is one "tap")
    const int num_k = cg.ntaps * kpt;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        tma_prefetch_desc(&tmD);
        if (SPLIT) tma_prefetch_desc(&tmD2);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full[i], 1);                  // the producer's arrive.expect_tx
            mbar_init(&empty[i], PP ? 4 : 8);        // one arrive per consumer warp that reads the stage
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ------------------------------------------------------------ TMA producer
        setmaxnreg_dec<PRODUCER_REGS>();             // the whole warpgroup, before warps 1..3 leave
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int i = 0; i < cta_tiles; ++i) {
                const int tile = blockIdx.x + i * gridDim.x;
                const int m0 = tile_m0(tile), n0 = tile_n0(tile);
                for (int tap = 0; tap < cg.ntaps; ++tap) {
                    const int arow = m0 + cg.tap_off[tap];       // may be negative / past the end: TMA zero-fills
                    const int bcol = tap * cg.k_per_tap;
                    for (int kk = 0; kk < kpt; ++kk) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        const bool lo_blk = NSPLIT == 2 && ((cg.lo_mask >> kk) & 1ull);    // W_lo not needed
                        mbar_expect_tx(&full[stage], Cfg::A_BYTES + (lo_blk ? Cfg::B_TILE : Cfg::B_BYTES));
                        tma_load_2d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], kk * BK, arow);
                        tma_load_2d(sB + stage * Cfg::B_BYTES, &tmB, &full[stage], bcol + kk * BK, n0);
                        if (NSPLIT == 2 && !lo_blk)   // the lo half of the weights lives ntaps*k_per_tap columns to the right
                            tma_load_2d(sB + stage * Cfg::B_BYTES + Cfg::B_TILE, &tmB, &full[stage],
                                        cg.ntaps * cg.k_per_tap + bcol + kk * BK, n0);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = (warp >> 2) - 1;              // ping-pong: 0 the CTA's even tiles, 1 its odd ones; else rows 0 / 64
    const int wq = warp & 3;                     // warp inside the warpgroup: 16 rows each
    constexpr int R = BN / 2;                    // accumulator registers per thread
    float acc[R];
    // Staging: two buffers per warpgroup.  Row r of a subtile is 128 bytes at r * 128 with its 16-byte chunk c at
    // position c ^ (r % 8) (CU_TENSOR_MAP_SWIZZLE_128B).  A thread's rows are wq * 16 + lane / 4 + 8h, so r % 8 = lane / 4.
    // Thread 0 of the warpgroup issues the stores and waits for them.
    const bool issuer = (threadIdx.x & 127) == 0;
    uint32_t buf = 0;                            // plain output: subtiles alternate between the buffers, across tiles too
    auto wg_sync = [&] {                         // literal ids: ptxas counts only the barriers used
        if (wg == 0) named_bar_sync(1, 128);
        else named_bar_sync(2, 128);
    };
    // Hand the subtile just written to buffer `buf` to the TMA unit.  Before the barrier the issuer waits until the
    // store issued before it has read its buffer, so once the barrier is passed the other buffer may be refilled.
    auto store_subtile = [&](int col, int row) {
        fence_proxy_async();                     // this thread's shared-memory writes -> visible to the async proxy
        if (issuer) bulk_wait_read<0>();
        wg_sync();
        if (issuer) {
            const uint8_t* src = sD + (wg * 2 + buf) * STG_BYTES;
            if (ep.accumulate) tma_reduce_add_2d(&tmD, src, col, row);   // one add per element: deterministic
            else tma_store_2d(&tmD, src, col, row);
            bulk_commit();
        }
        buf ^= 1;
    };
    // Main-loop turns: tile i > 0 starts its MMAs once the other warpgroup has issued every MMA of tile i - 1 (named
    // barrier 3 + owner of tile i: the owner syncs, the other warpgroup arrives).  Besides overlapping one epilogue with
    // the other main loop, this keeps a warpgroup from waiting on a `full` barrier more than one ring lap ahead of the
    // loads, where its parity would be ambiguous.  Only a tile that exists is waited for or signalled.
    auto wait_turn = [&] {
        if (wg == 0) named_bar_sync(3, 256);
        else named_bar_sync(4, 256);
    };
    auto pass_turn = [&] {
        if (wg == 0) named_bar_arrive(4, 256);
        else named_bar_arrive(3, 256);
    };
    for (int i = PP ? wg : 0; i < cta_tiles; i += PP ? 2 : 1) {
        const int tile = blockIdx.x + i * gridDim.x;
        const int m0 = tile_m0(tile) + (PP ? 0 : wg * 64), n0 = tile_n0(tile);   // this warpgroup's 64 rows
        // the producer fills the ring with the CTA's tiles in order: tile i starts at K block i * num_k of the sequence
        const uint64_t first = uint64_t(i) * uint64_t(num_k);
        int stage = int(first % STAGES);
        uint32_t phase = uint32_t(first / STAGES) & 1u;
        if (PP && i > 0) wait_turn();
        int prev = -1;
        for (int kb = 0, kk = 0; kb < num_k; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint64_t adesc = wgmma_desc_sw128(sA + stage * Cfg::A_BYTES + (PP ? 0 : wg * (64 * 128)));
            const uint64_t bdesc = wgmma_desc_sw128(sB + stage * Cfg::B_BYTES);
            const bool lo_blk = NSPLIT == 2 && ((cg.lo_mask >> kk) & 1ull);
            wgmma_fence_regs<R>(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                Wgmma<BN>::mma(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
                if (NSPLIT == 2 && !lo_blk) Wgmma<BN>::mma(acc, adesc + 2 * k, bdesc + (Cfg::B_TILE >> 4) + 2 * k, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();                     // the group of the previous K block has retired: its stage is free
            wgmma_fence_regs<R>(acc);
            if (prev >= 0) {
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
            if (++kk == kpt) kk = 0;              // K block index inside the current tap
        }
        if (PP && i + 1 < cta_tiles) pass_turn();
        wgmma_wait<0>();
        wgmma_fence_regs<R>(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);

        // ------------------------------------------------------------ epilogue through shared memory
        // accumulator register 4j + 2h + e: row (lane / 4) + 8h of this warp's 16, column 8j + 2 (lane % 4) + e.
        bool keep[2] = {true, true};   // rows outside the valid conv region become the next layer's zero padding
        if (cg.mask) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int mm = m0 + wq * 16 + (lane >> 2) + 8 * h - cg.row0;
                const int w = mm % cg.Wp, r1 = mm / cg.Wp;
                const int hh = r1 % cg.Hp, r2 = r1 / cg.Hp;
                const int tt = r2 % cg.Tp;
                keep[h] = (mm >= 0) && (w >= cg.w0) && (w < cg.w1) && (hh >= cg.h0) && (hh < cg.h1) && (tt >= cg.t0) && (tt < cg.t1);
            }
        }
        // scale / bias / activation / row mask of accumulator column group j, in place; columns at or past N are left
        // as they are (TMA clips them)
        auto finish = [&](int j) {
            const int n = n0 + 8 * j + 2 * (lane & 3);
            if (n >= N) return;                  // N % 8 == 0: n < N implies n + 1 < N
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if (ep.scale) {
                    const float2 s = __ldg(reinterpret_cast<const float2*>(ep.scale + n));
                    v0 *= s.x; v1 *= s.y;
                }
                if (ep.bias) {
                    const float2 b = __ldg(reinterpret_cast<const float2*>(ep.bias + n));
                    v0 += b.x; v1 += b.y;
                }
                if (ep.act != VF_ACT_NONE) { v0 = apply_act(v0, ep.act); v1 = apply_act(v1, ep.act); }
                if (!keep[h]) { v0 = 0.f; v1 = 0.f; }
                acc[4 * j + 2 * h] = v0;
                acc[4 * j + 2 * h + 1] = v1;
            }
        };
        // Subtiles of 128-byte rows, left to right; those wholly at or past N are skipped.
        const int row = m0;
        const uint32_t stg = smem_u32(sD) + wg * 2 * STG_BYTES + (wq * 16 + (lane >> 2)) * 128;
        const int swz = lane >> 2;
        if (!SPLIT && ep.out_f32) {              // (run_gemm refuses a split fp32 output)
#pragma unroll
            for (int s = 0; s < BN / 32; ++s) {  // 32 columns: j = 4s .. 4s + 3
                if (n0 + 32 * s >= N) break;
                const uint32_t d = stg + buf * STG_BYTES;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int j = 4 * s + c;
                    finish(j);
                    const int chunk = 2 * c + ((lane & 3) >> 1);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        st_shared_v2_f32(d + h * 8 * 128 + ((chunk ^ swz) << 4) + 8 * (lane & 1), acc[4 * j + 2 * h],
                                         acc[4 * j + 2 * h + 1]);
                }
                store_subtile(n0 + 32 * s, row);
            }
        } else {
#pragma unroll
            for (int s = 0; s < BN / 64; ++s) {  // 64 columns: j = 8s .. 8s + 7
                if (n0 + 64 * s >= N) break;
                if (SPLIT) {
                    // hi into buffer 0, lo = fp16(v - hi) into buffer 1, in one pass: finish the values first, then
                    // wait until both stores of the previous subtile have read their buffers
#pragma unroll
                    for (int c = 0; c < 8; ++c) finish(8 * s + c);
                    if (issuer) bulk_wait_read<0>();
                    wg_sync();
#pragma unroll
                    for (int c = 0; c < 8; ++c)
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int j = 8 * s + c;
                            const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                            const __half2 hi = __floats2half2_rn(v0, v1);
                            const uint32_t off = h * 8 * 128 + ((c ^ swz) << 4) + 4 * (lane & 3);
                            st_shared_b32(stg + off, *reinterpret_cast<const uint32_t*>(&hi));
                            st_shared_b32(stg + STG_BYTES + off, pack_half2(v0 - __low2float(hi), v1 - __high2float(hi)));
                        }
                    fence_proxy_async();
                    wg_sync();
                    if (issuer) {
                        tma_store_2d(&tmD, sD + wg * 2 * STG_BYTES, n0 + 64 * s, row);
                        tma_store_2d(&tmD2, sD + (wg * 2 + 1) * STG_BYTES, n0 + 64 * s, row);
                        bulk_commit();
                    }
                } else {
                    const uint32_t d = stg + buf * STG_BYTES;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const int j = 8 * s + c;
                        finish(j);
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            st_shared_b32(d + h * 8 * 128 + ((c ^ swz) << 4) + 4 * (lane & 3),
                                          pack_half2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
                    }
                    store_subtile(n0 + 64 * s, row);
                }
            }
        }
    }
    if (issuer) bulk_wait<0>();                  // the last stores have landed before the CTA exits
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

template <int BN, int NSPLIT, bool SPLIT, bool PP>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const CUtensorMap& tmD2,
                const GemmEpi& ep, int M, int N, const ConvGeom& cg, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, NSPLIT, PP>;
    // one handle per thread, but several threads (one per handle) may reach the same instantiation at once: the attribute
    // call is idempotent, the flag that remembers it is an atomic (acquire / release), so there is no data race
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        VF_CUDA(cudaFuncSetAttribute(gemm_f16_kernel<BN, NSPLIT, SPLIT, PP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg::SMEM_BYTES));
        if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    const int tiles = ((M + Cfg::BM - 1) / Cfg::BM) * ((N + BN - 1) / BN);
    const int sms = device_sm_count();
    const int grid = tiles < sms ? tiles : sms;
    gemm_f16_kernel<BN, NSPLIT, SPLIT, PP><<<grid, THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmD, tmD2, ep, M, N, cg);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

}  // namespace

int device_sm_count() {
    static std::atomic<int> sms[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    int v = sms[dev].load(std::memory_order_relaxed);
    if (v == 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        sms[dev].store(v, std::memory_order_relaxed);
    }
    return v;
}

int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols,
                 uint64_t row_pitch_bytes, uint32_t box_rows, uint32_t box_cols) {
    EncodeTiledFn enc = get_encode_tiled();
    if (!enc) return fail(VF_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (row_pitch_bytes & 15))
        return fail(VF_ERR_INVALID, "TMA operand must be 16-byte aligned with a 16-byte multiple row pitch");
    if (box_cols * uint32_t(elem_bytes) != 128) return fail(VF_ERR_INVALID, "TMA box rows must be 128 bytes");
    const CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {row_pitch_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(out, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(VF_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", int(r));
    return VF_OK;
}

// Roofline instrumentation shared by every handle (vf_gemm_profile): CUDA-event pairs around each GEMM launch on the
// launching stream, per host thread.
struct GemmProf {
    bool on = false;
    std::vector<cudaEvent_t> ev;
    size_t used = 0;
    double flops = 0.0;
};
static thread_local GemmProf g_prof;

template <bool PP>
static int run_gemm_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                           const CUtensorMap& tmD2, int bn, const GemmEpi& ep, int M, int N, const ConvGeom& cg,
                           cudaStream_t stream) {
    if (ep.split_off > 0 && !ep.out_f32) {
        if (cg.nsplit == 2) {
            if (bn == 256) return launch_gemm<256, 2, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
            if (bn == 192) return launch_gemm<192, 2, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
            if (bn == 128) return launch_gemm<128, 2, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
            return launch_gemm<64, 2, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        }
        if (bn == 256) return launch_gemm<256, 1, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        if (bn == 192) return launch_gemm<192, 1, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        if (bn == 128) return launch_gemm<128, 1, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        return launch_gemm<64, 1, true, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    }
    if (cg.nsplit == 2) {
        if (bn == 256) return launch_gemm<256, 2, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        if (bn == 192) return launch_gemm<192, 2, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        if (bn == 128) return launch_gemm<128, 2, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        return launch_gemm<64, 2, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    }
    if (bn == 256) return launch_gemm<256, 1, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    if (bn == 192) return launch_gemm<192, 1, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    if (bn == 128) return launch_gemm<128, 1, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    return launch_gemm<64, 1, false, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
}

// pp: the ping-pong schedule (64-row tiles, tmA boxes of 64 rows) or the cooperative one (128-row tiles, boxes of 128)
static int run_gemm(const CUtensorMap& tmA, bool pp, const __half* B, int ldb, int64_t Ktot, int M, int N,
                    const ConvGeom& cg, const GemmEpi& ep, cudaStream_t stream) {
    if (!ep.out) return fail(VF_ERR_INVALID, "gemm: null output");
    if (reinterpret_cast<uintptr_t>(ep.out) & 15) return fail(VF_ERR_INVALID, "gemm: output must be 16-byte aligned");
    if (ep.accumulate && !ep.out_f32) return fail(VF_ERR_INVALID, "gemm: accumulate needs fp32 output");
    if (N % 8) return fail(VF_ERR_INVALID, "gemm: N=%d must be a multiple of 8", N);
    if (ep.out_f32 ? (ep.ldo % 4) : (ep.ldo % 8)) return fail(VF_ERR_INVALID, "gemm: ldo breaks 16-byte rows");
    if (ep.split_off && (ep.out_f32 || ep.split_off < N || ep.split_off % 8))
        return fail(VF_ERR_INVALID, "gemm: split output needs fp16 out and split_off >= N, multiple of 8");
    // Tile width: the one whose busiest SM computes the fewest columns, i.e. rounds of tiles (64 rows ping-pong, 128
    // cooperative) over the SMs x width.  This counts both the padding of N and the idle SMs of a last partial wave; the
    // widest wins a tie.
    const int bm = tile_rows(pp);
    const int64_t num_m = (M + bm - 1) / bm, sms = device_sm_count();
    int bn = 256;
    int64_t best = INT64_MAX;
    for (int cand : {256, 192, 128, 64}) {
        const int64_t cost = (num_m * ((N + cand - 1) / cand) + sms - 1) / sms * cand;
        if (cost < best) { best = cost; bn = cand; }
    }
    CUtensorMap tmB, tmD, tmD2;
    VF_TRY(make_tmap_2d(&tmB, B, 2, uint64_t(N), uint64_t(Ktot), uint64_t(ldb) * 2, uint32_t(bn), BK));
    const int eb = ep.out_f32 ? 4 : 2;
    VF_TRY(make_tmap_2d(&tmD, ep.out, eb, uint64_t(M), uint64_t(N), uint64_t(ep.ldo) * eb, EPI_ROWS, 128 / eb));
    if (ep.split_off)
        VF_TRY(make_tmap_2d(&tmD2, static_cast<__half*>(ep.out) + ep.split_off, eb, uint64_t(M), uint64_t(N),
                            uint64_t(ep.ldo) * eb, EPI_ROWS, 128 / eb));
    else
        tmD2 = tmD;
    auto launch = [&] {
        return pp ? run_gemm_launch<true>(tmA, tmB, tmD, tmD2, bn, ep, M, N, cg, stream)
                  : run_gemm_launch<false>(tmA, tmB, tmD, tmD2, bn, ep, M, N, cg, stream);
    };
    if (!g_prof.on) return launch();
    if (g_prof.used + 2 > g_prof.ev.size())
        for (int i = 0; i < 2; ++i) {
            cudaEvent_t e;
            VF_CUDA(cudaEventCreate(&e));
            g_prof.ev.push_back(e);
        }
    VF_CUDA(cudaEventRecord(g_prof.ev[g_prof.used], stream));
    const int st = launch();
    VF_CUDA(cudaEventRecord(g_prof.ev[g_prof.used + 1], stream));
    g_prof.used += 2;
    double kexec = double(Ktot);
    if (cg.nsplit == 2 && cg.lo_mask) {      // K blocks whose W_lo pass is skipped
        const int kpt = (cg.k_per_tap + BK - 1) / BK;
        int skipped = 0;
        for (int kk = 0; kk < kpt && kk < 64; ++kk) skipped += int((cg.lo_mask >> kk) & 1ull);
        kexec -= double(cg.ntaps) * skipped * BK;
    }
    g_prof.flops += 2.0 * double(M) * double(N) * kexec;
    return st;
}

bool gemm_profile_on() { return g_prof.on; }
int gemm_profile(int enable) {
    g_prof.on = enable != 0;
    return VF_OK;
}
int gemm_profile_read(double* ms, int64_t* launches, double* flops) {
    VF_CUDA(cudaDeviceSynchronize());
    double t = 0.0;
    for (size_t i = 0; i + 1 < g_prof.used; i += 2) {
        float x = 0.f;
        VF_CUDA(cudaEventElapsedTime(&x, g_prof.ev[i], g_prof.ev[i + 1]));
        t += x;
    }
    if (ms) *ms = t;
    if (launches) *launches = int64_t(g_prof.used / 2);
    if (flops) *flops = g_prof.flops;
    g_prof.used = 0;
    g_prof.flops = 0.0;
    return VF_OK;
}

int gemm_f16(const __half* A, int lda, const __half* B, int ldb, int M, int N, int K, const GemmEpi& ep,
             cudaStream_t stream) {
    if (M <= 0 || N <= 0 || K <= 0) return fail(VF_ERR_INVALID, "gemm: empty problem %dx%dx%d", M, N, K);
    if (K % 8 || lda % 8 || ldb % 8) return fail(VF_ERR_INVALID, "gemm: K/lda/ldb must be multiples of 8");
    ConvGeom cg;
    memset(&cg, 0, sizeof(cg));
    cg.ntaps = 1;
    cg.k_per_tap = K;
    cg.nsplit = 1;
    CUtensorMap tmA;
    VF_TRY(make_tmap_2d(&tmA, A, 2, uint64_t(M), uint64_t(K), uint64_t(lda) * 2, tile_rows(true), BK));
    return run_gemm(tmA, true, B, ldb, K, M, N, cg, ep, stream);
}

int conv_gemm_f16(const __half* X, int C, int64_t P, const __half* Wt, int N, const ConvGeom& g, const GemmEpi& ep,
                  cudaStream_t stream) {
    if (P <= 0 || P > 0x7fffffff || N <= 0 || C <= 0) return fail(VF_ERR_INVALID, "conv_gemm: bad size");
    if (C % 8) return fail(VF_ERR_INVALID, "conv_gemm: C=%d must be a multiple of 8", C);
    if (g.ntaps < 1 || g.ntaps > 64 || g.k_per_tap < 8 || g.k_per_tap % 8)
        return fail(VF_ERR_INVALID, "conv_gemm: bad tap geometry (%d taps x %d)", g.ntaps, g.k_per_tap);
    if (g.nsplit != 1 && g.nsplit != 2) return fail(VF_ERR_INVALID, "conv_gemm: nsplit must be 1 or 2");
    // lo_mask bit kk names K block kk of a tap; the kernel tests it with lo_mask >> kk, so a tap of more than 64 blocks
    // cannot carry a mask, and a bit at or above the tap's block count would name a block that does not exist
    const int kpt = (g.k_per_tap + BK - 1) / BK;
    if (g.lo_mask && (kpt > 64 || (kpt < 64 && (g.lo_mask >> kpt) != 0)))
        return fail(VF_ERR_INVALID, "conv_gemm: lo_mask 0x%llx names K blocks beyond the %d of a tap", g.lo_mask, kpt);
    if (g.mask && (g.Tp < 1 || g.Hp < 1 || g.Wp < 1 || g.row0 < 0))
        return fail(VF_ERR_INVALID, "conv_gemm: bad mask volume %dx%dx%d, row0 %d", g.Tp, g.Hp, g.Wp, g.row0);
    // overlapping-row view: row p = k_per_tap contiguous elements starting at element p*C
    CUtensorMap tmA;
    VF_TRY(make_tmap_2d(&tmA, X, 2, uint64_t(P), uint64_t(g.k_per_tap), uint64_t(C) * 2, tile_rows(false), BK));
    const int64_t Ktot = int64_t(g.ntaps) * g.k_per_tap * g.nsplit;
    if (Ktot % 8) return fail(VF_ERR_INVALID, "conv_gemm: K must be a multiple of 8");
    return run_gemm(tmA, false, Wt, int(Ktot), Ktot, int(P), N, g, ep, stream);
}

}  // namespace vf
