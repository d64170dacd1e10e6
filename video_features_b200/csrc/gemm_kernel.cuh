// The wgmma GEMM kernel template (gemm_f16_kernel) and its launchers, shared by gemm.cu (the host side) and the
// gemm_inst_*.cu units that instantiate it.  The schedule, tile and epilogue are described at the top of gemm.cu.
#pragma once
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

// ACT is a template parameter of the kernel, so each instantiation carries the one expression it applies: a run-time
// switch here was compiled to a jump table and an indirect branch per output element, and inlined all four bodies at
// every accumulator position.
template <int ACT>
__device__ __forceinline__ float apply_act(float v) {
    if (ACT == VF_ACT_QUICKGELU) {
        return __fdividef(v, 1.0f + __expf(-1.702f * v));   // x * sigmoid(1.702 x)
    } else if (ACT == VF_ACT_RELU) {
        return fmaxf(v, 0.0f);
    } else if (ACT == VF_ACT_SIGMOID) {
        return __fdividef(1.0f, 1.0f + __expf(-v));
    } else if (ACT == VF_ACT_TANH) {
        return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * v));   // saturates cleanly to +-1
    }
    return v;
}

// SPLIT: split-fp16 output (GemmEpi::split_off) -- every fp16 pair is written twice, hi at column n (tmD) and lo at
// split_off + n (tmD2).  A compile-time switch keeps the plain epilogue free of it.
// ACT: the epilogue's activation (VF_ACT_*), fixed per instantiation; GemmEpi::act selects the instantiation.
// tmD / tmD2: the output as dims (N, M), row pitch ldo, 64-row x 128-byte boxes; TMA clips every store at N and M.
template <int BN, int NSPLIT, bool SPLIT, bool PP, int ACT>
__global__ void __launch_bounds__(THREADS, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmD2, const GemmEpi ep,
                const int M, const int N, const __grid_constant__ ConvGeom cg) {
    using Cfg = GemmCfg<BN, NSPLIT, PP>;
    static_assert(PP ? NSPLIT == 1 : true, "split weights run in the conv mode only");
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
        // Scale and bias of this thread's columns in the first 64-column subtile, loaded while the last MMAs run.  A
        // missing scale reads as 1 and a missing bias as -0: x * 1 and x + (-0) are x bit for bit (a +0 bias would turn
        // -0 into +0), so every launch runs the same branch-free arithmetic and gets the bits of skipping the operation.
        // A column pair at or past N (N % 8 == 0: a pair is wholly inside or outside) reads the scale / bias of the
        // last pair and is computed like the others, so there is no per-element bounds test: TMA clips those columns.
        float2 sc[8], bi[8];
        auto load_sb = [&](int s) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int n = min(n0 + 64 * s + 8 * c + 2 * (lane & 3), N - 2);
                sc[c] = ep.scale ? __ldg(reinterpret_cast<const float2*>(ep.scale + n)) : make_float2(1.f, 1.f);
                bi[c] = ep.bias ? __ldg(reinterpret_cast<const float2*>(ep.bias + n)) : make_float2(-0.f, -0.f);
            }
        };
        load_sb(0);
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
        // Subtiles of 64 columns (one fp16 or split box, two fp32 boxes), left to right; those wholly at or past N are
        // skipped.  Each is finished in registers by one copy of the scale / bias / activation / row-mask code, whatever
        // the output, and the next subtile's scale / bias loads are issued before this one is written out.  The product
        // and the sum are the separately rounded ones the epilogue has always computed; _rn keeps the compiler from
        // contracting them into an fma.
        const int row = m0;
        const uint32_t stg = smem_u32(sD) + wg * 2 * STG_BYTES + (wq * 16 + (lane >> 2)) * 128;
        const int swz = lane >> 2;
#pragma unroll
        for (int s = 0; s < BN / 64; ++s) {      // j = 8s .. 8s + 7
            if (n0 + 64 * s >= N) break;
#pragma unroll
            for (int c = 0; c < 8; ++c)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = 8 * s + c;
                    float v0 = __fadd_rn(__fmul_rn(acc[4 * j + 2 * h], sc[c].x), bi[c].x);
                    float v1 = __fadd_rn(__fmul_rn(acc[4 * j + 2 * h + 1], sc[c].y), bi[c].y);
                    v0 = apply_act<ACT>(v0);
                    v1 = apply_act<ACT>(v1);
                    acc[4 * j + 2 * h] = keep[h] ? v0 : 0.f;
                    acc[4 * j + 2 * h + 1] = keep[h] ? v1 : 0.f;
                }
            if (s + 1 < BN / 64) load_sb(s + 1);
            if (SPLIT) {
                // hi into buffer 0, lo = fp16(v - hi) into buffer 1, once both stores of the previous subtile have
                // read their buffers
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
            } else if (ep.out_f32) {             // (run_gemm refuses a split fp32 output)
#pragma unroll
                for (int q = 0; q < 2; ++q) {    // 32 columns: j = 8s + 4q .. 8s + 4q + 3
                    if (q == 1 && n0 + 64 * s + 32 >= N) break;
                    const uint32_t d = stg + buf * STG_BYTES;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const int j = 8 * s + 4 * q + c;
                        const int chunk = 2 * c + ((lane & 3) >> 1);
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            st_shared_v2_f32(d + h * 8 * 128 + ((chunk ^ swz) << 4) + 8 * (lane & 1), acc[4 * j + 2 * h],
                                             acc[4 * j + 2 * h + 1]);
                    }
                    store_subtile(n0 + 64 * s + 32 * q, row);
                }
            } else {
                const uint32_t d = stg + buf * STG_BYTES;
#pragma unroll
                for (int c = 0; c < 8; ++c)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int j = 8 * s + c;
                        st_shared_b32(d + h * 8 * 128 + ((c ^ swz) << 4) + 4 * (lane & 3),
                                      pack_half2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
                    }
                store_subtile(n0 + 64 * s, row);
            }
        }
    }
    if (issuer) bulk_wait<0>();                  // the last stores have landed before the CTA exits
}

template <int BN, int NSPLIT, bool SPLIT, bool PP, int ACT>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const CUtensorMap& tmD2,
                const GemmEpi& ep, int M, int N, const ConvGeom& cg, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, NSPLIT, PP>;
    // one handle per thread, but several threads (one per handle) may reach the same instantiation at once: the attribute
    // call is idempotent, the flag that remembers it is an atomic (acquire / release), so there is no data race
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        VF_CUDA(cudaFuncSetAttribute(gemm_f16_kernel<BN, NSPLIT, SPLIT, PP, ACT>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    const int tiles = ((M + Cfg::BM - 1) / Cfg::BM) * ((N + BN - 1) / BN);
    const int sms = device_sm_count();
    const int grid = tiles < sms ? tiles : sms;
    gemm_f16_kernel<BN, NSPLIT, SPLIT, PP, ACT><<<grid, THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmD, tmD2, ep, M,
                                                                                            N, cg);
    VF_CUDA(cudaGetLastError());
    return VF_OK;
}

// The epilogue's activation, chosen once per launch (run_gemm has checked ep.act).
template <int BN, int NSPLIT, bool SPLIT, bool PP>
int launch_act(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const CUtensorMap& tmD2,
               const GemmEpi& ep, int M, int N, const ConvGeom& cg, cudaStream_t stream) {
    switch (ep.act) {
        case VF_ACT_QUICKGELU:
            return launch_gemm<BN, NSPLIT, SPLIT, PP, VF_ACT_QUICKGELU>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        case VF_ACT_RELU:
            return launch_gemm<BN, NSPLIT, SPLIT, PP, VF_ACT_RELU>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        case VF_ACT_SIGMOID:
            return launch_gemm<BN, NSPLIT, SPLIT, PP, VF_ACT_SIGMOID>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        case VF_ACT_TANH:
            return launch_gemm<BN, NSPLIT, SPLIT, PP, VF_ACT_TANH>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
        default:
            return launch_gemm<BN, NSPLIT, SPLIT, PP, VF_ACT_NONE>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    }
}

}  // namespace

// One launch of the instantiation for (NSPLIT, SPLIT, PP), tile width bn and ep.act.  Each (NSPLIT, SPLIT, PP) is
// instantiated explicitly in one gemm_inst_*.cu unit; gemm.cu declares them extern.
#define GEMM_LAUNCH_ARGS                                                                                           \
    const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmD, const CUtensorMap &tmD2, int bn,       \
        const GemmEpi &ep, int M, int N, const ConvGeom &cg, cudaStream_t stream
template <int NSPLIT, bool SPLIT, bool PP>
int launch_bn(GEMM_LAUNCH_ARGS) {
    if (bn == 256) return launch_act<256, NSPLIT, SPLIT, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    if (bn == 192) return launch_act<192, NSPLIT, SPLIT, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    if (bn == 128) return launch_act<128, NSPLIT, SPLIT, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
    return launch_act<64, NSPLIT, SPLIT, PP>(tmA, tmB, tmD, tmD2, ep, M, N, cg, stream);
}

}  // namespace vf
