// Persistent warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = act( A[M,K] . B[N,K]^T * scale[n] + bias[n] )     A, B fp16 K-major; fp32 accumulate in registers;
//                                                              D fp16 or fp32
//
// A CTA owns a 128 x BN output tile at a time (tiles are strided over a grid of at most one CTA per SM).  Three
// warpgroups:
//   warpgroup 0    TMA producer (one lane): A and B tiles through a 128B-swizzled ring of STAGES stages, one mbarrier
//                  pair (full / empty) per stage.  It runs ahead into the next tile while the consumers store this one.
//   warpgroups 1,2 consumers: rows 0..63 and 64..127 of the tile.  Per 64-wide K block, four wgmma m64nBNk16 (eight with
//                  split weights), one commit group; the stage is released as soon as the group behind it has retired.
//                  Epilogue straight from the accumulator registers: scale / bias / activation, row mask, then fp16x2 or
//                  fp32x2 global stores (fp32x2 reductions for `accumulate`), M / N tails clipped per element.
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

constexpr int BM = 128;          // rows per CTA tile (64 per consumer warpgroup)
constexpr int BK = 64;           // 64 fp16 = one 128-byte swizzle row
constexpr int THREADS = 384;     // producer warpgroup + two consumer warpgroups
constexpr int CONSUMER_WARPS = 8;
constexpr uint32_t SMEM_BUDGET = 200 * 1024;   // operand ring; the rest of the 227 KB stays free

// NSPLIT = 2: the B stage holds the hi and the lo tile of a split-fp16 weight matrix and every K step issues two
// MMAs against the same A tile.
template <int BN, int NSPLIT>
struct GemmCfg {
    static constexpr uint32_t A_BYTES = BM * BK * 2;
    static constexpr uint32_t B_TILE = BN * BK * 2;           // one of hi / lo
    static constexpr uint32_t B_BYTES = NSPLIT * B_TILE;
    static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int STAGES = int(SMEM_BUDGET / STAGE_BYTES) > 8 ? 8 : int(SMEM_BUDGET / STAGE_BYTES);
    static constexpr uint32_t BAR_BYTES = 2 * STAGES * 8;
    static constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;   // + align slack
    static_assert(STAGES >= 2, "at least two pipeline stages");
    static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
    static_assert(A_BYTES % 1024 == 0 && B_TILE % 1024 == 0, "swizzle-128B tiles must stay 1024-byte aligned");
};

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

// SPLIT: split-fp16 output (GemmEpi::split_off) -- every fp16 pair is written twice, hi at column n and lo at
// split_off + n.  A compile-time switch keeps the plain epilogue free of it.
template <int BN, int NSPLIT, bool SPLIT>
__global__ void __launch_bounds__(THREADS, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmEpi ep,
                const int M, const int N, const __grid_constant__ ConvGeom cg) {
    using Cfg = GemmCfg<BN, NSPLIT>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_m = (M + BM - 1) / BM;
    const int num_n = (N + BN - 1) / BN;
    const int num_tiles = num_m * num_n;
    const int kpt = (cg.k_per_tap + BK - 1) / BK;    // K blocks per filter tap (a plain GEMM is one "tap")
    const int num_k = cg.ntaps * kpt;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full[i], 1);                  // the producer's arrive.expect_tx
            mbar_init(&empty[i], CONSUMER_WARPS);    // one arrive per consumer warp
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ------------------------------------------------------------ TMA producer
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int m0 = (tile % num_m) * BM, n0 = (tile / num_m) * BN;
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
    const int wg = (warp >> 2) - 1;              // 0: tile rows 0..63, 1: rows 64..127
    const int wq = warp & 3;                     // warp inside the warpgroup: 16 rows each
    constexpr int R = BN / 2;                    // accumulator registers per thread
    float acc[R];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile % num_m) * BM, n0 = (tile / num_m) * BN;
        int prev = -1;
        for (int kb = 0, kk = 0; kb < num_k; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint64_t adesc = wgmma_desc_sw128(sA + stage * Cfg::A_BYTES + wg * (64 * 128));
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
        wgmma_wait<0>();
        wgmma_fence_regs<R>(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);

        // ------------------------------------------------------------ epilogue from registers
        // accumulator register 4j + 2h + e: row (lane / 4) + 8h of this warp's 16, column 8j + 2 (lane % 4) + e
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
            if (m >= M) continue;
            bool keep = true;     // rows outside the valid conv region become the next layer's zero padding
            if (cg.mask) {
                const int mm = m - cg.row0;
                const int w = mm % cg.Wp, r1 = mm / cg.Wp;
                const int hh = r1 % cg.Hp, r2 = r1 / cg.Hp;
                const int tt = r2 % cg.Tp;
                keep = (mm >= 0) && (w >= cg.w0) && (w < cg.w1) && (hh >= cg.h0) && (hh < cg.h1) && (tt >= cg.t0) && (tt < cg.t1);
            }
            char* orow = static_cast<char*>(ep.out) + int64_t(m) * ep.ldo * (ep.out_f32 ? 4 : 2);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = n0 + 8 * j + 2 * (lane & 3);
                if (n >= N) continue;            // N % 8 == 0: n < N implies n + 1 < N
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
                if (!keep) { v0 = 0.f; v1 = 0.f; }
                if (ep.out_f32) {
                    float* p = reinterpret_cast<float*>(orow) + n;
                    if (ep.accumulate) atomicAdd(reinterpret_cast<float2*>(p), make_float2(v0, v1));   // one add per element: deterministic
                    else *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
                } else {
                    __half* p = reinterpret_cast<__half*>(orow) + n;
                    const __half2 hi = __floats2half2_rn(v0, v1);
                    *reinterpret_cast<__half2*>(p) = hi;
                    if (SPLIT)
                        *reinterpret_cast<__half2*>(p + ep.split_off) =
                            __floats2half2_rn(v0 - __low2float(hi), v1 - __high2float(hi));
                }
            }
        }
    }
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

template <int BN, int NSPLIT, bool SPLIT = false>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmEpi& ep, int M, int N, const ConvGeom& cg,
                cudaStream_t stream) {
    using Cfg = GemmCfg<BN, NSPLIT>;
    // one handle per thread, but several threads (one per handle) may reach the same instantiation at once: the attribute
    // call is idempotent, the flag that remembers it is an atomic (acquire / release), so there is no data race
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        VF_CUDA(cudaFuncSetAttribute(gemm_f16_kernel<BN, NSPLIT, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg::SMEM_BYTES));
        if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    const int sms = device_sm_count();
    const int grid = tiles < sms ? tiles : sms;
    gemm_f16_kernel<BN, NSPLIT, SPLIT><<<grid, THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, ep, M, N, cg);
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

static int run_gemm_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, int bn, const GemmEpi& ep, int M, int N,
                           const ConvGeom& cg, cudaStream_t stream) {
    if (ep.split_off > 0 && !ep.out_f32) {
        if (cg.nsplit == 2) {
            if (bn == 256) return launch_gemm<256, 2, true>(tmA, tmB, ep, M, N, cg, stream);
            if (bn == 192) return launch_gemm<192, 2, true>(tmA, tmB, ep, M, N, cg, stream);
            if (bn == 128) return launch_gemm<128, 2, true>(tmA, tmB, ep, M, N, cg, stream);
            return launch_gemm<64, 2, true>(tmA, tmB, ep, M, N, cg, stream);
        }
        if (bn == 256) return launch_gemm<256, 1, true>(tmA, tmB, ep, M, N, cg, stream);
        if (bn == 192) return launch_gemm<192, 1, true>(tmA, tmB, ep, M, N, cg, stream);
        if (bn == 128) return launch_gemm<128, 1, true>(tmA, tmB, ep, M, N, cg, stream);
        return launch_gemm<64, 1, true>(tmA, tmB, ep, M, N, cg, stream);
    }
    if (cg.nsplit == 2) {
        if (bn == 256) return launch_gemm<256, 2>(tmA, tmB, ep, M, N, cg, stream);
        if (bn == 192) return launch_gemm<192, 2>(tmA, tmB, ep, M, N, cg, stream);
        if (bn == 128) return launch_gemm<128, 2>(tmA, tmB, ep, M, N, cg, stream);
        return launch_gemm<64, 2>(tmA, tmB, ep, M, N, cg, stream);
    }
    if (bn == 256) return launch_gemm<256, 1>(tmA, tmB, ep, M, N, cg, stream);
    if (bn == 192) return launch_gemm<192, 1>(tmA, tmB, ep, M, N, cg, stream);
    if (bn == 128) return launch_gemm<128, 1>(tmA, tmB, ep, M, N, cg, stream);
    return launch_gemm<64, 1>(tmA, tmB, ep, M, N, cg, stream);
}

static int run_gemm(const CUtensorMap& tmA, const __half* B, int ldb, int64_t Ktot, int M, int N, const ConvGeom& cg,
                    const GemmEpi& ep, cudaStream_t stream) {
    if (!ep.out) return fail(VF_ERR_INVALID, "gemm: null output");
    if (reinterpret_cast<uintptr_t>(ep.out) & 15) return fail(VF_ERR_INVALID, "gemm: output must be 16-byte aligned");
    if (ep.accumulate && !ep.out_f32) return fail(VF_ERR_INVALID, "gemm: accumulate needs fp32 output");
    if (N % 8) return fail(VF_ERR_INVALID, "gemm: N=%d must be a multiple of 8", N);
    if (ep.out_f32 ? (ep.ldo % 4) : (ep.ldo % 8)) return fail(VF_ERR_INVALID, "gemm: ldo breaks 16-byte rows");
    if (ep.split_off && (ep.out_f32 || ep.split_off < N || ep.split_off % 8))
        return fail(VF_ERR_INVALID, "gemm: split output needs fp16 out and split_off >= N, multiple of 8");
    // tile width: the candidate that pads N least, the widest on a tie
    int bn = 64;
    if (N > 64) {
        int best = 0x7fffffff;
        for (int cand : {256, 192, 128}) {
            const int padded = (N + cand - 1) / cand * cand;
            if (padded < best) { best = padded; bn = cand; }
        }
    }
    CUtensorMap tmB;
    VF_TRY(make_tmap_2d(&tmB, B, 2, uint64_t(N), uint64_t(Ktot), uint64_t(ldb) * 2, uint32_t(bn), BK));
    if (!g_prof.on) return run_gemm_launch(tmA, tmB, bn, ep, M, N, cg, stream);
    if (g_prof.used + 2 > g_prof.ev.size())
        for (int i = 0; i < 2; ++i) {
            cudaEvent_t e;
            VF_CUDA(cudaEventCreate(&e));
            g_prof.ev.push_back(e);
        }
    VF_CUDA(cudaEventRecord(g_prof.ev[g_prof.used], stream));
    const int st = run_gemm_launch(tmA, tmB, bn, ep, M, N, cg, stream);
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
    VF_TRY(make_tmap_2d(&tmA, A, 2, uint64_t(M), uint64_t(K), uint64_t(lda) * 2, BM, BK));
    return run_gemm(tmA, B, ldb, K, M, N, cg, ep, stream);
}

int conv_gemm_f16(const __half* X, int C, int64_t P, const __half* Wt, int N, const ConvGeom& g, const GemmEpi& ep,
                  cudaStream_t stream) {
    if (P <= 0 || P > 0x7fffffff || N <= 0 || C <= 0) return fail(VF_ERR_INVALID, "conv_gemm: bad size");
    if (C % 8) return fail(VF_ERR_INVALID, "conv_gemm: C=%d must be a multiple of 8", C);
    if (g.ntaps < 1 || g.ntaps > 64 || g.k_per_tap < 8 || g.k_per_tap % 8)
        return fail(VF_ERR_INVALID, "conv_gemm: bad tap geometry (%d taps x %d)", g.ntaps, g.k_per_tap);
    // overlapping-row view: row p = k_per_tap contiguous elements starting at element p*C
    CUtensorMap tmA;
    VF_TRY(make_tmap_2d(&tmA, X, 2, uint64_t(P), uint64_t(g.k_per_tap), uint64_t(C) * 2, BM, BK));
    if (g.nsplit != 1 && g.nsplit != 2) return fail(VF_ERR_INVALID, "conv_gemm: nsplit must be 1 or 2");
    const int64_t Ktot = int64_t(g.ntaps) * g.k_per_tap * g.nsplit;
    if (Ktot % 8) return fail(VF_ERR_INVALID, "conv_gemm: K must be a multiple of 8");
    return run_gemm(tmA, Wt, int(Ktot), Ktot, int(P), N, g, ep, stream);
}

}  // namespace vf
