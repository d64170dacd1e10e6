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
//
// The kernel template is in gemm_kernel.cuh.  Its 120 instantiations (tile width x split weights x split output x
// schedule x activation) are compiled in three units that build in parallel: gemm_inst_pp.cu (the ping-pong schedule),
// gemm_inst_conv.cu and gemm_inst_conv_w2.cu (the conv mode with plain and split weights).  This file holds the host
// side: argument checks, tensor maps, tile-width choice and the profiling hooks.
#include "gemm_kernel.cuh"

namespace vf {

extern template int launch_bn<1, false, true>(GEMM_LAUNCH_ARGS);
extern template int launch_bn<1, true, true>(GEMM_LAUNCH_ARGS);
extern template int launch_bn<1, false, false>(GEMM_LAUNCH_ARGS);
extern template int launch_bn<1, true, false>(GEMM_LAUNCH_ARGS);
extern template int launch_bn<2, false, false>(GEMM_LAUNCH_ARGS);
extern template int launch_bn<2, true, false>(GEMM_LAUNCH_ARGS);

namespace {

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

// Everything the epilogue can settle per launch is a template parameter: tile width, split weights, split output,
// schedule and activation.  Split weights come only through conv_gemm_f16 (gemm_f16 sets nsplit = 1), so the ping-pong
// schedule is built without them.
template <bool PP>
static int run_gemm_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                           const CUtensorMap& tmD2, int bn, const GemmEpi& ep, int M, int N, const ConvGeom& cg,
                           cudaStream_t stream) {
    const bool split = ep.split_off > 0 && !ep.out_f32;
    if constexpr (!PP) {
        if (cg.nsplit == 2)
            return split ? launch_bn<2, true, PP>(tmA, tmB, tmD, tmD2, bn, ep, M, N, cg, stream)
                         : launch_bn<2, false, PP>(tmA, tmB, tmD, tmD2, bn, ep, M, N, cg, stream);
    }
    return split ? launch_bn<1, true, PP>(tmA, tmB, tmD, tmD2, bn, ep, M, N, cg, stream)
                 : launch_bn<1, false, PP>(tmA, tmB, tmD, tmD2, bn, ep, M, N, cg, stream);
}

// pp: the ping-pong schedule (64-row tiles, tmA boxes of 64 rows) or the cooperative one (128-row tiles, boxes of 128)
static int run_gemm(const CUtensorMap& tmA, bool pp, const __half* B, int ldb, int64_t Ktot, int M, int N,
                    const ConvGeom& cg, const GemmEpi& ep, cudaStream_t stream) {
    if (!ep.out) return fail(VF_ERR_INVALID, "gemm: null output");
    if (reinterpret_cast<uintptr_t>(ep.out) & 15) return fail(VF_ERR_INVALID, "gemm: output must be 16-byte aligned");
    if (ep.accumulate && !ep.out_f32) return fail(VF_ERR_INVALID, "gemm: accumulate needs fp32 output");
    if (N % 8) return fail(VF_ERR_INVALID, "gemm: N=%d must be a multiple of 8", N);
    if (ep.act < VF_ACT_NONE || ep.act > VF_ACT_TANH) return fail(VF_ERR_INVALID, "gemm: unknown activation %d", ep.act);
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
