// Host-side internals shared by the translation units of libvfeat.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include <array>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/vfeat.h"

namespace vf {

// thread-local last-error text behind vf_last_error()
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

#define VF_CUDA(expr)                                                                       \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess)                                                              \
            return vf::fail(VF_ERR_CUDA, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,      \
                            cudaGetErrorString(_e));                                        \
    } while (0)
#define VF_TRY(expr)                  \
    do {                              \
        int _s = (expr);              \
        if (_s != VF_OK) return _s;   \
    } while (0)

// ---- the host side every engine handle shares: device check, allocations, engine stream, graph cache, destroy.
// cudaSetDevice(device), then VF_ERR_UNSUPPORTED unless the device is sm_90 (the library is built for sm_90a only)
int check_device(int device);
bool graphs_enabled();   // false under VF_NO_GRAPH=1: every call runs eagerly
bool graph_trace();      // VF_GRAPH_TRACE=1: run_graphed reports every capture on stderr

// graph-cache key: (frames), (clips, T), (F, Hp, Wp) or (F, H, W, iters), unused slots zero
using GraphKey = std::array<int, 4>;
struct CachedGraph {
    cudaGraphExec_t exec = nullptr;
    int64_t launches = 0;     // kernel launches recorded during capture: what one replay adds to the count
};

struct EngineCore {
    const char* who = "";                          // prefixes error messages ("resnet_create", ...)
    int device = 0;
    std::vector<void*> allocs;                     // freed by release()
    int64_t launches = 0;                          // every kernel launch, eager or inside a replayed graph
    cudaStream_t cs = nullptr;                     // engine stream (open_stream), ordered against the caller's
    cudaEvent_t ev_in = nullptr, ev_out = nullptr; // stream by enter() / leave()
    bool use_graph = graphs_enabled();
    bool trace_graphs = graph_trace();
    std::map<GraphKey, CachedGraph> graphs;        // run_graphed's cache
    // run_graphed's admission policy: a key is captured on its capture_after-th sighting (earlier ones run eagerly); at
    // most max_graphs are kept, and once that many are, a new key evicts the smallest (evict_when_full) or runs eagerly
    int capture_after = 1;
    size_t max_graphs = 16;
    bool evict_when_full = true;
    std::map<GraphKey, int> seen;                  // sightings of keys not in the cache
    uint8_t *resized = nullptr, *resize_tmp = nullptr;   // the frame towers' resize scratch (resize_frames)
    size_t resized_cap = 0, tmp_cap = 0;
};

// cudaMalloc'd, zero-filled, + 64 KB: the overlapping-row TMA view of a conv input extends up to (k_per_tap - C)
// elements past its last row; zero-filled so that those elements are finite (they only feed masked border rows)
int engine_alloc(EngineCore* h, void** p, size_t bytes);
template <typename Tp>
int ralloc(EngineCore* h, Tp** p, size_t count) {
    void* q = nullptr;
    VF_TRY(engine_alloc(h, &q, count * sizeof(Tp)));
    *p = static_cast<Tp*>(q);
    return VF_OK;
}
int open_stream(EngineCore* h);                    // the engine stream and its ev_in / ev_out pair
int enter(EngineCore* h, cudaStream_t user);       // the engine stream waits for the work queued on `user`
int leave(EngineCore* h, cudaStream_t user);       // `user` waits for the work queued on the engine stream
// waits for the device, frees every allocation, graph and the resize scratch, destroys the stream and events (the
// handle is not deleted)
void release(EngineCore* h);
// a device buffer of at least `need` bytes; the engine stream is drained before an old one is freed
int grow(EngineCore* h, uint8_t** p, size_t* cap, size_t need);
// fp32 host -> device (a null source fails: a missing weight tensor)
int upload_f32(EngineCore* h, float** dst, const float* src, size_t count);
// fp32 host [rows, cols] -> fp16 device [rows, ld] (ld 0: cols; columns cols..ld-1 zero; transpose: src is
// [cols, rows]), round-to-nearest-even
int upload_f16(EngineCore* h, __half** dst, const float* src, size_t rows, size_t cols, size_t ld = 0,
               bool transpose = false);
// captures run() on stream s into an instantiated graph; h->launches is left as it was, g->launches gets what run()
// counted
int capture_graph(EngineCore* h, cudaStream_t s, const std::function<int()>& run, CachedGraph* g);
// run() on the engine stream through the graph cache: eager under VF_NO_GRAPH=1 or GEMM profiling (event-bracketed
// launches cannot be captured); otherwise a key is captured as h's admission policy says and then replayed.  The
// defaults capture on first use and keep 16 graphs, the smallest key evicted first.
int run_graphed(EngineCore* h, const GraphKey& key, const std::function<int()>& run);

// ---- the front end of the towers that take single frames (CLIP ViT-B / ViT-L / ResNet, DINOv2)
// Resize(resize_to, bicubic) of the short side, then CenterCrop(crop): the resized size, the crop offset and whether the
// frame is resized at all; filter: the Pillow filter resize_frames applies
struct FrameGeom { int rh, rw, cy, cx; bool resize; int filter = VF_FILTER_BICUBIC; };
int frame_geometry(const char* who, int H, int W, int resize_to, int crop, FrameGeom* g);
// n u8 frames of (H, W) -> *src, the frames the patchify kernel reads ((g.rh, g.rw) each): the frames themselves, or
// their Pillow-exact bicubic resize into h->resized (grown for max_frames frames)
int resize_frames(EngineCore* h, const uint8_t* frames, int n, int H, int W, const FrameGeom& g, int max_frames,
                  cudaStream_t s, const uint8_t** src);
// frames per chunk for a call of n: as few chunks as max_frames allows, all (nearly) the same size, so no ragged tail
// chunk runs the whole tower on a handful of rows
int balanced_step(int n, int max_frames);
// the argument check of a debug entry: h, a and b set, 1 .. limit frames (limit_name: what the limit is called)
int debug_frames(const EngineCore* h, const void* a, const void* b, int n, int limit, const char* limit_name,
                 const char* what);

// ---- tensor maps (driver entry point fetched at run time; the library does not link libcuda).
// 2-D row-major tensor of 2- or 4-byte elements, 128-byte-swizzled boxes of box_rows x (128 / elem_bytes) columns.
int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t rows, uint64_t cols,
                 uint64_t row_pitch_bytes, uint32_t box_rows, uint32_t box_cols);

// ---- GEMM: D[M,N] = act(A[M,K] . B[N,K]^T * scale[n] + bias[n]), fp16 operands, fp32 accumulate (wgmma)
struct GemmEpi {
    void* out;              // fp16 or fp32, row pitch ldo elements, 16-byte aligned rows
    const float* bias;      // [N] or null
    const float* scale;     // [N] or null
    int ldo;
    int out_f32;            // 0: fp16 out, 1: fp32 out
    int act;                // VF_ACT_*
    int split_off;          // fp16 out only: > 0 writes the result as a split-fp16 pair, hi at column n and
                            // lo = fp16(v - hi) at column split_off + n of the same row (0: plain fp16)
    int accumulate;         // fp32 out only: 1 = out += result (fp32 TMA reduce-adds from the epilogue; every element
                            // is added exactly once, so the sum is deterministic) -- the residual-stream update of the ViT blocks
};
GemmEpi linear_epi(void* out, int ldo, int out_f32, const float* bias, int act, int accumulate = 0);
int gemm_f16(const __half* A, int lda, const __half* B, int ldb, int M, int N, int K, const GemmEpi& ep,
             cudaStream_t stream);

// ---- shifted-row ("implicit GEMM") convolution on the same kernel.
// Activations live channels-last in a zero-bordered volume [n][Tp][Hp][Wp][C] flattened to P rows of C channels.
// A filter tap (dt,dh,dw) is then a constant row shift of the whole matrix, and because consecutive w positions are
// consecutive rows, the kw taps of one (dt,dh) form ONE contiguous run of kw*C elements: the A operand of tap j is
// the overlapping-row view  A_j[p, 0:k_per_tap] = X[(p + tap_off[j]) * C : ... + k_per_tap].
// Rows whose position lies outside the valid region [t0,t1)x[h0,h1)x[w0,w1) are written as zeros (they are the
// zero padding the next layer reads).
struct ConvGeom {
    int ntaps;          // number of (dt,dh) taps (1 for a 1x1x1 conv)
    int k_per_tap;      // contiguous K elements per tap (kw * C)
    int tap_off[64];    // row shift of each tap (includes the shift to the first kw tap)
    int nsplit;         // 1, or 2: weights are a hi+lo fp16 pair, Wt = [hi (ntaps*k_per_tap) | lo (same)] along K; every
                        // A tile is loaded once and multiplied with both (A.W_hi + A.W_lo)
    unsigned long long lo_mask;   // nsplit == 2 only: bit kk set = K block kk of every tap holds only lo halves of split-fp16
                        // activations (or unused columns): the W_lo pass is skipped there (a_lo.w_lo is below fp32 eps)
    int row0;           // leading guard rows: row m of the matrix is position m - row0 of the volume (rows < row0 are zeroed)
    int mask;           // 1: zero the rows outside the valid region
    int Tp, Hp, Wp;     // padded volume extents (rows per sample = Tp*Hp*Wp)
    int t0, t1, h0, h1, w0, w1;
};
// X: [P, C] fp16 (row pitch C), Wt: [N, ntaps*k_per_tap] fp16, output rows = P
int conv_gemm_f16(const __half* X, int C, int64_t P, const __half* Wt, int N, const ConvGeom& g, const GemmEpi& ep,
                  cudaStream_t stream);
// ---- QKV projection fused with the 50-token attention (csrc/attn_gemm.cu): h [n_frames*50, 768] fp16 -> att [.., heads*64]
// w_perm: in_proj rows regrouped per head, row h*192 + part*64 + d = in_proj row part*768 + h*64 + d (bias likewise)
int qkv_attention(const __half* h, int lda, const __half* w_perm, const float* bias_perm, __half* att, int n_frames, int heads,
                  cudaStream_t stream);
int device_sm_count();
int gemm_profile(int enable);
bool gemm_profile_on();   // event-bracketed launches cannot be captured into a graph: callers fall back to eager
int gemm_profile_read(double* ms, int64_t* launches, double* flops);

// ---- elementwise / reduction kernels
// patch = 32 (ViT-B/32: [n*49, 3072] patch rows) or 16 (ViT-B/16: [n*196, 768])
int launch_clip_patchify(const uint8_t* src, int n, int src_h, int src_w, int crop_y, int crop_x, __half* patches,
                         int patch, cudaStream_t s);
int launch_clip_patchify_f32(const float* src_chw, int n, __half* patches, int patch, cudaStream_t s);
int launch_clip_normalize_f32(const uint8_t* src, int n, int src_h, int src_w, int crop_y, int crop_x, float* dst_chw,
                              cudaStream_t s);
// x (+= y) ; out = LayerNorm(x) -- rows of 768 fp32.  y may be null; write_x stores the summed residual stream back.
int launch_add_layernorm(float* x, int64_t x_row_stride, const __half* y, int64_t y_row_stride, int write_x,
                         const float* gamma, const float* beta, void* out, int64_t out_row_stride, int out_f32, int rows,
                         cudaStream_t s);
// ViT embedding rows: token 0 = cls_pos0, token t>0 = emb[frame*(tokens-1) + t-1] + pos[t]; x = ln_pre(row) (fp32)
int launch_embed_layernorm(const float* emb, const float* pos, const float* cls_pos0, const float* gamma,
                           const float* beta, float* x, int n_frames, int tokens, cudaStream_t s);
// self-attention per (frame, head) on a [n_frames*tokens, 3*heads*64] QKV matrix: tokens == 50 or 65..208
int launch_attention(const __half* qkv, __half* out, int n_frames, int tokens, int heads, cudaStream_t s);
int launch_resample(const uint8_t* src, int n, int in_h, int in_w, uint8_t* tmp, uint8_t* dst, int out_h, int out_w,
                    const int* kh_bounds, const int* kh_coef, int kh_size, const int* kv_bounds, const int* kv_coef,
                    int kv_size, cudaStream_t s);

// host: Pillow-compatible resize (coefficient tables built in float64, cached on the device per geometry)
int resize_u8(const uint8_t* src, int n, int in_h, int in_w, uint8_t* dst, int out_h, int out_w, int filter,
              uint8_t* tmp, cudaStream_t s);
// torchvision CenterCrop offset: int(round((dim - crop) / 2.0)), Python round-half-to-even
int center_crop_offset(int dim, int crop);

}  // namespace vf
