// CLIP ViT-B image tower (patch 32: the north-star model; patch 16: the reference's 'CLIP-ViT-B/16' feature type, same
// width / depth, 197 tokens) on the wgmma GEMM + memory-bound kernels.
// Replaces `clip.load("ViT-B/32")` + `model.encode_image(frames)` (reference: models/CLIP/extract_clip.py:47,128;
// algorithm: third-party openai/CLIP clip/model.py VisionTransformer.forward, restated in oracle/clip_tower.py).
//
// Numerics: GEMM operands fp16, accumulation fp32 (wgmma registers), residual stream / LayerNorm / softmax fp32.
// Frames are packed along M (row = frame*tokens + token) and processed in chunks (default 256 frames, chosen by
// measurement: vf_clip_create_vit).
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <map>
#include <vector>

#include "internal.h"

namespace vf {

constexpr int W = 768, L = 12, H = 12, MLPW = 3072, E = 512;

struct ClipLayerDev {
    float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *b_qkv, *b_o, *b_fc, *b_proj;
    __half *w_qkv, *w_o, *w_fc, *w_proj;
    // in_proj regrouped per head ([q_h | k_h | v_h] rows contiguous) for the fused QKV + attention kernel
    __half* w_qkv_heads;
    float* b_qkv_heads;
};

}  // namespace vf

struct vf_clip {
    int device = 0;
    int chunk = 0;
    int patch = 32, T = 50, P = 49, PK = 3072;   // patch size, tokens (P + 1), patches per frame, patch-matrix columns
    int64_t launches = 0;
    std::vector<void*> allocs;
    // weights
    __half* w_patch = nullptr;   // [768, PK]
    __half* w_proj = nullptr;    // [512, 768]  (proj^T)
    float *pos = nullptr, *cls_pos0 = nullptr, *lnpre_w = nullptr, *lnpre_b = nullptr, *lnpost_w = nullptr,
          *lnpost_b = nullptr;
    vf::ClipLayerDev layer[12];
    // workspace (per chunk)
    __half *patches = nullptr, *h = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr, *cls = nullptr;
    float *x = nullptr, *emb = nullptr;   // residual stream (fp32), patch embeddings (fp32)
    __half* y = nullptr;                  // residual-branch increment written by out-proj / fc2 (fp16)
    // transform scratch (grown on demand)
    uint8_t *stage_u8 = nullptr, *resized = nullptr, *resize_tmp = nullptr;
    size_t stage_cap = 0, resized_cap = 0, tmp_cap = 0;
    size_t stage_fbytes = 0;      // frame size the two staging slots were last laid out for
    float* out_dev = nullptr;
    size_t out_cap = 0;
    // roofline instrumentation (vf_clip_profile)
    bool prof = false;
    std::vector<cudaEvent_t> prof_events;   // pairs
    std::vector<int> prof_cat;              // category of each pair: 0 gemm, 1 layernorm, 2 attention, 3 transform
    double prof_cat_ms[4] = {0, 0, 0, 0};
    size_t prof_used = 0;
    double prof_flops = 0.0;
    // All work of a call runs on the engine's own compute stream `cs` (ordered against the caller's stream with a
    // pair of events), so that the per-chunk tower can be captured once into a CUDA graph and replayed: ~90 kernel
    // launches and ~150 tensor-map encodes per chunk collapse into one cudaGraphLaunch (the legacy NULL stream, which
    // is what torch hands over by default, cannot be captured).
    //
    // Two LANES (stream + private workspace) take the chunks of a call alternately.  A GEMM owns every SM's shared
    // memory, so GEMMs of the two lanes serialise, but the memory-bound kernels of one lane (LayerNorm, attention,
    // transform: no shared memory to speak of) co-reside with the tensor-bound GEMM of the other and fill its tails.
    struct Lane {
        __half *patches = nullptr, *h = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr, *cls = nullptr, *y = nullptr;
        float *x = nullptr, *emb = nullptr, *feat = nullptr;
        uint8_t *resized = nullptr, *resize_tmp = nullptr;
        size_t resized_cap = 0, tmp_cap = 0;
        cudaStream_t cs = nullptr;
        cudaEvent_t ev_out = nullptr;
        std::map<int, cudaGraphExec_t> graphs;   // frames in chunk -> instantiated tower graph (writes feat)
        std::map<int, int> seen;                 // frames in chunk -> times this size has been run without a graph
    } lanes[2];
    int n_lanes = 2, cur = 0;
    cudaStream_t cs = nullptr;                // stream of the active lane
    cudaEvent_t ev_in = nullptr;
    bool use_graph = true;
    bool acc_o = true, acc_m = true;          // residual adds in the GEMM epilogue (fp32 reductions) instead of an fp16 y
    bool fused_attn = true;                   // QKV projection + attention in one kernel (VF_CLIP_ATTN=split: GEMM + kernel)
    float* feat = nullptr;                    // [chunk, 512] tower output of the active lane
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copy[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
    // asynchronous host calls (vf_clip_encode_u8_host_async): completion events of the last kTickets calls
    static constexpr int kTickets = 4;
    cudaEvent_t ev_ticket[kTickets] = {nullptr, nullptr, nullptr, nullptr};
    std::atomic<int64_t> seq{0};              // vf_clip_wait may run on another host thread than the enqueuing one
};

namespace vf {

template <typename Tp>
static int dev_alloc(vf_clip* h, Tp** p, size_t count) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(Tp));
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", count * sizeof(Tp), cudaGetErrorString(e));
    h->allocs.push_back(q);
    *p = static_cast<Tp*>(q);
    return VF_OK;
}
static int upload_f32(vf_clip* h, float** dst, const float* src, size_t count) {
    if (!src) return fail(VF_ERR_INVALID, "clip_create: missing weight tensor");
    VF_TRY(dev_alloc(h, dst, count));
    VF_CUDA(cudaMemcpy(*dst, src, count * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}
// fp32 host [rows, cols] (optionally transposed on the way) -> fp16 device, round-to-nearest-even
static int upload_f16(vf_clip* h, __half** dst, const float* src, size_t rows, size_t cols, bool transpose) {
    if (!src) return fail(VF_ERR_INVALID, "clip_create: missing weight tensor");
    std::vector<__half> tmp(rows * cols);
    if (!transpose) {
        for (size_t i = 0; i < rows * cols; ++i) tmp[i] = __float2half_rn(src[i]);
    } else {   // src is [rows, cols]; produce [cols, rows]
        for (size_t r = 0; r < rows; ++r)
            for (size_t c = 0; c < cols; ++c) tmp[c * rows + r] = __float2half_rn(src[r * cols + c]);
    }
    VF_TRY(dev_alloc(h, dst, rows * cols));
    VF_CUDA(cudaMemcpy(*dst, tmp.data(), tmp.size() * sizeof(__half), cudaMemcpyHostToDevice));
    return VF_OK;
}

static int grow(uint8_t** p, size_t* cap, size_t need) {
    if (need <= *cap) return VF_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), need);
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", need, cudaGetErrorString(e));
    *cap = need;
    return VF_OK;
}

static GemmEpi epi(void* out, int ldo, int out_f32, const float* bias, int act, int accumulate = 0) {
    GemmEpi e;
    memset(&e, 0, sizeof(e));
    e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.bias = bias; e.act = act; e.accumulate = accumulate;
    return e;
}

// event bracket around one launch when profiling is on (vf_clip_profile): category 0 gemm, 1 layernorm,
// 2 attention, 3 transform
struct ProfScope {
    vf_clip* h; cudaStream_t s; bool on;
    ProfScope(vf_clip* h_, int cat, cudaStream_t s_) : h(h_), s(s_), on(h_->prof) {
        if (!on) return;
        if (h->prof_used + 2 > h->prof_events.size()) {
            for (int i = 0; i < 2; ++i) {
                cudaEvent_t e;
                if (cudaEventCreate(&e) != cudaSuccess) { on = false; return; }
                h->prof_events.push_back(e);
            }
        }
        cudaEventRecord(h->prof_events[h->prof_used], s);
        h->prof_cat.resize(h->prof_used / 2 + 1);
        h->prof_cat[h->prof_used / 2] = cat;
    }
    ~ProfScope() {
        if (!on) return;
        cudaEventRecord(h->prof_events[h->prof_used + 1], s);
        h->prof_used += 2;
    }
};

static int tower_gemm(vf_clip* h, const __half* A, int lda, const __half* B, int ldb, int M, int N, int K,
                      const GemmEpi& ep, cudaStream_t s) {
    ProfScope p(h, 0, s);
    if (h->prof) h->prof_flops += 2.0 * double(M) * double(N) * double(K);
    return gemm_f16(A, lda, B, ldb, M, N, K, ep, s);
}
static int tower_embed_ln(vf_clip* h, int c, cudaStream_t s) {
    ProfScope p(h, 1, s);
    return launch_embed_layernorm(h->emb, h->pos, h->cls_pos0, h->lnpre_w, h->lnpre_b, h->x, c, h->T, s);
}
static int tower_add_ln(vf_clip* h, float* x, int64_t x_stride, const __half* y, int64_t y_stride, int write_x,
                        const float* g, const float* b, void* out, int64_t ostride, int rows, cudaStream_t s) {
    ProfScope p(h, 1, s);
    return launch_add_layernorm(x, x_stride, y, y_stride, write_x, g, b, out, ostride, 0, rows, s);
}
static int tower_qkv_attention(vf_clip* h, const ClipLayerDev& w, int c, cudaStream_t s) {
    ProfScope p(h, 2, s);      // its own category: QKV projection + attention core in one kernel
    return qkv_attention(h->h, W, w.w_qkv_heads, w.b_qkv_heads, h->att, c, H, s);
}
static int tower_attention(vf_clip* h, int c, cudaStream_t s) {
    ProfScope p(h, 2, s);
    return launch_attention(h->qkv, h->att, c, h->T, H, s);
}

// The tower on one chunk whose patch matrix is already in h->patches; writes c x 512 fp32 to out.
// GEMM epilogues never read global memory: bias / QuickGELU in registers, then global stores -- or, for the two GEMMs
// that end a residual branch, fp32 reductions that add the tile into the fp32 residual stream x.
static int clip_tower_eager(vf_clip* h, int c, float* out, cudaStream_t s) {
    const int T = h->T, P = h->P, PK = h->PK;
    const int M = c * T;
    // patch embedding: [c*P, PK] x [768, PK]^T -> emb (fp32)
    VF_TRY(tower_gemm(h, h->patches, PK, h->w_patch, PK, c * P, W, PK, epi(h->emb, W, 1, nullptr, VF_ACT_NONE), s));
    // token assembly (+ class / positional embedding) fused with ln_pre -> x
    VF_TRY(tower_embed_ln(h, c, s));
    h->launches += 2;
    // The residual stream x stays fp32 in HBM.  A GEMM that ends a residual branch either ADDS its result into x from the
    // epilogue (fp32 global reductions; the LayerNorm pass that follows then only reads x and writes h: 6 bytes per
    // element), or writes an fp16 increment y that the LayerNorm kernel adds ("x += y; h = LN(x)": 12 bytes per element).
    // acc_o / acc_m select the form for the attention out-projection / the MLP's second GEMM (VF_CLIP_RESID=acc|y|mix).
    const bool acc_o = h->acc_o, acc_m = h->acc_m;
    for (int l = 0; l < L; ++l) {
        const ClipLayerDev& w = h->layer[l];
        // h = ln_1(x)   (y form: x += y of the previous block's MLP first)
        VF_TRY(tower_add_ln(h, h->x, W, (acc_m || l == 0) ? nullptr : h->y, W, 1, w.ln1_w, w.ln1_b, h->h, W, M, s));
        if (h->fused_attn) {
            VF_TRY(tower_qkv_attention(h, w, c, s));
        } else {
            VF_TRY(tower_gemm(h, h->h, W, w.w_qkv, W, M, 3 * W, W, epi(h->qkv, 3 * W, 0, w.b_qkv, VF_ACT_NONE), s));
            VF_TRY(tower_attention(h, c, s));
        }
        // Last block: only the CLS token reaches ln_post / proj (encode_image returns x[:, 0]), so after the attention
        // everything runs on the c CLS rows: A operands and the residual rows are strided views (row pitch T*768), h /
        // mlp / y are compact c-row buffers.  Saves (T-1)/T of out-proj + MLP of this block (5.9 % of the FLOPs at T = 50).
        const bool last = l + 1 == L;
        const int rows = last ? c : M;
        const int a_ld = last ? T * W : W;                    // row pitch of att / x when only the CLS rows are read
        if (acc_o) {
            VF_TRY(tower_gemm(h, h->att, a_ld, w.w_o, W, rows, W, W, epi(h->x, a_ld, 1, w.b_o, VF_ACT_NONE, 1), s));
            VF_TRY(tower_add_ln(h, h->x, a_ld, nullptr, W, 0, w.ln2_w, w.ln2_b, h->h, W, rows, s));
        } else {
            VF_TRY(tower_gemm(h, h->att, a_ld, w.w_o, W, rows, W, W, epi(h->y, W, 0, w.b_o, VF_ACT_NONE), s));
            VF_TRY(tower_add_ln(h, h->x, a_ld, h->y, W, 1, w.ln2_w, w.ln2_b, h->h, W, rows, s));
        }
        VF_TRY(tower_gemm(h, h->h, W, w.w_fc, W, rows, MLPW, W, epi(h->mlp, MLPW, 0, w.b_fc, VF_ACT_QUICKGELU), s));
        if (acc_m) VF_TRY(tower_gemm(h, h->mlp, MLPW, w.w_proj, MLPW, rows, W, MLPW, epi(h->x, a_ld, 1, w.b_proj, VF_ACT_NONE, 1), s));
        else       VF_TRY(tower_gemm(h, h->mlp, MLPW, w.w_proj, MLPW, rows, W, MLPW, epi(h->y, W, 0, w.b_proj, VF_ACT_NONE), s));
        h->launches += h->fused_attn ? 6 : 7;
    }
    // CLS rows: (y form: x += y of the last MLP;) ln_post; then the 768 -> 512 projection
    VF_TRY(tower_add_ln(h, h->x, int64_t(T) * W, acc_m ? nullptr : h->y, W, 0, h->lnpost_w, h->lnpost_b, h->cls, W, c, s));
    VF_TRY(tower_gemm(h, h->cls, W, h->w_proj, W, c, E, W, epi(out, E, 1, nullptr, VF_ACT_NONE), s));
    h->launches += 2;
    return VF_OK;
}

constexpr int TOWER_LAUNCHES_SPLIT = 2 + 7 * L + 2, TOWER_LAUNCHES_FUSED = 2 + 6 * L + 2;
constexpr size_t kMaxTowerGraphs = 32;    // per lane; further sizes run eagerly

// Tower on one chunk: replay (capturing on first use) the CUDA graph for this chunk size, then copy the features out.
static int clip_tower_chunk(vf_clip* h, int c, float* out, cudaStream_t s) {
    if (!h->use_graph || h->prof) return clip_tower_eager(h, c, out, s);
    auto& graphs = h->lanes[h->cur].graphs;
    auto it = graphs.find(c);
    if (it == graphs.end()) {
        // A chunk size is captured the SECOND time it shows up: one-off sizes (the ragged tail of a list, batches of
        // videos of unequal length) run eagerly instead of paying capture + instantiation for a graph that is never
        // replayed, and the cache stays bounded.
        auto& seen = h->lanes[h->cur].seen;
        if (seen.size() > 4096) seen.clear();
        if (++seen[c] < 2 || graphs.size() >= kMaxTowerGraphs) return clip_tower_eager(h, c, out, s);
        const int64_t before = h->launches;
        cudaGraph_t graph = nullptr;
        VF_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
        const int st = clip_tower_eager(h, c, h->feat, s);
        const cudaError_t ce = cudaStreamEndCapture(s, &graph);
        h->launches = before;
        if (st != VF_OK) { if (graph) cudaGraphDestroy(graph); return st; }
        if (ce != cudaSuccess) return fail(VF_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(ce));
        cudaGraphExec_t exec = nullptr;
        const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) return fail(VF_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ie));
        it = graphs.emplace(c, exec).first;
    }
    VF_CUDA(cudaGraphLaunch(it->second, s));
    VF_CUDA(cudaMemcpyAsync(out, h->feat, size_t(c) * E * sizeof(float), cudaMemcpyDeviceToDevice, s));
    h->launches += h->fused_attn ? TOWER_LAUNCHES_FUSED : TOWER_LAUNCHES_SPLIT;
    return VF_OK;
}

// frames per chunk for a batch of n: as few chunks as the workspace allows, all (nearly) the same size, so no
// ragged tail chunk runs the 12-layer launch sequence on a handful of rows
static int balanced_chunk(const vf_clip* h, int n) {
    const int nchunks = (n + h->chunk - 1) / h->chunk;
    return nchunks > 0 ? (n + nchunks - 1) / nchunks : h->chunk;
}

// make lane `l` the active one: its workspace pointers and stream become the ones the launch helpers use
static cudaStream_t activate(vf_clip* h, int l) {
    vf_clip::Lane& L = h->lanes[l];
    h->cur = l;
    h->patches = L.patches; h->h = L.h; h->qkv = L.qkv; h->att = L.att; h->mlp = L.mlp; h->cls = L.cls; h->y = L.y;
    h->x = L.x; h->emb = L.emb; h->feat = L.feat;
    h->resized = L.resized; h->resize_tmp = L.resize_tmp; h->resized_cap = L.resized_cap; h->tmp_cap = L.tmp_cap;
    h->cs = L.cs;
    return L.cs;
}
static void deactivate(vf_clip* h) {      // keep the (possibly grown) resize scratch with its lane
    vf_clip::Lane& L = h->lanes[h->cur];
    L.resized = h->resized; L.resize_tmp = h->resize_tmp; L.resized_cap = h->resized_cap; L.tmp_cap = h->tmp_cap;
}
// keeps a lane's (possibly re-allocated) resize scratch with the lane on EVERY exit path of a chunk, early error returns
// included: a lane left holding pointers that grow() has already freed would be a use-after-free on the next call
struct LaneScope {
    vf_clip* h;
    cudaStream_t s;
    LaneScope(vf_clip* h_, int l) : h(h_), s(activate(h_, l)) {}
    ~LaneScope() { deactivate(h); }
};
// order the lane streams after the caller's stream (enter) and the caller's stream after the lanes (leave)
static int enter(vf_clip* h, cudaStream_t user) {
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaEventRecord(h->ev_in, user));
    for (int l = 0; l < h->n_lanes; ++l) VF_CUDA(cudaStreamWaitEvent(h->lanes[l].cs, h->ev_in, 0));
    return VF_OK;
}
static int leave(vf_clip* h, cudaStream_t user) {
    for (int l = 0; l < h->n_lanes; ++l) {
        VF_CUDA(cudaEventRecord(h->lanes[l].ev_out, h->lanes[l].cs));
        VF_CUDA(cudaStreamWaitEvent(user, h->lanes[l].ev_out, 0));
    }
    return VF_OK;
}

// transform geometry of the CLIP preprocess for a (src_h, src_w) frame
struct ClipGeom { int rh, rw, cy, cx; bool resize; };
static int clip_geometry(int src_h, int src_w, ClipGeom* g) {
    if (src_h <= 0 || src_w <= 0) return fail(VF_ERR_INVALID, "clip: bad frame geometry %dx%d", src_h, src_w);
    VF_TRY(vf_resize_geometry(src_h, src_w, 224, 1, &g->rh, &g->rw));
    g->resize = (g->rh != src_h) || (g->rw != src_w);
    g->cy = center_crop_offset(g->rh, 224);
    g->cx = center_crop_offset(g->rw, 224);
    return VF_OK;
}

// device uint8 frames (c of them, original geometry) -> h->patches
static int clip_transform_chunk(vf_clip* h, const uint8_t* frames, int c, int src_h, int src_w, const ClipGeom& g,
                                cudaStream_t s) {
    ProfScope p(h, 3, s);
    const uint8_t* cur = frames;
    int ch = src_h, cw = src_w;
    if (g.resize) {
        VF_TRY(grow(&h->resized, &h->resized_cap, size_t(h->chunk) * g.rh * g.rw * 3));
        VF_TRY(grow(&h->resize_tmp, &h->tmp_cap, size_t(h->chunk) * src_h * g.rw * 3));
        VF_TRY(resize_u8(frames, c, src_h, src_w, h->resized, g.rh, g.rw, VF_FILTER_BICUBIC, h->resize_tmp, s));
        h->launches += (g.rh != src_h) + (g.rw != src_w);
        cur = h->resized; ch = g.rh; cw = g.rw;
    }
    VF_TRY(launch_clip_patchify(cur, c, ch, cw, g.cy, g.cx, h->patches, h->patch, s));
    h->launches += 1;
    return VF_OK;
}

}  // namespace vf

using namespace vf;

extern "C" {

int vf_clip_create(vf_clip_t** out, const vf_clip_weights* w, int device, int chunk_frames) {
    return vf_clip_create_vit(out, w, device, chunk_frames, 32);
}

int vf_clip_create_vit(vf_clip_t** out, const vf_clip_weights* w, int device, int chunk_frames, int patch_size) {
    if (!out || !w) return fail(VF_ERR_INVALID, "clip_create: null argument");
    *out = nullptr;
    if (patch_size != 32 && patch_size != 16)
        return fail(VF_ERR_UNSUPPORTED, "clip_create: patch size %d (ViT-B/32 and ViT-B/16 are built)", patch_size);
    // default chunk: 256 frames (a 1000-frame call runs as 4 balanced chunks of 250 = 12.5 k token rows, 98 M-tiles of
    // 128 rows: 9 waves of the fc1 GEMM over 132 SMs, 1500 fused QKV + attention tiles).  Measured on one H100 at a 400 W
    // power limit (bench.py --chunk, 20 steps): 128 / 250 / 500 / 1000 frames per chunk give 21.5 / 23.0 / 22.3 / 21.9 k
    // frames/s -- larger chunks gain no GEMM efficiency and lose overlap of the copies with the tower.
    if (chunk_frames <= 0) chunk_frames = patch_size == 32 ? 256 : 126;
    if (chunk_frames > 4096) return fail(VF_ERR_INVALID, "clip_create: chunk_frames %d too large", chunk_frames);
    VF_CUDA(cudaSetDevice(device));
    int major = 0, minor = 0;
    VF_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    VF_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    if (major != 9 || minor != 0)
        return fail(VF_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device, major, minor);
    vf_clip* h = new vf_clip();
    h->device = device;
    h->chunk = chunk_frames;
    h->patch = patch_size;
    h->P = (224 / patch_size) * (224 / patch_size);
    h->T = h->P + 1;
    h->PK = 3 * patch_size * patch_size;
    const int T = h->T, P = h->P, PK = h->PK;
    int st = VF_OK;
    auto body = [&]() -> int {
        VF_TRY(upload_f16(h, &h->w_patch, w->conv1_w, W, PK, false));
        VF_TRY(upload_f16(h, &h->w_proj, w->proj, W, E, true));
        VF_TRY(upload_f32(h, &h->pos, w->positional_embedding, size_t(T) * W));
        if (!w->class_embedding) return fail(VF_ERR_INVALID, "clip_create: missing class_embedding");
        {
            std::vector<float> c0(W);
            for (int i = 0; i < W; ++i) c0[i] = w->class_embedding[i] + w->positional_embedding[i];
            VF_TRY(upload_f32(h, &h->cls_pos0, c0.data(), W));
        }
        VF_TRY(upload_f32(h, &h->lnpre_w, w->ln_pre_w, W));
        VF_TRY(upload_f32(h, &h->lnpre_b, w->ln_pre_b, W));
        VF_TRY(upload_f32(h, &h->lnpost_w, w->ln_post_w, W));
        VF_TRY(upload_f32(h, &h->lnpost_b, w->ln_post_b, W));
        for (int l = 0; l < L; ++l) {
            const vf_clip_layer_weights& s = w->layers[l];
            ClipLayerDev& d = h->layer[l];
            VF_TRY(upload_f32(h, &d.ln1_w, s.ln_1_w, W));
            VF_TRY(upload_f32(h, &d.ln1_b, s.ln_1_b, W));
            VF_TRY(upload_f32(h, &d.ln2_w, s.ln_2_w, W));
            VF_TRY(upload_f32(h, &d.ln2_b, s.ln_2_b, W));
            VF_TRY(upload_f32(h, &d.b_qkv, s.in_proj_b, 3 * W));
            VF_TRY(upload_f32(h, &d.b_o, s.out_proj_b, W));
            VF_TRY(upload_f32(h, &d.b_fc, s.c_fc_b, MLPW));
            VF_TRY(upload_f32(h, &d.b_proj, s.c_proj_b, W));
            VF_TRY(upload_f16(h, &d.w_qkv, s.in_proj_w, 3 * W, W, false));
            {
                if (!s.in_proj_w || !s.in_proj_b) return fail(VF_ERR_INVALID, "clip_create: missing weight tensor");
                std::vector<float> wp(size_t(3) * W * W), bp(3 * W);
                for (int hd = 0; hd < H; ++hd)
                    for (int part = 0; part < 3; ++part)
                        for (int dd = 0; dd < 64; ++dd) {
                            const size_t src = size_t(part) * W + hd * 64 + dd, dst = size_t(hd) * 192 + part * 64 + dd;
                            memcpy(&wp[dst * W], &s.in_proj_w[src * W], W * sizeof(float));
                            bp[dst] = s.in_proj_b[src];
                        }
                VF_TRY(upload_f16(h, &d.w_qkv_heads, wp.data(), 3 * W, W, false));
                VF_TRY(upload_f32(h, &d.b_qkv_heads, bp.data(), 3 * W));
            }
            VF_TRY(upload_f16(h, &d.w_o, s.out_proj_w, W, W, false));
            VF_TRY(upload_f16(h, &d.w_fc, s.c_fc_w, MLPW, W, false));
            VF_TRY(upload_f16(h, &d.w_proj, s.c_proj_w, W, MLPW, false));
        }
        const size_t C = size_t(chunk_frames);
        {
            // the persistent GEMM leaves no room for co-resident blocks, so one lane is the default and the second is
            // opt-in for experiments
            const char* e = getenv("VF_CLIP_LANES");
            h->n_lanes = (e && e[0] == '2') ? 2 : 1;
        }
        for (int l = 0; l < h->n_lanes; ++l) {
            vf_clip::Lane& L = h->lanes[l];
            VF_TRY(dev_alloc(h, &L.patches, C * P * PK));
            VF_TRY(dev_alloc(h, &L.x, C * T * W));
            VF_TRY(dev_alloc(h, &L.y, C * T * W));
            VF_TRY(dev_alloc(h, &L.emb, C * P * W));
            VF_TRY(dev_alloc(h, &L.h, C * T * W));
            VF_TRY(dev_alloc(h, &L.qkv, C * T * 3 * W));
            VF_TRY(dev_alloc(h, &L.att, C * T * W));
            VF_TRY(dev_alloc(h, &L.mlp, C * T * MLPW));
            VF_TRY(dev_alloc(h, &L.cls, C * W));
            VF_TRY(dev_alloc(h, &L.feat, C * E));
            VF_CUDA(cudaStreamCreateWithFlags(&L.cs, cudaStreamNonBlocking));
            VF_CUDA(cudaEventCreateWithFlags(&L.ev_out, cudaEventDisableTiming));
        }
        VF_CUDA(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
        {
            const char* e = getenv("VF_NO_GRAPH");
            h->use_graph = !(e && e[0] == '1');
            const char* r = getenv("VF_CLIP_RESID");     // acc (default) | y | mix (reduction for the MLP only)
            h->acc_o = !(r && (r[0] == 'y' || r[0] == 'm'));
            h->acc_m = !(r && r[0] == 'y');
            const char* a = getenv("VF_CLIP_ATTN");
            h->fused_attn = !(a && a[0] == 's') && T == 50;     // the fused kernel is built for 50-token frames
        }
        activate(h, 0);
        VF_CUDA(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            VF_CUDA(cudaEventCreateWithFlags(&h->ev_copy[i], cudaEventDisableTiming));
            VF_CUDA(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
        }
        for (int i = 0; i < vf_clip::kTickets; ++i)
            VF_CUDA(cudaEventCreateWithFlags(&h->ev_ticket[i], cudaEventDisableTiming | cudaEventBlockingSync));
        return VF_OK;
    };
    st = body();
    if (st != VF_OK) { vf_clip_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_clip_destroy(vf_clip_t* h) {
    if (!h) return VF_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (void* p : h->allocs) cudaFree(p);
    if (h->stage_u8) cudaFree(h->stage_u8);
    if (h->out_dev) cudaFree(h->out_dev);
    for (cudaEvent_t e : h->prof_events) cudaEventDestroy(e);
    deactivate(h);
    for (int l = 0; l < 2; ++l) {
        vf_clip::Lane& L = h->lanes[l];
        for (auto& kv : L.graphs) cudaGraphExecDestroy(kv.second);
        if (L.cs) cudaStreamDestroy(L.cs);
        if (L.ev_out) cudaEventDestroy(L.ev_out);
        if (L.resized) cudaFree(L.resized);
        if (L.resize_tmp) cudaFree(L.resize_tmp);
    }
    h->resized = nullptr; h->resize_tmp = nullptr;
    if (h->ev_in) cudaEventDestroy(h->ev_in);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    for (int i = 0; i < 2; ++i) {
        if (h->ev_copy[i]) cudaEventDestroy(h->ev_copy[i]);
        if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]);
    }
    for (int i = 0; i < vf_clip::kTickets; ++i)
        if (h->ev_ticket[i]) cudaEventDestroy(h->ev_ticket[i]);
    delete h;
    return VF_OK;
}

int vf_clip_encode_f32(vf_clip_t* h, const float* frames, int n, float* out, void* stream) {
    if (!h || (n > 0 && (!frames || !out))) return fail(VF_ERR_INVALID, "clip_encode_f32: null argument");
    if (n <= 0) return VF_OK;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    VF_TRY(enter(h, user));
    const int step = balanced_chunk(h, n);
    for (int b0 = 0, i = 0; b0 < n; b0 += step, ++i) {
        const int c = (n - b0 < step) ? (n - b0) : step;
        LaneScope lane(h, i % h->n_lanes);
        cudaStream_t s = lane.s;
        VF_TRY(launch_clip_patchify_f32(frames + size_t(b0) * 3 * 224 * 224, c, h->patches, h->patch, s));
        h->launches += 1;
        VF_TRY(clip_tower_chunk(h, c, out + size_t(b0) * E, s));
    }
    return leave(h, user);
}

int vf_clip_encode_u8(vf_clip_t* h, const uint8_t* frames, int n, int src_h, int src_w, float* out, void* stream) {
    if (!h || (n > 0 && (!frames || !out))) return fail(VF_ERR_INVALID, "clip_encode_u8: null argument");
    if (n <= 0) return VF_OK;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    ClipGeom g;
    VF_TRY(clip_geometry(src_h, src_w, &g));
    VF_TRY(enter(h, user));
    const size_t fbytes = size_t(src_h) * src_w * 3;
    const int step = balanced_chunk(h, n);
    for (int b0 = 0, i = 0; b0 < n; b0 += step, ++i) {
        const int c = (n - b0 < step) ? (n - b0) : step;
        LaneScope lane(h, i % h->n_lanes);
        cudaStream_t s = lane.s;
        VF_TRY(clip_transform_chunk(h, frames + size_t(b0) * fbytes, c, src_h, src_w, g, s));
        VF_TRY(clip_tower_chunk(h, c, out + size_t(b0) * E, s));
    }
    return leave(h, user);
}

// ticket == nullptr: synchronous (returns when the host buffers may be reused / read).  Otherwise the call returns once
// everything is enqueued and *ticket names it for vf_clip_wait; the staging slots, the feature buffer and the streams
// are shared with the calls still in flight, ordered by events, so the first H2D copy of call k+1 overlaps the last
// tower chunk of call k.
static int clip_encode_u8_host(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_host,
                               float* out_dev, void* stream, int64_t* ticket) {
    if (!h || (n > 0 && (!frames_host || (!out_host && !out_dev))))
        return fail(VF_ERR_INVALID, "clip_encode_u8_host: null argument");
    if (n <= 0) {
        if (ticket) *ticket = -1;              // nothing enqueued: vf_clip_wait(-1) returns at once
        return VF_OK;
    }
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    ClipGeom g;
    VF_TRY(clip_geometry(src_h, src_w, &g));
    VF_TRY(enter(h, user));
    const size_t fbytes = size_t(src_h) * src_w * 3;
    // two staging slots: the H2D copy of chunk i+1 (copy stream) overlaps the tower on chunk i (compute stream).
    // (a re-allocation frees the old buffer with cudaFree, which waits for the calls in flight)
    VF_TRY(grow(&h->stage_u8, &h->stage_cap, 2 * size_t(h->chunk) * fbytes));
    float* feats = out_dev;                 // the caller's device buffer, else the handle's own
    if (!feats) {
        if (h->out_cap < size_t(n) * E * sizeof(float)) {
            if (h->out_dev) cudaFree(h->out_dev);
            h->out_dev = nullptr; h->out_cap = 0;
            VF_CUDA(cudaMalloc(reinterpret_cast<void**>(&h->out_dev), size_t(n) * E * sizeof(float)));
            h->out_cap = size_t(n) * E * sizeof(float);
        }
        feats = h->out_dev;
    }
    const int step = balanced_chunk(h, n);
    const int nchunks = (n + step - 1) / step;
    // the staging copies read HOST memory that is ready now: they are not ordered behind the caller's stream (which, after
    // an asynchronous call, waits for that call's tower) -- only behind the staging slot's previous user
    if (fbytes != h->stage_fbytes) {
        // another frame size moves the boundary between the two slots: a slot of this call may overlap EITHER slot of a
        // call still in flight, so the first copy waits for both
        VF_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_done[0], 0));
        VF_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_done[1], 0));
        h->stage_fbytes = fbytes;
    }
    for (int i = 0; i < nchunks; ++i) {
        const int b0 = i * step;
        const int c = (n - b0 < step) ? (n - b0) : step;
        const int slot = i & 1;
        LaneScope lane(h, i % h->n_lanes);
        cudaStream_t s = lane.s;
        uint8_t* dst = h->stage_u8 + size_t(slot) * h->chunk * fbytes;
        // slot free again: its previous user (an earlier chunk of this call, or of a call still in flight) has been
        // transformed.  Waiting on a never-recorded event is a no-op.
        VF_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_done[slot], 0));
        VF_CUDA(cudaMemcpyAsync(dst, frames_host + size_t(b0) * fbytes, size_t(c) * fbytes, cudaMemcpyHostToDevice,
                                h->copy_stream));
        VF_CUDA(cudaEventRecord(h->ev_copy[slot], h->copy_stream));
        VF_CUDA(cudaStreamWaitEvent(s, h->ev_copy[slot], 0));
        VF_TRY(clip_transform_chunk(h, dst, c, src_h, src_w, g, s));
        VF_CUDA(cudaEventRecord(h->ev_done[slot], s));   // staging slot consumed
        VF_TRY(clip_tower_chunk(h, c, feats + size_t(b0) * E, s));
    }
    // gather point: lane 0 waits for lane 1, then one D2H of all features
    cudaStream_t s0 = h->lanes[0].cs;
    if (h->n_lanes > 1) {
        VF_CUDA(cudaEventRecord(h->lanes[1].ev_out, h->lanes[1].cs));
        VF_CUDA(cudaStreamWaitEvent(s0, h->lanes[1].ev_out, 0));
    }
    if (out_host)
        VF_CUDA(cudaMemcpyAsync(out_host, feats, size_t(n) * E * sizeof(float), cudaMemcpyDeviceToHost, s0));
    if (ticket) {
        // everything this call reads from / writes to the host is complete once s0 reaches this point (the tower
        // depends on every staging copy)
        const int64_t t = h->seq.load();
        cudaEvent_t ev = h->ev_ticket[t % vf_clip::kTickets];
        if (t >= vf_clip::kTickets) VF_CUDA(cudaEventSynchronize(ev));          // at most kTickets calls in flight
        VF_CUDA(cudaEventRecord(ev, s0));
        *ticket = t;
        h->seq.store(t + 1);
        return leave(h, user);
    }
    VF_TRY(leave(h, user));
    // the host frames may be reused (and out_host read) as soon as this returns
    VF_CUDA(cudaStreamSynchronize(out_host ? s0 : h->copy_stream));
    return VF_OK;
}

int vf_clip_encode_u8_host(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_host,
                           void* stream) {
    if (n > 0 && !out_host) return fail(VF_ERR_INVALID, "clip_encode_u8_host: null argument");
    return clip_encode_u8_host(h, frames_host, n, src_h, src_w, out_host, nullptr, stream, nullptr);
}

int vf_clip_encode_u8_host_dev(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_dev,
                               float* out_host, void* stream) {
    if (n > 0 && !out_dev) return fail(VF_ERR_INVALID, "clip_encode_u8_host_dev: null device output");
    return clip_encode_u8_host(h, frames_host, n, src_h, src_w, out_host, out_dev, stream, nullptr);
}

int vf_clip_encode_u8_host_async(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_dev,
                                 float* out_host, void* stream, int64_t* ticket) {
    if (!ticket) return fail(VF_ERR_INVALID, "clip_encode_u8_host_async: null ticket");
    return clip_encode_u8_host(h, frames_host, n, src_h, src_w, out_host, out_dev, stream, ticket);
}

int vf_clip_wait(vf_clip_t* h, int64_t ticket) {
    if (!h) return fail(VF_ERR_INVALID, "clip_wait: null handle");
    if (ticket < 0) return VF_OK;
    if (ticket >= h->seq.load()) return fail(VF_ERR_INVALID, "clip_wait: ticket %lld was never issued", (long long)ticket);
    if (ticket + vf_clip::kTickets < h->seq.load())
        return VF_OK;                          // its event has been reused: that only happens after it completed
    VF_CUDA(cudaEventSynchronize(h->ev_ticket[ticket % vf_clip::kTickets]));
    return VF_OK;
}

int vf_clip_block_attention(vf_clip_t* h, int layer, const void* x, int n_frames, void* out, int fused, void* stream) {
    if (!h || !x || !out) return fail(VF_ERR_INVALID, "clip_block_attention: null argument");
    if (layer < 0 || layer >= L || n_frames <= 0 || n_frames > h->chunk)
        return fail(VF_ERR_INVALID, "clip_block_attention: layer %d / %d frames outside the handle's limits", layer, n_frames);
    if (fused && h->T != 50) return fail(VF_ERR_UNSUPPORTED, "clip_block_attention: the fused kernel needs 50-token frames");
    const int T = h->T;
    VF_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const ClipLayerDev& w = h->layer[layer];
    const __half* xin = static_cast<const __half*>(x);
    __half* o = static_cast<__half*>(out);
    if (fused) return qkv_attention(xin, W, w.w_qkv_heads, w.b_qkv_heads, o, n_frames, H, s);
    __half* qkv = h->lanes[0].qkv;
    VF_TRY(gemm_f16(xin, W, w.w_qkv, W, n_frames * T, 3 * W, W, epi(qkv, 3 * W, 0, w.b_qkv, VF_ACT_NONE), s));
    return launch_attention(qkv, o, n_frames, T, H, s);
}

int64_t vf_clip_launch_count(const vf_clip_t* h) { return h ? h->launches : 0; }

int vf_clip_profile(vf_clip_t* h, int enable) {
    if (!h) return fail(VF_ERR_INVALID, "clip_profile: null handle");
    h->prof = enable != 0;
    return VF_OK;
}

int vf_clip_profile_read(vf_clip_t* h, double* gemm_ms, int64_t* gemm_launches, double* gemm_flops) {
    if (!h) return fail(VF_ERR_INVALID, "clip_profile_read: null handle");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaDeviceSynchronize());
    double ms[4] = {0, 0, 0, 0};
    int64_t n_gemm = 0;
    for (size_t i = 0; i + 1 < h->prof_used; i += 2) {
        float t = 0.f;
        VF_CUDA(cudaEventElapsedTime(&t, h->prof_events[i], h->prof_events[i + 1]));
        const int cat = h->prof_cat[i / 2];
        ms[cat] += t;
        n_gemm += (cat == 0);
    }
    for (int i = 0; i < 4; ++i) h->prof_cat_ms[i] = ms[i];
    if (gemm_ms) *gemm_ms = ms[0];
    if (gemm_launches) *gemm_launches = n_gemm;
    if (gemm_flops) *gemm_flops = h->prof_flops;
    h->prof_used = 0;
    h->prof_flops = 0.0;
    return VF_OK;
}

int vf_clip_profile_categories(const vf_clip_t* h, double* ms4) {
    if (!h || !ms4) return fail(VF_ERR_INVALID, "clip_profile_categories: null argument");
    for (int i = 0; i < 4; ++i) ms4[i] = h->prof_cat_ms[i];
    return VF_OK;
}

}  // extern "C"
