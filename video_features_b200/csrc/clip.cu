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

struct vf_clip : vf::EngineCore {
    int chunk = 0;
    int patch = 32, T = 50, P = 49, PK = 3072;   // patch size, tokens (P + 1), patches per frame, patch-matrix columns
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
    float* feat = nullptr;                // [chunk, 512] tower output
    // host-buffer entries: two staging slots of frames (grown on demand)
    uint8_t* stage_u8 = nullptr;
    size_t stage_cap = 0;
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
    // All work of a call runs on the engine stream `cs` (ordered against the caller's stream with a pair of events), so
    // that the per-chunk tower can be captured once into a CUDA graph and replayed: ~90 kernel launches and ~150
    // tensor-map encodes per chunk collapse into one cudaGraphLaunch (the legacy NULL stream, which is what torch hands
    // over by default, cannot be captured).
    bool acc_o = true, acc_m = true;          // residual adds in the GEMM epilogue (fp32 reductions) instead of an fp16 y
    bool fused_attn = true;                   // QKV projection + attention in one kernel (VF_CLIP_ATTN=split: GEMM + kernel)
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copy[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
    // asynchronous host calls (vf_clip_encode_u8_host_async): completion events of the last kTickets calls
    static constexpr int kTickets = 4;
    cudaEvent_t ev_ticket[kTickets] = {nullptr, nullptr, nullptr, nullptr};
    std::atomic<int64_t> seq{0};              // vf_clip_wait may run on another host thread than the enqueuing one
};

namespace vf {

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

// The tower on one chunk is three pieces -- embed, blocks, head -- that vf_clip_debug_embed / _blocks / _head also run one
// at a time (the float64 tests hold each to a reference of its own).
// GEMM epilogues never read global memory: bias / QuickGELU in registers, then global stores -- or, for the two GEMMs
// that end a residual branch, fp32 reductions that add the tile into the fp32 residual stream x.

// h->patches (c frames) -> h->x: the patch-embedding GEMM, then token assembly + ln_pre
static int tower_embed(vf_clip* h, int c, cudaStream_t s) {
    const int P = h->P, PK = h->PK;
    // patch embedding: [c*P, PK] x [768, PK]^T -> emb (fp32)
    VF_TRY(tower_gemm(h, h->patches, PK, h->w_patch, PK, c * P, W, PK, linear_epi(h->emb, W, 1, nullptr, VF_ACT_NONE), s));
    // token assembly (+ class / positional embedding) fused with ln_pre -> x
    VF_TRY(tower_embed_ln(h, c, s));
    h->launches += 2;
    return VF_OK;
}

// resblocks [l0, l1) on h->x.  In the y forms the MLP increment of block l1 - 1 is left in h->y, not yet added (the next
// ln_1, or the head, adds it); h->x must hold no such pending increment on entry.
static int tower_blocks(vf_clip* h, int c, int l0, int l1, cudaStream_t s) {
    const int T = h->T;
    const int M = c * T;
    // The residual stream x stays fp32 in HBM.  A GEMM that ends a residual branch either ADDS its result into x from the
    // epilogue (fp32 global reductions; the LayerNorm pass that follows then only reads x and writes h: 6 bytes per
    // element), or writes an fp16 increment y that the LayerNorm kernel adds ("x += y; h = LN(x)": 12 bytes per element).
    // acc_o / acc_m select the form for the attention out-projection / the MLP's second GEMM (VF_CLIP_RESID=acc|y|mix).
    const bool acc_o = h->acc_o, acc_m = h->acc_m;
    for (int l = l0; l < l1; ++l) {
        const ClipLayerDev& w = h->layer[l];
        // h = ln_1(x)   (y form: x += y of the previous block's MLP first)
        VF_TRY(tower_add_ln(h, h->x, W, (acc_m || l == l0) ? nullptr : h->y, W, 1, w.ln1_w, w.ln1_b, h->h, W, M, s));
        if (h->fused_attn) {
            VF_TRY(tower_qkv_attention(h, w, c, s));
        } else {
            VF_TRY(tower_gemm(h, h->h, W, w.w_qkv, W, M, 3 * W, W, linear_epi(h->qkv, 3 * W, 0, w.b_qkv, VF_ACT_NONE), s));
            VF_TRY(tower_attention(h, c, s));
        }
        // Last block: only the CLS token reaches ln_post / proj (encode_image returns x[:, 0]), so after the attention
        // everything runs on the c CLS rows: A operands and the residual rows are strided views (row pitch T*768), h /
        // mlp / y are compact c-row buffers.  Saves (T-1)/T of out-proj + MLP of this block (5.9 % of the FLOPs at T = 50).
        const bool last = l + 1 == L;
        const int rows = last ? c : M;
        const int a_ld = last ? T * W : W;                    // row pitch of att / x when only the CLS rows are read
        if (acc_o) {
            VF_TRY(tower_gemm(h, h->att, a_ld, w.w_o, W, rows, W, W, linear_epi(h->x, a_ld, 1, w.b_o, VF_ACT_NONE, 1), s));
            VF_TRY(tower_add_ln(h, h->x, a_ld, nullptr, W, 0, w.ln2_w, w.ln2_b, h->h, W, rows, s));
        } else {
            VF_TRY(tower_gemm(h, h->att, a_ld, w.w_o, W, rows, W, W, linear_epi(h->y, W, 0, w.b_o, VF_ACT_NONE), s));
            VF_TRY(tower_add_ln(h, h->x, a_ld, h->y, W, 1, w.ln2_w, w.ln2_b, h->h, W, rows, s));
        }
        VF_TRY(tower_gemm(h, h->h, W, w.w_fc, W, rows, MLPW, W, linear_epi(h->mlp, MLPW, 0, w.b_fc, VF_ACT_QUICKGELU), s));
        if (acc_m) VF_TRY(tower_gemm(h, h->mlp, MLPW, w.w_proj, MLPW, rows, W, MLPW, linear_epi(h->x, a_ld, 1, w.b_proj, VF_ACT_NONE, 1), s));
        else       VF_TRY(tower_gemm(h, h->mlp, MLPW, w.w_proj, MLPW, rows, W, MLPW, linear_epi(h->y, W, 0, w.b_proj, VF_ACT_NONE), s));
        h->launches += h->fused_attn ? 6 : 7;
    }
    return VF_OK;
}

// CLS rows of h->x (row pitch T*768): (y != nullptr: + the last MLP's increment, compact rows of pitch 768;) ln_post; then
// the 768 -> 512 projection -> out (c x 512 fp32)
static int tower_head(vf_clip* h, int c, const __half* y, float* out, cudaStream_t s) {
    VF_TRY(tower_add_ln(h, h->x, int64_t(h->T) * W, y, W, 0, h->lnpost_w, h->lnpost_b, h->cls, W, c, s));
    VF_TRY(tower_gemm(h, h->cls, W, h->w_proj, W, c, E, W, linear_epi(out, E, 1, nullptr, VF_ACT_NONE), s));
    h->launches += 2;
    return VF_OK;
}

// The tower on one chunk whose patch matrix is already in h->patches; writes c x 512 fp32 to out.
static int clip_tower_eager(vf_clip* h, int c, float* out, cudaStream_t s) {
    VF_TRY(tower_embed(h, c, s));
    VF_TRY(tower_blocks(h, c, 0, L, s));
    return tower_head(h, c, h->acc_m ? nullptr : h->y, out, s);
}

// device uint8 frames (c of them, original geometry) -> h->patches
static int clip_transform_chunk(vf_clip* h, const uint8_t* frames, int c, int src_h, int src_w, const FrameGeom& g,
                                cudaStream_t s) {
    ProfScope p(h, 3, s);
    const uint8_t* src;
    VF_TRY(resize_frames(h, frames, c, src_h, src_w, g, h->chunk, s, &src));
    VF_TRY(launch_clip_patchify(src, c, g.rh, g.rw, g.cy, g.cx, h->patches, h->patch, s));
    h->launches += 1;
    return VF_OK;
}

// The tower on one chunk whose patch matrix is in h->patches -> out (c x 512): through the graph cache (a chunk size is
// captured the second time it shows up, so one-off sizes -- the ragged tail of a list, batches of videos of unequal
// length -- run eagerly instead of paying capture + instantiation for a graph that is never replayed), eagerly while
// profiling (vf_clip_profile brackets launches with events).
static int clip_tower_run(vf_clip* h, int c, float* out) {
    auto tower = [&] { return clip_tower_eager(h, c, h->feat, h->cs); };
    VF_TRY(h->prof ? tower() : run_graphed(h, {c, 0, 0, 0}, tower));
    VF_CUDA(cudaMemcpyAsync(out, h->feat, size_t(c) * E * sizeof(float), cudaMemcpyDeviceToDevice, h->cs));
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
    VF_TRY(check_device(device));
    vf_clip* h = new vf_clip();
    h->who = "clip_create";
    h->device = device;
    h->chunk = chunk_frames;
    h->capture_after = 2;            // one-off chunk sizes run eagerly
    h->max_graphs = 32;
    h->evict_when_full = false;
    h->patch = patch_size;
    h->P = (224 / patch_size) * (224 / patch_size);
    h->T = h->P + 1;
    h->PK = 3 * patch_size * patch_size;
    const int T = h->T, P = h->P, PK = h->PK;
    int st = VF_OK;
    auto body = [&]() -> int {
        VF_TRY(upload_f16(h, &h->w_patch, w->conv1_w, W, PK));
        VF_TRY(upload_f16(h, &h->w_proj, w->proj, E, W, W, true));
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
            VF_TRY(upload_f16(h, &d.w_qkv, s.in_proj_w, 3 * W, W));
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
                VF_TRY(upload_f16(h, &d.w_qkv_heads, wp.data(), 3 * W, W));
                VF_TRY(upload_f32(h, &d.b_qkv_heads, bp.data(), 3 * W));
            }
            VF_TRY(upload_f16(h, &d.w_o, s.out_proj_w, W, W));
            VF_TRY(upload_f16(h, &d.w_fc, s.c_fc_w, MLPW, W));
            VF_TRY(upload_f16(h, &d.w_proj, s.c_proj_w, W, MLPW));
        }
        const size_t C = size_t(chunk_frames);
        VF_TRY(ralloc(h, &h->patches, C * P * PK));
        VF_TRY(ralloc(h, &h->x, C * T * W));
        VF_TRY(ralloc(h, &h->y, C * T * W));
        VF_TRY(ralloc(h, &h->emb, C * P * W));
        VF_TRY(ralloc(h, &h->h, C * T * W));
        VF_TRY(ralloc(h, &h->qkv, C * T * 3 * W));
        VF_TRY(ralloc(h, &h->att, C * T * W));
        VF_TRY(ralloc(h, &h->mlp, C * T * MLPW));
        VF_TRY(ralloc(h, &h->cls, C * W));
        VF_TRY(ralloc(h, &h->feat, C * E));
        VF_TRY(open_stream(h));
        {
            const char* r = getenv("VF_CLIP_RESID");     // acc (default) | y | mix (reduction for the MLP only)
            h->acc_o = !(r && (r[0] == 'y' || r[0] == 'm'));
            h->acc_m = !(r && r[0] == 'y');
            const char* a = getenv("VF_CLIP_ATTN");
            h->fused_attn = !(a && a[0] == 's') && T == 50;     // the fused kernel is built for 50-token frames
        }
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
    release(h);
    if (h->stage_u8) cudaFree(h->stage_u8);
    if (h->out_dev) cudaFree(h->out_dev);
    for (cudaEvent_t e : h->prof_events) cudaEventDestroy(e);
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
    const int step = balanced_step(n, h->chunk);
    for (int b0 = 0; b0 < n; b0 += step) {
        const int c = (n - b0 < step) ? (n - b0) : step;
        VF_TRY(launch_clip_patchify_f32(frames + size_t(b0) * 3 * 224 * 224, c, h->patches, h->patch, h->cs));
        h->launches += 1;
        VF_TRY(clip_tower_run(h, c, out + size_t(b0) * E));
    }
    return leave(h, user);
}

int vf_clip_encode_u8(vf_clip_t* h, const uint8_t* frames, int n, int src_h, int src_w, float* out, void* stream) {
    if (!h || (n > 0 && (!frames || !out))) return fail(VF_ERR_INVALID, "clip_encode_u8: null argument");
    if (n <= 0) return VF_OK;
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    FrameGeom g;
    VF_TRY(frame_geometry("clip", src_h, src_w, 224, 224, &g));
    VF_TRY(enter(h, user));
    const size_t fbytes = size_t(src_h) * src_w * 3;
    const int step = balanced_step(n, h->chunk);
    for (int b0 = 0; b0 < n; b0 += step) {
        const int c = (n - b0 < step) ? (n - b0) : step;
        VF_TRY(clip_transform_chunk(h, frames + size_t(b0) * fbytes, c, src_h, src_w, g, h->cs));
        VF_TRY(clip_tower_run(h, c, out + size_t(b0) * E));
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
    FrameGeom g;
    VF_TRY(frame_geometry("clip", src_h, src_w, 224, 224, &g));
    VF_TRY(enter(h, user));
    const size_t fbytes = size_t(src_h) * src_w * 3;
    // two staging slots: the H2D copy of chunk i+1 (copy stream) overlaps the tower on chunk i (engine stream).
    // (a re-allocation frees the old buffer with cudaFree, which waits for the calls in flight)
    VF_TRY(grow(h, &h->stage_u8, &h->stage_cap, 2 * size_t(h->chunk) * fbytes));
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
    const int step = balanced_step(n, h->chunk);
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
        uint8_t* dst = h->stage_u8 + size_t(slot) * h->chunk * fbytes;
        // slot free again: its previous user (an earlier chunk of this call, or of a call still in flight) has been
        // transformed.  Waiting on a never-recorded event is a no-op.
        VF_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_done[slot], 0));
        VF_CUDA(cudaMemcpyAsync(dst, frames_host + size_t(b0) * fbytes, size_t(c) * fbytes, cudaMemcpyHostToDevice,
                                h->copy_stream));
        VF_CUDA(cudaEventRecord(h->ev_copy[slot], h->copy_stream));
        VF_CUDA(cudaStreamWaitEvent(h->cs, h->ev_copy[slot], 0));
        VF_TRY(clip_transform_chunk(h, dst, c, src_h, src_w, g, h->cs));
        VF_CUDA(cudaEventRecord(h->ev_done[slot], h->cs));   // staging slot consumed
        VF_TRY(clip_tower_run(h, c, feats + size_t(b0) * E));
    }
    if (out_host)
        VF_CUDA(cudaMemcpyAsync(out_host, feats, size_t(n) * E * sizeof(float), cudaMemcpyDeviceToHost, h->cs));
    if (ticket) {
        // everything this call reads from / writes to the host is complete once the engine stream reaches this point (the tower
        // depends on every staging copy)
        const int64_t t = h->seq.load();
        cudaEvent_t ev = h->ev_ticket[t % vf_clip::kTickets];
        if (t >= vf_clip::kTickets) VF_CUDA(cudaEventSynchronize(ev));          // at most kTickets calls in flight
        VF_CUDA(cudaEventRecord(ev, h->cs));
        *ticket = t;
        h->seq.store(t + 1);
        return leave(h, user);
    }
    VF_TRY(leave(h, user));
    // the host frames may be reused (and out_host read) as soon as this returns
    VF_CUDA(cudaStreamSynchronize(out_host ? h->cs : h->copy_stream));
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
    VF_TRY(gemm_f16(xin, W, w.w_qkv, W, n_frames * T, 3 * W, W, linear_epi(h->qkv, 3 * W, 0, w.b_qkv, VF_ACT_NONE), s));
    return launch_attention(h->qkv, o, n_frames, T, H, s);
}

// The three pieces of the tower one at a time, eagerly, on the handle's workspace and the caller's stream.
int vf_clip_debug_embed_f32(vf_clip_t* h, const float* frames, int n, float* x_out, void* stream) {
    VF_TRY(debug_frames(h, frames, x_out, n, h ? h->chunk : 0, "chunk", "clip_debug_embed_f32"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_TRY(launch_clip_patchify_f32(frames, n, h->patches, h->patch, s));
    h->launches += 1;
    VF_TRY(tower_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * h->T * W * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_clip_debug_embed_u8(vf_clip_t* h, const uint8_t* frames, int n, int src_h, int src_w, float* x_out, void* stream) {
    VF_TRY(debug_frames(h, frames, x_out, n, h ? h->chunk : 0, "chunk", "clip_debug_embed_u8"));
    FrameGeom g;
    VF_TRY(frame_geometry("clip", src_h, src_w, 224, 224, &g));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_TRY(clip_transform_chunk(h, frames, n, src_h, src_w, g, s));
    VF_TRY(tower_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * h->T * W * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_clip_debug_blocks(vf_clip_t* h, float* x, int n_frames, int layer_begin, int layer_end, void* stream) {
    VF_TRY(debug_frames(h, x, x, n_frames, h ? h->chunk : 0, "chunk", "clip_debug_blocks"));
    if (layer_begin < 0 || layer_begin >= layer_end || layer_end > L)
        return fail(VF_ERR_INVALID, "clip_debug_blocks: layers [%d, %d) are not a range within [0, %d)", layer_begin, layer_end, L);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int T = h->T;
    const size_t bytes = size_t(n_frames) * T * W * sizeof(float);
    VF_CUDA(cudaMemcpyAsync(h->x, x, bytes, cudaMemcpyDeviceToDevice, s));
    VF_TRY(tower_blocks(h, n_frames, layer_begin, layer_end, s));
    if (!h->acc_m) {
        // y forms: add the last MLP's pending increment the way the tower does, with the add + LayerNorm kernel writing x
        // back (x += y); its LayerNorm output lands in scratch (cls / h) and is dropped.  After block 11 the increment is
        // the compact CLS-row buffer and x is addressed at the CLS rows, as the head would.
        const bool cls_only = layer_end == L;
        VF_TRY(tower_add_ln(h, h->x, cls_only ? int64_t(T) * W : W, h->y, W, 1, h->lnpost_w, h->lnpost_b,
                            cls_only ? h->cls : h->h, W, cls_only ? n_frames : n_frames * T, s));
        h->launches += 1;
    }
    VF_CUDA(cudaMemcpyAsync(x, h->x, bytes, cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_clip_debug_head(vf_clip_t* h, const float* x, int n_frames, float* out, void* stream) {
    VF_TRY(debug_frames(h, x, out, n_frames, h ? h->chunk : 0, "chunk", "clip_debug_head"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaMemcpyAsync(h->x, x, size_t(n_frames) * h->T * W * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return tower_head(h, n_frames, nullptr, out, s);
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
