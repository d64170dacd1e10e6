// CLIP ViT-L/14 image towers (224 px: 257 tokens; 336 px: 577 tokens) on the wgmma GEMM, the key-streaming attention
// and 1024-wide LayerNorms of clip_vitl_kernels.cu.  Replaces `clip.load("ViT-L/14" | "ViT-L/14@336px")` and
// `model.encode_image(preprocess(frame))`, the transform Resize(n_px, bicubic) -> CenterCrop(n_px) -> ToTensor ->
// Normalize included (algorithm: third-party openai/CLIP clip/model.py VisionTransformer.forward).  The configuration is
// inferred from the weights' sizes as clip.model.build_model does.
//
// Numerics (as the ViT-B towers of clip.cu): GEMM operands fp16, accumulation fp32; the residual stream, LayerNorm
// statistics, softmax max / sum fp32.  Rounded to fp16: weights, patches, the outputs of ln_1 / ln_2 / ln_post, q / k / v,
// the per-key-block P = exp(s - running max), the attention output and the MLP hidden layer.  The out-projection and
// c_proj add their tiles into the fp32 residual stream from the GEMM epilogue (fp32 reductions).
// Frames are packed along M (row = frame * tokens + token) and run in chunks of at most max_frames frames; each chunk
// size is captured into a CUDA graph the second time it is seen.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "clip_vitl_kernels.h"
#include "internal.h"
#include "split_conv.h"

namespace vf {

constexpr int VL_LAYERS = 24, VL_HEADS = 16, VL_MLP = 4096, VL_EMBED = 768;

struct VitlLayer {
    float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *b_qkv, *b_o, *b_fc, *b_proj;
    __half *w_qkv, *w_o, *w_fc, *w_proj;
};

}  // namespace vf

using namespace vf;

struct vf_clip_vitl : vf::EngineCore {
    int max_frames = 0, npx = 0, tokens = 0, patches_per_frame = 0;
    // weights
    __half* w_patch = nullptr;      // [1024, VITL_PK] (conv1, zero columns 588..591)
    __half* w_proj = nullptr;       // [768, 1024] (proj^T)
    float *pos = nullptr, *cls_pos0 = nullptr, *lnpre_w = nullptr, *lnpre_b = nullptr, *lnpost_w = nullptr,
          *lnpost_b = nullptr;
    VitlLayer layer[VL_LAYERS];
    // workspace (max_frames frames)
    __half *patches = nullptr, *h = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr, *cls = nullptr;
    float *x = nullptr, *emb = nullptr, *feat = nullptr;
};

namespace vf {

// h->patches (c frames) -> h->x: patch-embedding GEMM, then token assembly + ln_pre
static int vl_embed(vf_clip_vitl* h, int c, cudaStream_t s) {
    const int P = h->patches_per_frame;
    VF_TRY(gemm_f16(h->patches, VITL_PK, h->w_patch, VITL_PK, c * P, VITL_W, VITL_PK,
                    linear_epi(h->emb, VITL_W, 1, nullptr, VF_ACT_NONE), s));
    VF_TRY(vitl_embed_layernorm(h->emb, h->pos, h->cls_pos0, h->lnpre_w, h->lnpre_b, h->x, c, h->tokens, s));
    h->launches += 2;
    return VF_OK;
}

// resblocks [l0, l1) on h->x.  The last block of the tower runs its out-projection and MLP on the c class rows only
// (encode_image returns x[:, 0]); those rows of x are then read in place with a row pitch of T tokens.
static int vl_blocks(vf_clip_vitl* h, int c, int l0, int l1, cudaStream_t s) {
    const int T = h->tokens, W = VITL_W, M = c * T;
    for (int l = l0; l < l1; ++l) {
        const VitlLayer& w = h->layer[l];
        VF_TRY(vitl_layernorm(h->x, W, w.ln1_w, w.ln1_b, h->h, W, M, s));
        VF_TRY(gemm_f16(h->h, W, w.w_qkv, W, M, 3 * W, W, linear_epi(h->qkv, 3 * W, 0, w.b_qkv, VF_ACT_NONE), s));
        VF_TRY(vitl_attention(h->qkv, h->att, c, T, VL_HEADS, s));
        const bool last = l + 1 == VL_LAYERS;
        const int rows = last ? c : M, a_ld = last ? T * W : W;
        VF_TRY(gemm_f16(h->att, a_ld, w.w_o, W, rows, W, W, linear_epi(h->x, a_ld, 1, w.b_o, VF_ACT_NONE, 1), s));
        VF_TRY(vitl_layernorm(h->x, a_ld, w.ln2_w, w.ln2_b, h->h, W, rows, s));
        VF_TRY(gemm_f16(h->h, W, w.w_fc, W, rows, VL_MLP, W, linear_epi(h->mlp, VL_MLP, 0, w.b_fc, VF_ACT_QUICKGELU), s));
        VF_TRY(gemm_f16(h->mlp, VL_MLP, w.w_proj, VL_MLP, rows, W, VL_MLP, linear_epi(h->x, a_ld, 1, w.b_proj, VF_ACT_NONE, 1), s));
        h->launches += 6;
    }
    return VF_OK;
}

// class rows of h->x (row pitch T * 1024): ln_post, then the 1024 -> 768 projection -> out (c x 768 fp32)
static int vl_head(vf_clip_vitl* h, int c, float* out, cudaStream_t s) {
    VF_TRY(vitl_layernorm(h->x, int64_t(h->tokens) * VITL_W, h->lnpost_w, h->lnpost_b, h->cls, VITL_W, c, s));
    VF_TRY(gemm_f16(h->cls, VITL_W, h->w_proj, VITL_W, c, VL_EMBED, VITL_W, linear_epi(out, VL_EMBED, 1, nullptr, VF_ACT_NONE), s));
    h->launches += 2;
    return VF_OK;
}

static int vl_tower(vf_clip_vitl* h, int c, float* out, cudaStream_t s) {
    VF_TRY(vl_embed(h, c, s));
    VF_TRY(vl_blocks(h, c, 0, VL_LAYERS, s));
    return vl_head(h, c, out, s);
}

static int vl_encode(vf_clip_vitl* h, const void* frames, int is_u8, int n, int H, int W, float* out, void* stream) {
    if (!h || (n > 0 && (!frames || !out))) return fail(VF_ERR_INVALID, "clip_vitl_encode: null argument");
    if (n < 0) return fail(VF_ERR_INVALID, "clip_vitl_encode: %d frames", n);
    if (n == 0) return VF_OK;
    FrameGeom g{h->npx, h->npx, 0, 0, false};
    if (is_u8) VF_TRY(frame_geometry("clip_vitl", H, W, h->npx, h->npx, &g));
    const size_t frame_elems = is_u8 ? size_t(H) * W * 3 : size_t(3) * h->npx * h->npx;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    const int step = balanced_step(n, h->max_frames);
    for (int off = 0; off < n; off += step) {
        const int c = n - off < step ? n - off : step;
        if (is_u8) {
            const uint8_t* src;
            VF_TRY(resize_frames(h, static_cast<const uint8_t*>(frames) + off * frame_elems, c, H, W, g, h->max_frames,
                                 s, &src));
            VF_TRY(vitl_patchify_u8(src, c, g.rh, g.rw, g.cy, g.cx, h->npx, h->patches, s));
        } else {
            VF_TRY(vitl_patchify_f32(static_cast<const float*>(frames) + off * frame_elems, c, h->npx, h->patches, s));
        }
        h->launches += 1;
        VF_TRY(run_graphed(h, {c, 0, 0, 0}, [&] { return vl_tower(h, c, h->feat, s); }));
        VF_CUDA(cudaMemcpyAsync(out + size_t(off) * VL_EMBED, h->feat, size_t(c) * VL_EMBED * sizeof(float),
                                cudaMemcpyDeviceToDevice, s));
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_clip_vitl_destroy(vf_clip_vitl_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_clip_vitl_create(vf_clip_vitl_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "clip_vitl_create: null argument");
    *out = nullptr;
    const ResTensors T{tensors, n_tensors, "clip_vitl_create"};
    // clip.model.build_model: width from conv1 (its output channels, here the class embedding's length, which must
    // agree), patch from conv1's kernel, depth from the resblock keys, heads = width / 64, resolution from the
    // positional embedding, output width from proj
    const int W = VITL_W;
    const int64_t n_cls = T.numel("visual.class_embedding");
    if (n_cls <= 0) return fail(VF_ERR_INVALID, "clip_vitl_create: missing tensor 'visual.class_embedding'");
    const int64_t n_conv = T.numel("visual.conv1.weight");
    if (n_conv <= 0) return fail(VF_ERR_INVALID, "clip_vitl_create: missing tensor 'visual.conv1.weight'");
    if (n_cls != W || n_conv % (3 * n_cls))
        return fail(VF_ERR_UNSUPPORTED, "clip_vitl_create: tensors 'visual.conv1.weight' (%lld elements) and "
                    "'visual.class_embedding' (%lld) give width %lld; the ViT-L/14 towers are %d wide",
                    (long long)n_conv, (long long)n_cls, (long long)n_cls, W);
    const int64_t kk = n_conv / (3 * W);
    const int patch = int(lround(sqrt(double(kk))));
    if (int64_t(patch) * patch != kk || patch != VITL_PATCH)
        return fail(VF_ERR_UNSUPPORTED, "clip_vitl_create: tensor 'visual.conv1.weight' has %lld elements, not "
                    "%d x 3 x 14 x 14 (patch 14 is built)", (long long)n_conv, W);
    int depth = 0;
    while (T.numel("visual.transformer.resblocks." + std::to_string(depth) + ".attn.in_proj_weight") > 0) ++depth;
    if (depth != VL_LAYERS)
        return fail(depth < VL_LAYERS ? VF_ERR_INVALID : VF_ERR_UNSUPPORTED,
                    "clip_vitl_create: tensor 'visual.transformer.resblocks.%d.attn.in_proj_weight' %s: %d resblocks "
                    "(24 are built)", depth < VL_LAYERS ? depth : VL_LAYERS, depth < VL_LAYERS ? "missing" : "present",
                    depth);
    const int64_t n_pos = T.numel("visual.positional_embedding");
    if (n_pos <= 0) return fail(VF_ERR_INVALID, "clip_vitl_create: missing tensor 'visual.positional_embedding'");
    const int64_t cells = n_pos / W - 1;
    const int grid = int(lround(sqrt(double(cells > 0 ? cells : 0))));
    if (n_pos % W || cells < 1 || int64_t(grid) * grid != cells)
        return fail(VF_ERR_INVALID, "clip_vitl_create: tensor 'visual.positional_embedding' has %lld elements, not "
                    "(g^2 + 1) x %d (a square patch grid)", (long long)n_pos, W);
    const int npx = VITL_PATCH * grid;
    if (npx != 224 && npx != 336)
        return fail(VF_ERR_UNSUPPORTED, "clip_vitl_create: tensor 'visual.positional_embedding' gives n_px %d "
                    "(224 and 336 are built)", npx);
    const int64_t n_proj = T.numel("visual.proj");
    if (n_proj != int64_t(W) * VL_EMBED)
        return fail(n_proj <= 0 ? VF_ERR_INVALID : VF_ERR_UNSUPPORTED, "clip_vitl_create: tensor 'visual.proj' has %lld "
                    "elements, not %d x %d", (long long)n_proj, W, VL_EMBED);
    // workspace per frame: patches 2 * 592 P, emb 4 * 1024 P, x 4 * 1024 T, h / att 2 * 1024 T each, qkv 2 * 3072 T,
    // mlp 2 * 4096 T bytes (+ 2 * 1024 + 4 * 768 of class rows): 7.1 MB at 224 px, 16.0 MB at 336 px.  The default keeps
    // it near 2.5 GB.
    if (max_frames <= 0) max_frames = npx == 224 ? 352 : 160;
    if (max_frames > 4096) return fail(VF_ERR_INVALID, "clip_vitl_create: max_frames %d too large", max_frames);
    VF_TRY(check_device(device));
    vf_clip_vitl* h = new vf_clip_vitl();
    h->who = "clip_vitl_create";
    h->device = device; h->max_frames = max_frames; h->npx = npx;
    h->patches_per_frame = grid * grid; h->tokens = grid * grid + 1;
    h->capture_after = 2;            // one-off chunk sizes run eagerly
    h->evict_when_full = false;
    auto body = [&]() -> int {
        const int Tk = h->tokens, P = h->patches_per_frame;
        const float *conv, *cls, *pos, *proj, *a, *b;
        VF_TRY(T.get("visual.conv1.weight", int64_t(W) * 588, &conv));
        VF_TRY(upload_f16(h, &h->w_patch, conv, W, 588, VITL_PK));
        VF_TRY(T.get("visual.proj", int64_t(W) * VL_EMBED, &proj));
        VF_TRY(upload_f16(h, &h->w_proj, proj, VL_EMBED, W, W, true));
        VF_TRY(T.get("visual.positional_embedding", int64_t(Tk) * W, &pos));
        VF_TRY(upload_f32(h, &h->pos, pos, size_t(Tk) * W));
        VF_TRY(T.get("visual.class_embedding", W, &cls));
        std::vector<float> c0(W);
        for (int i = 0; i < W; ++i) c0[i] = cls[i] + pos[i];
        VF_TRY(upload_f32(h, &h->cls_pos0, c0.data(), W));
        VF_TRY(T.get("visual.ln_pre.weight", W, &a)); VF_TRY(upload_f32(h, &h->lnpre_w, a, W));
        VF_TRY(T.get("visual.ln_pre.bias", W, &a)); VF_TRY(upload_f32(h, &h->lnpre_b, a, W));
        VF_TRY(T.get("visual.ln_post.weight", W, &a)); VF_TRY(upload_f32(h, &h->lnpost_w, a, W));
        VF_TRY(T.get("visual.ln_post.bias", W, &a)); VF_TRY(upload_f32(h, &h->lnpost_b, a, W));
        for (int l = 0; l < VL_LAYERS; ++l) {
            const std::string p = "visual.transformer.resblocks." + std::to_string(l) + ".";
            VitlLayer& d = h->layer[l];
            const struct { const char* name; int64_t n; float** dst; } vecs[] = {
                {"ln_1.weight", W, &d.ln1_w}, {"ln_1.bias", W, &d.ln1_b}, {"ln_2.weight", W, &d.ln2_w},
                {"ln_2.bias", W, &d.ln2_b}, {"attn.in_proj_bias", 3 * W, &d.b_qkv}, {"attn.out_proj.bias", W, &d.b_o},
                {"mlp.c_fc.bias", VL_MLP, &d.b_fc}, {"mlp.c_proj.bias", W, &d.b_proj}};
            for (const auto& v : vecs) {
                VF_TRY(T.get(p + v.name, v.n, &a));
                VF_TRY(upload_f32(h, v.dst, a, size_t(v.n)));
            }
            const struct { const char* name; int rows, cols; __half** dst; } mats[] = {
                {"attn.in_proj_weight", 3 * W, W, &d.w_qkv}, {"attn.out_proj.weight", W, W, &d.w_o},
                {"mlp.c_fc.weight", VL_MLP, W, &d.w_fc}, {"mlp.c_proj.weight", W, VL_MLP, &d.w_proj}};
            for (const auto& m : mats) {
                VF_TRY(T.get(p + m.name, int64_t(m.rows) * m.cols, &b));
                VF_TRY(upload_f16(h, m.dst, b, m.rows, m.cols));
            }
        }
        const size_t F = size_t(max_frames);
        VF_TRY(ralloc(h, &h->patches, F * P * VITL_PK));
        VF_TRY(ralloc(h, &h->emb, F * P * W));
        VF_TRY(ralloc(h, &h->x, F * Tk * W));
        VF_TRY(ralloc(h, &h->h, F * Tk * W));
        VF_TRY(ralloc(h, &h->qkv, F * Tk * 3 * W));
        VF_TRY(ralloc(h, &h->att, F * Tk * W));
        VF_TRY(ralloc(h, &h->mlp, F * Tk * VL_MLP));
        VF_TRY(ralloc(h, &h->cls, F * W));
        VF_TRY(ralloc(h, &h->feat, F * VL_EMBED));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_clip_vitl_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_clip_vitl_info(const vf_clip_vitl_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "clip_vitl_info: null argument");
    const int v[8] = {VL_EMBED, h->npx, VITL_W, VL_LAYERS, VL_HEADS, VITL_PATCH, h->tokens, h->max_frames};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

int vf_clip_vitl_encode_f32(vf_clip_vitl_t* h, const float* frames, int n, float* out, void* stream) {
    return vl_encode(h, frames, 0, n, 0, 0, out, stream);
}

int vf_clip_vitl_encode_u8(vf_clip_vitl_t* h, const uint8_t* frames, int n, int H, int W, float* out, void* stream) {
    return vl_encode(h, frames, 1, n, H, W, out, stream);
}

// The three pieces of the tower one at a time, eagerly, on the handle's workspace and the caller's stream.
int vf_clip_vitl_debug_embed_f32(vf_clip_vitl_t* h, const float* frames, int n, float* x_out, void* stream) {
    VF_TRY(debug_frames(h, frames, x_out, n, h ? h->max_frames : 0, "max_frames", "clip_vitl_debug_embed_f32"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_TRY(vitl_patchify_f32(frames, n, h->npx, h->patches, s));
    h->launches += 1;
    VF_TRY(vl_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * h->tokens * VITL_W * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_clip_vitl_debug_embed_u8(vf_clip_vitl_t* h, const uint8_t* frames, int n, int H, int W, float* x_out,
                                void* stream) {
    VF_TRY(debug_frames(h, frames, x_out, n, h ? h->max_frames : 0, "max_frames", "clip_vitl_debug_embed_u8"));
    FrameGeom g;
    VF_TRY(frame_geometry("clip_vitl", H, W, h->npx, h->npx, &g));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaStreamSynchronize(h->cs));       // a resize buffer may be re-allocated: the engine stream is idle
    const uint8_t* src;
    VF_TRY(resize_frames(h, frames, n, H, W, g, h->max_frames, s, &src));
    VF_TRY(vitl_patchify_u8(src, n, g.rh, g.rw, g.cy, g.cx, h->npx, h->patches, s));
    h->launches += 1;
    VF_TRY(vl_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * h->tokens * VITL_W * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_clip_vitl_debug_blocks(vf_clip_vitl_t* h, float* x, int n, int layer_begin, int layer_end, void* stream) {
    VF_TRY(debug_frames(h, x, x, n, h ? h->max_frames : 0, "max_frames", "clip_vitl_debug_blocks"));
    if (layer_begin < 0 || layer_begin >= layer_end || layer_end > VL_LAYERS)
        return fail(VF_ERR_INVALID, "clip_vitl_debug_blocks: layers [%d, %d) are not a range within [0, %d)", layer_begin,
                    layer_end, VL_LAYERS);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t bytes = size_t(n) * h->tokens * VITL_W * sizeof(float);
    VF_CUDA(cudaMemcpyAsync(h->x, x, bytes, cudaMemcpyDeviceToDevice, s));
    VF_TRY(vl_blocks(h, n, layer_begin, layer_end, s));
    VF_CUDA(cudaMemcpyAsync(x, h->x, bytes, cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_clip_vitl_debug_head(vf_clip_vitl_t* h, const float* x, int n, float* out, void* stream) {
    VF_TRY(debug_frames(h, x, out, n, h ? h->max_frames : 0, "max_frames", "clip_vitl_debug_head"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaMemcpyAsync(h->x, x, size_t(n) * h->tokens * VITL_W * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return vl_head(h, n, out, s);
}

int vf_clip_vitl_attention(vf_clip_vitl_t* h, const void* qkv, int n_frames, int tokens, void* out, void* stream) {
    if (!h || !qkv || !out) return fail(VF_ERR_INVALID, "clip_vitl_attention: null argument");
    VF_CUDA(cudaSetDevice(h->device));
    VF_TRY(vitl_attention(static_cast<const __half*>(qkv), static_cast<__half*>(out), n_frames, tokens, VL_HEADS,
                          static_cast<cudaStream_t>(stream)));
    h->launches += 1;
    return VF_OK;
}

int64_t vf_clip_vitl_launch_count(const vf_clip_vitl_t* h) { return h ? h->launches : 0; }

}  // extern "C"
