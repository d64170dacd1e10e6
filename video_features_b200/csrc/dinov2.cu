// DINOv2 frame features (`torch.hub.load('facebookresearch/dinov2', 'dinov2_vit{s,b,l,g}14[_reg]')(x)` at 224 px: the
// class token after the final norm) on the split-weight wgmma GEMM, clip_vitl_kernels.cu's key-streaming attention,
// swin3d_kernels.cu's width-generic LayerNorm and the kernels of dinov2_kernels.cu.  The fused u8 transform is the hub's
// eval preset: Resize(256, bicubic) on the PIL image, CenterCrop(224), ToTensor, Normalize (ImageNet).
//
// Block: x += ls1 * proj(attn(norm1(x))); x += ls2 * ffn(norm2(x)), ffn = fc2(GELU(fc1)) for S / B / L and
// w3(silu(a) * b), (a, b) = w12(.), for g.  LayerNorm eps 1e-6, attention scale 1/8, no LayerNorm before block 0.
//
// Numerics: every GEMM weight is a split-fp16 pair W_hi | W_lo, run as a 1-tap split-weight linear on the conv-mode GEMM;
// accumulation fp32; the residual stream, LayerNorm statistics, softmax max / sum fp32.  LayerScale is folded into the
// epilogue of proj and fc2 / w3: scale gamma[n], bias fp32(gamma[n] * b[n]), added into the fp32 residual stream (fp32
// reductions, each element once).  Rounded to one fp16 value: patch rows, norm1 / norm2 outputs, q / k / v, P per
// 64-key block, the attention output and the FFN hidden layer; g's w12 output (a, b) stays fp32 and the SwiGLU kernel
// rounds silu(a) * b once.  scripts/precision/emulate_dinov2.py decided the scheme (DESIGN.md §4.17).
// The last block runs its out-projection and FFN on the class rows only, gathered into a compact buffer.
// Frames are packed along M (row = frame * S + token) and run in chunks of at most max_frames frames; each chunk size
// is one CUDA graph.
#include <string.h>

#include <string>
#include <vector>

#include "clip_vitl_kernels.h"
#include "dinov2_kernels.h"
#include "internal.h"
#include "split_conv.h"
#include "swin3d_kernels.h"

namespace vf {

constexpr float DV_EPS = 1e-6f;
constexpr int DV_REG = 4, DV_SWIGLU_HIDDEN = 4096;

struct DvBlock {
    float *n1w, *n1b, *n2w, *n2b, *bqkv, *ls1, *bproj, *ls2, *bfc1, *bfc2;   // bproj / bfc2: gamma * b
    __half *wqkv, *wproj, *wfc1, *wfc2;          // fc1 / fc2: mlp.fc1 / fc2 or mlp.w12 / w3
};

}  // namespace vf

using namespace vf;

struct vf_dinov2 : vf::EngineCore {
    int D = 0, depth = 0, heads = 0, S = 0, n_reg = 0, swiglu = 0, hidden = 0, max_frames = 0;
    __half* w_patch = nullptr;
    float *b_patch = nullptr, *pos = nullptr, *cls_pos0 = nullptr, *reg = nullptr, *norm_w = nullptr, *norm_b = nullptr;
    std::vector<DvBlock> blocks;
    // workspace (max_frames frames)
    __half *patches = nullptr, *hbuf = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr, *attc = nullptr;
    float *emb = nullptr, *x = nullptr, *ab = nullptr, *xc = nullptr, *feat = nullptr;
    uint8_t *resized = nullptr, *resize_tmp = nullptr;        // grown on demand for the u8 entry's resize
    size_t resized_cap = 0, tmp_cap = 0;
};

namespace vf {

static GemmEpi ls_epi(float* out, int ldo, const float* gamma, const float* bias) {
    GemmEpi e = linear_epi(out, ldo, 1, bias, VF_ACT_NONE, 1);
    e.scale = gamma;
    return e;
}

// rows of `ld`-element class rows: row f of dst (pitch D) <-> row f * S of src (pitch S * D)
static int dv_gather(void* dst, const void* src, size_t elem, int c, const vf_dinov2* h, cudaStream_t s) {
    VF_CUDA(cudaMemcpy2DAsync(dst, elem * h->D, src, elem * h->D * h->S, elem * h->D, c, cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}
static int dv_scatter(void* dst, const void* src, size_t elem, int c, const vf_dinov2* h, cudaStream_t s) {
    VF_CUDA(cudaMemcpy2DAsync(dst, elem * h->D * h->S, src, elem * h->D, elem * h->D, c, cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

// the FFN of block w on `rows` fp16 rows in h->hbuf, its LayerScale'd result added into x (pitch D)
static int dv_ffn(vf_dinov2* h, const DvBlock& w, int rows, float* x, cudaStream_t s) {
    const int D = h->D, H = h->hidden;
    if (h->swiglu) {
        VF_TRY(split_linear(h->hbuf, rows, 2 * H, D, w.wfc1, linear_epi(h->ab, 2 * H, 1, w.bfc1, VF_ACT_NONE), s));
        VF_TRY(dinov2_swiglu(h->ab, rows, H, h->mlp, s));
        h->launches += 1;
    } else {
        VF_TRY(split_linear(h->hbuf, rows, H, D, w.wfc1, linear_epi(h->mlp, H, 0, w.bfc1, VF_ACT_GELU), s));
    }
    VF_TRY(split_linear(h->mlp, rows, D, H, w.wfc2, ls_epi(x, D, w.ls2, w.bfc2), s));
    h->launches += 2;
    return VF_OK;
}

// blocks [l0, l1) on h->x (c frames)
static int dv_blocks(vf_dinov2* h, int c, int l0, int l1, cudaStream_t s) {
    const int D = h->D, M = c * h->S;
    for (int l = l0; l < l1; ++l) {
        const DvBlock& w = h->blocks[l];
        VF_TRY(swin3d_layernorm(h->x, D, w.n1w, w.n1b, h->hbuf, 0, M, s, nullptr, DV_EPS));
        VF_TRY(split_linear(h->hbuf, M, 3 * D, D, w.wqkv, linear_epi(h->qkv, 3 * D, 0, w.bqkv, VF_ACT_NONE), s));
        VF_TRY(vitl_attention(h->qkv, h->att, c, h->S, h->heads, s));
        h->launches += 3;
        if (l + 1 < h->depth) {
            VF_TRY(split_linear(h->att, M, D, D, w.wproj, ls_epi(h->x, D, w.ls1, w.bproj), s));
            VF_TRY(swin3d_layernorm(h->x, D, w.n2w, w.n2b, h->hbuf, 0, M, s, nullptr, DV_EPS));
            h->launches += 2;
            VF_TRY(dv_ffn(h, w, M, h->x, s));
        } else {            // the feature reads the class rows only: the rest of the last block runs on them alone
            VF_TRY(dv_gather(h->attc, h->att, sizeof(__half), c, h, s));
            VF_TRY(dv_gather(h->xc, h->x, sizeof(float), c, h, s));
            VF_TRY(split_linear(h->attc, c, D, D, w.wproj, ls_epi(h->xc, D, w.ls1, w.bproj), s));
            VF_TRY(swin3d_layernorm(h->xc, D, w.n2w, w.n2b, h->hbuf, 0, c, s, nullptr, DV_EPS));
            h->launches += 2;
            VF_TRY(dv_ffn(h, w, c, h->xc, s));
            VF_TRY(dv_scatter(h->x, h->xc, sizeof(float), c, h, s));
        }
    }
    return VF_OK;
}

// h->patches (c frames) -> h->x
static int dv_embed(vf_dinov2* h, int c, cudaStream_t s) {
    VF_TRY(split_linear(h->patches, c * DV_PATCHES, h->D, DV_PK, h->w_patch,
                        linear_epi(h->emb, h->D, 1, h->b_patch, VF_ACT_NONE), s));
    VF_TRY(dinov2_tokens(h->emb, h->pos, h->cls_pos0, h->reg, h->n_reg, h->x, c, h->D, s));
    h->launches += 2;
    return VF_OK;
}

// the final norm of the class rows of h->x -> out (c x D fp32)
static int dv_head(vf_dinov2* h, int c, float* out, cudaStream_t s) {
    VF_TRY(dv_gather(h->xc, h->x, sizeof(float), c, h, s));
    VF_TRY(swin3d_layernorm(h->xc, h->D, h->norm_w, h->norm_b, out, 1, c, s, nullptr, DV_EPS));
    h->launches += 1;
    return VF_OK;
}

static int dv_net(vf_dinov2* h, int c, cudaStream_t s) {
    VF_TRY(dv_embed(h, c, s));
    VF_TRY(dv_blocks(h, c, 0, h->depth, s));
    return dv_head(h, c, h->feat, s);
}

// a resize buffer of at least `need` bytes; the engine stream is drained before an old one is freed
static int dv_grow(vf_dinov2* h, uint8_t** p, size_t* cap, size_t need) {
    if (need <= *cap) return VF_OK;
    if (*p) {
        VF_CUDA(cudaStreamSynchronize(h->cs));
        VF_CUDA(cudaFree(*p));
        *p = nullptr; *cap = 0;
    }
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, need);
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "dinov2: cudaMalloc(%zu bytes): %s", need, cudaGetErrorString(e));
    *p = static_cast<uint8_t*>(q);
    *cap = need;
    return VF_OK;
}

// Resize(256): the short side to 256 (bicubic, Pillow-exact), then the centre 224 crop
struct DvGeom { int rh, rw, cy, cx; bool resize; };
static int dv_geometry(int H, int W, DvGeom* g) {
    if (H <= 0 || W <= 0) return fail(VF_ERR_INVALID, "dinov2: bad frame geometry %dx%d", H, W);
    VF_TRY(vf_resize_geometry(H, W, DV_RESIZE, 1, &g->rh, &g->rw));
    if (g->rh < DV_CROP || g->rw < DV_CROP)
        return fail(VF_ERR_INVALID, "dinov2: a %dx%d frame resizes to %dx%d, smaller than the 224 crop", H, W, g->rh, g->rw);
    g->resize = g->rh != H || g->rw != W;
    g->cy = center_crop_offset(g->rh, DV_CROP);
    g->cx = center_crop_offset(g->rw, DV_CROP);
    return VF_OK;
}

// c device uint8 BGR frames of geometry (H, W) -> h->patches
static int dv_transform(vf_dinov2* h, const uint8_t* frames, int c, int H, int W, const DvGeom& g, cudaStream_t s) {
    const uint8_t* cur = frames;
    int ch = H, cw = W;
    if (g.resize) {
        VF_TRY(dv_grow(h, &h->resized, &h->resized_cap, size_t(h->max_frames) * g.rh * g.rw * 3));
        VF_TRY(dv_grow(h, &h->resize_tmp, &h->tmp_cap, size_t(h->max_frames) * H * g.rw * 3));
        VF_TRY(resize_u8(frames, c, H, W, h->resized, g.rh, g.rw, VF_FILTER_BICUBIC, h->resize_tmp, s));
        h->launches += (g.rh != H) + (g.rw != W);
        cur = h->resized; ch = g.rh; cw = g.rw;
    }
    VF_TRY(dinov2_patchify_u8(cur, c, ch, cw, g.cy, g.cx, h->patches, s));
    h->launches += 1;
    return VF_OK;
}

static int dv_encode(vf_dinov2* h, const void* frames, int is_u8, int n, int H, int W, float* out, void* stream) {
    if (!h || (n > 0 && (!frames || !out))) return fail(VF_ERR_INVALID, "dinov2_encode: null argument");
    if (n < 0) return fail(VF_ERR_INVALID, "dinov2_encode: %d frames", n);
    if (n == 0) return VF_OK;
    DvGeom g{DV_CROP, DV_CROP, 0, 0, false};
    if (is_u8) VF_TRY(dv_geometry(H, W, &g));
    const size_t frame_elems = is_u8 ? size_t(H) * W * 3 : size_t(3) * DV_CROP * DV_CROP;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    // as few chunks as the workspace allows, all (nearly) the same size
    const int nchunks = (n + h->max_frames - 1) / h->max_frames, step = (n + nchunks - 1) / nchunks;
    for (int off = 0; off < n; off += step) {
        const int c = n - off < step ? n - off : step;
        if (is_u8) {
            VF_TRY(dv_transform(h, static_cast<const uint8_t*>(frames) + off * frame_elems, c, H, W, g, s));
        } else {
            VF_TRY(dinov2_patchify_f32(static_cast<const float*>(frames) + off * frame_elems, c, h->patches, s));
            h->launches += 1;
        }
        VF_TRY(run_graphed(h, {c, 0, 0, 0}, [&] { return dv_net(h, c, s); }));
        VF_CUDA(cudaMemcpyAsync(out + size_t(off) * h->D, h->feat, size_t(c) * h->D * sizeof(float),
                                cudaMemcpyDeviceToDevice, s));
    }
    return leave(h, user);
}

static int dv_debug_args(vf_dinov2* h, const void* a, const void* b, int n, const char* what) {
    if (!h || !a || !b) return fail(VF_ERR_INVALID, "%s: null argument", what);
    if (n <= 0 || n > h->max_frames)
        return fail(VF_ERR_INVALID, "%s: %d frames (1 .. %d, the handle's max_frames)", what, n, h->max_frames);
    VF_CUDA(cudaSetDevice(h->device));
    return VF_OK;
}

static int dv_upload_f32(vf_dinov2* h, float** dst, const float* src, size_t count) {
    VF_TRY(ralloc(h, dst, count));
    VF_CUDA(cudaMemcpy(*dst, src, count * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

// the LayerScale fold of a residual-branch output linear: gamma and fp32(gamma * b)
static int dv_upload_ls(vf_dinov2* h, const ResTensors& T, const std::string& gamma, const std::string& bias, int D,
                        float** g_dst, float** b_dst) {
    const float *g, *b;
    VF_TRY(T.get(gamma, D, &g));
    VF_TRY(T.get(bias, D, &b));
    std::vector<float> gb(D);
    for (int i = 0; i < D; ++i) gb[i] = g[i] * b[i];
    VF_TRY(dv_upload_f32(h, g_dst, g, D));
    return dv_upload_f32(h, b_dst, gb.data(), D);
}

}  // namespace vf

extern "C" {

int vf_dinov2_destroy(vf_dinov2_t* h) {
    if (!h) return VF_OK;
    release(h);
    if (h->resized) cudaFree(h->resized);
    if (h->resize_tmp) cudaFree(h->resize_tmp);
    delete h;
    return VF_OK;
}

int vf_dinov2_create(vf_dinov2_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "dinov2_create: null argument");
    *out = nullptr;
    const ResTensors T{tensors, n_tensors, "dinov2_create"};
    // the hub's shapes: width from cls_token, depth from the block keys, heads = width / 64, the FFN from its keys
    const vf_named_tensor* cls = T.find("cls_token");
    if (!cls) return fail(VF_ERR_INVALID, "dinov2_create: missing tensor 'cls_token'");
    const int64_t D = cls->numel;
    int want_depth = 0;
    bool want_swiglu = false;
    if (D == 384 || D == 768) want_depth = 12;
    else if (D == 1024) want_depth = 24;
    else if (D == 1536) { want_depth = 40; want_swiglu = true; }
    else
        return fail(VF_ERR_UNSUPPORTED, "dinov2_create: tensor 'cls_token' gives width %lld (384, 768, 1024 and 1536 "
                    "are built)", (long long)D);
    int depth = 0;
    while (T.find("blocks." + std::to_string(depth) + ".norm1.weight")) ++depth;
    if (depth != want_depth)
        return fail(depth < want_depth ? VF_ERR_INVALID : VF_ERR_UNSUPPORTED,
                    "dinov2_create: tensor 'blocks.%d.norm1.weight' %s: %d blocks at width %lld (%d are built)",
                    depth < want_depth ? depth : want_depth, depth < want_depth ? "missing" : "present", depth,
                    (long long)D, want_depth);
    const bool swiglu = T.find("blocks.0.mlp.w12.weight") != nullptr;
    if (swiglu != want_swiglu)
        return fail(VF_ERR_UNSUPPORTED, "dinov2_create: tensor 'blocks.0.mlp.w12.weight' %s: width %lld is built with %s",
                    swiglu ? "present" : "missing", (long long)D,
                    want_swiglu ? "the SwiGLU FFN (mlp.w12 / mlp.w3)" : "the GELU MLP (mlp.fc1 / mlp.fc2)");
    if (!swiglu && !T.find("blocks.0.mlp.fc1.weight"))
        return fail(VF_ERR_INVALID, "dinov2_create: missing tensor 'blocks.0.mlp.fc1.weight' (width %lld is built with "
                    "the GELU MLP)", (long long)D);
    const vf_named_tensor* rg = T.find("register_tokens");
    if (rg && rg->numel != DV_REG * D)
        return fail(VF_ERR_UNSUPPORTED, "dinov2_create: tensor 'register_tokens' has %lld elements, not 4 x %lld",
                    (long long)rg->numel, (long long)D);
    const vf_named_tensor* pt = T.find("pos_embed_224");
    if (!pt || pt->numel != int64_t(1 + DV_PATCHES) * D)
        return fail(VF_ERR_INVALID, "dinov2_create: tensor 'pos_embed_224' %s (the 257 x %lld positional table of a 224-px "
                    "input)", pt ? "has the wrong size" : "missing", (long long)D);
    const int hidden = swiglu ? DV_SWIGLU_HIDDEN : int(4 * D);
    const int n_reg = rg ? DV_REG : 0, S = 1 + n_reg + DV_PATCHES;
    // workspace per frame: patches 2 * 592 * 256, emb 4 D * 256, x 4 D S, hbuf / att 2 D S each, qkv 6 D S, mlp 2 H S
    // (+ 8 H S of w12 output for g) bytes: 2.9 MB (S/14), 5.4 MB (B/14), 7.1 MB (L/14), 18.2 MB (g/14) at 257 / 261
    // tokens.  The default keeps it near 2.5 GB: 864 (832 with registers) / 448 / 320 / 128 frames.
    const size_t per_frame = size_t(2) * DV_PK * DV_PATCHES + size_t(4) * D * DV_PATCHES +
                             size_t(S) * (4 * D + 4 * D + 6 * D + 2 * hidden + (swiglu ? 8 * hidden : 0));
    if (max_frames <= 0) max_frames = int(2500000000ull / per_frame) / 32 * 32;
    if (max_frames > 4096) return fail(VF_ERR_INVALID, "dinov2_create: max_frames %d too large", max_frames);
    VF_TRY(check_device(device));
    vf_dinov2* h = new vf_dinov2();
    h->who = "dinov2_create";
    h->device = device; h->D = int(D); h->depth = depth; h->heads = int(D / 64); h->S = S; h->n_reg = n_reg;
    h->swiglu = swiglu; h->hidden = hidden; h->max_frames = max_frames;
    auto body = [&]() -> int {
        const int W = int(D);
        const float *a, *pos;
        VF_TRY(upload_split_mat(h, T, "patch_embed.proj.weight", W, 3 * DV_PATCH * DV_PATCH, &h->w_patch, DV_PK));
        VF_TRY(upload_vec(h, T, "patch_embed.proj.bias", W, &h->b_patch));
        VF_TRY(T.get("pos_embed_224", int64_t(1 + DV_PATCHES) * W, &pos));
        VF_TRY(dv_upload_f32(h, &h->pos, pos, size_t(1 + DV_PATCHES) * W));
        VF_TRY(T.get("cls_token", W, &a));
        std::vector<float> c0(W);
        for (int i = 0; i < W; ++i) c0[i] = a[i] + pos[i];
        VF_TRY(dv_upload_f32(h, &h->cls_pos0, c0.data(), W));
        if (n_reg) VF_TRY(upload_vec(h, T, "register_tokens", int64_t(n_reg) * W, &h->reg));
        VF_TRY(upload_vec(h, T, "norm.weight", W, &h->norm_w));
        VF_TRY(upload_vec(h, T, "norm.bias", W, &h->norm_b));
        const std::string f1 = swiglu ? "mlp.w12." : "mlp.fc1.", f2 = swiglu ? "mlp.w3." : "mlp.fc2.";
        const int n1 = swiglu ? 2 * hidden : hidden;
        for (int l = 0; l < depth; ++l) {
            const std::string p = "blocks." + std::to_string(l) + ".";
            DvBlock w;
            VF_TRY(upload_vec(h, T, p + "norm1.weight", W, &w.n1w));
            VF_TRY(upload_vec(h, T, p + "norm1.bias", W, &w.n1b));
            VF_TRY(upload_vec(h, T, p + "norm2.weight", W, &w.n2w));
            VF_TRY(upload_vec(h, T, p + "norm2.bias", W, &w.n2b));
            VF_TRY(upload_vec(h, T, p + "attn.qkv.bias", 3 * W, &w.bqkv));
            VF_TRY(upload_vec(h, T, p + f1 + "bias", n1, &w.bfc1));
            VF_TRY(dv_upload_ls(h, T, p + "ls1.gamma", p + "attn.proj.bias", W, &w.ls1, &w.bproj));
            VF_TRY(dv_upload_ls(h, T, p + "ls2.gamma", p + f2 + "bias", W, &w.ls2, &w.bfc2));
            VF_TRY(upload_split_mat(h, T, p + "attn.qkv.weight", 3 * W, W, &w.wqkv));
            VF_TRY(upload_split_mat(h, T, p + "attn.proj.weight", W, W, &w.wproj));
            VF_TRY(upload_split_mat(h, T, p + f1 + "weight", n1, W, &w.wfc1));
            VF_TRY(upload_split_mat(h, T, p + f2 + "weight", W, hidden, &w.wfc2));
            h->blocks.push_back(w);
        }
        const size_t F = size_t(max_frames), R = F * S;
        VF_TRY(ralloc(h, &h->patches, F * DV_PATCHES * DV_PK));
        VF_TRY(ralloc(h, &h->emb, F * DV_PATCHES * W));
        VF_TRY(ralloc(h, &h->x, R * W));
        VF_TRY(ralloc(h, &h->hbuf, R * W));
        VF_TRY(ralloc(h, &h->qkv, R * 3 * W));
        VF_TRY(ralloc(h, &h->att, R * W));
        VF_TRY(ralloc(h, &h->mlp, R * hidden));
        if (swiglu) VF_TRY(ralloc(h, &h->ab, R * 2 * hidden));
        VF_TRY(ralloc(h, &h->attc, F * W));
        VF_TRY(ralloc(h, &h->xc, F * W));
        VF_TRY(ralloc(h, &h->feat, F * W));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_dinov2_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_dinov2_info(const vf_dinov2_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "dinov2_info: null argument");
    const int v[7] = {h->D, h->depth, h->heads, h->S, h->n_reg, h->swiglu, h->max_frames};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

int vf_dinov2_encode_f32(vf_dinov2_t* h, const float* frames, int n, float* out, void* stream) {
    return dv_encode(h, frames, 0, n, 0, 0, out, stream);
}

int vf_dinov2_encode_u8(vf_dinov2_t* h, const uint8_t* frames, int n, int H, int W, float* out, void* stream) {
    return dv_encode(h, frames, 1, n, H, W, out, stream);
}

int vf_dinov2_debug_embed_f32(vf_dinov2_t* h, const float* frames, int n, float* x_out, void* stream) {
    VF_TRY(dv_debug_args(h, frames, x_out, n, "dinov2_debug_embed_f32"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_TRY(dinov2_patchify_f32(frames, n, h->patches, s));
    h->launches += 1;
    VF_TRY(dv_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * h->S * h->D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_dinov2_debug_embed_u8(vf_dinov2_t* h, const uint8_t* frames, int n, int H, int W, float* x_out, void* stream) {
    VF_TRY(dv_debug_args(h, frames, x_out, n, "dinov2_debug_embed_u8"));
    DvGeom g;
    VF_TRY(dv_geometry(H, W, &g));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaStreamSynchronize(h->cs));       // a resize buffer may be re-allocated: the engine stream is idle
    VF_TRY(dv_transform(h, frames, n, H, W, g, s));
    VF_TRY(dv_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * h->S * h->D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_dinov2_debug_blocks(vf_dinov2_t* h, float* x, int n, int layer_begin, int layer_end, void* stream) {
    VF_TRY(dv_debug_args(h, x, x, n, "dinov2_debug_blocks"));
    if (layer_begin < 0 || layer_begin >= layer_end || layer_end > h->depth)
        return fail(VF_ERR_INVALID, "dinov2_debug_blocks: layers [%d, %d) are not a range within [0, %d)", layer_begin,
                    layer_end, h->depth);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t bytes = size_t(n) * h->S * h->D * sizeof(float);
    VF_CUDA(cudaMemcpyAsync(h->x, x, bytes, cudaMemcpyDeviceToDevice, s));
    VF_TRY(dv_blocks(h, n, layer_begin, layer_end, s));
    VF_CUDA(cudaMemcpyAsync(x, h->x, bytes, cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_dinov2_debug_head(vf_dinov2_t* h, const float* x, int n, float* out, void* stream) {
    VF_TRY(dv_debug_args(h, x, out, n, "dinov2_debug_head"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaMemcpyAsync(h->x, x, size_t(n) * h->S * h->D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return dv_head(h, n, out, s);
}

int vf_dinov2_swiglu(const float* ab, int rows, int hidden, void* out, void* stream) {
    if (!ab || !out) return fail(VF_ERR_INVALID, "dinov2_swiglu: null argument");
    return dinov2_swiglu(ab, rows, hidden, static_cast<__half*>(out), static_cast<cudaStream_t>(stream));
}

int vf_dinov2_attention(const void* qkv, int n, int S, int heads, void* out, void* stream) {
    if (!qkv || !out) return fail(VF_ERR_INVALID, "dinov2_attention: null argument");
    return vitl_attention(static_cast<const __half*>(qkv), static_cast<__half*>(out), n, S, heads,
                          static_cast<cudaStream_t>(stream));
}

int64_t vf_dinov2_launch_count(const vf_dinov2_t* h) { return h ? h->launches : 0; }

}  // extern "C"
