// openai/CLIP's text tower (`CLIP.encode_text`, clip/model.py) on the wgmma GEMM and the kernels of
// clip_text_kernels.cu: prompts of token ids -> L2-normalised text features, what the zero-shot `--show_pred` of the
// CLIP feature types compares each frame's image feature with.
//
// Geometry from the state dict, as clip.build_model reads it: width = ln_final.weight size, heads = width / 64, layers =
// the count of transformer.resblocks.*, context = positional_embedding rows, embed = text_projection columns.  The
// released towers are 512 / 8 (ViT-B, RN50, RN101), 640 / 10 (RN50x4) and 768 / 12 (RN50x16, ViT-L), all 12 blocks.
//
// Numerics (scripts/precision/emulate_clip_text.py, DESIGN.md §4.16): every GEMM weight is a split-fp16 pair W_hi | W_lo,
// run as a 1-tap split-weight linear on the conv-mode GEMM; accumulation fp32; the residual stream, LayerNorm statistics,
// scores, softmax and P.V fp32.  Rounded to one fp16 value: the LayerNorm outputs, q / k / v, the attention output and
// fc1 after QuickGELU.  out_proj and c_proj add into the fp32 residual stream from the GEMM epilogue.
//
// Length cut: under openai's causal mask row i reads rows 0..i only, so rows after the last EOT of a call never reach
// an EOT row.  A call runs on L = 1 + its largest EOT position rows per prompt instead of the context's 77.
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "clip_text_kernels.h"
#include "internal.h"
#include "split_conv.h"
#include "swin3d_kernels.h"

namespace vf {

struct CtBlock {
    float *ln1w, *ln1b, *ln2w, *ln2b, *bqkv, *bout, *bfc1, *bfc2;
    __half *wqkv, *wout, *wfc1, *wfc2;
};

}  // namespace vf

using namespace vf;

struct vf_clip_text : vf::EngineCore {
    int width = 0, heads = 0, layers = 0, ctx = 0, embed = 0, vocab = 0, max_rows = 0;
    float *tok_emb = nullptr, *pos = nullptr, *lnf_w = nullptr, *lnf_b = nullptr;
    __half* wproj = nullptr;                       // text_projection^T as a split pair: embed rows of [hi W | lo W]
    std::vector<CtBlock> blocks;
    // workspace, max_rows token rows
    int32_t *tokens = nullptr, *eot = nullptr;
    float *x = nullptr, *pooled = nullptr, *proj = nullptr;
    __half *hbuf = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr;
};

namespace vf {

// blocks [first, first + count) on the stream x of n prompts of L rows
static int run_blocks(vf_clip_text* h, float* x, int n, int L, int first, int count, cudaStream_t s) {
    const int W = h->width, R = n * L;
    for (int i = first; i < first + count; ++i) {
        const CtBlock& w = h->blocks[i];
        VF_TRY(swin3d_layernorm(x, W, w.ln1w, w.ln1b, h->hbuf, 0, R, s));
        VF_TRY(split_linear(h->hbuf, R, 3 * W, W, w.wqkv, linear_epi(h->qkv, 3 * W, 0, w.bqkv, VF_ACT_NONE), s));
        VF_TRY(clip_text_attention(h->qkv, n, L, h->heads, h->att, s));
        VF_TRY(split_linear(h->att, R, W, W, w.wout, linear_epi(x, W, 1, w.bout, VF_ACT_NONE, 1), s));
        VF_TRY(swin3d_layernorm(x, W, w.ln2w, w.ln2b, h->hbuf, 0, R, s));
        VF_TRY(split_linear(h->hbuf, R, 4 * W, W, w.wfc1, linear_epi(h->mlp, 4 * W, 0, w.bfc1, VF_ACT_QUICKGELU), s));
        VF_TRY(split_linear(h->mlp, R, W, 4 * W, w.wfc2, linear_epi(x, W, 1, w.bfc2, VF_ACT_NONE, 1), s));
        h->launches += 7;
    }
    return VF_OK;
}

static int check_rows(const vf_clip_text* h, int n, int L, const char* who) {
    if (n < 0 || L < 1 || L > h->ctx || int64_t(n) * L > h->max_rows)
        return fail(VF_ERR_INVALID, "%s: %d prompts of %d rows (context %d, workspace %d rows)", who, n, L, h->ctx,
                    h->max_rows);
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_clip_text_destroy(vf_clip_text_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_clip_text_create(vf_clip_text_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_rows) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "clip_text_create: null argument");
    *out = nullptr;
    if (max_rows <= 0) max_rows = 8192;
    const ResTensors Tn{tensors, n_tensors, "clip_text_create"};
    const vf_named_tensor *lnf = Tn.find("ln_final.weight"), *pe = Tn.find("positional_embedding"),
                          *te = Tn.find("token_embedding.weight"), *tp = Tn.find("text_projection");
    const char* missing = !lnf ? "ln_final.weight" : !pe ? "positional_embedding" : !te ? "token_embedding.weight"
                          : !tp ? "text_projection" : nullptr;
    if (missing) return fail(VF_ERR_INVALID, "clip_text_create: missing tensor '%s'", missing);
    const int W = int(lnf->numel);
    if (W != 512 && W != 640 && W != 768)
        return fail(VF_ERR_UNSUPPORTED, "clip_text_create: text width %d (ln_final.weight); the released towers are "
                    "512 / 8 heads, 640 / 10 and 768 / 12", W);
    int layers = 0;
    while (Tn.find("transformer.resblocks." + std::to_string(layers) + ".ln_1.weight")) ++layers;
    if (layers != 12 || pe->numel % W || te->numel % W || tp->numel % W)
        return fail(VF_ERR_UNSUPPORTED, "clip_text_create: %d blocks, positional_embedding %lld, token_embedding %lld "
                    "and text_projection %lld elements at width %d (the released towers have 12 blocks)", layers,
                    (long long)pe->numel, (long long)te->numel, (long long)tp->numel, W);
    const int ctx = int(pe->numel / W), embed = int(tp->numel / W);
    const int64_t vocab = te->numel / W;
    if (ctx < 2 || ctx > CT_MAX_CTX || embed < 8 || embed % 8 || vocab < 2 || vocab > INT32_MAX)
        return fail(VF_ERR_UNSUPPORTED, "clip_text_create: context %d (2..%d), embed %d (a multiple of 8), vocabulary "
                    "%lld", ctx, CT_MAX_CTX, embed, (long long)vocab);
    if (max_rows < ctx) return fail(VF_ERR_INVALID, "clip_text_create: workspace of %d rows < context %d", max_rows, ctx);
    VF_TRY(check_device(device));
    vf_clip_text* h = new vf_clip_text();
    h->who = "clip_text_create";
    h->device = device;
    h->width = W; h->heads = W / CT_HEAD_DIM; h->layers = layers; h->ctx = ctx; h->embed = embed;
    h->vocab = int(vocab); h->max_rows = max_rows;
    auto body = [&]() -> int {
        VF_TRY(upload_vec(h, Tn, "token_embedding.weight", vocab * W, &h->tok_emb));
        VF_TRY(upload_vec(h, Tn, "positional_embedding", int64_t(ctx) * W, &h->pos));
        VF_TRY(upload_vec(h, Tn, "ln_final.weight", W, &h->lnf_w));
        VF_TRY(upload_vec(h, Tn, "ln_final.bias", W, &h->lnf_b));
        {   // x @ text_projection: the GEMM's weight rows are its columns
            std::vector<float> t(size_t(embed) * W);
            for (int r = 0; r < W; ++r)
                for (int c = 0; c < embed; ++c) t[size_t(c) * W + r] = tp->data[size_t(r) * embed + c];
            const vf_named_tensor nt{"text_projection^T", t.data(), int64_t(t.size())};
            VF_TRY(upload_split_mat(h, ResTensors{&nt, 1, "clip_text_create"}, "text_projection^T", embed, W, &h->wproj));
        }
        h->blocks.resize(layers);
        for (int i = 0; i < layers; ++i) {
            CtBlock& w = h->blocks[i];
            const std::string p = "transformer.resblocks." + std::to_string(i) + ".";
            VF_TRY(upload_vec(h, Tn, p + "ln_1.weight", W, &w.ln1w));
            VF_TRY(upload_vec(h, Tn, p + "ln_1.bias", W, &w.ln1b));
            VF_TRY(upload_vec(h, Tn, p + "ln_2.weight", W, &w.ln2w));
            VF_TRY(upload_vec(h, Tn, p + "ln_2.bias", W, &w.ln2b));
            VF_TRY(upload_split_mat(h, Tn, p + "attn.in_proj_weight", 3 * W, W, &w.wqkv));
            VF_TRY(upload_vec(h, Tn, p + "attn.in_proj_bias", 3 * W, &w.bqkv));
            VF_TRY(upload_split_mat(h, Tn, p + "attn.out_proj.weight", W, W, &w.wout));
            VF_TRY(upload_vec(h, Tn, p + "attn.out_proj.bias", W, &w.bout));
            VF_TRY(upload_split_mat(h, Tn, p + "mlp.c_fc.weight", 4 * W, W, &w.wfc1));
            VF_TRY(upload_vec(h, Tn, p + "mlp.c_fc.bias", 4 * W, &w.bfc1));
            VF_TRY(upload_split_mat(h, Tn, p + "mlp.c_proj.weight", W, 4 * W, &w.wfc2));
            VF_TRY(upload_vec(h, Tn, p + "mlp.c_proj.bias", W, &w.bfc2));
        }
        const size_t R = size_t(max_rows);
        VF_TRY(ralloc(h, &h->tokens, R));
        VF_TRY(ralloc(h, &h->eot, R));
        VF_TRY(ralloc(h, &h->x, R * W));
        VF_TRY(ralloc(h, &h->hbuf, R * W));
        VF_TRY(ralloc(h, &h->qkv, R * 3 * W));
        VF_TRY(ralloc(h, &h->att, R * W));
        VF_TRY(ralloc(h, &h->mlp, R * 4 * W));
        VF_TRY(ralloc(h, &h->pooled, R * W));
        VF_TRY(ralloc(h, &h->proj, R * size_t(embed)));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_clip_text_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_clip_text_info(const vf_clip_text_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "clip_text_info: null argument");
    const int v[7] = {h->width, h->heads, h->layers, h->ctx, h->embed, h->vocab, h->max_rows};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

int vf_clip_text_encode(vf_clip_text_t* h, const int32_t* tokens, int n, float* out, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "clip_text_encode: null handle");
    if (n < 0 || (n > 0 && (!tokens || !out))) return fail(VF_ERR_INVALID, "clip_text_encode: null argument");
    if (n == 0) return VF_OK;
    // EOT = the argmax id of each prompt (its first occurrence, as torch.argmax); L covers every EOT of the call
    std::vector<int32_t> eot(size_t(n), 0);
    int L = 1;
    for (int b = 0; b < n; ++b) {
        const int32_t* r = tokens + int64_t(b) * h->ctx;
        for (int t = 0; t < h->ctx; ++t) {
            if (r[t] < 0 || r[t] >= h->vocab)
                return fail(VF_ERR_INVALID, "clip_text_encode: prompt %d, position %d: token id %d outside the "
                            "vocabulary of %d", b, t, r[t], h->vocab);
            if (r[t] > r[eot[b]]) eot[b] = t;
        }
        L = std::max(L, eot[b] + 1);
    }
    const int per_chunk = h->max_rows / L, W = h->width;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n; off += per_chunk) {
        const int m = std::min(per_chunk, n - off);
        // the first L ids of each prompt (m * L <= max_rows); pageable sources are staged before the copy returns
        VF_CUDA(cudaMemcpy2DAsync(h->tokens, size_t(L) * sizeof(int32_t), tokens + int64_t(off) * h->ctx,
                                  size_t(h->ctx) * sizeof(int32_t), size_t(L) * sizeof(int32_t), size_t(m),
                                  cudaMemcpyHostToDevice, s));
        VF_CUDA(cudaMemcpyAsync(h->eot, eot.data() + off, size_t(m) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        VF_TRY(clip_text_embed(h->tokens, L, m, L, h->tok_emb, h->pos, W, h->x, s));
        h->launches += 1;
        VF_TRY(run_blocks(h, h->x, m, L, 0, h->layers, s));
        VF_TRY(clip_text_gather(h->x, h->eot, m, L, W, h->pooled, s));
        VF_TRY(swin3d_layernorm(h->pooled, W, h->lnf_w, h->lnf_b, h->hbuf, 0, m, s));
        VF_TRY(split_linear(h->hbuf, m, h->embed, W, h->wproj, linear_epi(h->proj, h->embed, 1, nullptr, VF_ACT_NONE), s));
        VF_TRY(l2_normalize_rows(h->proj, m, h->embed, out + int64_t(off) * h->embed, s));
        h->launches += 4;
    }
    return leave(h, user);
}

int vf_clip_text_blocks(vf_clip_text_t* h, float* x, int n, int L, int first, int count, void* stream) {
    if (!h || !x) return fail(VF_ERR_INVALID, "clip_text_blocks: null argument");
    VF_TRY(check_rows(h, n, L, "clip_text_blocks"));
    if (first < 0 || count < 0 || first + count > h->layers)
        return fail(VF_ERR_INVALID, "clip_text_blocks: blocks %d..%d of %d", first, first + count - 1, h->layers);
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    VF_TRY(enter(h, user));
    VF_TRY(run_blocks(h, x, n, L, first, count, h->cs));
    return leave(h, user);
}

int vf_clip_text_attention(const void* qkv, int n, int L, int heads, void* out, void* stream) {
    if (!qkv || !out) return fail(VF_ERR_INVALID, "clip_text_attention: null argument");
    return clip_text_attention(static_cast<const __half*>(qkv), n, L, heads, static_cast<__half*>(out),
                               static_cast<cudaStream_t>(stream));
}

int vf_l2_normalize_rows(const float* x, int n, int C, float* out, void* stream) {
    if (!x || !out) return fail(VF_ERR_INVALID, "l2_normalize_rows: null argument");
    return l2_normalize_rows(x, n, C, out, static_cast<cudaStream_t>(stream));
}

int64_t vf_clip_text_launch_count(const vf_clip_text_t* h) { return h ? h->launches : 0; }

}  // extern "C"
