// torchvision MViT-V1-B / MViT-V2-S (`torchvision.models.video.mvit_v1_b` / `mvit_v2_s`, eval) on the wgmma GEMM and
// the kernels of mvit_kernels.cu: the clip feature `norm(x)[:, 0]` (the class token after the final norm, 768-d),
// torchvision's forward without `head`.  The fused input transform is the MViT_*_Weights.KINETICS400_V1 preset.
//
// Numerics: every GEMM weight is a split-fp16 pair W_hi | W_lo, run as a 1-tap split-weight linear on the conv-mode GEMM;
// accumulation fp32; the residual stream, LayerNorm statistics, the head-pooling conv, the rel-pos dot products and
// softmax max / sum fp32.  Rounded to one fp16 value: patch rows, the outputs of norm1 / norm2, qkv, pooled q / k / v
// (after their LayerNorm), P per 32-key block, the attention output and the MLP hidden layer
// (scripts/precision/emulate_mvit.py, DESIGN.md §4.15).  proj, mlp.3 and (v1) project add into the fp32 residual stream
// from the GEMM epilogue.
// Token rows are per clip [class | 8 x S x S tokens]; stage s (0..3) has S = 56 >> s.  Each stage owns two fp32 stream
// buffers: a block that pools or widens writes a buffer other than its input, so the embedding and every stage's output
// stay intact for vf_mvit_read_stage.  Per clip count one CUDA graph covers the patch GEMM to the final norm.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"
#include "mvit_kernels.h"
#include "split_conv.h"
#include "swin3d_kernels.h"

namespace vf {

constexpr int MV_BLOCKS = 16;
// torchvision's block settings (mvit.py): heads, input / output channels, q stride, kv stride; v1 pools q only at the
// stride blocks, v2 everywhere
constexpr int kHeads[MV_BLOCKS] = {1, 2, 2, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 8, 8};
constexpr int kCinV1[MV_BLOCKS] = {96, 192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768, 768};
constexpr int kCoutV1[MV_BLOCKS] = {192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768, 768, 768};
constexpr int kCinV2[MV_BLOCKS] = {96, 96, 192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768};
constexpr int kCoutV2[MV_BLOCKS] = {96, 192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768, 768};
constexpr int kStrideQ[MV_BLOCKS] = {1, 2, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 1};
constexpr int kStrideKV[MV_BLOCKS] = {8, 4, 4, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1};

struct MvPool {
    float *w = nullptr, *g = nullptr, *b = nullptr;     // depthwise weight [96][27], LayerNorm(96)
};
struct MvBlock {
    int heads = 0, cin = 0, cout = 0, ad = 0, sq = 1, skv = 1, s_in = 56;   // ad: the attention width
    bool pool_q = false, project = false;
    float *n1w, *n1b, *n2w, *n2b, *bqkv, *bproj, *bfc1, *bfc2, *bprj = nullptr;
    float *rel_h = nullptr, *rel_w = nullptr, *rel_t = nullptr;
    __half *wqkv, *wproj, *wfc1, *wfc2, *wprj = nullptr;
    MvPool pq, pk, pv;
    int s_q() const { return (s_in - 1) / sq + 1; }
    int s_kv() const { return (s_in - 1) / skv + 1; }
};

static int64_t rows_of(int S) { return 1 + int64_t(MV_TQ) * S * S; }

}  // namespace vf

using namespace vf;

struct vf_mvit : vf::EngineCore {
    int v2 = 0, max_clips = 0;
    __half* w_patch = nullptr;
    float *b_patch = nullptr, *cls = nullptr, *cls_pos = nullptr, *tpos = nullptr, *spos = nullptr;
    float *norm_w = nullptr, *norm_b = nullptr;
    MvBlock blocks[MV_BLOCKS];
    // workspace: embed (the stage-0 tap), two fp32 stream buffers per stage, the final norm
    __half *patches = nullptr, *hbuf = nullptr, *qkv = nullptr, *qp = nullptr, *kp = nullptr, *vp = nullptr,
           *att = nullptr, *mlp = nullptr;
    float *emb = nullptr, *embed = nullptr, *buf[4][2] = {}, *normed = nullptr;
    const float* tap[5] = {};       // stage outputs of the last chunk (tap[0] = embed)
    int tap_C[5] = {};
    int last_m = 0;
};

namespace vf {

static int other(int j) { return 1 - j; }

// one MultiscaleBlock; (st, j) names the stream buffer holding the input and receives the one holding the output
static int run_block(vf_mvit* h, const MvBlock& w, int m, int& st, int& j, cudaStream_t s) {
    const int S = w.s_in, Sq = w.s_q(), Skv = w.s_kv(), ad = w.ad;
    const int64_t n_in = rows_of(S), n_q = rows_of(Sq);
    const int R = int(m * n_in), Rq = int(m * n_q);
    float* x = h->buf[st][j];
    VF_TRY(swin3d_layernorm(x, w.cin, w.n1w, w.n1b, h->hbuf, 0, R, s, nullptr, 1e-6f));
    VF_TRY(split_linear(h->hbuf, R, 3 * ad, w.cin, w.wqkv, linear_epi(h->qkv, 3 * ad, 0, w.bqkv, VF_ACT_NONE), s));
    VF_TRY(mvit_head_pool(h->qkv + ad, 3 * ad, m, w.heads, MV_TQ, S, S, w.skv, w.pk.w, w.pk.g, w.pk.b, h->kp, s));
    VF_TRY(mvit_head_pool(h->qkv + 2 * ad, 3 * ad, m, w.heads, MV_TQ, S, S, w.skv, w.pv.w, w.pv.g, w.pv.b, h->vp, s));
    h->launches += 4;
    const __half* q = h->qkv;
    int ldq = 3 * ad;
    if (w.pool_q) {
        VF_TRY(mvit_head_pool(h->qkv, 3 * ad, m, w.heads, MV_TQ, S, S, w.sq, w.pq.w, w.pq.g, w.pq.b, h->qp, s));
        q = h->qp;
        ldq = ad;
        h->launches += 1;
    }
    MViTAttnGeom g;
    g.n = m; g.heads = w.heads; g.ldq = ldq; g.rel = h->v2; g.resid = h->v2;
    g.q_thw[0] = MV_TQ; g.q_thw[1] = g.q_thw[2] = Sq;
    g.k_thw[0] = MV_TQ; g.k_thw[1] = g.k_thw[2] = Skv;
    VF_TRY(mvit_attention(q, h->kp, h->vp, w.rel_h, w.rel_w, w.rel_t, h->att, g, s));
    h->launches += 1;
    // the skip path: v2 widens norm1's output first; a stride block max-pools into the next stage's buffer
    const float* src = x;
    int sj = j;
    if (h->v2 && w.project) {
        sj = other(j);
        VF_TRY(split_linear(h->hbuf, R, w.cout, w.cin, w.wprj,
                            linear_epi(h->buf[st][sj], w.cout, 1, w.bprj, VF_ACT_NONE), s));
        src = h->buf[st][sj];
        h->launches += 1;
    }
    int yst = st, yj = sj;
    if (w.sq > 1) {
        yst = st + 1; yj = 0;
        VF_TRY(mvit_skip_pool(src, m, ad, MV_TQ, S, S, h->buf[yst][yj], s));
        h->launches += 1;
    }
    float* y = h->buf[yst][yj];
    VF_TRY(split_linear(h->att, Rq, ad, ad, w.wproj, linear_epi(y, ad, 1, w.bproj, VF_ACT_NONE, 1), s));
    VF_TRY(swin3d_layernorm(y, ad, w.n2w, w.n2b, h->hbuf, 0, Rq, s, nullptr, 1e-6f));
    h->launches += 2;
    if (!h->v2 && w.project) {          // v1 widens norm2's output into the stream's other buffer
        yj = other(yj);
        VF_TRY(split_linear(h->hbuf, Rq, w.cout, ad, w.wprj,
                            linear_epi(h->buf[yst][yj], w.cout, 1, w.bprj, VF_ACT_NONE), s));
        h->launches += 1;
    }
    VF_TRY(split_linear(h->hbuf, Rq, 4 * ad, ad, w.wfc1, linear_epi(h->mlp, 4 * ad, 0, w.bfc1, VF_ACT_GELU), s));
    VF_TRY(split_linear(h->mlp, Rq, w.cout, 4 * ad, w.wfc2,
                        linear_epi(h->buf[yst][yj], w.cout, 1, w.bfc2, VF_ACT_NONE, 1), s));
    h->launches += 2;
    st = yst; j = yj;
    return VF_OK;
}

// patch rows of m clips in h->patches -> h->normed (m x 393 x 768) and the stage taps
static int run_net(vf_mvit* h, int m, cudaStream_t s) {
    const int R = m * MV_TQ * 3136;
    VF_TRY(split_linear(h->patches, R, 96, MV_PK, h->w_patch, linear_epi(h->emb, 96, 1, h->b_patch, VF_ACT_NONE), s));
    VF_TRY(mvit_embed(h->emb, h->cls, h->cls_pos, h->tpos, h->spos, m, h->embed, h->buf[0][0], s));
    h->launches += 2;
    h->tap[0] = h->embed;
    h->tap_C[0] = 96;
    int st = 0, j = 0;
    for (int i = 0; i < MV_BLOCKS; ++i) {
        VF_TRY(run_block(h, h->blocks[i], m, st, j, s));
        if (i == MV_BLOCKS - 1 || h->blocks[i + 1].sq > 1) {
            h->tap[st + 1] = h->buf[st][j];
            h->tap_C[st + 1] = h->blocks[i].cout;
        }
    }
    VF_TRY(swin3d_layernorm(h->buf[st][j], 768, h->norm_w, h->norm_b, h->normed, 1, m * rows_of(7), s, nullptr, 1e-6f));
    h->launches += 1;
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_mvit_destroy(vf_mvit_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_mvit_create(vf_mvit_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "mvit_create: null argument");
    *out = nullptr;
    if (max_clips <= 0) max_clips = 4;
    if (max_clips > R21D_MAX_CHUNK) return fail(VF_ERR_INVALID, "mvit_create: workspace of %d clips", max_clips);
    const ResTensors Tn{tensors, n_tensors, "mvit_create"};
    // v2 from its relative-position tables, v1 from its absolute position embeddings; every key's size is checked below
    const bool v2 = Tn.find("blocks.0.attn.rel_pos_h") != nullptr;
    if (!v2 && !Tn.find("pos_encoding.spatial_pos"))
        return fail(VF_ERR_UNSUPPORTED, "mvit_create: neither 'blocks.0.attn.rel_pos_h' (mvit_v2_s) nor "
                    "'pos_encoding.spatial_pos' (mvit_v1_b) is present");
    if (Tn.find("blocks.16.norm1.weight"))
        return fail(VF_ERR_UNSUPPORTED, "mvit_create: tensor 'blocks.16.norm1.weight': 16 blocks are built");
    if (v2 && Tn.find("pos_encoding.spatial_pos"))
        return fail(VF_ERR_UNSUPPORTED, "mvit_create: tensor 'pos_encoding.spatial_pos' with relative positions (neither "
                    "mvit_v1_b nor mvit_v2_s)");
    VF_TRY(check_device(device));
    vf_mvit* h = new vf_mvit();
    h->who = "mvit_create";
    h->device = device; h->v2 = v2; h->max_clips = max_clips;
    auto body = [&]() -> int {
        auto pool = [&](const std::string& p, MvPool& o) -> int {
            VF_TRY(upload_vec(h, Tn, p + ".pool.weight", 96 * 27, &o.w));
            VF_TRY(upload_vec(h, Tn, p + ".norm_act.0.weight", 96, &o.g));
            return upload_vec(h, Tn, p + ".norm_act.0.bias", 96, &o.b);
        };
        VF_TRY(upload_split_mat(h, Tn, "conv_proj.weight", 96, MV_PATCH_K, &h->w_patch, MV_PK));
        VF_TRY(upload_vec(h, Tn, "conv_proj.bias", 96, &h->b_patch));
        VF_TRY(upload_vec(h, Tn, "pos_encoding.class_token", 96, &h->cls));
        if (!v2) {
            VF_TRY(upload_vec(h, Tn, "pos_encoding.class_pos", 96, &h->cls_pos));
            VF_TRY(upload_vec(h, Tn, "pos_encoding.temporal_pos", MV_TQ * 96, &h->tpos));
            VF_TRY(upload_vec(h, Tn, "pos_encoding.spatial_pos", 3136 * 96, &h->spos));
        }
        VF_TRY(upload_vec(h, Tn, "norm.weight", 768, &h->norm_w));
        VF_TRY(upload_vec(h, Tn, "norm.bias", 768, &h->norm_b));
        size_t hb = 0, qk = 0, qp = 0, kv = 0, at = 0, ml = 0;
        int S = 56;
        for (int i = 0; i < MV_BLOCKS; ++i) {
            MvBlock& w = h->blocks[i];
            w.heads = kHeads[i];
            w.cin = v2 ? kCinV2[i] : kCinV1[i];
            w.cout = v2 ? kCoutV2[i] : kCoutV1[i];
            w.ad = v2 ? w.cout : w.cin;
            w.sq = kStrideQ[i]; w.skv = kStrideKV[i]; w.s_in = S;
            w.pool_q = v2 || w.sq > 1;
            w.project = w.cin != w.cout;
            const std::string p = "blocks." + std::to_string(i) + ".";
            const int64_t ad = w.ad;
            VF_TRY(upload_vec(h, Tn, p + "norm1.weight", w.cin, &w.n1w));
            VF_TRY(upload_vec(h, Tn, p + "norm1.bias", w.cin, &w.n1b));
            VF_TRY(upload_vec(h, Tn, p + "norm2.weight", ad, &w.n2w));
            VF_TRY(upload_vec(h, Tn, p + "norm2.bias", ad, &w.n2b));
            VF_TRY(upload_split_mat(h, Tn, p + "attn.qkv.weight", 3 * ad, w.cin, &w.wqkv));
            VF_TRY(upload_vec(h, Tn, p + "attn.qkv.bias", 3 * ad, &w.bqkv));
            VF_TRY(upload_split_mat(h, Tn, p + "attn.project.0.weight", ad, ad, &w.wproj));
            VF_TRY(upload_vec(h, Tn, p + "attn.project.0.bias", ad, &w.bproj));
            VF_TRY(upload_split_mat(h, Tn, p + "mlp.0.weight", 4 * ad, ad, &w.wfc1));
            VF_TRY(upload_vec(h, Tn, p + "mlp.0.bias", 4 * ad, &w.bfc1));
            VF_TRY(upload_split_mat(h, Tn, p + "mlp.3.weight", w.cout, 4 * ad, &w.wfc2));
            VF_TRY(upload_vec(h, Tn, p + "mlp.3.bias", w.cout, &w.bfc2));
            if (w.project) {
                VF_TRY(upload_split_mat(h, Tn, p + "project.weight", w.cout, w.cin, &w.wprj));
                VF_TRY(upload_vec(h, Tn, p + "project.bias", w.cout, &w.bprj));
            }
            if (w.pool_q) VF_TRY(pool(p + "attn.pool_q", w.pq));
            else if (Tn.find(p + "attn.pool_q.pool.weight"))
                return fail(VF_ERR_UNSUPPORTED, "mvit_create: tensor '%sattn.pool_q.pool.weight' in an mvit_v1_b block "
                            "without q pooling", p.c_str());
            VF_TRY(pool(p + "attn.pool_k", w.pk));
            VF_TRY(pool(p + "attn.pool_v", w.pv));
            if (v2) {
                const int sp = 2 * std::max(w.s_q(), w.s_kv()) - 1;
                VF_TRY(upload_vec(h, Tn, p + "attn.rel_pos_h", int64_t(sp) * 96, &w.rel_h));
                VF_TRY(upload_vec(h, Tn, p + "attn.rel_pos_w", int64_t(sp) * 96, &w.rel_w));
                VF_TRY(upload_vec(h, Tn, p + "attn.rel_pos_t", int64_t(2 * MV_TQ - 1) * 96, &w.rel_t));
            }
            const size_t n_in = size_t(rows_of(S)), n_q = size_t(rows_of(w.s_q()));
            hb = std::max({hb, n_in * w.cin, n_q * ad});
            qk = std::max(qk, n_in * 3 * ad);
            if (w.pool_q) qp = std::max(qp, n_q * ad);
            kv = std::max(kv, size_t(rows_of(w.s_kv())) * ad);
            at = std::max(at, n_q * ad);
            ml = std::max(ml, n_q * 4 * ad);
            S = w.s_q();
        }
        const size_t M = size_t(max_clips);
        VF_TRY(ralloc(h, &h->patches, M * MV_TQ * 3136 * MV_PK));
        VF_TRY(ralloc(h, &h->emb, M * MV_TQ * 3136 * 96));
        VF_TRY(ralloc(h, &h->embed, M * rows_of(56) * 96));
        for (int st = 0; st < 4; ++st)      // stage st holds rows of up to min(192 << st, 768) channels
            for (int j = 0; j < 2; ++j) VF_TRY(ralloc(h, &h->buf[st][j], M * rows_of(56 >> st) * std::min(192 << st, 768)));
        VF_TRY(ralloc(h, &h->hbuf, M * hb));
        VF_TRY(ralloc(h, &h->qkv, M * qk));
        VF_TRY(ralloc(h, &h->qp, M * qp));
        VF_TRY(ralloc(h, &h->kp, M * kv));
        VF_TRY(ralloc(h, &h->vp, M * kv));
        VF_TRY(ralloc(h, &h->att, M * at));
        VF_TRY(ralloc(h, &h->mlp, M * ml));
        VF_TRY(ralloc(h, &h->normed, M * rows_of(7) * 768));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_mvit_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_mvit_info(const vf_mvit_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "mvit_info: null argument");
    const int v[4] = {768, h->v2 ? 2 : 1, MV_T, h->max_clips};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

}  // extern "C"

namespace vf {

// u8: frames n_frames x H x W x 3 and host starts[n]; f32: clips n x 3 x 16 x 224 x 224
static int mv_forward(vf_mvit* h, const void* src, int is_u8, int n_frames, int H, int W, const int* starts, int n,
                      int T, float* out, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "mvit_forward: null handle");
    if (n < 0 || T != MV_T)
        return fail(VF_ERR_INVALID, "mvit_forward: %d clips of %d frames (the position tables fix 16 frames)", n, T);
    if (n > 0 && (!src || !out || (is_u8 && !starts))) return fail(VF_ERR_INVALID, "mvit_forward: null argument");
    const int per_chunk = std::min(h->max_clips, R21D_MAX_CHUNK);
    int rh = MV_CROP, rw = MV_CROP, cy = 0, cx = 0;
    if (is_u8) {
        if (H < 1 || W < 1) return fail(VF_ERR_INVALID, "mvit_forward: frame size %dx%d", H, W);
        for (int i = 0; i < n; ++i)
            if (starts[i] < 0 || int64_t(starts[i]) + T > n_frames)
                return fail(VF_ERR_INVALID, "mvit_forward: clip %d (frames %d..%d) outside the %d frames", i, starts[i],
                            starts[i] + T - 1, n_frames);
        VF_TRY(vf_resize_geometry(H, W, MV_RESIZE, 1, &rh, &rw));     // Resize([256]): the short side to 256
        cy = center_crop_offset(rh, MV_CROP);
        cx = center_crop_offset(rw, MV_CROP);
    }
    if (n == 0) return VF_OK;
    const int64_t per_clip = rows_of(7) * 768;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n;) {      // calls beyond the workspace run in chunks
        int m = 0;
        if (is_u8) {
            int lo = 0, hi = 0;
            R21DStarts st;
            // the patch kernel reads the caller's frames in place: any frame span fits
            VF_TRY(clip_window("mvit_forward", starts + off, n - off, T, per_chunk, INT_MAX, &m, &lo, &hi, &st));
            const uint8_t* f0 = static_cast<const uint8_t*>(src) + int64_t(lo) * H * W * 3;
            VF_TRY(mvit_patch_u8(f0, st, m, H, W, rh, rw, cy, cx, h->patches, s));
        } else {
            m = std::min(per_chunk, n - off);
            VF_TRY(mvit_patch_f32(static_cast<const float*>(src) + int64_t(off) * 3 * T * MV_CROP * MV_CROP, m,
                                  h->patches, s));
        }
        h->launches += 1;
        VF_TRY(run_graphed(h, {m, 0, 0, 0}, [&] { return run_net(h, m, s); }));
        // the feature: the class-token row of each clip's final norm
        VF_CUDA(cudaMemcpy2DAsync(out + int64_t(off) * 768, 768 * sizeof(float), h->normed, per_clip * sizeof(float),
                                  768 * sizeof(float), size_t(m), cudaMemcpyDeviceToDevice, s));
        h->last_m = m;
        off += m;
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_mvit_forward_f32(vf_mvit_t* h, const float* clips, int n, int T, float* out, void* stream) {
    return mv_forward(h, clips, 0, 0, MV_CROP, MV_CROP, nullptr, n, T, out, stream);
}

int vf_mvit_forward_u8(vf_mvit_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n, int T,
                       float* out, void* stream) {
    return mv_forward(h, frames, 1, n_frames, H, W, starts, n, T, out, stream);
}

int vf_mvit_read_stage(vf_mvit_t* h, int stage, float* out, int64_t capacity, int* dims3, void* stream) {
    if (!h || !dims3 || h->last_m <= 0) return fail(VF_ERR_INVALID, "mvit_read_stage: no forward has run");
    if (stage < 0 || stage > 5) return fail(VF_ERR_INVALID, "mvit_read_stage: unknown stage %d", stage);
    const int S = stage == 0 ? 56 : stage == 5 ? 7 : 56 >> (stage - 1);
    const int C = stage == 5 ? 768 : h->tap_C[stage];
    dims3[0] = h->last_m; dims3[1] = int(rows_of(S)); dims3[2] = C;
    if (!out) return VF_OK;
    const int64_t count = int64_t(dims3[0]) * dims3[1] * C;
    if (capacity < count) return fail(VF_ERR_INVALID, "mvit_read_stage: capacity too small");
    const float* src = stage == 5 ? h->normed : h->tap[stage];
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));      // diagnostics only: the engine stream has finished the last call
    VF_CUDA(cudaMemcpyAsync(out, src, size_t(count) * sizeof(float), cudaMemcpyDeviceToDevice,
                            static_cast<cudaStream_t>(stream)));
    return VF_OK;
}

int vf_mvit_attention(const void* q, int ldq, const void* k, const void* v, const float* rel_h, const float* rel_w,
                      const float* rel_t, int n, int heads, const int* q_thw, const int* k_thw, int rel, int resid,
                      void* out, void* stream) {
    if (!q || !k || !v || !out || !q_thw || !k_thw) return fail(VF_ERR_INVALID, "mvit_attention: null argument");
    MViTAttnGeom g;
    g.n = n; g.heads = heads; g.ldq = ldq; g.rel = rel != 0; g.resid = resid != 0;
    for (int i = 0; i < 3; ++i) { g.q_thw[i] = q_thw[i]; g.k_thw[i] = k_thw[i]; }
    return mvit_attention(static_cast<const __half*>(q), static_cast<const __half*>(k), static_cast<const __half*>(v),
                          rel_h, rel_w, rel_t, static_cast<__half*>(out), g, static_cast<cudaStream_t>(stream));
}

int vf_mvit_head_pool(const void* src, int ld_src, int n, int heads, int T, int H, int W, int stride,
                      const float* weight, const float* gamma, const float* beta, void* dst, void* stream) {
    if (!src || !weight || !gamma || !beta || !dst) return fail(VF_ERR_INVALID, "mvit_head_pool: null argument");
    return mvit_head_pool(static_cast<const __half*>(src), ld_src, n, heads, T, H, W, stride, weight, gamma, beta,
                          static_cast<__half*>(dst), static_cast<cudaStream_t>(stream));
}

int vf_mvit_skip_pool(const float* x, int n, int C, int T, int H, int W, float* y, void* stream) {
    if (!x || !y) return fail(VF_ERR_INVALID, "mvit_skip_pool: null argument");
    return mvit_skip_pool(x, n, C, T, H, W, y, static_cast<cudaStream_t>(stream));
}

int64_t vf_mvit_launch_count(const vf_mvit_t* h) { return h ? h->launches : 0; }

}  // extern "C"
