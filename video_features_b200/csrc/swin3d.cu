// torchvision Swin3D-T / S / B (`torchvision.models.video.swin3d_{t,s,b}`, eval) on the wgmma GEMM and the kernels of
// swin3d_kernels.cu: the clip feature `flatten(avgpool(norm(features(patch_embed(x)))))`, torchvision's forward without
// `head` (the classifier is class_head.cu's).  The fused input transform is the Swin3D_*_Weights.KINETICS400_V1 preset.
//
// Numerics: every GEMM weight is a split-fp16 pair W_hi | W_lo (lo = fp16(w - hi)), run as a 1-tap split-weight
// linear on the conv-mode GEMM (each A tile multiplied by both halves); accumulation fp32; the residual stream,
// LayerNorm statistics, softmax max / sum fp32.  Rounded to one fp16 value: patch rows, the outputs of norm1 / norm2 /
// the merge norm, q / k / v, P per 64-key block, the attention output and the MLP hidden layer.
// scripts/precision/emulate_swin3d.py shows why: fp16 weights alone put swin3d_b's features at 1.14e-3 max-abs / max,
// over the 1e-3 bar, while every other class alone in fp16 costs under 5e-5 (DESIGN.md §4.14).  proj and mlp.3 add their
// tiles into the fp32 residual stream from the GEMM epilogue (fp32 reductions, each element once); the merge reduction
// writes the next stage's fp32 stream.
// Rows are in natural (clip, t', h', w') order throughout; the window attention kernel owns the padding, cyclic shift
// and partition.  patch_embed.norm writes both the stage-0 tap and stage 1's residual stream.  Per (clips, T) one CUDA
// graph covers the patch-embedding GEMM to the final norm and clip mean.
// Geometry at 224 x 224, T frames: T' = ceil(T / 2); stage s (0..3) has C << s channels on T' x (56 >> s)^2 tokens.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"
#include "split_conv.h"
#include "swin3d_kernels.h"

namespace vf {

struct SwBlock {
    float *n1w, *n1b, *n2w, *n2b, *bqkv, *bproj, *bfc1, *bfc2, *table;
    __half *wqkv, *wproj, *wfc1, *wfc2;
};
struct SwMerge {
    float *nw, *nb;
    __half* wred;
};

}  // namespace vf

using namespace vf;

struct vf_swin3d : vf::EngineCore {
    int dim = 0, depths[4] = {0, 0, 0, 0}, max_clips = 0, max_T = 0;
    int64_t cap_rows = 0;                          // stage-1 rows the workspace holds: max_clips x T'(max_T) x 3136
    __half* w_patch = nullptr;
    float *b_patch = nullptr, *pe_w = nullptr, *pe_b = nullptr, *norm_w = nullptr, *norm_b = nullptr;
    std::vector<SwBlock> blocks[4];
    SwMerge merge[3];
    // workspace; x[0] (patch embedding + norm), x[1..4] (stage outputs) and normed are kept for vf_swin3d_read_stage
    __half *patches = nullptr, *hbuf = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr;
    float *emb = nullptr, *x[5] = {nullptr, nullptr, nullptr, nullptr, nullptr}, *normed = nullptr, *feat = nullptr;
    int last_m = 0, last_T = 0;
};

namespace vf {

static int tq_of(int T) { return (T + 1) / 2; }

// one SwinTransformerBlock on the stage's residual stream x (rows R of C), in place
static int run_block(vf_swin3d* h, const SwBlock& w, float* x, int m, int Tq, int S, int C, bool shifted, cudaStream_t s) {
    const int R = m * Tq * S * S;
    VF_TRY(swin3d_layernorm(x, C, w.n1w, w.n1b, h->hbuf, 0, R, s));
    VF_TRY(split_linear(h->hbuf, R, 3 * C, C, w.wqkv, linear_epi(h->qkv, 3 * C, 0, w.bqkv, VF_ACT_NONE), s));
    VF_TRY(swin3d_attention(h->qkv, w.bqkv, w.table, h->att, swin3d_attn_geom(m, Tq, S, S, C, shifted), s));
    VF_TRY(split_linear(h->att, R, C, C, w.wproj, linear_epi(x, C, 1, w.bproj, VF_ACT_NONE, 1), s));
    VF_TRY(swin3d_layernorm(x, C, w.n2w, w.n2b, h->hbuf, 0, R, s));
    VF_TRY(split_linear(h->hbuf, R, 4 * C, C, w.wfc1, linear_epi(h->mlp, 4 * C, 0, w.bfc1, VF_ACT_GELU), s));
    VF_TRY(split_linear(h->mlp, R, C, 4 * C, w.wfc2, linear_epi(x, C, 1, w.bfc2, VF_ACT_NONE, 1), s));
    h->launches += 7;
    return VF_OK;
}

// patch rows of m clips of T frames in h->patches -> h->feat (m x 8C) and the retained stages
static int run_net(vf_swin3d* h, int m, int T, cudaStream_t s) {
    const int Tq = tq_of(T), C = h->dim;
    const int R = m * Tq * 3136;
    VF_TRY(split_linear(h->patches, R, C, SW_PK, h->w_patch, linear_epi(h->emb, C, 1, h->b_patch, VF_ACT_NONE), s));
    VF_TRY(swin3d_layernorm(h->emb, C, h->pe_w, h->pe_b, h->x[0], 1, R, s, h->x[1]));
    h->launches += 2;
    for (int st = 0; st < 4; ++st) {
        const int Cs = C << st, S = 56 >> st;
        for (int d = 0; d < h->depths[st]; ++d)
            VF_TRY(run_block(h, h->blocks[st][d], h->x[st + 1], m, Tq, S, Cs, d % 2 == 1, s));
        if (st < 3) {
            const int Rn = m * Tq * (S / 2) * (S / 2);
            VF_TRY(swin3d_merge_layernorm(h->x[st + 1], m, Tq, S, S, Cs, h->merge[st].nw, h->merge[st].nb, h->hbuf, s));
            VF_TRY(split_linear(h->hbuf, Rn, 2 * Cs, 4 * Cs, h->merge[st].wred,
                                linear_epi(h->x[st + 2], 2 * Cs, 1, nullptr, VF_ACT_NONE), s));
            h->launches += 2;
        }
    }
    VF_TRY(swin3d_norm_mean(h->x[4], m, Tq * 49, 8 * C, h->norm_w, h->norm_b, h->normed, h->feat, s));
    h->launches += 1;
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_swin3d_destroy(vf_swin3d_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_swin3d_create(vf_swin3d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips,
                     int max_T) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "swin3d_create: null argument");
    *out = nullptr;
    if (max_clips <= 0) max_clips = 4;
    if (max_T <= 0) max_T = 32;
    if (max_clips > R21D_MAX_CHUNK || max_T > 4096)
        return fail(VF_ERR_INVALID, "swin3d_create: workspace of %d clips x %d frames", max_clips, max_T);
    const ResTensors Tn{tensors, n_tensors, "swin3d_create"};
    // the shape from the weights: embed dim from the patch embedding, depths from the block keys, heads = dim / 32;
    // patch (2,4,4) from the conv weight's size and window (8,7,7) from the bias-table size
    const vf_named_tensor* pb = Tn.find("patch_embed.proj.bias");
    if (!pb) return fail(VF_ERR_INVALID, "swin3d_create: missing tensor 'patch_embed.proj.bias'");
    const int dim = int(pb->numel);
    if (dim != 96 && dim != 128)
        return fail(VF_ERR_UNSUPPORTED, "swin3d_create: tensor 'patch_embed.proj.bias' gives embed dim %lld (96 and 128 "
                    "are built)", (long long)pb->numel);
    const vf_named_tensor* pw = Tn.find("patch_embed.proj.weight");
    if (!pw) return fail(VF_ERR_INVALID, "swin3d_create: missing tensor 'patch_embed.proj.weight'");
    if (pw->numel != int64_t(dim) * SW_PK)
        return fail(VF_ERR_UNSUPPORTED, "swin3d_create: tensor 'patch_embed.proj.weight' has %lld elements, not %d x 3 x "
                    "2 x 4 x 4 (patch (2,4,4) is built)", (long long)pw->numel, dim);
    int depths[4];
    for (int st = 0; st < 4; ++st) {
        int d = 0;
        while (Tn.find("features." + std::to_string(2 * st) + "." + std::to_string(d) + ".norm1.weight")) ++d;
        depths[st] = d;
    }
    const bool t_or_s = dim == 96 && depths[0] == 2 && depths[1] == 2 && (depths[2] == 6 || depths[2] == 18) &&
                        depths[3] == 2;
    const bool b = dim == 128 && depths[0] == 2 && depths[1] == 2 && depths[2] == 18 && depths[3] == 2;
    if (!t_or_s && !b) {
        int st = 0;
        const int want[4] = {2, 2, dim == 96 && depths[2] == 6 ? 6 : 18, 2};
        while (st < 3 && depths[st] == want[st]) ++st;
        return fail(VF_ERR_UNSUPPORTED, "swin3d_create: tensors 'features.%d.*.norm1.weight' give %d blocks in stage %d "
                    "at embed dim %d (depths (2,2,6,2) or (2,2,18,2) at 96, (2,2,18,2) at 128 are built)", 2 * st,
                    depths[st], st + 1, dim);
    }
    for (int st = 0; st < 4; ++st) {
        const std::string key = "features." + std::to_string(2 * st) + ".0.attn.relative_position_bias_table";
        const vf_named_tensor* tb = Tn.find(key);
        const int heads = (dim << st) / SW_HEAD_DIM;
        if (!tb) return fail(VF_ERR_INVALID, "swin3d_create: missing tensor '%s'", key.c_str());
        if (tb->numel != int64_t(SW_TABLE) * heads)
            return fail(VF_ERR_UNSUPPORTED, "swin3d_create: tensor '%s' has %lld elements, not 15 x 13 x 13 x %d (window "
                        "(8,7,7) with heads = dim / 32 is built)", key.c_str(), (long long)tb->numel, heads);
    }
    VF_TRY(check_device(device));
    vf_swin3d* h = new vf_swin3d();
    h->who = "swin3d_create";
    h->device = device; h->dim = dim; h->max_clips = max_clips; h->max_T = max_T;
    memcpy(h->depths, depths, sizeof(depths));
    h->cap_rows = int64_t(max_clips) * tq_of(max_T) * 3136;
    auto body = [&]() -> int {
        const int C = dim;
        VF_TRY(upload_split_mat(h, Tn, "patch_embed.proj.weight", C, SW_PK, &h->w_patch));   // [C][c kt kh kw] pairs
        VF_TRY(upload_vec(h, Tn, "patch_embed.proj.bias", C, &h->b_patch));
        VF_TRY(upload_vec(h, Tn, "patch_embed.norm.weight", C, &h->pe_w));
        VF_TRY(upload_vec(h, Tn, "patch_embed.norm.bias", C, &h->pe_b));
        VF_TRY(upload_vec(h, Tn, "norm.weight", 8 * C, &h->norm_w));
        VF_TRY(upload_vec(h, Tn, "norm.bias", 8 * C, &h->norm_b));
        for (int st = 0; st < 4; ++st) {
            const int64_t Cs = C << st, heads = Cs / SW_HEAD_DIM;
            for (int d = 0; d < depths[st]; ++d) {
                const std::string p = "features." + std::to_string(2 * st) + "." + std::to_string(d) + ".";
                SwBlock w;
                VF_TRY(upload_vec(h, Tn, p + "norm1.weight", Cs, &w.n1w));
                VF_TRY(upload_vec(h, Tn, p + "norm1.bias", Cs, &w.n1b));
                VF_TRY(upload_vec(h, Tn, p + "norm2.weight", Cs, &w.n2w));
                VF_TRY(upload_vec(h, Tn, p + "norm2.bias", Cs, &w.n2b));
                VF_TRY(upload_vec(h, Tn, p + "attn.qkv.bias", 3 * Cs, &w.bqkv));
                VF_TRY(upload_vec(h, Tn, p + "attn.proj.bias", Cs, &w.bproj));
                VF_TRY(upload_vec(h, Tn, p + "mlp.0.bias", 4 * Cs, &w.bfc1));
                VF_TRY(upload_vec(h, Tn, p + "mlp.3.bias", Cs, &w.bfc2));
                VF_TRY(upload_vec(h, Tn, p + "attn.relative_position_bias_table", SW_TABLE * heads, &w.table));
                VF_TRY(upload_split_mat(h, Tn, p + "attn.qkv.weight", 3 * Cs, Cs, &w.wqkv));
                VF_TRY(upload_split_mat(h, Tn, p + "attn.proj.weight", Cs, Cs, &w.wproj));
                VF_TRY(upload_split_mat(h, Tn, p + "mlp.0.weight", 4 * Cs, Cs, &w.wfc1));
                VF_TRY(upload_split_mat(h, Tn, p + "mlp.3.weight", Cs, 4 * Cs, &w.wfc2));
                h->blocks[st].push_back(w);
            }
            if (st < 3) {
                const std::string p = "features." + std::to_string(2 * st + 1) + ".";
                VF_TRY(upload_vec(h, Tn, p + "norm.weight", 4 * Cs, &h->merge[st].nw));
                VF_TRY(upload_vec(h, Tn, p + "norm.bias", 4 * Cs, &h->merge[st].nb));
                VF_TRY(upload_split_mat(h, Tn, p + "reduction.weight", 2 * Cs, 4 * Cs, &h->merge[st].wred));
            }
        }
        // workspace for cap_rows stage-1 rows R: stage s has R / 4^s rows of C << s, so every per-row buffer is largest
        // in stage 1 (the merge norm's R / 4 rows of 4C included)
        const size_t R = size_t(h->cap_rows);
        VF_TRY(ralloc(h, &h->patches, R * SW_PK));
        VF_TRY(ralloc(h, &h->emb, R * C));
        for (int i = 0; i < 5; ++i) VF_TRY(ralloc(h, &h->x[i], i == 0 ? R * C : (R >> (2 * (i - 1))) * (size_t(C) << (i - 1))));
        VF_TRY(ralloc(h, &h->hbuf, R * C));
        VF_TRY(ralloc(h, &h->qkv, R * 3 * C));
        VF_TRY(ralloc(h, &h->att, R * C));
        VF_TRY(ralloc(h, &h->mlp, R * 4 * C));
        VF_TRY(ralloc(h, &h->normed, (R / 64) * 8 * C));
        VF_TRY(ralloc(h, &h->feat, size_t(max_clips) * 8 * C));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_swin3d_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_swin3d_info(const vf_swin3d_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "swin3d_info: null argument");
    const int v[8] = {8 * h->dim, h->dim, h->depths[0], h->depths[1], h->depths[2], h->depths[3], h->max_clips, h->max_T};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

}  // extern "C"

namespace vf {

// u8: frames n_frames x H x W x 3 and host starts[n]; f32: clips n x 3 x T x 224 x 224
static int sw_forward(vf_swin3d* h, const void* src, int is_u8, int n_frames, int H, int W, const int* starts, int n,
                      int T, float* out, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "swin3d_forward: null handle");
    if (n < 0 || T < 1) return fail(VF_ERR_INVALID, "swin3d_forward: %d clips of %d frames", n, T);
    if (n > 0 && (!src || !out || (is_u8 && !starts))) return fail(VF_ERR_INVALID, "swin3d_forward: null argument");
    const int64_t per_clip = int64_t(tq_of(T)) * 3136;
    const int per_chunk = int(std::min<int64_t>(h->cap_rows / per_clip, std::min(h->max_clips, R21D_MAX_CHUNK)));
    if (per_chunk < 1)
        return fail(VF_ERR_INVALID, "swin3d_forward: a %d-frame clip exceeds the workspace (%d clips x %d frames)", T,
                    h->max_clips, h->max_T);
    FrameGeom g{SW_CROP, SW_CROP, 0, 0, false};
    if (is_u8) {
        if (H < 1 || W < 1) return fail(VF_ERR_INVALID, "swin3d_forward: frame size %dx%d", H, W);
        for (int i = 0; i < n; ++i)
            if (starts[i] < 0 || int64_t(starts[i]) + T > n_frames)
                return fail(VF_ERR_INVALID, "swin3d_forward: clip %d (frames %d..%d) outside the %d frames", i, starts[i],
                            starts[i] + T - 1, n_frames);
        VF_TRY(frame_geometry("swin3d_forward", H, W, SW_RESIZE, SW_CROP, &g));     // Resize([256]), CenterCrop(224)
    }
    if (n == 0) return VF_OK;
    const int C8 = 8 * h->dim;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n;) {      // calls beyond the workspace run in chunks
        int m = 0;
        if (is_u8) {
            int lo = 0, hi = 0;
            R21DStarts st;
            // the patch kernel reads the caller's frames in place: any frame span fits
            VF_TRY(clip_window("swin3d_forward", starts + off, n - off, T, per_chunk, INT_MAX, &m, &lo, &hi, &st));
            const uint8_t* f0 = static_cast<const uint8_t*>(src) + int64_t(lo) * H * W * 3;
            VF_TRY(swin3d_patch_u8(f0, st, m, T, H, W, g.rh, g.rw, g.cy, g.cx, h->patches, s));
        } else {
            m = std::min(per_chunk, n - off);
            VF_TRY(swin3d_patch_f32(static_cast<const float*>(src) + int64_t(off) * 3 * T * SW_CROP * SW_CROP, m, T,
                                    h->patches, s));
        }
        h->launches += 1;
        VF_TRY(run_graphed(h, {m, T, 0, 0}, [&] { return run_net(h, m, T, s); }));
        VF_CUDA(cudaMemcpyAsync(out + int64_t(off) * C8, h->feat, size_t(m) * C8 * sizeof(float),
                                cudaMemcpyDeviceToDevice, s));
        h->last_m = m; h->last_T = T;
        off += m;
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_swin3d_forward_f32(vf_swin3d_t* h, const float* clips, int n, int T, float* out, void* stream) {
    return sw_forward(h, clips, 0, 0, SW_CROP, SW_CROP, nullptr, n, T, out, stream);
}

int vf_swin3d_forward_u8(vf_swin3d_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n,
                         int T, float* out, void* stream) {
    return sw_forward(h, frames, 1, n_frames, H, W, starts, n, T, out, stream);
}

int vf_swin3d_read_stage(vf_swin3d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream) {
    if (!h || !dims5 || h->last_m <= 0) return fail(VF_ERR_INVALID, "swin3d_read_stage: no forward has run");
    if (stage < 0 || stage > 5) return fail(VF_ERR_INVALID, "swin3d_read_stage: unknown stage %d", stage);
    const int si = stage == 0 ? 0 : stage == 5 ? 3 : stage - 1;       // the stage whose geometry the tap has
    const int S = 56 >> si, C = h->dim << si;
    dims5[0] = h->last_m; dims5[1] = tq_of(h->last_T); dims5[2] = S; dims5[3] = S; dims5[4] = C;
    if (!out) return VF_OK;
    const int64_t count = int64_t(dims5[0]) * dims5[1] * S * S * C;
    if (capacity < count) return fail(VF_ERR_INVALID, "swin3d_read_stage: capacity too small");
    const float* src = stage == 5 ? h->normed : h->x[stage == 0 ? 0 : stage];
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));      // diagnostics only: the engine stream has finished the last call
    VF_CUDA(cudaMemcpyAsync(out, src, size_t(count) * sizeof(float), cudaMemcpyDeviceToDevice,
                            static_cast<cudaStream_t>(stream)));
    return VF_OK;
}

int vf_swin3d_attention(const void* qkv, const float* bias_qkv, const float* table, int n, int Tq, int H, int W, int C,
                        int shifted, void* out, void* stream) {
    if (!qkv || !bias_qkv || !table || !out) return fail(VF_ERR_INVALID, "swin3d_attention: null argument");
    return swin3d_attention(static_cast<const __half*>(qkv), bias_qkv, table, static_cast<__half*>(out),
                            swin3d_attn_geom(n, Tq, H, W, C, shifted != 0), static_cast<cudaStream_t>(stream));
}

int64_t vf_swin3d_launch_count(const vf_swin3d_t* h) { return h ? h->launches : 0; }

}  // extern "C"
