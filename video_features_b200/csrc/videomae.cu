// VideoMAE clip features (Hugging Face `VideoMAEForVideoClassification`, Kinetics-400 fine-tuned ViT-S / B / L with
// 16 x 16 patches, 2-frame tubelets, 16 frames at 224 px: 1568 tokens): the classifier's input
// fc_norm(mean over tokens of the last hidden state), on the split-weight wgmma GEMM, swin3d_kernels.cu's LayerNorm and
// the kernels of videomae_kernels.cu.  The fused u8 transform is the processor's: Resize(shortest_edge 224, Pillow
// bilinear), a center crop at the floor offset, BGR->RGB, rescale 1 / 255, Normalize (the checkpoint's mean / std).
//
// Block (pre-LN): x += proj(attn(ln_before(x))); x += fc2(GELU(fc1(ln_after(x)))), LayerNorm eps from the config; qkv is
// one GEMM with bias [q_bias | 0 | v_bias] (the key has no bias).  fc_norm is nn.LayerNorm's default eps 1e-5.
//
// Numerics: every GEMM weight is a split-fp16 pair W_hi | W_lo, run as a 1-tap split-weight linear on the conv-mode GEMM;
// accumulation fp32; the residual stream, LayerNorm statistics, softmax max / sum, the positional table and the clip
// mean fp32.  Rounded to one fp16 value: tubelet rows, ln_before / ln_after outputs, q / k / v, P per 64-key block, the
// attention output and the MLP hidden layer (DESIGN.md §4.18).  proj and fc2 add into the fp32 residual stream from the
// GEMM epilogue.
// Clips are packed along M (row = clip * 1568 + token); per clip count one CUDA graph covers tubelet GEMM to fc_norm.
#include <limits.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"
#include "split_conv.h"
#include "swin3d_kernels.h"
#include "videomae_kernels.h"

namespace vf {

constexpr int VM_MAX_CLIPS = 64;
constexpr float VM_FC_NORM_EPS = 1e-5f;

struct VmBlock {
    float *n1w, *n1b, *n2w, *n2b, *bqkv, *bproj, *bfc1, *bfc2;
    __half *wqkv, *wproj, *wfc1, *wfc2;
};

}  // namespace vf

using namespace vf;

struct vf_videomae : vf::EngineCore {
    int D = 0, depth = 0, heads = 0, hidden = 0, max_clips = 0;
    float eps = 1e-12f;
    VmNorm nm{};
    __half* w_patch = nullptr;
    float *b_patch = nullptr, *pos = nullptr, *fcn_w = nullptr, *fcn_b = nullptr;
    std::vector<VmBlock> blocks;
    struct SplitMat { __half* w; int64_t rows, cols; };
    std::vector<SplitMat> split_mats;     // every split-fp16 weight, for vf_videomae_debug_drop_lo
    // workspace (max_clips clips)
    __half *tubes = nullptr, *hbuf = nullptr, *qkv = nullptr, *att = nullptr, *mlp = nullptr;
    float *x = nullptr, *pooled = nullptr, *feat = nullptr;
};

namespace vf {

static const std::string kPre = "videomae.";

// blocks [l0, l1) on h->x (m clips)
static int vm_blocks(vf_videomae* h, int m, int l0, int l1, cudaStream_t s) {
    const int D = h->D, M = m * VM_TOKENS;
    for (int l = l0; l < l1; ++l) {
        const VmBlock& w = h->blocks[l];
        VF_TRY(swin3d_layernorm(h->x, D, w.n1w, w.n1b, h->hbuf, 0, M, s, nullptr, h->eps));
        VF_TRY(split_linear(h->hbuf, M, 3 * D, D, w.wqkv, linear_epi(h->qkv, 3 * D, 0, w.bqkv, VF_ACT_NONE), s));
        VF_TRY(videomae_attention(h->qkv, h->att, m, VM_TOKENS, h->heads, s));
        VF_TRY(split_linear(h->att, M, D, D, w.wproj, linear_epi(h->x, D, 1, w.bproj, VF_ACT_NONE, 1), s));
        VF_TRY(swin3d_layernorm(h->x, D, w.n2w, w.n2b, h->hbuf, 0, M, s, nullptr, h->eps));
        VF_TRY(split_linear(h->hbuf, M, h->hidden, D, w.wfc1, linear_epi(h->mlp, h->hidden, 0, w.bfc1, VF_ACT_GELU), s));
        VF_TRY(split_linear(h->mlp, M, D, h->hidden, w.wfc2, linear_epi(h->x, D, 1, w.bfc2, VF_ACT_NONE, 1), s));
        h->launches += 7;
    }
    return VF_OK;
}

// h->tubes (m clips) -> h->x
static int vm_embed(vf_videomae* h, int m, cudaStream_t s) {
    VF_TRY(split_linear(h->tubes, m * VM_TOKENS, h->D, VM_PK, h->w_patch,
                        linear_epi(h->x, h->D, 1, h->b_patch, VF_ACT_NONE), s));
    VF_TRY(videomae_add_pos(h->x, h->pos, m, h->D, s));
    h->launches += 2;
    return VF_OK;
}

// fc_norm(mean over the tokens of h->x) -> out (m x D fp32)
static int vm_head(vf_videomae* h, int m, float* out, cudaStream_t s) {
    VF_TRY(videomae_mean(h->x, m, h->D, h->pooled, s));
    VF_TRY(swin3d_layernorm(h->pooled, h->D, h->fcn_w, h->fcn_b, out, 1, m, s, nullptr, VM_FC_NORM_EPS));
    h->launches += 2;
    return VF_OK;
}

static int vm_net(vf_videomae* h, int m, cudaStream_t s) {
    VF_TRY(vm_embed(h, m, s));
    VF_TRY(vm_blocks(h, m, 0, h->depth, s));
    return vm_head(h, m, h->feat, s);
}

// Resize(shortest_edge 224, bilinear) and the processor's center crop, which starts at the floor of half the margin
static int vm_geometry(const char* who, int H, int W, FrameGeom* g) {
    VF_TRY(frame_geometry(who, H, W, VM_CROP, VM_CROP, g));
    g->filter = VF_FILTER_BILINEAR;
    g->cy = (g->rh - VM_CROP) / 2;
    g->cx = (g->rw - VM_CROP) / 2;
    return VF_OK;
}

// u8: frames n_frames x H x W x 3 and host starts[n]; f32: clips n x 16 x 3 x 224 x 224
static int vm_forward(vf_videomae* h, const void* src, int is_u8, int n_frames, int H, int W, const int* starts, int n,
                      int T, float* out, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "videomae_forward: null handle");
    if (n < 0 || T != VM_T)
        return fail(VF_ERR_INVALID, "videomae_forward: %d clips of %d frames (the positional table fixes 16 frames)", n,
                    T);
    if (n > 0 && (!src || !out || (is_u8 && !starts))) return fail(VF_ERR_INVALID, "videomae_forward: null argument");
    FrameGeom g{VM_CROP, VM_CROP, 0, 0, false};
    if (is_u8) {
        for (int i = 0; i < n; ++i)
            if (starts[i] < 0 || int64_t(starts[i]) + T > n_frames)
                return fail(VF_ERR_INVALID, "videomae_forward: clip %d (frames %d..%d) outside the %d frames", i,
                            starts[i], starts[i] + T - 1, n_frames);
        VF_TRY(vm_geometry("videomae_forward", H, W, &g));
    }
    if (n == 0) return VF_OK;
    const int slots = h->max_clips * VM_T;       // frames the resize scratch holds
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n;) {
        int m = 0;
        if (is_u8) {
            int lo = 0, hi = 0;
            R21DStarts st;
            VF_TRY(clip_window("videomae_forward", starts + off, n - off, T, h->max_clips, slots, &m, &lo, &hi, &st));
            const uint8_t* fr;
            VF_TRY(resize_frames(h, static_cast<const uint8_t*>(src) + int64_t(lo) * H * W * 3, hi - lo, H, W, g, slots,
                                 s, &fr));
            VF_TRY(videomae_tubelets_u8(fr, st, m, g.rh, g.rw, g.cy, g.cx, h->nm, h->tubes, s));
        } else {
            m = std::min(h->max_clips, n - off);
            VF_TRY(videomae_tubelets_f32(static_cast<const float*>(src) + int64_t(off) * VM_T * 3 * VM_CROP * VM_CROP, m,
                                         h->tubes, s));
        }
        h->launches += 1;
        VF_TRY(run_graphed(h, {m, 0, 0, 0}, [&] { return vm_net(h, m, s); }));
        VF_CUDA(cudaMemcpyAsync(out + int64_t(off) * h->D, h->feat, size_t(m) * h->D * sizeof(float),
                                cudaMemcpyDeviceToDevice, s));
        off += m;
    }
    return leave(h, user);
}

static int vm_upload_vec(vf_videomae* h, const ResTensors& T, const std::string& name, int64_t n, float** dst) {
    return upload_vec(h, T, kPre + name, n, dst);
}
static int vm_upload_split(vf_videomae* h, const ResTensors& T, const std::string& name, int64_t rows, int64_t cols,
                           __half** dst) {
    VF_TRY(upload_split_mat(h, T, name, rows, cols, dst));
    h->split_mats.push_back({*dst, rows, cols});
    return VF_OK;
}
static int vm_upload_mat(vf_videomae* h, const ResTensors& T, const std::string& name, int64_t rows, int64_t cols,
                         __half** dst) {
    return vm_upload_split(h, T, kPre + name, rows, cols, dst);
}

}  // namespace vf

extern "C" {

int vf_videomae_destroy(vf_videomae_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_videomae_create(vf_videomae_t** out, const vf_named_tensor* tensors, int n_tensors, const float* config,
                       int device, int max_clips) {
    if (!out || !tensors || n_tensors <= 0 || !config) return fail(VF_ERR_INVALID, "videomae_create: null argument");
    *out = nullptr;
    const ResTensors T{tensors, n_tensors, "videomae_create"};
    // config: hidden size, depth, heads, MLP width, LayerNorm eps, qkv_bias (0 / 1)
    const double cD = config[0], cdepth = config[1], cheads = config[2], chidden = config[3];
    if (cD != 384 && cD != 768 && cD != 1024)
        return fail(VF_ERR_UNSUPPORTED, "videomae_create: hidden size %g (384, 768 and 1024 are built)", cD);
    const int D = int(cD);
    if (cheads < 1 || cheads * 64 != cD)
        return fail(VF_ERR_UNSUPPORTED, "videomae_create: %g heads at hidden size %d give head dim %g (64 is built)",
                    cheads, D, cheads >= 1 ? cD / cheads : 0.0);
    if (cdepth < 1 || cdepth > 64 || chidden < 64 || chidden > 8192 || int(chidden) % 64 || !(config[4] > 0.f))
        return fail(VF_ERR_INVALID, "videomae_create: depth %g, MLP width %g, eps %g", cdepth, chidden, double(config[4]));
    const int depth = int(cdepth), hidden = int(chidden);
    if (config[5] != 0.f && config[5] != 1.f)
        return fail(VF_ERR_INVALID, "videomae_create: qkv_bias %g (0 or 1)", double(config[5]));
    const bool qkv_bias = config[5] != 0.f;
    if (T.find(kPre + "encoder.layer." + std::to_string(depth) + ".layernorm_before.weight"))
        return fail(VF_ERR_INVALID, "videomae_create: tensor '%sencoder.layer.%d.layernorm_before.weight' present: the "
                    "config has %d layers", kPre.c_str(), depth, depth);
    if (T.find(kPre + "layernorm.weight"))
        return fail(VF_ERR_UNSUPPORTED, "videomae_create: tensor '%slayernorm.weight' (use_mean_pooling = false) is not "
                    "built", kPre.c_str());
    if (max_clips <= 0) max_clips = 16;
    if (max_clips > VM_MAX_CLIPS)
        return fail(VF_ERR_INVALID, "videomae_create: workspace of %d clips (at most %d)", max_clips, VM_MAX_CLIPS);
    VF_TRY(check_device(device));
    vf_videomae* h = new vf_videomae();
    h->who = "videomae_create";
    h->device = device; h->D = D; h->depth = depth; h->heads = D / 64; h->hidden = hidden; h->max_clips = max_clips;
    h->eps = config[4];
    auto body = [&]() -> int {
        const float *mean, *std_;
        VF_TRY(T.get("image_mean", 3, &mean));
        VF_TRY(T.get("image_std", 3, &std_));
        for (int c = 0; c < 3; ++c) {
            if (!(std_[c] > 0.f)) return fail(VF_ERR_INVALID, "videomae_create: image_std[%d] = %g", c, double(std_[c]));
            h->nm.mean[c] = mean[c]; h->nm.std[c] = std_[c];
        }
        const float* pos;
        VF_TRY(T.get("position_embeddings", int64_t(VM_TOKENS) * D, &pos));
        VF_TRY(upload_f32(h, &h->pos, pos, size_t(VM_TOKENS) * D));
        VF_TRY(vm_upload_mat(h, T, "embeddings.patch_embeddings.projection.weight", D, VM_PK, &h->w_patch));
        VF_TRY(vm_upload_vec(h, T, "embeddings.patch_embeddings.projection.bias", D, &h->b_patch));
        VF_TRY(upload_vec(h, T, "fc_norm.weight", D, &h->fcn_w));
        VF_TRY(upload_vec(h, T, "fc_norm.bias", D, &h->fcn_b));
        for (int l = 0; l < depth; ++l) {
            const std::string p = "encoder.layer." + std::to_string(l) + ".", a = p + "attention.attention.";
            VmBlock w;
            VF_TRY(vm_upload_vec(h, T, p + "layernorm_before.weight", D, &w.n1w));
            VF_TRY(vm_upload_vec(h, T, p + "layernorm_before.bias", D, &w.n1b));
            VF_TRY(vm_upload_vec(h, T, p + "layernorm_after.weight", D, &w.n2w));
            VF_TRY(vm_upload_vec(h, T, p + "layernorm_after.bias", D, &w.n2b));
            // q / k / v as one [3D][D] weight; the bias [q_bias | 0 | v_bias] (no bias at all without qkv_bias)
            const float *wq, *wk, *wv, *bq = nullptr, *bv = nullptr;
            VF_TRY(T.get(kPre + a + "query.weight", int64_t(D) * D, &wq));
            VF_TRY(T.get(kPre + a + "key.weight", int64_t(D) * D, &wk));
            VF_TRY(T.get(kPre + a + "value.weight", int64_t(D) * D, &wv));
            if (qkv_bias) {
                VF_TRY(T.get(kPre + a + "q_bias", D, &bq));
                VF_TRY(T.get(kPre + a + "v_bias", D, &bv));
            } else if (T.find(kPre + a + "q_bias") || T.find(kPre + a + "v_bias")) {
                return fail(VF_ERR_INVALID, "videomae_create: tensor '%s%sq_bias' / 'v_bias' present with qkv_bias = "
                            "false", kPre.c_str(), a.c_str());
            }
            std::vector<float> wqkv(size_t(3) * D * D), bqkv(size_t(3) * D, 0.f);
            memcpy(wqkv.data(), wq, sizeof(float) * D * D);
            memcpy(wqkv.data() + size_t(D) * D, wk, sizeof(float) * D * D);
            memcpy(wqkv.data() + size_t(2) * D * D, wv, sizeof(float) * D * D);
            if (bq) {
                memcpy(bqkv.data(), bq, sizeof(float) * D);
                memcpy(bqkv.data() + 2 * D, bv, sizeof(float) * D);
            }
            const vf_named_tensor qkv_t[2] = {{"qkv.weight", wqkv.data(), int64_t(wqkv.size())},
                                              {"qkv.bias", bqkv.data(), int64_t(bqkv.size())}};
            const ResTensors Q{qkv_t, 2, "videomae_create"};
            VF_TRY(vm_upload_split(h, Q, "qkv.weight", 3 * D, D, &w.wqkv));
            VF_TRY(upload_vec(h, Q, "qkv.bias", 3 * D, &w.bqkv));
            VF_TRY(vm_upload_mat(h, T, p + "attention.output.dense.weight", D, D, &w.wproj));
            VF_TRY(vm_upload_vec(h, T, p + "attention.output.dense.bias", D, &w.bproj));
            VF_TRY(vm_upload_mat(h, T, p + "intermediate.dense.weight", hidden, D, &w.wfc1));
            VF_TRY(vm_upload_vec(h, T, p + "intermediate.dense.bias", hidden, &w.bfc1));
            VF_TRY(vm_upload_mat(h, T, p + "output.dense.weight", D, hidden, &w.wfc2));
            VF_TRY(vm_upload_vec(h, T, p + "output.dense.bias", D, &w.bfc2));
            h->blocks.push_back(w);
        }
        const size_t R = size_t(max_clips) * VM_TOKENS;
        VF_TRY(ralloc(h, &h->tubes, R * VM_PK));
        VF_TRY(ralloc(h, &h->x, R * D));
        VF_TRY(ralloc(h, &h->hbuf, R * D));
        VF_TRY(ralloc(h, &h->qkv, R * 3 * D));
        VF_TRY(ralloc(h, &h->att, R * D));
        VF_TRY(ralloc(h, &h->mlp, R * hidden));
        VF_TRY(ralloc(h, &h->pooled, size_t(max_clips) * D));
        VF_TRY(ralloc(h, &h->feat, size_t(max_clips) * D));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_videomae_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_videomae_info(const vf_videomae_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "videomae_info: null argument");
    const int v[5] = {h->D, h->depth, h->heads, h->hidden, h->max_clips};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

int vf_videomae_forward_f32(vf_videomae_t* h, const float* clips, int n, int T, float* out, void* stream) {
    return vm_forward(h, clips, 0, 0, VM_CROP, VM_CROP, nullptr, n, T, out, stream);
}

int vf_videomae_forward_u8(vf_videomae_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n,
                           int T, float* out, void* stream) {
    return vm_forward(h, frames, 1, n_frames, H, W, starts, n, T, out, stream);
}

int vf_videomae_debug_tubelets_u8(vf_videomae_t* h, const uint8_t* frames, int n_frames, int H, int W,
                                  const int* starts, int n, void* tubelets, void* stream) {
    VF_TRY(debug_frames(h, frames, tubelets, n, h ? h->max_clips : 0, "max_clips", "videomae_debug_tubelets_u8"));
    if (!starts) return fail(VF_ERR_INVALID, "videomae_debug_tubelets_u8: null argument");
    FrameGeom g;
    VF_TRY(vm_geometry("videomae_debug_tubelets_u8", H, W, &g));
    R21DStarts st;
    for (int i = 0; i < n; ++i) {
        if (starts[i] < 0 || int64_t(starts[i]) + VM_T > n_frames)
            return fail(VF_ERR_INVALID, "videomae_debug_tubelets_u8: clip %d outside the %d frames", i, n_frames);
        st.first[i] = starts[i];
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaStreamSynchronize(h->cs));       // a resize buffer may be re-allocated: the engine stream is idle
    const uint8_t* fr;
    VF_TRY(resize_frames(h, frames, n_frames, H, W, g, n_frames, s, &fr));
    VF_TRY(videomae_tubelets_u8(fr, st, n, g.rh, g.rw, g.cy, g.cx, h->nm, static_cast<__half*>(tubelets), s));
    h->launches += 1;
    return VF_OK;
}

int vf_videomae_debug_tubelets_f32(vf_videomae_t* h, const float* clips, int n, void* tubelets, void* stream) {
    VF_TRY(debug_frames(h, clips, tubelets, n, h ? h->max_clips : 0, "max_clips", "videomae_debug_tubelets_f32"));
    VF_TRY(videomae_tubelets_f32(clips, n, static_cast<__half*>(tubelets), static_cast<cudaStream_t>(stream)));
    h->launches += 1;
    return VF_OK;
}

int vf_videomae_debug_embed(vf_videomae_t* h, const void* tubelets, int n, float* x_out, void* stream) {
    VF_TRY(debug_frames(h, tubelets, x_out, n, h ? h->max_clips : 0, "max_clips", "videomae_debug_embed"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaMemcpyAsync(h->tubes, tubelets, size_t(n) * VM_TOKENS * VM_PK * sizeof(__half),
                            cudaMemcpyDeviceToDevice, s));
    VF_TRY(vm_embed(h, n, s));
    VF_CUDA(cudaMemcpyAsync(x_out, h->x, size_t(n) * VM_TOKENS * h->D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_videomae_debug_blocks(vf_videomae_t* h, float* x, int n, int layer_begin, int layer_end, void* stream) {
    VF_TRY(debug_frames(h, x, x, n, h ? h->max_clips : 0, "max_clips", "videomae_debug_blocks"));
    if (layer_begin < 0 || layer_begin >= layer_end || layer_end > h->depth)
        return fail(VF_ERR_INVALID, "videomae_debug_blocks: layers [%d, %d) are not a range within [0, %d)", layer_begin,
                    layer_end, h->depth);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t bytes = size_t(n) * VM_TOKENS * h->D * sizeof(float);
    VF_CUDA(cudaMemcpyAsync(h->x, x, bytes, cudaMemcpyDeviceToDevice, s));
    VF_TRY(vm_blocks(h, n, layer_begin, layer_end, s));
    VF_CUDA(cudaMemcpyAsync(x, h->x, bytes, cudaMemcpyDeviceToDevice, s));
    return VF_OK;
}

int vf_videomae_debug_head(vf_videomae_t* h, const float* x, int n, float* out, void* stream) {
    VF_TRY(debug_frames(h, x, out, n, h ? h->max_clips : 0, "max_clips", "videomae_debug_head"));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaMemcpyAsync(h->x, x, size_t(n) * VM_TOKENS * h->D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return vm_head(h, n, out, s);
}

int vf_videomae_debug_drop_lo(vf_videomae_t* h) {
    if (!h) return fail(VF_ERR_INVALID, "videomae_debug_drop_lo: null handle");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));
    for (const auto& m : h->split_mats)      // rows [hi cols | lo cols]: zero the lo columns
        VF_CUDA(cudaMemset2D(m.w + m.cols, size_t(2 * m.cols) * sizeof(__half), 0, size_t(m.cols) * sizeof(__half),
                             size_t(m.rows)));
    VF_CUDA(cudaDeviceSynchronize());
    return VF_OK;
}

int vf_videomae_attention(const void* qkv, int n, int S, int heads, void* out, void* stream) {
    if (!qkv || !out) return fail(VF_ERR_INVALID, "videomae_attention: null argument");
    return videomae_attention(static_cast<const __half*>(qkv), static_cast<__half*>(out), n, S, heads,
                              static_cast<cudaStream_t>(stream));
}

int64_t vf_videomae_launch_count(const vf_videomae_t* h) { return h ? h->launches : 0; }

}  // extern "C"
