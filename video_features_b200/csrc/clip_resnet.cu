// CLIP ResNet image towers (openai/CLIP ModifiedResNet: RN50, RN101, RN50x4, RN50x16) on the wgmma conv-GEMM.
// Replaces `clip.load("RN50" | "RN101" | "RN50x4" | "RN50x16")` and `model.encode_image(preprocess(frame))`
// (reference: models/CLIP/extract_clip.py:45-64), the transform Resize(n_px, bicubic) -> CenterCrop(n_px) -> ToTensor
// -> Normalize included.  The configuration is inferred from the weights' sizes as clip.model.build_model does.
//
// Layout: as resnet.cu -- every activation is a split-fp16 pair row [hi C | lo C] of a zero-bordered channels-last 2-D
// volume with a one-position border, every weight a hi + lo fp16 pair, BatchNorm folded into the epilogue.
//   stem conv1 (3x3/2 pad 1): 2 taps (kernel row pairs) over the phase volume the transform writes (rows of
//     [16 hi | 16 lo], 4 channels per phase, 3 used), each a run of 2 phase positions x 32 elements;
//   stem conv2 / conv3 and every stride-1 3x3 / 1x1: prep_same;
//   AvgPool2d(2) + 1x1 conv + BatchNorm (the stem's pool feeding layer1.0's conv1 and downsample, and conv3 / the
//     downsample of every stride-2 block): ONE conv over the phase repack (raft_phase_repack) of the unpooled input, one
//     tap of 8C elements with the same weight in all four phase slots and the 1/4 folded into the fp32 BatchNorm scale
//     (a power of two: exact, and the fp16 weight pair keeps every bit it would have without the pool).  No
//     stand-alone pool kernel runs; the pooled stem is never materialised.
//   AttentionPool2d: clip_rn_tokens writes T = HW + 1 token rows [hi E | lo E] (mean first, positional embedding
//     added); K|V is one GEMM over all token rows (N = 2E, k and v weights concatenated, biases in the epilogue, fp32
//     out); Q is a GEMM over token 0 of every frame, read in place with a row pitch of T tokens; clip_rn_attention runs
//     one query per (frame, head); c_proj writes fp32 into the caller's feature rows.
// Geometry at n_px: stem [n][n_px/2 + 2]^2, then [n][S+2]^2 with S = n_px/4, /8, /16, /32 for layer1..4.  Everything
// from the stem conv to the attention is replayed as one CUDA graph per frame count; the resize / transform (which
// depend on the caller's frames) and c_proj (which writes the caller's rows) run around it.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "clip_resnet_kernels.h"
#include "internal.h"
#include "split_conv.h"

namespace vf {

struct RnBlock {
    int cin = 0, width = 0, cout = 0, stride = 1;
    bool pool_in = false;      // layer1.0: its input is the stem's AvgPool2d(2), fused into conv1 and the downsample
    bool down = false;
    ResConv c1, c2, c3, dn;
};

}  // namespace vf

using namespace vf;

struct vf_clip_rn : vf::EngineCore {
    int max_frames = 0, npx = 0, width = 0, embed = 0, heads = 0, out_dim = 0, tokens = 0;
    int layers[4] = {0, 0, 0, 0};
    ResConv stem[3];
    std::vector<RnBlock> blocks;
    ResConv q, kv, cproj;
    float* pos = nullptr;
    // workspace: s0 = stem phase volume; stem_out and the stage outputs are kept for vf_clip_rn_read_stage
    __half *s0 = nullptr, *stem_out = nullptr, *stage_out[4] = {nullptr, nullptr, nullptr, nullptr};
    __half *bufA = nullptr, *bufB = nullptr, *t1 = nullptr, *t2 = nullptr, *ds = nullptr, *ph1 = nullptr, *ph2 = nullptr;
    __half *tok = nullptr, *att = nullptr;
    float *kvo = nullptr, *qo = nullptr;
    int last_n = 0;
    int attn_n = 0;           // frames of the last vf_clip_rn_debug_attnpool (its intermediates stay readable)
};

namespace vf {

static const double kEps = 1e-5;                                // BatchNorm2d

static Vol2 stem_vol(const vf_clip_rn* h, int n) {
    const int S = h->npx / 2;
    return Vol2{n, S + 2, S + 2, 1, S + 1, 1, S + 1};
}
static Vol2 stage_vol(const vf_clip_rn* h, int n, int L) {
    const int S = h->npx / (4 << L);
    return Vol2{n, S + 2, S + 2, 1, S + 1, 1, S + 1};
}

// stem conv1 3x3/2 pad 1 on the transform's phase volume: phase row q holds x[2(q-1)+p]; tap a (kernel rows 2a-1,
// 2a) reads phase row q + a - 1 from column q' - 1 on, 2 phase positions x 32 elements
static int prep_stem1(vf_clip_rn* h, ResConv& cw, const ResTensors& T, int co) {
    cw.ntaps = 2; cw.k_per_tap = 64;
    for (int a = 0; a < 2; ++a) { cw.dh[a] = a - 1; cw.dw[a] = -1; }
    return upload_conv(h, cw, T, "visual.conv1", "visual.bn1", kEps, {co, 3, 1, 3, 3}, 16, [](int, int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return a * 64 + b * 32 + (ph * 2 + pw) * 4 + c;
    });
}

// AvgPool2d(2) -> 1x1 conv -> BatchNorm on the phase repack of split rows of 2*ci: one tap of the four phases, the
// weight in each, 1/4 in the scale
static int prep_pooled(vf_clip_rn* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                       int co, int ci) {
    cw.ntaps = 1; cw.k_per_tap = 8 * ci;
    return upload_conv(h, cw, T, name, bn, kEps, {co, ci, 1, 1, 1}, ci, [](int, int, int, int c) { return c; }, 0, 4, 2 * ci,
                       0.25f);
}

// nn.Linear (weight [co][ci], bias [co]) on split rows of 2*ci; w / b are host pointers already checked
static int prep_linear(vf_clip_rn* h, ResConv& cw, const float* w, const float* b, int co, int ci) {
    cw.ntaps = 1; cw.k_per_tap = 2 * ci;
    const std::vector<float> sc(size_t(co), 1.f), sh(b, b + co);
    return upload_weights(h, cw, w, {co, ci, 1, 1, 1}, ci, [](int, int, int, int c) { return c; }, sc, sh);
}

// one linear on M rows of X (row pitch `pitch` elements) -> fp32 rows of ldo
static int run_linear(vf_clip_rn* h, const ResConv& cw, const __half* X, int pitch, int M, float* out, int ldo,
                      cudaStream_t s) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = 1; g.k_per_tap = cw.k_per_tap; g.nsplit = 2; g.lo_mask = cw.lo_mask; g.mask = 0;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.ldo = ldo; ep.out_f32 = 1; ep.bias = cw.bias; ep.scale = cw.scale; ep.act = VF_ACT_NONE;
    h->launches += 1;
    return conv_gemm_f16(X, pitch, M, cw.w, cw.n_out, g, ep, s);
}

// openai Bottleneck: 1x1, 3x3 (stride 1), AvgPool2d(stride) fused into the 1x1 conv3, the downsample AvgPool2d(stride)
// fused into its 1x1 conv.  x (valid region vi, cin channels) -> dst (vo, cout channels)
static int run_block(vf_clip_rn* h, const RnBlock& B, const __half* x, const Vol2& vi, const Vol2& vo, __half* dst,
                     cudaStream_t s) {
    const __half* res = x;
    const Vol2& vc = B.pool_in ? vo : vi;           // where conv1 / conv2 run
    if (B.pool_in) {
        VF_TRY(raft_phase_repack(x, vi, 2 * B.cin, h->ph2, vo, s));
        VF_TRY(run_conv(h, B.c1, h->ph2, 8 * B.cin, vo, h->t1, true, s));
        h->launches += 1;
    } else {
        VF_TRY(run_conv(h, B.c1, x, 2 * B.cin, vi, h->t1, true, s));
    }
    VF_TRY(run_conv(h, B.c2, h->t1, 2 * B.width, vc, h->t2, true, s));
    if (B.stride == 2) {
        VF_TRY(raft_phase_repack(h->t2, vi, 2 * B.width, h->ph1, vo, s));
        VF_TRY(run_conv(h, B.c3, h->ph1, 8 * B.width, vo, h->t1, false, s));
        h->launches += 1;
    } else {
        VF_TRY(run_conv(h, B.c3, h->t2, 2 * B.width, vo, h->t1, false, s));
    }
    if (B.down) {
        if (B.stride == 2) {
            VF_TRY(raft_phase_repack(x, vi, 2 * B.cin, h->ph2, vo, s));
            h->launches += 1;
        }
        if (B.stride == 2 || B.pool_in) VF_TRY(run_conv(h, B.dn, h->ph2, 8 * B.cin, vo, h->ds, false, s));
        else                            VF_TRY(run_conv(h, B.dn, x, 2 * B.cin, vo, h->ds, false, s));
        res = h->ds;
    }
    VF_TRY(raft_add_relu(res, h->t1, dst, vo, B.cout, s));
    h->launches += 1;
    return VF_OK;
}

// AttentionPool2d up to c_proj's input, on m frames of the layer4 pair volume x4: tokens (h->tok), K|V (h->kvo), Q
// (h->qo: token 0 of every frame, read in place with a pitch of T tokens), attention (h->att).  The trunk graph and
// vf_clip_rn_debug_attnpool run it; run_cproj follows outside the graph, since it writes the caller's rows.
static int run_attention(vf_clip_rn* h, const __half* x4, int m, cudaStream_t s) {
    const int E = h->embed, T = h->tokens;
    VF_TRY(clip_rn_tokens(x4, stage_vol(h, m, 3), E, h->pos, h->tok, s));
    VF_TRY(run_linear(h, h->kv, h->tok, 2 * E, m * T, h->kvo, 2 * E, s));
    VF_TRY(run_linear(h, h->q, h->tok, T * 2 * E, m, h->qo, E, s));
    VF_TRY(clip_rn_attention(h->kvo, h->qo, m, T, E, h->att, s));
    h->launches += 2;
    return VF_OK;
}

// c_proj of the m attention rows in h->att -> m fp32 rows of out_dim
static int run_cproj(vf_clip_rn* h, int m, float* out, cudaStream_t s) {
    return run_linear(h, h->cproj, h->att, 2 * h->embed, m, out, h->out_dim, s);
}

// stem conv1 .. attention on m frames whose stem phase volume is in h->s0
static int run_trunk(vf_clip_rn* h, int m, cudaStream_t s) {
    const Vol2 sv = stem_vol(h, m);
    const int w = h->width;
    VF_TRY(run_conv(h, h->stem[0], h->s0, 32, sv, h->t1, true, s));
    VF_TRY(run_conv(h, h->stem[1], h->t1, w, sv, h->t2, true, s));
    VF_TRY(run_conv(h, h->stem[2], h->t2, w, sv, h->stem_out, true, s));
    const __half* x = h->stem_out;
    size_t bi = 0;
    for (int L = 0; L < 4; ++L)
        for (int b = 0; b < h->layers[L]; ++b, ++bi) {
            const Vol2 vo = stage_vol(h, m, L), vi = b > 0 ? vo : L == 0 ? sv : stage_vol(h, m, L - 1);
            __half* dst = b == h->layers[L] - 1 ? h->stage_out[L] : (x == h->bufA ? h->bufB : h->bufA);
            VF_TRY(run_block(h, h->blocks[bi], x, vi, vo, dst, s));
            x = dst;
        }
    return run_attention(h, h->stage_out[3], m, s);
}

static int clip_rn_encode(vf_clip_rn* h, const void* frames, int is_u8, int n, int H, int W, float* out, void* stream) {
    if (!h || !frames || !out) return fail(VF_ERR_INVALID, "clip_rn_encode: null argument");
    if (n < 0) return fail(VF_ERR_INVALID, "clip_rn_encode: %d frames", n);
    const int npx = h->npx;
    FrameGeom g{npx, npx, 0, 0, false};
    if (is_u8) VF_TRY(frame_geometry("clip_rn_encode", H, W, npx, npx, &g));
    if (n == 0) return VF_OK;
    const size_t frame_elems = is_u8 ? size_t(H) * W * 3 : size_t(3) * npx * npx;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n; off += h->max_frames) {      // calls beyond the workspace run in chunks
        const int m = std::min(h->max_frames, n - off);
        const uint8_t* u8 = nullptr;
        if (is_u8)
            VF_TRY(resize_frames(h, static_cast<const uint8_t*>(frames) + off * frame_elems, m, H, W, g, h->max_frames,
                                 s, &u8));
        const void* src = is_u8 ? static_cast<const void*>(u8) : static_cast<const float*>(frames) + off * frame_elems;
        VF_TRY(clip_rn_input_pack(src, is_u8, m, g.rh, g.rw, g.cy, g.cx, npx, h->s0, s));
        VF_TRY(run_graphed(h, {m, 0, 0, 0}, [&] { return run_trunk(h, m, s); }));
        VF_TRY(run_cproj(h, m, out + size_t(off) * h->out_dim, s));
        h->launches += 1;       // the input pack
        h->last_n = m;
        h->attn_n = 0;
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_clip_rn_destroy(vf_clip_rn_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_clip_rn_create(vf_clip_rn_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "clip_rn_create: null argument");
    *out = nullptr;
    const ResTensors T{tensors, n_tensors, "clip_rn_create"};
    // clip.model.build_model: width from the stem, depths from the block keys, resolution from the positional embedding
    const int64_t n_bn1 = T.numel("visual.bn1.weight");
    if (n_bn1 <= 0) return fail(VF_ERR_INVALID, "clip_rn_create: missing tensor 'visual.bn1.weight'");
    const int width = int(2 * n_bn1), E = 32 * width;
    if (width % 16 || E % 64)
        return fail(VF_ERR_UNSUPPORTED, "clip_rn_create: width %d is not a multiple of 16", width);
    int layers[4];
    for (int L = 0; L < 4; ++L) {
        int b = 0;
        while (T.numel("visual.layer" + std::to_string(L + 1) + "." + std::to_string(b) + ".conv1.weight") > 0) ++b;
        if (b == 0) return fail(VF_ERR_INVALID, "clip_rn_create: missing tensor 'visual.layer%d.0.conv1.weight'", L + 1);
        layers[L] = b;
    }
    const int64_t n_pos = T.numel("visual.attnpool.positional_embedding");
    if (n_pos <= 0) return fail(VF_ERR_INVALID, "clip_rn_create: missing tensor 'visual.attnpool.positional_embedding'");
    const int side = int(lround(sqrt(double(n_pos / E - 1))));
    if (side < 1 || n_pos != int64_t(side * side + 1) * E)
        return fail(VF_ERR_INVALID, "clip_rn_create: tensor 'visual.attnpool.positional_embedding' has %lld elements, "
                    "not (s^2 + 1) x %d", (long long)n_pos, E);
    const int64_t n_cp = T.numel("visual.attnpool.c_proj.weight");
    if (n_cp <= 0) return fail(VF_ERR_INVALID, "clip_rn_create: missing tensor 'visual.attnpool.c_proj.weight'");
    if (n_cp % E || n_cp / E % 8)
        return fail(VF_ERR_INVALID, "clip_rn_create: tensor 'visual.attnpool.c_proj.weight' has %lld elements, not a "
                    "multiple of 8 x %d", (long long)n_cp, E);
    const int npx = 32 * side;
    if (max_frames <= 0) max_frames = npx <= 224 ? 64 : npx <= 288 ? 32 : 16;
    VF_TRY(check_device(device));
    vf_clip_rn* h = new vf_clip_rn();
    h->who = "clip_rn_create";
    h->device = device; h->max_frames = max_frames; h->npx = npx; h->width = width; h->embed = E;
    h->heads = E / 64; h->out_dim = int(n_cp / E); h->tokens = side * side + 1;
    for (int L = 0; L < 4; ++L) h->layers[L] = layers[L];
    auto body = [&]() -> int {
        auto rows = [](const Vol2& v) { return size_t(v.rows()); };
        const Vol2 sv = stem_vol(h, 1);
        VF_TRY(prep_stem1(h, h->stem[0], T, width / 2));
        VF_TRY(prep_same(h, h->stem[1], T, "visual.conv2", "visual.bn2", kEps, width / 2, width / 2, 3));
        VF_TRY(prep_same(h, h->stem[2], T, "visual.conv3", "visual.bn3", kEps, width, width / 2, 3));
        // per-frame element counts of the working buffers, found while walking the blocks
        size_t e_act = rows(sv) * 2 * width, e_ph = 8;
        int cin = width;
        for (int L = 0; L < 4; ++L) {
            const int planes = width << L, cout = 4 * planes;
            const Vol2 vo = stage_vol(h, 1, L);
            for (int b = 0; b < layers[L]; ++b) {
                RnBlock B;
                B.cin = b == 0 ? cin : cout; B.width = planes; B.cout = cout;
                B.stride = (b == 0 && L > 0) ? 2 : 1;
                B.pool_in = b == 0 && L == 0;
                B.down = B.stride != 1 || B.cin != cout;
                const Vol2 vi = b > 0 ? vo : L == 0 ? sv : stage_vol(h, 1, L - 1);
                const Vol2& vc = B.pool_in ? vo : vi;
                const std::string p = "visual.layer" + std::to_string(L + 1) + "." + std::to_string(b);
                if (B.pool_in) VF_TRY(prep_pooled(h, B.c1, T, p + ".conv1", p + ".bn1", planes, B.cin));
                else           VF_TRY(prep_same(h, B.c1, T, p + ".conv1", p + ".bn1", kEps, planes, B.cin, 1));
                VF_TRY(prep_same(h, B.c2, T, p + ".conv2", p + ".bn2", kEps, planes, planes, 3));
                if (B.stride == 2) VF_TRY(prep_pooled(h, B.c3, T, p + ".conv3", p + ".bn3", cout, planes));
                else               VF_TRY(prep_same(h, B.c3, T, p + ".conv3", p + ".bn3", kEps, cout, planes, 1));
                if (B.down) {
                    if (B.stride == 2 || B.pool_in)
                        VF_TRY(prep_pooled(h, B.dn, T, p + ".downsample.0", p + ".downsample.1", cout, B.cin));
                    else
                        VF_TRY(prep_same(h, B.dn, T, p + ".downsample.0", p + ".downsample.1", kEps, cout, B.cin, 1));
                }
                e_act = std::max({e_act, rows(vc) * 2 * planes, rows(vo) * 2 * cout});
                if (B.stride == 2) e_ph = std::max(e_ph, rows(vo) * 8 * planes);
                if (B.stride == 2 || B.pool_in) e_ph = std::max(e_ph, rows(vo) * 8 * B.cin);
                h->blocks.push_back(B);
            }
            cin = cout;
        }
        if (cin != E) return fail(VF_ERR_INVALID, "clip_rn_create: layer4 has %d channels, the attention pool %d", cin, E);
        // attention pool: q on token 0, k | v concatenated into one projection, c_proj
        const float *qw, *qb, *kw, *kb, *vw, *vb, *cw, *cb, *pos;
        const std::string a = "visual.attnpool.";
        VF_TRY(T.get(a + "q_proj.weight", int64_t(E) * E, &qw)); VF_TRY(T.get(a + "q_proj.bias", E, &qb));
        VF_TRY(T.get(a + "k_proj.weight", int64_t(E) * E, &kw)); VF_TRY(T.get(a + "k_proj.bias", E, &kb));
        VF_TRY(T.get(a + "v_proj.weight", int64_t(E) * E, &vw)); VF_TRY(T.get(a + "v_proj.bias", E, &vb));
        VF_TRY(T.get(a + "c_proj.weight", int64_t(h->out_dim) * E, &cw)); VF_TRY(T.get(a + "c_proj.bias", h->out_dim, &cb));
        VF_TRY(T.get(a + "positional_embedding", int64_t(h->tokens) * E, &pos));
        VF_TRY(prep_linear(h, h->q, qw, qb, E, E));
        std::vector<float> kvw(size_t(2) * E * E), kvb(size_t(2) * E);
        std::copy(kw, kw + size_t(E) * E, kvw.begin());
        std::copy(vw, vw + size_t(E) * E, kvw.begin() + size_t(E) * E);
        std::copy(kb, kb + E, kvb.begin());
        std::copy(vb, vb + E, kvb.begin() + E);
        VF_TRY(prep_linear(h, h->kv, kvw.data(), kvb.data(), 2 * E, E));
        VF_TRY(prep_linear(h, h->cproj, cw, cb, h->out_dim, E));
        VF_TRY(ralloc(h, &h->pos, size_t(h->tokens) * E));
        VF_CUDA(cudaMemcpy(h->pos, pos, size_t(h->tokens) * E * sizeof(float), cudaMemcpyHostToDevice));
        const size_t F = size_t(max_frames), TE = size_t(h->tokens) * 2 * E;
        VF_TRY(ralloc(h, &h->s0, F * rows(sv) * 32));
        VF_TRY(ralloc(h, &h->stem_out, F * rows(sv) * 2 * width));
        for (int L = 0; L < 4; ++L) VF_TRY(ralloc(h, &h->stage_out[L], F * rows(stage_vol(h, 1, L)) * 8 * (width << L)));
        for (__half** b : {&h->bufA, &h->bufB, &h->t1, &h->t2, &h->ds}) VF_TRY(ralloc(h, b, F * e_act));
        VF_TRY(ralloc(h, &h->ph1, F * e_ph));
        VF_TRY(ralloc(h, &h->ph2, F * e_ph));
        VF_TRY(ralloc(h, &h->tok, F * TE));
        VF_TRY(ralloc(h, &h->kvo, F * TE));
        VF_TRY(ralloc(h, &h->qo, F * E));
        VF_TRY(ralloc(h, &h->att, F * 2 * E));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_clip_rn_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_clip_rn_info(const vf_clip_rn_t* h, int* info) {
    if (!h || !info) return fail(VF_ERR_INVALID, "clip_rn_info: null argument");
    const int v[11] = {h->out_dim, h->npx, h->width, h->embed, h->heads, h->tokens, h->max_frames,
                       h->layers[0], h->layers[1], h->layers[2], h->layers[3]};
    memcpy(info, v, sizeof(v));
    return VF_OK;
}

int vf_clip_rn_encode_f32(vf_clip_rn_t* h, const float* frames, int n, float* out, void* stream) {
    return clip_rn_encode(h, frames, 0, n, 0, 0, out, stream);
}

int vf_clip_rn_encode_u8(vf_clip_rn_t* h, const uint8_t* frames, int n, int H, int W, float* out, void* stream) {
    return clip_rn_encode(h, frames, 1, n, H, W, out, stream);
}

int vf_clip_rn_read_stage(vf_clip_rn_t* h, int stage, float* out, int64_t capacity, int* dims4, void* stream) {
    if (!h || !dims4 || h->last_n <= 0)
        return fail(VF_ERR_INVALID, "clip_rn_read_stage: no encode has run (since the last debug call)");
    if (stage < 0 || stage > 6) return fail(VF_ERR_INVALID, "clip_rn_read_stage: unknown stage %d", stage);
    const int n = h->last_n, E = h->embed;
    Vol2 v;
    int C, ld;
    const __half* src;
    if (stage == 0) { v = stem_vol(h, n); C = h->width; src = h->stem_out; ld = 2 * C; }
    else if (stage <= 4) { v = stage_vol(h, n, stage - 1); C = 4 * (h->width << (stage - 1)); src = h->stage_out[stage - 1]; ld = 2 * C; }
    else if (stage == 5) { v = Vol2{n, h->tokens, 1, 0, h->tokens, 0, 1}; C = E; src = h->tok; ld = 2 * E; }
    else { v = Vol2{n, 1, 1, 0, 1, 0, 1}; C = E; src = h->att; ld = 2 * E; }
    dims4[0] = n; dims4[1] = C; dims4[2] = v.H(); dims4[3] = v.W();
    if (!out) return VF_OK;
    if (capacity < int64_t(n) * C * v.H() * v.W()) return fail(VF_ERR_INVALID, "clip_rn_read_stage: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));      // diagnostics only: the engine stream has finished the last call
    return raft_unpack2d(src, v, ld, 0, C, C, out, static_cast<cudaStream_t>(stream));
}

int vf_clip_rn_debug_block(vf_clip_rn_t* h, int block, const void* x_pairs, int n, void* out_pairs, void* branch_out,
                           void* shortcut_out, void* stream) {
    if (!h || !x_pairs || !out_pairs || !branch_out) return fail(VF_ERR_INVALID, "clip_rn_debug_block: null argument");
    if (block < 0 || block >= int(h->blocks.size()) || n <= 0 || n > h->max_frames)
        return fail(VF_ERR_INVALID, "clip_rn_debug_block: block %d of %d, %d frames (max_frames %d)", block,
                    int(h->blocks.size()), n, h->max_frames);
    int L = 0, b = block;
    while (b >= h->layers[L]) b -= h->layers[L++];
    const RnBlock& B = h->blocks[size_t(block)];
    const Vol2 vo = stage_vol(h, n, L), vi = b > 0 ? vo : L == 0 ? stem_vol(h, n) : stage_vol(h, n, L - 1);
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_CUDA(cudaSetDevice(h->device));
    // the trunk's own buffers: bufA holds every block input (the workspace sizes it for the stem volume too), bufB the
    // output; run_block leaves bn3's output in t1 and the downsample's in ds.  The retained stages are not written,
    // but read_stage is refused until the next encode, as for I3D and S3D.
    h->last_n = 0;
    h->attn_n = 0;
    const size_t in_h = size_t(vi.rows()) * 2 * B.cin, out_h = size_t(vo.rows()) * 2 * B.cout;
    VF_TRY(enter(h, user));
    VF_CUDA(cudaMemcpyAsync(h->bufA, x_pairs, in_h * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    VF_TRY(run_block(h, B, h->bufA, vi, vo, h->bufB, s));
    VF_CUDA(cudaMemcpyAsync(out_pairs, h->bufB, out_h * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    VF_CUDA(cudaMemcpyAsync(branch_out, h->t1, out_h * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    if (B.down && shortcut_out)
        VF_CUDA(cudaMemcpyAsync(shortcut_out, h->ds, out_h * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    return leave(h, user);
}

int vf_clip_rn_debug_attnpool(vf_clip_rn_t* h, const void* x_pairs, int n, float* features, void* stream) {
    if (!h || !x_pairs || !features) return fail(VF_ERR_INVALID, "clip_rn_debug_attnpool: null argument");
    if (n <= 0 || n > h->max_frames)
        return fail(VF_ERR_INVALID, "clip_rn_debug_attnpool: %d frames (max_frames %d)", n, h->max_frames);
    const Vol2 v4 = stage_vol(h, n, 3);
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_CUDA(cudaSetDevice(h->device));
    h->last_n = 0;
    VF_TRY(enter(h, user));
    VF_CUDA(cudaMemcpyAsync(h->bufA, x_pairs, size_t(v4.rows()) * 2 * h->embed * sizeof(__half),
                            cudaMemcpyDeviceToDevice, s));
    VF_TRY(run_attention(h, h->bufA, n, s));
    VF_TRY(run_cproj(h, n, features, s));
    VF_TRY(leave(h, user));
    h->attn_n = n;
    return VF_OK;
}

int vf_clip_rn_debug_attnpool_read(vf_clip_rn_t* h, int what, void* out, int64_t capacity, void* stream) {
    if (!h || !out) return fail(VF_ERR_INVALID, "clip_rn_debug_attnpool_read: null argument");
    if (h->attn_n <= 0) return fail(VF_ERR_INVALID, "clip_rn_debug_attnpool_read: no vf_clip_rn_debug_attnpool has run");
    const int64_t n = h->attn_n, T = h->tokens, E = h->embed;
    const void* src;
    int64_t count, size;
    switch (what) {
        case 0: src = h->tok; count = n * T * 2 * E; size = sizeof(__half); break;
        case 1: src = h->kvo; count = n * T * 2 * E; size = sizeof(float); break;
        case 2: src = h->qo; count = n * E; size = sizeof(float); break;
        case 3: src = h->att; count = n * 2 * E; size = sizeof(__half); break;
        default: return fail(VF_ERR_INVALID, "clip_rn_debug_attnpool_read: unknown intermediate %d", what);
    }
    if (capacity < count) return fail(VF_ERR_INVALID, "clip_rn_debug_attnpool_read: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));
    VF_CUDA(cudaMemcpyAsync(out, src, size_t(count * size), cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    return VF_OK;
}

int vf_debug_clip_rn_attention(const float* kv, const float* q, int n, int T, int E, void* out_pairs, void* stream) {
    if (!kv || !q || !out_pairs) return fail(VF_ERR_INVALID, "debug_clip_rn_attention: null argument");
    if (n <= 0 || n > 65535 || E <= 0 || E % 64 || E / 64 > 65535)
        return fail(VF_ERR_INVALID, "debug_clip_rn_attention: %d frames, E %d (a multiple of 64)", n, E);
    return clip_rn_attention(kv, q, n, T, E, static_cast<__half*>(out_pairs), static_cast<cudaStream_t>(stream));
}

int vf_clip_rn_read_pairs(vf_clip_rn_t* h, int stage, void* out, int64_t capacity, void* stream) {
    if (!h || !out || h->last_n <= 0)
        return fail(VF_ERR_INVALID, "clip_rn_read_pairs: no encode has run (since the last debug call)");
    if (stage < 0 || stage > 4) return fail(VF_ERR_INVALID, "clip_rn_read_pairs: unknown stage %d", stage);
    const int n = h->last_n;
    const Vol2 v = stage == 0 ? stem_vol(h, n) : stage_vol(h, n, stage - 1);
    const int C = stage == 0 ? h->width : 4 * (h->width << (stage - 1));
    const int64_t count = int64_t(v.rows()) * 2 * C;
    if (capacity < count) return fail(VF_ERR_INVALID, "clip_rn_read_pairs: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));
    VF_CUDA(cudaMemcpyAsync(out, stage == 0 ? h->stem_out : h->stage_out[stage - 1], size_t(count) * sizeof(__half),
                            cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    return VF_OK;
}

int64_t vf_clip_rn_launch_count(const vf_clip_rn_t* h) { return h ? h->launches : 0; }

int vf_clip_rn_conv(const vf_clip_rn_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "clip_rn_conv: null argument");
    std::vector<const ResConv*> cs{&h->stem[0], &h->stem[1], &h->stem[2]};
    for (const RnBlock& B : h->blocks) {
        for (const ResConv* c : {&B.c1, &B.c2, &B.c3}) cs.push_back(c);
        if (B.down) cs.push_back(&B.dn);
    }
    for (const ResConv* c : {&h->q, &h->kv, &h->cproj}) cs.push_back(c);
    if (index < 0 || index >= int(cs.size()))
        return fail(VF_ERR_INVALID, "clip_rn_conv: index %d outside the %d convs", index, int(cs.size()));
    return read_back_conv(h->device, *cs[index], geom, lo_mask, w, scale, bias);
}

}  // extern "C"
