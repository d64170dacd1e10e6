// torchvision ResNet-18/34/50/101/152 trunk (fc = Identity) on the wgmma conv-GEMM.
// Replaces `models.resnetXX(pretrained=True)` with `model.fc = Identity()` in eval mode (reference:
// models/resnet/extract_resnet.py:52-72, called at :108) together with its per-frame transform (:32-38).
//
// Layout: every activation is a split-fp16 pair row [hi C | lo C] of a zero-bordered channels-last 2-D volume
// (raft_kernels.h Vol2), written by the GEMM epilogue's split output; BatchNorm is folded into the epilogue scale /
// bias, every weight is a hi + lo fp16 pair (nsplit 2) whose W_lo pass is skipped on K blocks that only meet lo halves.
// That is emulated-fp32 arithmetic on the fp16 tensor cores: with single fp16 operands ResNet-50 and deeper miss the
// 1e-3 parity bar (DESIGN.md §4.6, scripts/precision/emulate_resnet.py).
// Convolutions (all shifted-row GEMMs, conv_gemm_f16):
//   stride-1 3x3: 3 taps (kernel rows), the 3 columns of a row one contiguous run of 3 * 2C elements;
//   1x1: one tap of 2C elements;
//   stride-2 3x3 / 1x1: on the space-to-depth ("phase") repack of the input (raft_phase_repack, 4 phases of 2C);
//     the 3x3 is 4 taps of 8C elements (phase rows (a, b) in {q-1, q}^2), the 1x1 reads phase (0, 0);
//   stem 7x7/2 pad 3: 4 taps over the phase volume the transform kernel writes (rows of [16 hi | 16 lo]).
// Geometry at 224x224: stem output [n][115][115] (valid [2,114)^2), then [n][S+2][S+2] (valid [1,S+1)^2) with
// S = 56, 28, 14, 7 for layer1..4.  Residual add + ReLU: raft_add_relu.  Everything from the stem conv to layer4 is
// replayed as one CUDA graph per frame count.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#include "internal.h"
#include "resnet_kernels.h"
#include "split_conv.h"

namespace vf {

struct ResBlock {
    int cin = 0, width = 0, cout = 0, stride = 1;
    bool down = false;
    ResConv c1, c2, c3, dn;
};

}  // namespace vf

using namespace vf;

struct vf_resnet : vf::EngineCore {
    int depth = 0, max_frames = 0, out_dim = 0;
    bool bottleneck = false;
    int nblocks[4] = {0, 0, 0, 0}, cout[4] = {0, 0, 0, 0};
    ResConv stem;
    std::vector<ResBlock> blocks;
    // workspace: s0 = stem phase volume; stage outputs are kept for vf_resnet_read_stage
    __half *s0 = nullptr, *stem_out = nullptr, *pool_out = nullptr, *stage_out[4] = {nullptr, nullptr, nullptr, nullptr};
    __half *bufA = nullptr, *bufB = nullptr, *t1 = nullptr, *t2 = nullptr, *ds = nullptr, *ph1 = nullptr, *ph2 = nullptr;
    int last_n = 0;
};

namespace vf {

static const int kStemQ = 115;                                  // stem phase / output volume side (112 + 3)
static const int kSide[4] = {56, 28, 14, 7};

static Vol2 stem_vol(int n) { return Vol2{n, kStemQ, kStemQ, 2, 114, 2, 114}; }
static Vol2 stage_vol(int n, int L) { return Vol2{n, kSide[L] + 2, kSide[L] + 2, 1, kSide[L] + 1, 1, kSide[L] + 1}; }

static const double kEps = 1e-5;                                // torchvision BatchNorm2d

// torchvision BasicBlock / Bottleneck (v1.5: the stride sits on the 3x3): x (valid region vi, cin channels) ->
// dst (vo, cout channels)
static int run_block(vf_resnet* h, const ResBlock& B, const __half* x, const Vol2& vi, const Vol2& vo, __half* dst,
                     cudaStream_t s) {
    const __half* res = x;
    if (!h->bottleneck) {
        if (B.stride == 2) {
            VF_TRY(raft_phase_repack(x, vi, 2 * B.cin, h->ph2, vo, s));
            VF_TRY(run_conv(h, B.c1, h->ph2, 8 * B.cin, vo, h->t1, true, s));
        } else {
            VF_TRY(run_conv(h, B.c1, x, 2 * B.cin, vo, h->t1, true, s));
        }
        VF_TRY(run_conv(h, B.c2, h->t1, 2 * B.width, vo, h->t2, false, s));
        if (B.down) {
            VF_TRY(run_conv(h, B.dn, B.stride == 2 ? h->ph2 : x, (B.stride == 2 ? 8 : 2) * B.cin, vo, h->ds, false, s));
            res = h->ds;
        }
        VF_TRY(raft_add_relu(res, h->t2, dst, vo, B.cout, s));
        h->launches += 1 + (B.stride == 2);
        return VF_OK;
    }
    VF_TRY(run_conv(h, B.c1, x, 2 * B.cin, vi, h->t1, true, s));
    if (B.stride == 2) {
        VF_TRY(raft_phase_repack(h->t1, vi, 2 * B.width, h->ph1, vo, s));
        VF_TRY(run_conv(h, B.c2, h->ph1, 8 * B.width, vo, h->t2, true, s));
        h->launches += 1;
    } else {
        VF_TRY(run_conv(h, B.c2, h->t1, 2 * B.width, vo, h->t2, true, s));
    }
    VF_TRY(run_conv(h, B.c3, h->t2, 2 * B.width, vo, h->t1, false, s));
    if (B.down) {
        if (B.stride == 2) {
            VF_TRY(raft_phase_repack(x, vi, 2 * B.cin, h->ph2, vo, s));
            VF_TRY(run_conv(h, B.dn, h->ph2, 8 * B.cin, vo, h->ds, false, s));
            h->launches += 1;
        } else {
            VF_TRY(run_conv(h, B.dn, x, 2 * B.cin, vo, h->ds, false, s));
        }
        res = h->ds;
    }
    VF_TRY(raft_add_relu(res, h->t1, dst, vo, B.cout, s));
    h->launches += 1;
    return VF_OK;
}

// stem conv .. layer4 on m frames whose stem phase volume is in h->s0
static int run_trunk(vf_resnet* h, int m, cudaStream_t s) {
    const Vol2 g2 = stem_vol(m);
    VF_TRY(run_conv(h, h->stem, h->s0, 32, g2, h->stem_out, true, s));
    VF_TRY(resnet_maxpool(h->stem_out, g2, 64, h->pool_out, stage_vol(m, 0), s));
    h->launches += 1;
    const __half* x = h->pool_out;
    size_t bi = 0;
    for (int L = 0; L < 4; ++L)
        for (int b = 0; b < h->nblocks[L]; ++b, ++bi) {
            const Vol2 vo = stage_vol(m, L), vi = (b == 0 && L > 0) ? stage_vol(m, L - 1) : vo;
            __half* dst = b == h->nblocks[L] - 1 ? h->stage_out[L] : (x == h->bufA ? h->bufB : h->bufA);
            VF_TRY(run_block(h, h->blocks[bi], x, vi, vo, dst, s));
            x = dst;
        }
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_resnet_create(vf_resnet_t** out, const vf_named_tensor* tensors, int n_tensors, int depth, int device,
                     int max_frames) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "resnet_create: null argument");
    *out = nullptr;
    int layers[4];
    bool bottleneck;
    switch (depth) {     // torchvision resnet.py: _resnet(BasicBlock / Bottleneck, layers)
        case 18: bottleneck = false; layers[0] = 2; layers[1] = 2; layers[2] = 2; layers[3] = 2; break;
        case 34: bottleneck = false; layers[0] = 3; layers[1] = 4; layers[2] = 6; layers[3] = 3; break;
        case 50: bottleneck = true; layers[0] = 3; layers[1] = 4; layers[2] = 6; layers[3] = 3; break;
        case 101: bottleneck = true; layers[0] = 3; layers[1] = 4; layers[2] = 23; layers[3] = 3; break;
        case 152: bottleneck = true; layers[0] = 3; layers[1] = 8; layers[2] = 36; layers[3] = 3; break;
        default: return fail(VF_ERR_INVALID, "resnet_create: depth %d is not one of 18, 34, 50, 101, 152", depth);
    }
    if (max_frames <= 0) max_frames = 64;
    VF_TRY(check_device(device));
    vf_resnet* h = new vf_resnet();
    h->who = "resnet_create";
    h->device = device; h->depth = depth; h->max_frames = max_frames; h->bottleneck = bottleneck;
    const ResTensors T{tensors, n_tensors, "resnet_create"};
    auto body = [&]() -> int {
        VF_TRY(prep_stem(h, h->stem, T, "conv1", "bn1", kEps, 64));
        // per-frame element counts of the working buffers, found while walking the blocks
        size_t e_act = 0, e_ph = 0;
        auto rows = [](const Vol2& v) { return size_t(v.rows()); };
        int cin = 64;
        for (int L = 0; L < 4; ++L) {
            const int width = 64 << L, cout = bottleneck ? 4 * width : width;
            h->nblocks[L] = layers[L]; h->cout[L] = cout;
            const Vol2 vo = stage_vol(1, L);
            for (int b = 0; b < layers[L]; ++b) {
                ResBlock B;
                B.cin = b == 0 ? cin : cout; B.width = width; B.cout = cout;
                B.stride = (b == 0 && L > 0) ? 2 : 1;
                B.down = B.stride != 1 || B.cin != cout;
                const Vol2 vi = B.stride == 2 ? stage_vol(1, L - 1) : vo;
                const std::string p = "layer" + std::to_string(L + 1) + "." + std::to_string(b);
                if (!bottleneck) {
                    if (B.stride == 2) VF_TRY(prep_stride2(h, B.c1, T, p + ".conv1", p + ".bn1", kEps, width, B.cin));
                    else               VF_TRY(prep_same(h, B.c1, T, p + ".conv1", p + ".bn1", kEps, width, B.cin, 3));
                    VF_TRY(prep_same(h, B.c2, T, p + ".conv2", p + ".bn2", kEps, width, width, 3));
                } else {
                    VF_TRY(prep_same(h, B.c1, T, p + ".conv1", p + ".bn1", kEps, width, B.cin, 1));
                    if (B.stride == 2) VF_TRY(prep_stride2(h, B.c2, T, p + ".conv2", p + ".bn2", kEps, width, width));
                    else               VF_TRY(prep_same(h, B.c2, T, p + ".conv2", p + ".bn2", kEps, width, width, 3));
                    VF_TRY(prep_same(h, B.c3, T, p + ".conv3", p + ".bn3", kEps, cout, width, 1));
                    e_act = std::max(e_act, rows(vi) * 2 * width);                  // c1 output at the input geometry
                    if (B.stride == 2) e_ph = std::max(e_ph, rows(vo) * 8 * width);
                }
                if (B.down) VF_TRY(prep_same(h, B.dn, T, p + ".downsample.0", p + ".downsample.1", kEps, cout, B.cin, 1));
                if (B.stride == 2) e_ph = std::max(e_ph, rows(vo) * 8 * B.cin);
                e_act = std::max(e_act, rows(vo) * 2 * std::max(width, cout));
                h->blocks.push_back(B);
            }
            cin = cout;
        }
        h->out_dim = h->cout[3];
        const size_t F = size_t(max_frames);
        VF_TRY(ralloc(h, &h->s0, F * rows(stem_vol(1)) * 32));
        VF_TRY(ralloc(h, &h->stem_out, F * rows(stem_vol(1)) * 128));
        VF_TRY(ralloc(h, &h->pool_out, F * rows(stage_vol(1, 0)) * 128));
        for (int L = 0; L < 4; ++L) VF_TRY(ralloc(h, &h->stage_out[L], F * rows(stage_vol(1, L)) * 2 * h->cout[L]));
        for (__half** b : {&h->bufA, &h->bufB, &h->t1, &h->t2, &h->ds}) VF_TRY(ralloc(h, b, F * e_act));
        VF_TRY(ralloc(h, &h->ph1, F * std::max<size_t>(e_ph, 8)));
        VF_TRY(ralloc(h, &h->ph2, F * std::max<size_t>(e_ph, 8)));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_resnet_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_resnet_destroy(vf_resnet_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

}  // extern "C"

namespace vf {

static int resnet_forward(vf_resnet* h, const void* frames, int is_u8, int n, int Hr, int Wr, float* out, void* stream) {
    if (!h || !frames || !out) return fail(VF_ERR_INVALID, "resnet_forward: null argument");
    if (n < 0) return fail(VF_ERR_INVALID, "resnet_forward: %d frames", n);
    if (is_u8 && (Hr < 224 || Wr < 224))
        return fail(VF_ERR_INVALID, "resnet_forward: resized frame %dx%d is smaller than the 224 crop", Hr, Wr);
    if (n == 0) return VF_OK;
    const int cy = is_u8 ? center_crop_offset(Hr, 224) : 0, cx = is_u8 ? center_crop_offset(Wr, 224) : 0;
    const size_t frame_elems = is_u8 ? size_t(Hr) * Wr * 3 : size_t(3) * 224 * 224;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n; off += h->max_frames) {      // calls beyond the workspace run in chunks
        const int m = std::min(h->max_frames, n - off);
        const void* src = is_u8 ? static_cast<const void*>(static_cast<const uint8_t*>(frames) + off * frame_elems)
                                : static_cast<const void*>(static_cast<const float*>(frames) + off * frame_elems);
        VF_TRY(resnet_input_pack(src, is_u8, m, Hr, Wr, cy, cx, h->s0, s));
        VF_TRY(run_graphed(h, {m, 0, 0, 0}, [&] { return run_trunk(h, m, s); }));
        VF_TRY(resnet_avgpool(h->stage_out[3], stage_vol(m, 3), h->out_dim, out + size_t(off) * h->out_dim, s));
        h->launches += 2;
        h->last_n = m;
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_resnet_forward_f32(vf_resnet_t* h, const float* frames, int n, float* out, void* stream) {
    return resnet_forward(h, frames, 0, n, 224, 224, out, stream);
}

int vf_resnet_forward_u8(vf_resnet_t* h, const uint8_t* frames, int n, int Hr, int Wr, float* out, void* stream) {
    return resnet_forward(h, frames, 1, n, Hr, Wr, out, stream);
}

int vf_resnet_read_stage(vf_resnet_t* h, int stage, float* out, int64_t capacity, int* dims4, void* stream) {
    if (!h || !dims4 || h->last_n <= 0) return fail(VF_ERR_INVALID, "resnet_read_stage: no forward has run");
    if (stage < 0 || stage > 5) return fail(VF_ERR_INVALID, "resnet_read_stage: unknown stage %d", stage);
    const int n = h->last_n;
    const Vol2 v = stage == 0 ? stem_vol(n) : stage_vol(n, stage < 2 ? 0 : stage - 2);
    const int C = stage < 2 ? 64 : h->cout[stage - 2];
    const __half* src = stage == 0 ? h->stem_out : stage == 1 ? h->pool_out : h->stage_out[stage - 2];
    dims4[0] = n; dims4[1] = C; dims4[2] = v.H(); dims4[3] = v.W();
    if (!out) return VF_OK;
    if (capacity < int64_t(n) * C * v.H() * v.W()) return fail(VF_ERR_INVALID, "resnet_read_stage: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));      // diagnostics only: the engine stream has finished the last call
    return raft_unpack2d(src, v, 2 * C, 0, C, C, out, static_cast<cudaStream_t>(stream));
}

int64_t vf_resnet_launch_count(const vf_resnet_t* h) { return h ? h->launches : 0; }

int vf_resnet_conv(const vf_resnet_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "resnet_conv: null argument");
    std::vector<const ResConv*> cs{&h->stem};
    for (const ResBlock& B : h->blocks) {
        cs.push_back(&B.c1);
        cs.push_back(&B.c2);
        if (h->bottleneck) cs.push_back(&B.c3);
        if (B.down) cs.push_back(&B.dn);
    }
    if (index < 0 || index >= int(cs.size()))
        return fail(VF_ERR_INVALID, "resnet_conv: index %d outside the %d convs", index, int(cs.size()));
    return read_back_conv(h->device, *cs[index], geom, lo_mask, w, scale, bias);
}

}  // extern "C"
