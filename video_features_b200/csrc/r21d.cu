// torchvision R(2+1)D trunk (`VideoResNet` with `Conv2Plus1D` blocks, fc = Identity) on the wgmma conv-GEMM.
// Replaces `r2plus1d_18(pretrained=True)` with `model.fc = Identity()` in eval mode (reference:
// models/r21d/extract_r21d.py) together with its clip transform ToFloatTensorInZeroOne -> Resize((128, 171)) ->
// Normalize -> CenterCrop(112).  The depth is read from the state dict: blocks per stage, each Conv2Plus1D's mid width
// and the downsamples, so the IG65M R(2+1)D-34 models (layers 3, 4, 6, 3; conv1 and conv2 of a block with different
// mid widths; BatchNorm eps 1e-3) run on the same code.
//
// Layout: every activation is a split-fp16 pair row [hi C | lo C] of a zero-bordered channels-last 3-D volume
// [clip][T+2][Hp][Wp] (r21d_kernels.h Vol3), written by the GEMM epilogue's split output; BatchNorm is folded into the
// epilogue scale / bias, every weight is a hi + lo fp16 pair (nsplit 2) whose W_lo pass is skipped on K blocks that
// only meet lo halves -- the ResNet scheme, chosen by the same kind of emulation (DESIGN.md §4.7,
// scripts/precision/emulate_r21d.py).  Odd widths (45, 230, 460, 921 mid-planes) are padded to a multiple of 8 with
// zero filters, zero scale and zero bias, so the pad channels are exact zeros.
// Convolutions (all shifted-row GEMMs, conv_gemm_f16, on the 3-D geometry; border frames are masked to zero):
//   spatial (1,3,3) stride 1: 3 taps (kernel rows), the 3 columns of a row one run of 3 * 2C elements;
//   spatial (1,3,3) stride (1,2,2): on the 2-D phase repack (raft_phase_repack) with every (clip, t) a frame, 4 taps;
//   temporal (3,1,1) stride 1: 3 taps of 2C elements, Hp * Wp rows apart;
//   temporal (3,1,1) stride (2,1,1): on the temporal phase repack (rows [t even | t odd]), 2 taps of 4C elements;
//   downsample 1x1x1 stride 2: one tap of 2C over the (2,2,2) subsample of the block input;
//   stem (1,7,7)/(1,2,2): 4 taps over the per-frame phase volume the transform kernel writes (rows [16 hi | 16 lo]).
// Geometry at 112 x 112: stem and layer1 on [clip][T+2][59][59] (valid [1,T+1) x [2,58)^2, 56 x 56), layer2..4 on
// [clip][T'+2][S+2][S+2] (valid border 1) with S = 28, 14, 7 and T' = (T-1)/2 + 1 per stride-2 stage.  Residual
// add + ReLU: raft_add_relu.  Everything from the stem conv to layer4 is one CUDA graph per (clips, T).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"
#include "r21d_kernels.h"
#include "split_conv.h"

namespace vf {

int launch_unpack_ndhwc_raw(const __half* in, const void* vi, int C, int c_off, int c_cnt, int ld, int lo_off, float* out,
                            cudaStream_t s);     // i3d_kernels.cu

struct R21Block {
    int cin = 0, mid1 = 0, mid2 = 0, cout = 0, stride = 1;     // conv1's / conv2's mid width, padded to a multiple of 8
    bool down = false;
    ResConv c1s, c1t, c2s, c2t, dn;
};

}  // namespace vf

using namespace vf;

struct vf_r21d : vf::EngineCore {
    int max_clips = 0, max_T = 0, slots = 0;
    double bn_eps = 1e-5;
    ResConv stem_s, stem_t;
    std::vector<R21Block> blocks;
    int nblocks[4] = {0, 0, 0, 0};   // blocks per stage, in the order of `blocks`
    // workspace, in frame slots (max_clips * (max_T + 2)); stage outputs are kept for vf_r21d_read_stage
    __half *s0 = nullptr, *pf = nullptr, *stem_mid = nullptr, *stem_out = nullptr;
    __half *stage_out[4] = {nullptr, nullptr, nullptr, nullptr};
    __half *bufA = nullptr, *bufB = nullptr, *t1 = nullptr, *t2 = nullptr, *t3 = nullptr, *ds = nullptr;
    __half *ph = nullptr, *tph = nullptr, *sub = nullptr;
    int last_m = 0, last_T = 0;
};

namespace vf {

static const int kSide[4] = {56, 28, 14, 7};
static const int kCout[4] = {64, 128, 256, 512};

static int pad8(int c) { return (c + 7) / 8 * 8; }
static int t_next(int T) { return (T - 1) / 2 + 1; }            // (3,1,1) stride 2 pad 1 / 1x1x1 stride 2
static int stage_T(int T, int L) { for (int i = 0; i < L; ++i) T = t_next(T); return T; }

static Vol3 stage_vol(int m, int T, int L) {
    const int TL = stage_T(T, L);
    if (L == 0) return Vol3{m, TL + 2, R21D_Q, R21D_Q, 1, TL + 1, 2, 58, 2, 58};
    const int S = kSide[L];
    return Vol3{m, TL + 2, S + 2, S + 2, 1, TL + 1, 1, S + 1, 1, S + 1};
}
// the volume with vo's spatial geometry and vi's frames (output of a stride-(1,2,2) spatial conv)
static Vol3 mix_vol(const Vol3& vi, const Vol3& vo) {
    return Vol3{vi.n, vi.Tp, vo.Hp, vo.Wp, vi.t0, vi.t1, vo.h0, vo.h1, vo.w0, vo.w1};
}
static Vol2 frames2d(const Vol3& v) { return Vol2{v.n * v.Tp, v.Hp, v.Wp, v.h0, v.h1, v.w0, v.w1}; }

// (3,1,1) stride (2,1,1) pad 1 on the temporal phase repack (rows [even frame 2ci_p | odd frame 2ci_p]): output frame
// t reads frames 2t-1 (odd phase of row q-1), 2t and 2t+1 (both phases of row q)
static int prep_temporal2(vf_r21d* h, ResConv& cw, const ResTensors& T, const std::string& p, const std::string& bn,
                          int co, int ci, int ci_p) {
    cw.ntaps = 2; cw.k_per_tap = 4 * ci_p;
    cw.dt[0] = -1; cw.dt[1] = 0;
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, p, bn, h->bn_eps, {co, ci, 3, 1, 1}, ci_p, [=](int kt, int, int, int c) {
        return kt == 0 ? 2 * ci_p + c : kpt + (kt - 1) * 2 * ci_p + c;
    }, pad8(co));
}

// torchvision video BasicBlock with Conv2Plus1D: x (volume vi, cin channels) -> dst (vo, cout channels)
static int run_block(vf_r21d* h, const R21Block& B, const __half* x, const Vol3& vi, const Vol3& vo, __half* dst,
                     cudaStream_t s) {
    const int mid1 = B.mid1, cout = B.cout;
    if (B.stride == 2) {
        const Vol3 vm = mix_vol(vi, vo);           // the spatial conv keeps the frames
        VF_TRY(raft_phase_repack(x, frames2d(vi), 2 * B.cin, h->ph, frames2d(vm), s));
        VF_TRY(run_conv(h, B.c1s, h->ph, 8 * B.cin, vm, h->t1, true, s));
        VF_TRY(r21d_temporal_phase(h->t1, vm, 2 * mid1, h->tph, vo, s));
        VF_TRY(run_conv(h, B.c1t, h->tph, 4 * mid1, vo, h->t2, true, s));
        h->launches += 2;
    } else {
        VF_TRY(run_conv(h, B.c1s, x, 2 * B.cin, vi, h->t1, true, s));
        VF_TRY(run_conv(h, B.c1t, h->t1, 2 * mid1, vi, h->t2, true, s));
    }
    VF_TRY(run_conv(h, B.c2s, h->t2, 2 * cout, vo, h->t1, true, s));
    VF_TRY(run_conv(h, B.c2t, h->t1, 2 * B.mid2, vo, h->t3, false, s));
    const __half* res = x;
    if (B.down) {
        VF_TRY(r21d_subsample(x, vi, 2 * B.cin, h->sub, vo, s));
        VF_TRY(run_conv(h, B.dn, h->sub, 2 * B.cin, vo, h->ds, false, s));
        res = h->ds;
        h->launches += 1;
    }
    // border frames of both operands are zero, so relu(0 + 0) keeps them zero
    VF_TRY(raft_add_relu(res, h->t3, dst, frames2d(vo), cout, s));
    h->launches += 1;
    return VF_OK;
}

// stem .. layer4 on m clips of T frames whose clip phase volume is in h->s0
static int run_trunk(vf_r21d* h, int m, int T, cudaStream_t s) {
    const Vol3 v0 = stage_vol(m, T, 0);
    VF_TRY(run_conv(h, h->stem_s, h->s0, 32, v0, h->stem_mid, true, s));
    VF_TRY(run_conv(h, h->stem_t, h->stem_mid, 96, v0, h->stem_out, true, s));
    const __half* x = h->stem_out;
    for (int L = 0, bi = 0; L < 4; ++L)
        for (int b = 0; b < h->nblocks[L]; ++b, ++bi) {
            const Vol3 vo = stage_vol(m, T, L), vi = (b == 0 && L > 0) ? stage_vol(m, T, L - 1) : vo;
            // the stage's last block writes the stage output vf_r21d_read_stage returns
            __half* dst = b == h->nblocks[L] - 1 ? h->stage_out[L] : (x == h->bufA ? h->bufB : h->bufA);
            VF_TRY(run_block(h, h->blocks[bi], x, vi, vo, dst, s));
            x = dst;
        }
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_r21d_create(vf_r21d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips, int max_T) {
    return vf_r21d_create2(out, tensors, n_tensors, device, max_clips, max_T, 1e-5);
}

int vf_r21d_create2(vf_r21d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips, int max_T,
                    double bn_eps) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "r21d_create: null argument");
    *out = nullptr;
    if (!(bn_eps > 0.0 && bn_eps < 1.0)) return fail(VF_ERR_INVALID, "r21d_create: BatchNorm eps %g outside (0, 1)", bn_eps);
    if (max_clips <= 0) max_clips = 4;
    if (max_T <= 0) max_T = 16;
    VF_TRY(check_device(device));
    vf_r21d* h = new vf_r21d();
    h->who = "r21d_create";
    h->device = device; h->max_clips = max_clips; h->max_T = max_T; h->bn_eps = bn_eps;
    h->slots = max_clips * (max_T + 2);
    const ResTensors Tn{tensors, n_tensors, "r21d_create"};
    const double eps = bn_eps;
    auto body = [&]() -> int {
        VF_TRY(prep_stem(h, h->stem_s, Tn, "stem.0", "stem.1", eps, 45, 48));
        VF_TRY(prep_temporal(h, h->stem_t, Tn, "stem.3", "stem.4", eps, 64, 45, 48));
        // per-frame-slot element counts of the working buffers, found while walking the blocks
        auto rows = [](const Vol3& v) { return size_t(v.Hp) * v.Wp; };
        size_t e_act = rows(stage_vol(1, 1, 0)) * 2 * 64, e_mid = 0, e_ph = 8, e_tph = 8, e_sub = 8;
        int cin = 64;
        for (int L = 0; L < 4; ++L) {
            const int cout = kCout[L];
            const Vol3 vo = stage_vol(1, 1, L);
            // blocks layerL.0, layerL.1, ... as far as the state dict has them (r2plus1d_18: 2 per stage; R(2+1)D-34:
            // 3, 4, 6, 3)
            int nb = 0;
            while (nb < 64 && Tn.find("layer" + std::to_string(L + 1) + "." + std::to_string(nb) + ".conv1.0.0.weight"))
                ++nb;
            if (nb == 0) return fail(VF_ERR_INVALID, "r21d_create: missing tensor 'layer%d.0.conv1.0.0.weight'", L + 1);
            h->nblocks[L] = nb;
            for (int b = 0; b < nb; ++b) {
                R21Block B;
                B.cin = b == 0 ? cin : cout; B.cout = cout;
                B.stride = (b == 0 && L > 0) ? 2 : 1;
                B.down = B.stride != 1 || B.cin != cout;
                const std::string p = "layer" + std::to_string(L + 1) + "." + std::to_string(b);
                if (!B.down && Tn.find(p + ".downsample.0.weight"))
                    return fail(VF_ERR_INVALID, "r21d_create: '%s.downsample.0.weight' on a stride-1 block of equal "
                                "widths (%d -> %d); torchvision's VideoResNet has none there", p.c_str(), B.cin, cout);
                // each Conv2Plus1D's mid width is its spatial conv's output width: torchvision's BasicBlock gives both
                // (inplanes * planes * 27) // (inplanes * 9 + 3 * planes), IG65M's R(2+1)D-34 widens conv2's in the
                // first block of layer2..4 (288, 576, 1152 instead of 230, 460, 921)
                int mid1 = 0, mid2 = 0;
                VF_TRY(Tn.spatial_width(p + ".conv1.0.0.weight", B.cin, &mid1));
                VF_TRY(Tn.spatial_width(p + ".conv2.0.0.weight", cout, &mid2));
                B.mid1 = pad8(mid1); B.mid2 = pad8(mid2);
                if (B.stride == 2) {
                    VF_TRY(prep_stride2(h, B.c1s, Tn, p + ".conv1.0.0", p + ".conv1.0.1", eps, mid1, B.cin, pad8(mid1)));
                    VF_TRY(prep_temporal2(h, B.c1t, Tn, p + ".conv1.0.3", p + ".conv1.1", cout, mid1, B.mid1));
                    e_ph = std::max(e_ph, rows(vo) * 8 * B.cin);
                    e_tph = std::max(e_tph, rows(vo) * 4 * B.mid1);
                    e_sub = std::max(e_sub, rows(vo) * 2 * B.cin);
                } else {
                    VF_TRY(prep_same(h, B.c1s, Tn, p + ".conv1.0.0", p + ".conv1.0.1", eps, mid1, B.cin, 3, B.cin, pad8(mid1)));
                    VF_TRY(prep_temporal(h, B.c1t, Tn, p + ".conv1.0.3", p + ".conv1.1", eps, cout, mid1, B.mid1, pad8(cout)));
                }
                VF_TRY(prep_same(h, B.c2s, Tn, p + ".conv2.0.0", p + ".conv2.0.1", eps, mid2, cout, 3, cout, pad8(mid2)));
                VF_TRY(prep_temporal(h, B.c2t, Tn, p + ".conv2.0.3", p + ".conv2.1", eps, cout, mid2, B.mid2, pad8(cout)));
                if (B.down) VF_TRY(prep_same(h, B.dn, Tn, p + ".downsample.0", p + ".downsample.1", eps, cout, B.cin, 1));
                // t1 holds both spatial convs' outputs
                e_mid = std::max(e_mid, rows(vo) * 2 * std::max(B.mid1, B.mid2));
                e_act = std::max(e_act, rows(vo) * 2 * cout);
                h->blocks.push_back(B);
            }
            cin = cout;
        }
        const size_t F = size_t(h->slots);
        const size_t e_s0 = size_t(R21D_Q) * R21D_Q * 32;
        VF_TRY(ralloc(h, &h->s0, F * e_s0));
        VF_TRY(ralloc(h, &h->pf, F * e_s0));
        VF_TRY(ralloc(h, &h->stem_mid, F * e_s0 * 3));
        VF_TRY(ralloc(h, &h->stem_out, F * e_s0 * 4));
        for (int L = 0; L < 4; ++L) VF_TRY(ralloc(h, &h->stage_out[L], F * rows(stage_vol(1, 1, L)) * 2 * kCout[L]));
        for (__half** b : {&h->bufA, &h->bufB, &h->t2, &h->t3, &h->ds}) VF_TRY(ralloc(h, b, F * e_act));
        VF_TRY(ralloc(h, &h->t1, F * e_mid));
        VF_TRY(ralloc(h, &h->ph, F * e_ph));
        VF_TRY(ralloc(h, &h->tph, F * e_tph));
        VF_TRY(ralloc(h, &h->sub, F * e_sub));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_r21d_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_r21d_destroy(vf_r21d_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

}  // extern "C"

namespace vf {

// u8: frames n_frames x H x W x 3 and host starts[n]; f32: clips n x 3 x T x 112 x 112
static int r21d_forward(vf_r21d* h, const void* src, int is_u8, int n_frames, int H, int W, const int* starts, int n,
                        int T, float* out, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "r21d_forward: null handle");
    if (n < 0 || T < 1) return fail(VF_ERR_INVALID, "r21d_forward: %d clips of %d frames", n, T);
    if (n > 0 && (!src || !out || (is_u8 && !starts))) return fail(VF_ERR_INVALID, "r21d_forward: null argument");
    const int per_chunk = std::min(R21D_MAX_CHUNK, h->slots / (T + 2));
    if (per_chunk < 1)
        return fail(VF_ERR_INVALID, "r21d_forward: a %d-frame clip exceeds the workspace (%d clips x %d frames)", T,
                    h->max_clips, h->max_T);
    if (is_u8) {
        if (H < 1 || W < 1) return fail(VF_ERR_INVALID, "r21d_forward: frame size %dx%d", H, W);
        for (int i = 0; i < n; ++i)
            if (starts[i] < 0 || int64_t(starts[i]) + T > n_frames)
                return fail(VF_ERR_INVALID, "r21d_forward: clip %d (frames %d..%d) outside the %d frames", i, starts[i],
                            starts[i] + T - 1, n_frames);
    }
    if (n == 0) return VF_OK;
    const int cy = center_crop_offset(128, 112), cx = center_crop_offset(171, 112);
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n;) {      // calls beyond the workspace run in chunks
        int m = 0;
        if (is_u8) {
            int lo = 0, hi = 0;
            R21DStarts st;
            VF_TRY(clip_window("r21d_forward", starts + off, n - off, T, per_chunk, h->slots, &m, &lo, &hi, &st));
            const uint8_t* f0 = static_cast<const uint8_t*>(src) + int64_t(lo) * H * W * 3;
            VF_TRY(r21d_frames_u8(f0, hi - lo, H, W, cy, cx, h->pf, s));
            VF_TRY(r21d_clip_gather(h->pf, st, m, T, h->s0, s));
            h->launches += 2;
        } else {
            m = std::min(per_chunk, n - off);
            VF_TRY(r21d_pack_f32(static_cast<const float*>(src) + int64_t(off) * 3 * T * 112 * 112, m, T, h->s0, s));
            h->launches += 1;
        }
        VF_TRY(run_graphed(h, {m, T, 0, 0}, [&] { return run_trunk(h, m, T, s); }));
        VF_TRY(r21d_avgpool(h->stage_out[3], stage_vol(m, T, 3), 512, out + int64_t(off) * 512, s));
        h->launches += 1;
        h->last_m = m; h->last_T = T;
        off += m;
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_r21d_forward_f32(vf_r21d_t* h, const float* clips, int n, int T, float* out, void* stream) {
    return r21d_forward(h, clips, 0, 0, 112, 112, nullptr, n, T, out, stream);
}

int vf_r21d_forward_u8(vf_r21d_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n, int T,
                       float* out, void* stream) {
    return r21d_forward(h, frames, 1, n_frames, H, W, starts, n, T, out, stream);
}

int vf_r21d_read_stage(vf_r21d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream) {
    if (!h || !dims5 || h->last_m <= 0) return fail(VF_ERR_INVALID, "r21d_read_stage: no forward has run");
    if (stage < 0 || stage > 4) return fail(VF_ERR_INVALID, "r21d_read_stage: unknown stage %d", stage);
    const int L = stage == 0 ? 0 : stage - 1;
    const Vol3 v = stage_vol(h->last_m, h->last_T, L);
    const int C = kCout[L];
    const __half* src = stage == 0 ? h->stem_out : h->stage_out[L];
    dims5[0] = v.n; dims5[1] = C; dims5[2] = v.T(); dims5[3] = v.H(); dims5[4] = v.W();
    if (!out) return VF_OK;
    if (capacity < int64_t(v.n) * C * v.T() * v.H() * v.W())
        return fail(VF_ERR_INVALID, "r21d_read_stage: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));      // diagnostics only: the engine stream has finished the last call
    return launch_unpack_ndhwc_raw(src, &v, C, 0, C, 2 * C, C, out, static_cast<cudaStream_t>(stream));
}

int64_t vf_r21d_launch_count(const vf_r21d_t* h) { return h ? h->launches : 0; }

int vf_r21d_conv(const vf_r21d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "r21d_conv: null argument");
    std::vector<const ResConv*> cs{&h->stem_s, &h->stem_t};
    for (const R21Block& B : h->blocks) {
        for (const ResConv* c : {&B.c1s, &B.c1t, &B.c2s, &B.c2t}) cs.push_back(c);
        if (B.down) cs.push_back(&B.dn);
    }
    if (index < 0 || index >= int(cs.size()))
        return fail(VF_ERR_INVALID, "r21d_conv: index %d outside the %d convs", index, int(cs.size()));
    return read_back_conv(h->device, *cs[index], geom, lo_mask, w, scale, bias);
}

}  // extern "C"
