// torchvision S3D trunk (`torchvision.models.video.s3d`, eval) on the wgmma conv-GEMM: `model.features` followed by
// `model.avgpool` and the mean over (T, H, W), the 1024-d clip feature; the classifier is class_head.cu's.  The fused
// input transform is the S3D_Weights.KINETICS400_V1 preset (r21d_kernels.cu frames_u8_kernel at S3D's geometry).
//
// Layout: every activation is a split-fp16 pair row [hi C | lo C] of a zero-bordered channels-last 3-D volume
// (r21d_kernels.h Vol3), written by the GEMM epilogue's split output; BatchNorm (eps 1e-3) is folded into the epilogue
// scale / bias, every weight is a hi + lo fp16 pair (nsplit 2) whose W_lo pass is skipped on K blocks that only meet lo
// halves -- the R(2+1)D / ResNet scheme.  scripts/precision/emulate_s3d.py shows why: leaving any one tensor class
// (stem input, stem temporal input, features.2 input, spatial / temporal conv inputs, Mixed inputs, branch-3 pool
// outputs, weights) in single fp16 misses the 1e-3 feature bar by 3..25x (DESIGN.md §4.12).  Every channel count of
// S3D is a multiple of 8, so nothing is padded.
// Convolutions (all shifted-row GEMMs, conv_gemm_f16; border positions are masked to zero):
//   stem (1,7,7)/(1,2,2) pad (0,3,3): 4 taps over the per-frame phase volume the transform writes (rows [16 hi | 16 lo]),
//     as R(2+1)D's stem;
//   stem (7,1,1)/(2,1,1) pad (3,0,0): on R(2+1)D's temporal phase repack (rows [t even | t odd]) with a 2-frame
//     border, 4 taps of 4C elements one phase row apart; filter index kt = 2a + p - 1, the half-tap kt = -1 is zero;
//   (1,3,3) stride 1: 3 taps (kernel rows), the 3 columns of a row one run of 3 * 2C elements;
//   (3,1,1) stride 1: 3 taps of 2C elements, Hp * Wp rows apart;
//   1x1x1: one tap of 2C.
// Pools (i3d_kernels.cu launch_maxpool3d_raw, pair in and out; skipping padded positions equals -inf padding because
// every input is post-ReLU, and the output volume's extent is the floor-mode size):
//   (1,3,3)/(1,2,2) pad (0,1,1) and (3,3,3)/2 pad 1: the general bounds-checked kernel;
//   (2,2,2)/2 pad 0: the fixed-window fast kernel (every floor-mode window lies inside the valid region);
//   the Mixed blocks' (3,3,3)/1 pad 1: the rolling-max kernel (the zero border is the padding).
// Mixed blocks store each branch into its channel slice of the concat rows (I3D's scheme, ldo = 2 * concat width).
// Head: I3D's (2,7,7) average pool + temporal mean (launch_i3d_head_raw), fp32 out, fixed summation order.
// Geometry at 224 x 224, T input frames, T1 = (T-1)/2 + 1, T2 = (T1-1)/2 + 1, T3 = T2/2 (>= 2):
//   stem spatial on [clip][T+2][115][115] (valid [1,T+1) x [2,114)^2), stem temporal on [clip][T1+3][115][115]
//   (valid frames [2,T1+2)); then [clip][Tx+2][S+2][S+2] with border 1: S = 56 (T1), 28 (T1), 14 (T2), 7 (T3).
// Everything from the stem conv to Mixed 5c is one CUDA graph per (clips, T).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"
#include "s3d_kernels.h"
#include "split_conv.h"

namespace vf {

int launch_unpack_ndhwc_raw(const __half* in, const void* vi, int C, int c_off, int c_cnt, int ld, int lo_off, float* out,
                            cudaStream_t s);     // i3d_kernels.cu
int launch_maxpool3d_raw(const __half* in, const void* vi, __half* out, const void* vo, int C, int kt, int kh, int kw,
                         int st, int sh, int sw, int pt, int ph, int pw, cudaStream_t s);
int launch_i3d_head_raw(const __half* in, const void* vi, int C, float* out, cudaStream_t s);

// SepInceptionBlock3D: branch0 1x1x1; branch1 / branch2 1x1x1 -> (1,3,3) -> (3,1,1); branch3 pool -> 1x1x1
struct S3Mixed {
    int cin = 0, c[6] = {0, 0, 0, 0, 0, 0};     // b0, b1 mid, b1, b2 mid, b2, b3
    ResConv b0, b1a, b1s, b1t, b2a, b2s, b2t, b3;
    int ctot() const { return c[0] + c[2] + c[4] + c[5]; }
};

// element counts of the workspace buffers for m clips of T frames
struct S3Sizes { size_t s0, mid, tph, stem, v1, v1w, mixA, mixT, mixP, m3c, m4f, m5c; };

}  // namespace vf

using namespace vf;

struct vf_s3d : vf::EngineCore {
    int max_clips = 0, max_T = 0, slots = 0;
    ResConv stem_s, stem_t, f2, f3s, f3t;
    std::vector<S3Mixed> mixed;
    S3Sizes cap{};
    // workspace; stem_out, c3, m3c, m4f and m5c are kept for vf_s3d_read_stage
    __half *s0 = nullptr, *pf = nullptr, *stem_mid = nullptr, *tph = nullptr, *stem_out = nullptr;
    __half *p1 = nullptr, *c2 = nullptr, *c3a = nullptr, *c3 = nullptr;
    __half *bufA = nullptr, *bufB = nullptr, *ta = nullptr, *tb = nullptr, *tp = nullptr;
    __half *m3c = nullptr, *m4f = nullptr, *m5c = nullptr;
    int last_m = 0, last_T = 0;
};

namespace vf {

static const int kMixedCfg[9][7] = {
    // cin, b0, b1 mid, b1, b2 mid, b2, b3   (torchvision S3D.features 5, 6, 8..12, 14, 15)
    {192, 64, 96, 128, 16, 32, 32},   {256, 128, 128, 192, 32, 96, 64},  {480, 192, 96, 208, 16, 48, 64},
    {512, 160, 112, 224, 24, 64, 64}, {512, 128, 128, 256, 24, 64, 64},  {512, 112, 144, 288, 32, 64, 64},
    {528, 256, 160, 320, 32, 128, 128}, {832, 256, 160, 320, 32, 128, 128}, {832, 384, 192, 384, 48, 128, 128}};
static const int kMixedIdx[9] = {5, 6, 8, 9, 10, 11, 12, 14, 15};

static const double kEps = 1e-3;      // torchvision S3D's BatchNorm3d

static int t_half(int T) { return (T - 1) / 2 + 1; }     // (7,1,1)/2 pad 3 and (3,3,3)/2 pad 1, floor mode

struct S3Geom { Vol3 v0, vt, v1, v2, v3, v4; };
static S3Geom geom(int m, int T) {
    const int T1 = t_half(T), T2 = t_half(T1), T3 = T2 / 2;
    auto bordered = [m](int Tx, int S) { return Vol3{m, Tx + 2, S + 2, S + 2, 1, Tx + 1, 1, S + 1, 1, S + 1}; };
    S3Geom g;
    g.v0 = Vol3{m, T + 2, S3D_Q, S3D_Q, 1, T + 1, 2, 114, 2, 114};
    g.vt = Vol3{m, T1 + 3, S3D_Q, S3D_Q, 2, T1 + 2, 2, 114, 2, 114};
    g.v1 = bordered(T1, 56);
    g.v2 = bordered(T1, 28);
    g.v3 = bordered(T2, 14);
    g.v4 = bordered(T3, 7);
    return g;
}

static S3Sizes sizes(int m, int T) {
    const S3Geom g = geom(m, T);
    S3Sizes z{};
    z.s0 = size_t(g.v0.rows()) * 32;
    z.mid = size_t(g.v0.rows()) * 128;
    z.tph = size_t(g.vt.rows()) * 256;
    z.stem = size_t(g.vt.rows()) * 128;
    z.v1 = size_t(g.v1.rows()) * 128;                   // pool1 / features.2 outputs (64 channels)
    z.v1w = size_t(g.v1.rows()) * 384;                  // features.3 outputs (192 channels)
    const Vol3 mv[9] = {g.v2, g.v2, g.v3, g.v3, g.v3, g.v3, g.v3, g.v4, g.v4};
    z.mixA = std::max(size_t(g.v2.rows()) * 2 * 480, size_t(g.v4.rows()) * 2 * 832);   // pool outputs
    for (int i = 0; i < 9; ++i) {
        const int* c = kMixedCfg[i];
        const size_t r = size_t(mv[i].rows());
        z.mixA = std::max(z.mixA, r * 2 * (c[1] + c[3] + c[5] + c[6]));
        z.mixT = std::max(z.mixT, r * 2 * std::max({c[2], c[3], c[4], c[5]}));
        z.mixP = std::max(z.mixP, r * 2 * c[0]);
    }
    z.m3c = size_t(g.v2.rows()) * 2 * 480;
    z.m4f = size_t(g.v3.rows()) * 2 * 832;
    z.m5c = size_t(g.v4.rows()) * 2 * 1024;
    return z;
}
static bool fits(const S3Sizes& a, const S3Sizes& cap) {
    return a.s0 <= cap.s0 && a.mid <= cap.mid && a.tph <= cap.tph && a.stem <= cap.stem && a.v1 <= cap.v1 &&
           a.v1w <= cap.v1w && a.mixA <= cap.mixA && a.mixT <= cap.mixT && a.mixP <= cap.mixP && a.m3c <= cap.m3c &&
           a.m4f <= cap.m4f && a.m5c <= cap.m5c;
}

// torchvision Conv3dNormActivation `p`: conv p.0, BatchNorm p.1
static int prep_point(vf_s3d* h, ResConv& cw, const ResTensors& T, const std::string& p, int co, int ci) {
    return prep_same(h, cw, T, p + ".0", p + ".1", kEps, co, ci, 1);
}
static int prep_spatial(vf_s3d* h, ResConv& cw, const ResTensors& T, const std::string& p, int co, int ci) {
    return prep_same(h, cw, T, p + ".0", p + ".1", kEps, co, ci, 3);
}
static int prep_time(vf_s3d* h, ResConv& cw, const ResTensors& T, const std::string& p, int co, int ci) {
    return prep_temporal(h, cw, T, p + ".0", p + ".1", kEps, co, ci);
}

// stem (7,1,1) stride (2,1,1) pad (3,0,0) on the temporal phase repack (rows [even frame 128 | odd frame 128], a
// 2-frame border): output frame t reads frames 2t-3 .. 2t+3; tap a (row shift a - 2) holds frames 2t-4+2a+p, so
// kt = 2a + p - 1 and the half-tap (a, p) = (0, 0) is zero
static int prep_stem_t(vf_s3d* h, ResConv& cw, const ResTensors& T) {
    cw.ntaps = 4; cw.k_per_tap = 256;
    for (int a = 0; a < 4; ++a) cw.dt[a] = a - 2;
    return upload_conv(h, cw, T, "features.0.1.0", "features.0.1.1", kEps, {64, 64, 7, 1, 1}, 64,
                       [](int kt, int, int, int c) {
        const int a = (kt + 1) / 2, p = (kt + 1) % 2;
        return a * 256 + p * 128 + c;
    });
}

// SepInceptionBlock3D: x (volume v, cin channels) -> out (v, ctot channels, each branch in its slice)
static int run_mixed(vf_s3d* h, const S3Mixed& B, const __half* x, const Vol3& v, __half* out, cudaStream_t s) {
    const int* c = B.c;
    const int ld = 2 * B.ctot(), xp = 2 * B.cin;
    VF_TRY(run_conv(h, B.b0, x, xp, v, out, true, s, ld));
    VF_TRY(run_conv(h, B.b1a, x, xp, v, h->ta, true, s, 2 * c[1]));
    VF_TRY(run_conv(h, B.b1s, h->ta, 2 * c[1], v, h->tb, true, s, 2 * c[2]));
    VF_TRY(run_conv(h, B.b1t, h->tb, 2 * c[2], v, out + c[0], true, s, ld));
    VF_TRY(run_conv(h, B.b2a, x, xp, v, h->ta, true, s, 2 * c[3]));
    VF_TRY(run_conv(h, B.b2s, h->ta, 2 * c[3], v, h->tb, true, s, 2 * c[4]));
    VF_TRY(run_conv(h, B.b2t, h->tb, 2 * c[4], v, out + c[0] + c[2], true, s, ld));
    VF_TRY(launch_maxpool3d_raw(x, &v, h->tp, &v, B.cin, 3, 3, 3, 1, 1, 1, 1, 1, 1, s));
    h->launches += 1;
    VF_TRY(run_conv(h, B.b3, h->tp, xp, v, out + c[0] + c[2] + c[4], true, s, ld));
    return VF_OK;
}

// stem .. Mixed 5c on m clips of T frames whose clip phase volume is in h->s0
static int run_trunk(vf_s3d* h, int m, int T, cudaStream_t s) {
    const S3Geom g = geom(m, T);
    VF_TRY(run_conv(h, h->stem_s, h->s0, 32, g.v0, h->stem_mid, true, s, 128));
    VF_TRY(r21d_temporal_phase(h->stem_mid, g.v0, 128, h->tph, g.vt, s));
    VF_TRY(run_conv(h, h->stem_t, h->tph, 256, g.vt, h->stem_out, true, s, 128));
    VF_TRY(launch_maxpool3d_raw(h->stem_out, &g.vt, h->p1, &g.v1, 64, 1, 3, 3, 1, 2, 2, 0, 1, 1, s));
    VF_TRY(run_conv(h, h->f2, h->p1, 128, g.v1, h->c2, true, s, 128));
    VF_TRY(run_conv(h, h->f3s, h->c2, 128, g.v1, h->c3a, true, s, 384));
    VF_TRY(run_conv(h, h->f3t, h->c3a, 384, g.v1, h->c3, true, s, 384));
    VF_TRY(launch_maxpool3d_raw(h->c3, &g.v1, h->bufA, &g.v2, 192, 1, 3, 3, 1, 2, 2, 0, 1, 1, s));
    VF_TRY(run_mixed(h, h->mixed[0], h->bufA, g.v2, h->bufB, s));        // 3b -> 256
    VF_TRY(run_mixed(h, h->mixed[1], h->bufB, g.v2, h->m3c, s));         // 3c -> 480
    VF_TRY(launch_maxpool3d_raw(h->m3c, &g.v2, h->bufA, &g.v3, 480, 3, 3, 3, 2, 2, 2, 1, 1, 1, s));
    VF_TRY(run_mixed(h, h->mixed[2], h->bufA, g.v3, h->bufB, s));        // 4b -> 512
    VF_TRY(run_mixed(h, h->mixed[3], h->bufB, g.v3, h->bufA, s));        // 4c
    VF_TRY(run_mixed(h, h->mixed[4], h->bufA, g.v3, h->bufB, s));        // 4d
    VF_TRY(run_mixed(h, h->mixed[5], h->bufB, g.v3, h->bufA, s));        // 4e -> 528
    VF_TRY(run_mixed(h, h->mixed[6], h->bufA, g.v3, h->m4f, s));         // 4f -> 832
    VF_TRY(launch_maxpool3d_raw(h->m4f, &g.v3, h->bufA, &g.v4, 832, 2, 2, 2, 2, 2, 2, 0, 0, 0, s));
    VF_TRY(run_mixed(h, h->mixed[7], h->bufA, g.v4, h->bufB, s));        // 5b -> 832
    VF_TRY(run_mixed(h, h->mixed[8], h->bufB, g.v4, h->m5c, s));         // 5c -> 1024
    h->launches += 5;
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_s3d_create(vf_s3d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips, int max_T) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "s3d_create: null argument");
    *out = nullptr;
    if (max_clips <= 0) max_clips = 2;
    if (max_T <= 0) max_T = 64;
    if (max_T < 13) return fail(VF_ERR_INVALID, "s3d_create: max_T %d < 13, the smallest clip S3D accepts", max_T);
    VF_TRY(check_device(device));
    vf_s3d* h = new vf_s3d();
    h->who = "s3d_create";
    h->device = device; h->max_clips = max_clips; h->max_T = max_T;
    h->slots = max_clips * (max_T + 2);
    const ResTensors Tn{tensors, n_tensors, "s3d_create"};
    auto body = [&]() -> int {
        VF_TRY(prep_stem(h, h->stem_s, Tn, "features.0.0.0", "features.0.0.1", kEps, 64));
        VF_TRY(prep_stem_t(h, h->stem_t, Tn));
        VF_TRY(prep_point(h, h->f2, Tn, "features.2", 64, 64));
        VF_TRY(prep_spatial(h, h->f3s, Tn, "features.3.0", 192, 64));
        VF_TRY(prep_time(h, h->f3t, Tn, "features.3.1", 192, 192));
        for (int i = 0; i < 9; ++i) {
            S3Mixed B;
            const int* c = kMixedCfg[i];
            B.cin = c[0];
            for (int j = 0; j < 6; ++j) B.c[j] = c[j + 1];
            const std::string p = "features." + std::to_string(kMixedIdx[i]);
            VF_TRY(prep_point(h, B.b0, Tn, p + ".branch0", B.c[0], B.cin));
            VF_TRY(prep_point(h, B.b1a, Tn, p + ".branch1.0", B.c[1], B.cin));
            VF_TRY(prep_spatial(h, B.b1s, Tn, p + ".branch1.1.0", B.c[2], B.c[1]));
            VF_TRY(prep_time(h, B.b1t, Tn, p + ".branch1.1.1", B.c[2], B.c[2]));
            VF_TRY(prep_point(h, B.b2a, Tn, p + ".branch2.0", B.c[3], B.cin));
            VF_TRY(prep_spatial(h, B.b2s, Tn, p + ".branch2.1.0", B.c[4], B.c[3]));
            VF_TRY(prep_time(h, B.b2t, Tn, p + ".branch2.1.1", B.c[4], B.c[4]));
            VF_TRY(prep_point(h, B.b3, Tn, p + ".branch3.1", B.c[5], B.cin));
            h->mixed.push_back(B);
        }
        h->cap = sizes(max_clips, max_T);
        const S3Sizes& z = h->cap;
        VF_TRY(ralloc(h, &h->s0, z.s0));
        VF_TRY(ralloc(h, &h->pf, size_t(h->slots) * S3D_Q * S3D_Q * 32));
        VF_TRY(ralloc(h, &h->stem_mid, z.mid));
        VF_TRY(ralloc(h, &h->tph, z.tph));
        VF_TRY(ralloc(h, &h->stem_out, z.stem));
        VF_TRY(ralloc(h, &h->p1, z.v1));
        VF_TRY(ralloc(h, &h->c2, z.v1));
        VF_TRY(ralloc(h, &h->c3a, z.v1w));
        VF_TRY(ralloc(h, &h->c3, z.v1w));
        VF_TRY(ralloc(h, &h->bufA, z.mixA));
        VF_TRY(ralloc(h, &h->bufB, z.mixA));
        VF_TRY(ralloc(h, &h->ta, z.mixT));
        VF_TRY(ralloc(h, &h->tb, z.mixT));
        VF_TRY(ralloc(h, &h->tp, z.mixP));
        VF_TRY(ralloc(h, &h->m3c, z.m3c));
        VF_TRY(ralloc(h, &h->m4f, z.m4f));
        VF_TRY(ralloc(h, &h->m5c, z.m5c));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_s3d_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_s3d_destroy(vf_s3d_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

}  // extern "C"

namespace vf {

// u8: frames n_frames x H x W x 3 and host starts[n]; f32: clips n x 3 x T x 224 x 224
static int s3d_forward(vf_s3d* h, const void* src, int is_u8, int n_frames, int H, int W, const int* starts, int n,
                       int T, float* out, void* stream) {
    if (!h) return fail(VF_ERR_INVALID, "s3d_forward: null handle");
    if (n < 0) return fail(VF_ERR_INVALID, "s3d_forward: %d clips", n);
    if (T < 13) return fail(VF_ERR_INVALID, "s3d_forward: T=%d < 13 leaves no position for the (2,7,7) average pool", T);
    if (n > 0 && (!src || !out || (is_u8 && !starts))) return fail(VF_ERR_INVALID, "s3d_forward: null argument");
    int per_chunk = 0;
    while (per_chunk < R21D_MAX_CHUNK && fits(sizes(per_chunk + 1, T), h->cap))
        ++per_chunk;
    if (per_chunk < 1)
        return fail(VF_ERR_INVALID, "s3d_forward: a %d-frame clip exceeds the workspace (%d clips x %d frames)", T,
                    h->max_clips, h->max_T);
    if (is_u8) {
        if (H < 1 || W < 1) return fail(VF_ERR_INVALID, "s3d_forward: frame size %dx%d", H, W);
        for (int i = 0; i < n; ++i)
            if (starts[i] < 0 || int64_t(starts[i]) + T > n_frames)
                return fail(VF_ERR_INVALID, "s3d_forward: clip %d (frames %d..%d) outside the %d frames", i, starts[i],
                            starts[i] + T - 1, n_frames);
    }
    if (n == 0) return VF_OK;
    const int crop = center_crop_offset(S3D_RESIZE, S3D_CROP);
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int off = 0; off < n;) {      // calls beyond the workspace run in chunks
        int m = 0;
        if (is_u8) {
            int lo = 0, hi = 0;
            R21DStarts st;
            VF_TRY(clip_window("s3d_forward", starts + off, n - off, T, per_chunk, h->slots, &m, &lo, &hi, &st));
            const uint8_t* f0 = static_cast<const uint8_t*>(src) + int64_t(lo) * H * W * 3;
            VF_TRY(s3d_frames_u8(f0, hi - lo, H, W, crop, crop, h->pf, s));
            VF_TRY(s3d_clip_gather(h->pf, st, m, T, h->s0, s));
            h->launches += 2;
        } else {
            m = std::min(per_chunk, n - off);
            VF_TRY(s3d_pack_f32(static_cast<const float*>(src) + int64_t(off) * 3 * T * S3D_CROP * S3D_CROP, m, T,
                                h->s0, s));
            h->launches += 1;
        }
        VF_TRY(run_graphed(h, {m, T, 0, 0}, [&] { return run_trunk(h, m, T, s); }));
        const Vol3 v4 = geom(m, T).v4;
        VF_TRY(launch_i3d_head_raw(h->m5c, &v4, 1024, out + int64_t(off) * 1024, s));
        h->launches += 1;
        h->last_m = m; h->last_T = T;
        off += m;
    }
    return leave(h, user);
}

}  // namespace vf

extern "C" {

int vf_s3d_forward_f32(vf_s3d_t* h, const float* clips, int n, int T, float* out, void* stream) {
    return s3d_forward(h, clips, 0, 0, S3D_CROP, S3D_CROP, nullptr, n, T, out, stream);
}

int vf_s3d_forward_u8(vf_s3d_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n, int T,
                      float* out, void* stream) {
    return s3d_forward(h, frames, 1, n_frames, H, W, starts, n, T, out, stream);
}

int vf_s3d_read_stage(vf_s3d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream) {
    if (!h || !dims5 || h->last_m <= 0)
        return fail(VF_ERR_INVALID, "s3d_read_stage: no forward has run (since the last vf_s3d_debug_mixed)");
    if (stage < 0 || stage > 4) return fail(VF_ERR_INVALID, "s3d_read_stage: unknown stage %d", stage);
    const S3Geom g = geom(h->last_m, h->last_T);
    const Vol3 vols[5] = {g.vt, g.v1, g.v2, g.v3, g.v4};
    const int Cs[5] = {64, 192, 480, 832, 1024};
    const __half* srcs[5] = {h->stem_out, h->c3, h->m3c, h->m4f, h->m5c};
    const Vol3& v = vols[stage];
    const int C = Cs[stage];
    dims5[0] = v.n; dims5[1] = C; dims5[2] = v.T(); dims5[3] = v.H(); dims5[4] = v.W();
    if (!out) return VF_OK;
    if (capacity < int64_t(v.n) * C * v.T() * v.H() * v.W())
        return fail(VF_ERR_INVALID, "s3d_read_stage: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaStreamSynchronize(h->cs));      // diagnostics only: the engine stream has finished the last call
    return launch_unpack_ndhwc_raw(srcs[stage], &v, C, 0, C, 2 * C, C, out, static_cast<cudaStream_t>(stream));
}

int vf_s3d_debug_mixed(vf_s3d_t* h, int block, const void* x_pairs, int n, int T, void* out_pairs, void* stream) {
    if (!h || !x_pairs || !out_pairs) return fail(VF_ERR_INVALID, "s3d_debug_mixed: null argument");
    if (block < 0 || block > 8 || n < 1 || T < 1)
        return fail(VF_ERR_INVALID, "s3d_debug_mixed: block %d, %d clips of %d frames", block, n, T);
    const int S = block < 2 ? 28 : block < 7 ? 14 : 7;
    const Vol3 v{n, T + 2, S + 2, S + 2, 1, T + 1, 1, S + 1, 1, S + 1};
    const S3Mixed& B = h->mixed[block];
    const size_t r = size_t(v.rows());
    const int* c = B.c;
    // the buffers run_trunk gives a Mixed block: input bufA, output bufB, ta / tb the branch intermediates, tp the pool
    if (r * 2 * B.cin > h->cap.mixA || r * 2 * B.ctot() > h->cap.mixA ||
        r * 2 * std::max({c[1], c[2], c[3], c[4]}) > h->cap.mixT || r * 2 * B.cin > h->cap.mixP)
        return fail(VF_ERR_INVALID, "s3d_debug_mixed: %d clips of %d frames exceed the workspace", n, T);
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_CUDA(cudaSetDevice(h->device));
    // the retained stages (stem_out, c3, m3c, m4f, m5c) are not written here, but the block replaces bufA / bufB and
    // the branch intermediates, so read_stage is refused until a forward has run again, as for I3D
    h->last_m = 0;
    VF_TRY(enter(h, user));
    VF_CUDA(cudaMemcpyAsync(h->bufA, x_pairs, r * 2 * B.cin * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    VF_TRY(run_mixed(h, B, h->bufA, v, h->bufB, s));
    VF_CUDA(cudaMemcpyAsync(out_pairs, h->bufB, r * 2 * B.ctot() * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    return leave(h, user);
}

int64_t vf_s3d_launch_count(const vf_s3d_t* h) { return h ? h->launches : 0; }

int vf_s3d_conv(const vf_s3d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "s3d_conv: null argument");
    std::vector<const ResConv*> cs{&h->stem_s, &h->stem_t, &h->f2, &h->f3s, &h->f3t};
    for (const S3Mixed& B : h->mixed)
        for (const ResConv* c : {&B.b0, &B.b1a, &B.b1s, &B.b1t, &B.b2a, &B.b2s, &B.b2t, &B.b3}) cs.push_back(c);
    if (index < 0 || index >= int(cs.size()))
        return fail(VF_ERR_INVALID, "s3d_conv: index %d outside the %d convs", index, int(cs.size()));
    return read_back_conv(h->device, *cs[index], geom, lo_mask, w, scale, bias);
}

}  // extern "C"
