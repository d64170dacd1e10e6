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
#include <functional>
#include <map>
#include <string>
#include <utility>
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

struct S3Conv {
    int n_out = 0, ntaps = 0, k_per_tap = 0;
    int tap_kind = 0;            // tap offsets: 0 spatial (rows / columns), 1 temporal (frames)
    int dt[4] = {0, 0, 0, 0}, dh[4] = {0, 0, 0, 0}, dw[4] = {0, 0, 0, 0};
    unsigned long long lo_mask = 0;
    __half* w = nullptr;         // [n_out][2 * ntaps * k_per_tap]: hi pass | lo pass
    float *scale = nullptr, *bias = nullptr;
};

// SepInceptionBlock3D: branch0 1x1x1; branch1 / branch2 1x1x1 -> (1,3,3) -> (3,1,1); branch3 pool -> 1x1x1
struct S3Mixed {
    int cin = 0, c[6] = {0, 0, 0, 0, 0, 0};     // b0, b1 mid, b1, b2 mid, b2, b3
    S3Conv b0, b1a, b1s, b1t, b2a, b2s, b2t, b3;
    int ctot() const { return c[0] + c[2] + c[4] + c[5]; }
};

// element counts of the workspace buffers for m clips of T frames
struct S3Sizes { size_t s0, mid, tph, stem, v1, v1w, mixA, mixT, mixP, m3c, m4f, m5c; };

}  // namespace vf

using namespace vf;

struct vf_s3d {
    ConvHost ch;
    int device = 0, max_clips = 0, max_T = 0, slots = 0;
    S3Conv stem_s, stem_t, f2, f3s, f3t;
    std::vector<S3Mixed> mixed;
    S3Sizes cap{};
    // workspace; stem_out, c3, m3c, m4f and m5c are kept for vf_s3d_read_stage
    __half *s0 = nullptr, *pf = nullptr, *stem_mid = nullptr, *tph = nullptr, *stem_out = nullptr;
    __half *p1 = nullptr, *c2 = nullptr, *c3a = nullptr, *c3 = nullptr;
    __half *bufA = nullptr, *bufB = nullptr, *ta = nullptr, *tb = nullptr, *tp = nullptr;
    __half *m3c = nullptr, *m4f = nullptr, *m5c = nullptr;
    cudaStream_t cs = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    bool use_graph = true;
    std::map<std::pair<int, int>, std::pair<cudaGraphExec_t, int64_t>> graphs;   // (clips, T) -> (graph, launches)
    int last_m = 0, last_T = 0;
};

namespace vf {

static const int kMixedCfg[9][7] = {
    // cin, b0, b1 mid, b1, b2 mid, b2, b3   (torchvision S3D.features 5, 6, 8..12, 14, 15)
    {192, 64, 96, 128, 16, 32, 32},   {256, 128, 128, 192, 32, 96, 64},  {480, 192, 96, 208, 16, 48, 64},
    {512, 160, 112, 224, 24, 64, 64}, {512, 128, 128, 256, 24, 64, 64},  {512, 112, 144, 288, 32, 64, 64},
    {528, 256, 160, 320, 32, 128, 128}, {832, 256, 160, 320, 32, 128, 128}, {832, 384, 192, 384, 48, 128, 128}};
static const int kMixedIdx[9] = {5, 6, 8, 9, 10, 11, 12, 14, 15};

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

// Uploads conv `name` (weight [co][ci][kt][kh][kw], no bias) followed by BatchNorm3d `bn` (eval, eps 1e-3, folded in
// double) as a hi + lo weight pair.  col(kt, kh, kw, c) -> K column of the activation's hi half; its lo half sits lo_off
// columns further and gets the same weight.  cw.ntaps / k_per_tap and the tap shifts must be set.
static int upload_conv(vf_s3d* h, S3Conv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                       int co, int ci, int kt, int kh, int kw, int lo_off,
                       const std::function<int(int, int, int, int)>& col) {
    const float *w, *g, *b, *m, *v;
    VF_TRY(T.get(name + ".weight", int64_t(co) * ci * kt * kh * kw, &w));
    VF_TRY(T.get(bn + ".weight", co, &g)); VF_TRY(T.get(bn + ".bias", co, &b));
    VF_TRY(T.get(bn + ".running_mean", co, &m)); VF_TRY(T.get(bn + ".running_var", co, &v));
    std::vector<float> sc(co), sh(co);
    for (int i = 0; i < co; ++i) {
        const double s = double(g[i]) / sqrt(double(v[i]) + 1e-3);
        sc[i] = float(s);
        sh[i] = float(double(b[i]) - double(m[i]) * s);
    }
    const int Ktot = cw.ntaps * cw.k_per_tap;
    const size_t Kall = size_t(2) * Ktot;
    std::vector<__half> B(size_t(co) * Kall, __float2half_rn(0.f));
    std::vector<char> has_hi(size_t(Ktot), 0);
    for (int o = 0; o < co; ++o)
        for (int c = 0; c < ci; ++c)
            for (int a = 0; a < kt; ++a)
                for (int y = 0; y < kh; ++y)
                    for (int x = 0; x < kw; ++x) {
                        const int kc = col(a, y, x, c);
                        if (kc < 0 || kc + lo_off >= Ktot) return fail(VF_ERR_INVALID, "s3d_create: filter column out of range");
                        const float wf = w[(((size_t(o) * ci + c) * kt + a) * kh + y) * kw + x];
                        const __half wh = __float2half_rn(wf), wl = __float2half_rn(wf - __half2float(wh));
                        for (int kk : {kc, kc + lo_off}) {
                            B[size_t(o) * Kall + kk] = wh;
                            B[size_t(o) * Kall + Ktot + kk] = wl;
                        }
                        has_hi[kc] = 1;
                    }
    cw.n_out = co;
    // a K block none of whose columns meets a hi half needs only the W_hi pass (a_lo . w_lo < 2^-22 of the product)
    cw.lo_mask = 0;
    const int kpt_blocks = (cw.k_per_tap + 63) / 64;
    if (kpt_blocks <= 64) {
        unsigned long long msk = ~0ull;
        for (int t = 0; t < cw.ntaps; ++t)
            for (int kk = 0; kk < kpt_blocks; ++kk)
                for (int j = kk * 64; j < (kk + 1) * 64 && j < cw.k_per_tap; ++j)
                    if (has_hi[size_t(t) * cw.k_per_tap + j]) { msk &= ~(1ull << kk); break; }
        cw.lo_mask = kpt_blocks == 64 ? msk : (msk & ((1ull << kpt_blocks) - 1));
    }
    VF_TRY(ralloc(&h->ch, &cw.w, B.size()));
    VF_TRY(ralloc(&h->ch, &cw.scale, size_t(co)));
    VF_TRY(ralloc(&h->ch, &cw.bias, size_t(co)));
    VF_CUDA(cudaMemcpy(cw.w, B.data(), B.size() * sizeof(__half), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.scale, sc.data(), co * sizeof(float), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.bias, sh.data(), co * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

// torchvision Conv3dNormActivation `p`: conv p.0, BatchNorm p.1
static int prep(vf_s3d* h, S3Conv& cw, const ResTensors& T, const std::string& p, int co, int ci, int kt, int kh,
                int kw, int lo_off, const std::function<int(int, int, int, int)>& col) {
    return upload_conv(h, cw, T, p + ".0", p + ".1", co, ci, kt, kh, kw, lo_off, col);
}

// (1,3,3) stride 1 pad 1 on split rows of 2ci: one tap per kernel row of 3 * 2ci contiguous elements
static int prep_spatial(vf_s3d* h, S3Conv& cw, const ResTensors& T, const std::string& p, int co, int ci) {
    cw.ntaps = 3; cw.k_per_tap = 6 * ci;
    for (int a = 0; a < 3; ++a) { cw.dh[a] = a - 1; cw.dw[a] = -1; }
    return prep(h, cw, T, p, co, ci, 1, 3, 3, ci, [=](int, int kh, int kw, int c) { return kh * 6 * ci + kw * 2 * ci + c; });
}

// (3,1,1) stride 1 pad 1 on split rows of 2ci: 3 taps one frame apart
static int prep_temporal(vf_s3d* h, S3Conv& cw, const ResTensors& T, const std::string& p, int co, int ci) {
    cw.ntaps = 3; cw.k_per_tap = 2 * ci; cw.tap_kind = 1;
    for (int a = 0; a < 3; ++a) cw.dt[a] = a - 1;
    return prep(h, cw, T, p, co, ci, 3, 1, 1, ci, [=](int kt, int, int, int c) { return kt * 2 * ci + c; });
}

// 1x1x1 on split rows of 2ci
static int prep_point(vf_s3d* h, S3Conv& cw, const ResTensors& T, const std::string& p, int co, int ci) {
    cw.ntaps = 1; cw.k_per_tap = 2 * ci;
    return prep(h, cw, T, p, co, ci, 1, 1, 1, ci, [](int, int, int, int c) { return c; });
}

// stem (1,7,7) stride (1,2,2) pad (0,3,3) on the phase volume (rows [16 hi | 16 lo], 4 channels per phase, 3 used):
// phase row q holds x[2(q-2)+p]; 4 taps (kernel row pairs), each a run of 4 phase positions x 32 elements
static int prep_stem_s(vf_s3d* h, S3Conv& cw, const ResTensors& T) {
    cw.ntaps = 4; cw.k_per_tap = 128;
    for (int a = 0; a < 4; ++a) { cw.dh[a] = a - 2; cw.dw[a] = -2; }
    return prep(h, cw, T, "features.0.0", 64, 3, 1, 7, 7, 16, [](int, int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return a * 128 + b * 32 + (ph * 2 + pw) * 4 + c;
    });
}

// stem (7,1,1) stride (2,1,1) pad (3,0,0) on the temporal phase repack (rows [even frame 128 | odd frame 128], a
// 2-frame border): output frame t reads frames 2t-3 .. 2t+3; tap a (row shift a - 2) holds frames 2t-4+2a+p, so
// kt = 2a + p - 1 and the half-tap (a, p) = (0, 0) is zero
static int prep_stem_t(vf_s3d* h, S3Conv& cw, const ResTensors& T) {
    cw.ntaps = 4; cw.k_per_tap = 256; cw.tap_kind = 1;
    for (int a = 0; a < 4; ++a) cw.dt[a] = a - 2;
    return prep(h, cw, T, "features.0.1", 64, 64, 7, 1, 1, 64, [](int kt, int, int, int c) {
        const int a = (kt + 1) / 2, p = (kt + 1) % 2;
        return a * 256 + p * 128 + c;
    });
}

// one conv over the volume v (rows of `pitch` elements in X) -> split rows [hi n_out | lo n_out] at column 0 of rows
// of ldo elements (split_off = ldo / 2 apart: a channel slice of concat rows), rows outside the valid region zeroed
static int run_conv(vf_s3d* h, const S3Conv& cw, const __half* X, int pitch, const Vol3& v, __half* out, int ldo,
                    cudaStream_t s) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = cw.ntaps; g.k_per_tap = cw.k_per_tap; g.nsplit = 2; g.lo_mask = cw.lo_mask;
    for (int j = 0; j < cw.ntaps; ++j)
        g.tap_off[j] = cw.tap_kind ? cw.dt[j] * v.Hp * v.Wp : cw.dh[j] * v.Wp + cw.dw[j];
    g.mask = 1; g.row0 = 0;
    g.Tp = v.Tp; g.Hp = v.Hp; g.Wp = v.Wp;
    g.t0 = v.t0; g.t1 = v.t1; g.h0 = v.h0; g.h1 = v.h1; g.w0 = v.w0; g.w1 = v.w1;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.ldo = ldo; ep.out_f32 = 0; ep.bias = cw.bias; ep.scale = cw.scale;
    ep.act = VF_ACT_RELU; ep.split_off = ldo / 2;
    h->ch.launches += 1;
    return conv_gemm_f16(X, pitch, v.rows(), cw.w, cw.n_out, g, ep, s);
}

// SepInceptionBlock3D: x (volume v, cin channels) -> out (v, ctot channels, each branch in its slice)
static int run_mixed(vf_s3d* h, const S3Mixed& B, const __half* x, const Vol3& v, __half* out, cudaStream_t s) {
    const int* c = B.c;
    const int ld = 2 * B.ctot(), xp = 2 * B.cin;
    VF_TRY(run_conv(h, B.b0, x, xp, v, out, ld, s));
    VF_TRY(run_conv(h, B.b1a, x, xp, v, h->ta, 2 * c[1], s));
    VF_TRY(run_conv(h, B.b1s, h->ta, 2 * c[1], v, h->tb, 2 * c[2], s));
    VF_TRY(run_conv(h, B.b1t, h->tb, 2 * c[2], v, out + c[0], ld, s));
    VF_TRY(run_conv(h, B.b2a, x, xp, v, h->ta, 2 * c[3], s));
    VF_TRY(run_conv(h, B.b2s, h->ta, 2 * c[3], v, h->tb, 2 * c[4], s));
    VF_TRY(run_conv(h, B.b2t, h->tb, 2 * c[4], v, out + c[0] + c[2], ld, s));
    VF_TRY(launch_maxpool3d_raw(x, &v, h->tp, &v, B.cin, 3, 3, 3, 1, 1, 1, 1, 1, 1, s));
    h->ch.launches += 1;
    VF_TRY(run_conv(h, B.b3, h->tp, xp, v, out + c[0] + c[2] + c[4], ld, s));
    return VF_OK;
}

// stem .. Mixed 5c on m clips of T frames whose clip phase volume is in h->s0
static int run_trunk(vf_s3d* h, int m, int T, cudaStream_t s) {
    const S3Geom g = geom(m, T);
    VF_TRY(run_conv(h, h->stem_s, h->s0, 32, g.v0, h->stem_mid, 128, s));
    VF_TRY(r21d_temporal_phase(h->stem_mid, g.v0, 128, h->tph, g.vt, s));
    VF_TRY(run_conv(h, h->stem_t, h->tph, 256, g.vt, h->stem_out, 128, s));
    VF_TRY(launch_maxpool3d_raw(h->stem_out, &g.vt, h->p1, &g.v1, 64, 1, 3, 3, 1, 2, 2, 0, 1, 1, s));
    VF_TRY(run_conv(h, h->f2, h->p1, 128, g.v1, h->c2, 128, s));
    VF_TRY(run_conv(h, h->f3s, h->c2, 128, g.v1, h->c3a, 384, s));
    VF_TRY(run_conv(h, h->f3t, h->c3a, 384, g.v1, h->c3, 384, s));
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
    h->ch.launches += 5;
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
    VF_CUDA(cudaSetDevice(device));
    int major = 0, minor = 0;
    VF_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    VF_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    if (major != 9 || minor != 0)
        return fail(VF_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device, major, minor);
    vf_s3d* h = new vf_s3d();
    h->ch.who = "s3d_create";
    h->device = device; h->max_clips = max_clips; h->max_T = max_T;
    h->slots = max_clips * (max_T + 2);
    const ResTensors Tn{tensors, n_tensors, "s3d_create"};
    auto body = [&]() -> int {
        VF_TRY(prep_stem_s(h, h->stem_s, Tn));
        VF_TRY(prep_stem_t(h, h->stem_t, Tn));
        VF_TRY(prep_point(h, h->f2, Tn, "features.2", 64, 64));
        VF_TRY(prep_spatial(h, h->f3s, Tn, "features.3.0", 192, 64));
        VF_TRY(prep_temporal(h, h->f3t, Tn, "features.3.1", 192, 192));
        for (int i = 0; i < 9; ++i) {
            S3Mixed B;
            const int* c = kMixedCfg[i];
            B.cin = c[0];
            for (int j = 0; j < 6; ++j) B.c[j] = c[j + 1];
            const std::string p = "features." + std::to_string(kMixedIdx[i]);
            VF_TRY(prep_point(h, B.b0, Tn, p + ".branch0", B.c[0], B.cin));
            VF_TRY(prep_point(h, B.b1a, Tn, p + ".branch1.0", B.c[1], B.cin));
            VF_TRY(prep_spatial(h, B.b1s, Tn, p + ".branch1.1.0", B.c[2], B.c[1]));
            VF_TRY(prep_temporal(h, B.b1t, Tn, p + ".branch1.1.1", B.c[2], B.c[2]));
            VF_TRY(prep_point(h, B.b2a, Tn, p + ".branch2.0", B.c[3], B.cin));
            VF_TRY(prep_spatial(h, B.b2s, Tn, p + ".branch2.1.0", B.c[4], B.c[3]));
            VF_TRY(prep_temporal(h, B.b2t, Tn, p + ".branch2.1.1", B.c[4], B.c[4]));
            VF_TRY(prep_point(h, B.b3, Tn, p + ".branch3.1", B.c[5], B.cin));
            h->mixed.push_back(B);
        }
        h->cap = sizes(max_clips, max_T);
        const S3Sizes& z = h->cap;
        VF_TRY(ralloc(&h->ch, &h->s0, z.s0));
        VF_TRY(ralloc(&h->ch, &h->pf, size_t(h->slots) * S3D_Q * S3D_Q * 32));
        VF_TRY(ralloc(&h->ch, &h->stem_mid, z.mid));
        VF_TRY(ralloc(&h->ch, &h->tph, z.tph));
        VF_TRY(ralloc(&h->ch, &h->stem_out, z.stem));
        VF_TRY(ralloc(&h->ch, &h->p1, z.v1));
        VF_TRY(ralloc(&h->ch, &h->c2, z.v1));
        VF_TRY(ralloc(&h->ch, &h->c3a, z.v1w));
        VF_TRY(ralloc(&h->ch, &h->c3, z.v1w));
        VF_TRY(ralloc(&h->ch, &h->bufA, z.mixA));
        VF_TRY(ralloc(&h->ch, &h->bufB, z.mixA));
        VF_TRY(ralloc(&h->ch, &h->ta, z.mixT));
        VF_TRY(ralloc(&h->ch, &h->tb, z.mixT));
        VF_TRY(ralloc(&h->ch, &h->tp, z.mixP));
        VF_TRY(ralloc(&h->ch, &h->m3c, z.m3c));
        VF_TRY(ralloc(&h->ch, &h->m4f, z.m4f));
        VF_TRY(ralloc(&h->ch, &h->m5c, z.m5c));
        VF_CUDA(cudaStreamCreateWithFlags(&h->cs, cudaStreamNonBlocking));
        VF_CUDA(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
        VF_CUDA(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
        const char* e = getenv("VF_NO_GRAPH");
        h->use_graph = !(e && e[0] == '1');
        return VF_OK;
    };
    const int st = body();
    if (st != VF_OK) { vf_s3d_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_s3d_destroy(vf_s3d_t* h) {
    if (!h) return VF_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (void* p : h->ch.allocs) cudaFree(p);
    for (auto& kv : h->graphs) cudaGraphExecDestroy(kv.second.first);
    if (h->cs) cudaStreamDestroy(h->cs);
    if (h->ev_in) cudaEventDestroy(h->ev_in);
    if (h->ev_out) cudaEventDestroy(h->ev_out);
    delete h;
    return VF_OK;
}

}  // extern "C"

namespace vf {

static int trunk_graph(vf_s3d* h, int m, int T, cudaStream_t s) {
    if (!h->use_graph || gemm_profile_on()) return run_trunk(h, m, T, s);
    const auto key = std::make_pair(m, T);
    auto it = h->graphs.find(key);
    if (it == h->graphs.end()) {
        const int64_t before = h->ch.launches;
        cudaGraph_t graph = nullptr;
        VF_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
        const int st = run_trunk(h, m, T, s);
        const cudaError_t ce = cudaStreamEndCapture(s, &graph);
        const int64_t n_launch = h->ch.launches - before;
        h->ch.launches = before;
        if (st != VF_OK) { if (graph) cudaGraphDestroy(graph); return st; }
        if (ce != cudaSuccess) return fail(VF_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(ce));
        cudaGraphExec_t exec = nullptr;
        const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) return fail(VF_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ie));
        // bounded cache: ragged last chunks of many videos must not pile up executable graphs
        if (h->graphs.size() >= 16) {
            cudaGraphExecDestroy(h->graphs.begin()->second.first);
            h->graphs.erase(h->graphs.begin());
        }
        it = h->graphs.emplace(key, std::make_pair(exec, n_launch)).first;
    }
    VF_CUDA(cudaGraphLaunch(it->second.first, s));
    h->ch.launches += it->second.second;
    return VF_OK;
}

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
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaEventRecord(h->ev_in, user));
    VF_CUDA(cudaStreamWaitEvent(s, h->ev_in, 0));
    for (int off = 0; off < n;) {      // calls beyond the workspace run in chunks
        int m = 0;
        if (is_u8) {
            // the chunk's frames [lo, hi) are transformed once each, so they must fit the per-frame buffer
            int lo = starts[off], hi = starts[off] + T;
            while (off + m < n && m < per_chunk) {
                const int l2 = std::min(lo, starts[off + m]), h2 = std::max(hi, starts[off + m] + T);
                if (m > 0 && h2 - l2 > h->slots) break;
                lo = l2; hi = h2; ++m;
            }
            if (hi - lo > h->slots) return fail(VF_ERR_INVALID, "s3d_forward: clip exceeds the frame workspace");
            R21DStarts st;
            for (int b = 0; b < m; ++b) st.first[b] = starts[off + b] - lo;
            const uint8_t* f0 = static_cast<const uint8_t*>(src) + int64_t(lo) * H * W * 3;
            VF_TRY(s3d_frames_u8(f0, hi - lo, H, W, crop, crop, h->pf, s));
            VF_TRY(s3d_clip_gather(h->pf, st, m, T, h->s0, s));
            h->ch.launches += 2;
        } else {
            m = std::min(per_chunk, n - off);
            VF_TRY(s3d_pack_f32(static_cast<const float*>(src) + int64_t(off) * 3 * T * S3D_CROP * S3D_CROP, m, T,
                                h->s0, s));
            h->ch.launches += 1;
        }
        VF_TRY(trunk_graph(h, m, T, s));
        const Vol3 v4 = geom(m, T).v4;
        VF_TRY(launch_i3d_head_raw(h->m5c, &v4, 1024, out + int64_t(off) * 1024, s));
        h->ch.launches += 1;
        h->last_m = m; h->last_T = T;
        off += m;
    }
    VF_CUDA(cudaEventRecord(h->ev_out, s));
    VF_CUDA(cudaStreamWaitEvent(user, h->ev_out, 0));
    return VF_OK;
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
    if (!h || !dims5 || h->last_m <= 0) return fail(VF_ERR_INVALID, "s3d_read_stage: no forward has run");
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

int64_t vf_s3d_launch_count(const vf_s3d_t* h) { return h ? h->ch.launches : 0; }

int vf_s3d_conv(const vf_s3d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "s3d_conv: null argument");
    std::vector<const S3Conv*> cs{&h->stem_s, &h->stem_t, &h->f2, &h->f3s, &h->f3t};
    for (const S3Mixed& B : h->mixed)
        for (const S3Conv* c : {&B.b0, &B.b1a, &B.b1s, &B.b1t, &B.b2a, &B.b2s, &B.b2t, &B.b3}) cs.push_back(c);
    if (index < 0 || index >= int(cs.size()))
        return fail(VF_ERR_INVALID, "s3d_conv: index %d outside the %d convs", index, int(cs.size()));
    const S3Conv& c = *cs[index];
    geom[0] = c.n_out; geom[1] = c.ntaps; geom[2] = c.k_per_tap;
    for (int j = 0; j < 4; ++j) {
        geom[3 + 3 * j] = c.tap_kind ? c.dt[j] : 0;
        geom[4 + 3 * j] = c.tap_kind ? 0 : c.dh[j];
        geom[5 + 3 * j] = c.tap_kind ? 0 : c.dw[j];
    }
    *lo_mask = c.lo_mask;
    VF_CUDA(cudaSetDevice(h->device));
    const size_t nw = size_t(c.n_out) * 2 * c.ntaps * c.k_per_tap;
    if (w) VF_CUDA(cudaMemcpy(w, c.w, nw * sizeof(__half), cudaMemcpyDeviceToDevice));
    if (scale) VF_CUDA(cudaMemcpy(scale, c.scale, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    if (bias) VF_CUDA(cudaMemcpy(bias, c.bias, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    return VF_OK;
}

}  // extern "C"
