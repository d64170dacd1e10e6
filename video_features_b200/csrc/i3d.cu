// Inception-3D (I3D) feature extractor on the wgmma conv-GEMM.
// Replaces `I3D(num_classes=400, modality).forward(x, features=True)` (reference: models/i3d/i3d_src/i3d_net.py:238-264,
// called at models/i3d/extract_i3d.py:186) and the stream transforms around it (extract_i3d.py:62-73).
//
// Data layout: every activation is channels-last fp16 in a ZERO-BORDERED volume [n][Tp][Hp][Wp][C] (border 1 around
// the valid T x H x W region), flattened to rows of C channels.  With that layout
//   * a 1x1x1 conv is a plain GEMM over the rows,
//   * a 3x3x3 conv is 9 (dt,dh) "taps", each a constant row shift whose 3 kw neighbours are one contiguous run of
//     3*C elements (conv_gemm_f16), the zero border IS the SAME padding, and the epilogue re-zeroes border rows,
//   * the zero-padding max pools of the reference (MaxPool3dTFPadding pads with 0, i3d_net.py:114) read the border,
//   * the 7x7x7 stride-2 stem becomes a 4x4x4 stride-1 conv over the 8 space-time phases of the input; the phase volume
//     [n][T/2+3][115][115][4 x 8*C] carries the 4 h-taps inside each row, so the GEMM walks 4 t-taps of 4*32*C contiguous
//     elements (i3d_kernels.cu).
// BatchNorm (eval) is folded into the epilogue's per-channel scale/bias (fp32), ReLU fused; branch outputs of a Mixed
// block are written straight into their channel slice of the concat buffer (stored with the concat row pitch).
//
// Numerics: accumulate fp32.  With single-fp16 weights the 1024-d feature is 1.7e-3 off the fp32 reference (trained
// weights; CPU emulation in DESIGN.md); weights are therefore carried as a hi+lo fp16 pair and every K block is issued
// twice (A.W_hi + A.W_lo): 8e-4 .. 1.06e-3 with single-fp16 activations.  Of that, 6.8e-4 comes from the rounding of the
// tensors read by the 1x1x1 convs and the pools, so exactly those are "pair tensors", rows [hi C | lo C] of split-fp16
// pairs (written by the GEMM's split-output epilogue or by the pool kernels); the inputs of the 3x3x3 convs, which carry
// the FLOPs, stay single fp16: 1.5e-4 .. 4.0e-4.  VF_I3D_FAST=1 selects single-fp16 weights.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "internal.h"

namespace vf {

struct Vol {
    int n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1;
    int64_t rows() const { return int64_t(n) * Tp * Hp * Wp; }
    int T() const { return t1 - t0; }
    int H() const { return h1 - h0; }
    int W() const { return w1 - w0; }
};
static Vol bordered(int n, int T, int H, int W) { return Vol{n, T + 2, H + 2, W + 2, 1, 1 + T, 1, 1 + H, 1, 1 + W}; }

struct ConvUnit {
    int cout = 0, cin = 0, k = 0;     // k: 1, 3, or 7 (the stem)
    int ntaps = 0, k_per_tap = 0;     // base tap geometry (before the hi/lo split)
    int nsplit = 1;
    unsigned long long lo_mask = 0;   // K blocks that meet only lo halves of a pair input (ConvGeom::lo_mask)
    __half* w = nullptr;              // [cout, nsplit * ntaps * k_per_tap]
    float *scale = nullptr, *bias = nullptr;
};

// kernels (i3d_kernels.cu); volumes are passed as pointers to the 10 leading ints of Vol
int launch_i3d_phase_pack_f32(const float* x, int n, int C, int T, __half* out, int Tq, cudaStream_t s);
int launch_i3d_phase_pack_u8(const uint8_t* frames, int n, int T, int64_t stack_stride, int Hr, int Wr, int cy, int cx,
                             __half* out, int Tq,
                             cudaStream_t s);
int launch_i3d_phase_pack_flow(const float* flow, int n, int T, int H, int W, int cy, int cx, __half* out, int Tq,
                               cudaStream_t s);
int launch_maxpool3d_raw(const __half* in, const void* vi, __half* out, const void* vo, int C, int kt, int kh, int kw,
                         int st, int sh, int sw, int pt, int ph, int pw, cudaStream_t s);
int launch_i3d_head_raw(const __half* in, const void* vi, int C, float* out, cudaStream_t s);
int launch_unpack_ndhwc_raw(const __half* in, const void* vi, int C, int c_off, int c_cnt, int ld, int lo_off, float* out,
                            cudaStream_t s);
static int launch_maxpool3d(const __half* in, const Vol& vi, __half* out, const Vol& vo, int C, int kt, int kh, int kw,
                            int st, int sh, int sw, int pt, int ph, int pw, cudaStream_t s) {
    return launch_maxpool3d_raw(in, &vi, out, &vo, C, kt, kh, kw, st, sh, sw, pt, ph, pw, s);
}
static int launch_i3d_head(const __half* in, const Vol& vi, int C, float* out, cudaStream_t s) {
    return launch_i3d_head_raw(in, &vi, C, out, s);
}
static int launch_unpack_ndhwc(const __half* in, const Vol& vi, int C, int c_off, int c_cnt, int ld, int lo_off, float* out,
                               cudaStream_t s) {
    return launch_unpack_ndhwc_raw(in, &vi, C, c_off, c_cnt, ld, lo_off, out, s);
}

}  // namespace vf

using namespace vf;

static const int kMixed[9][7] = {
    // cin, b0, b1a, b1b, b2a, b2b, b3     (i3d_net.py:206-224)
    {192, 64, 96, 128, 16, 32, 32},   {256, 128, 128, 192, 32, 96, 64},  {480, 192, 96, 208, 16, 48, 64},
    {512, 160, 112, 224, 24, 64, 64}, {512, 128, 128, 256, 24, 64, 64},  {512, 112, 144, 288, 32, 64, 64},
    {528, 256, 160, 320, 32, 128, 128}, {832, 256, 160, 320, 32, 128, 128}, {832, 384, 192, 384, 48, 128, 128}};

struct vf_i3d : vf::EngineCore {
    int cin = 3, max_stacks = 0, max_T = 0;
    int nsplit = 2;
    ConvUnit units[VF_I3D_UNITS];
    // activation buffers (sized for max_stacks x max_T at create)
    __half *s0 = nullptr, *a1 = nullptr, *p1 = nullptr, *c2b = nullptr, *c2c = nullptr;
    __half *bufA = nullptr, *bufB = nullptr, *t1 = nullptr, *t2 = nullptr, *tp = nullptr;
    size_t cap_s0 = 0, cap_a1 = 0, cap_s1 = 0, cap_rows2 = 0;
    float* feat = nullptr;            // [max_stacks, 1024] trunk output
    // last forward's stage views, for vf_i3d_read_stage
    struct StageRef { const __half* p; Vol v; int C; } stages[5];
};

namespace vf {

// fold BN, re-lay the filter for the shifted-row GEMM, split into hi/lo fp16, upload
static int prepare_unit(vf_i3d* h, ConvUnit& u, const vf_conv_unit& src, int idx) {
    if (!src.w || !src.bn_w || !src.bn_b || !src.bn_mean || !src.bn_var)
        return fail(VF_ERR_INVALID, "i3d_create: unit %d has a null tensor", idx);
    u.cout = src.cout; u.cin = src.cin; u.k = src.k;
    const int co = u.cout, ci = u.cin, k = u.k;
    std::vector<float> wt;   // [co][ntaps*k_per_tap]
    if (k == 1) {
        // every 1x1x1 conv reads a pair tensor, rows [hi ci | lo ci]: the filter is laid over both halves, and K blocks
        // that fall entirely into the lo half skip the W_lo pass
        u.ntaps = 1; u.k_per_tap = 2 * ci;
        wt.resize(size_t(co) * 2 * ci);
        for (int o = 0; o < co; ++o)
            for (int c = 0; c < ci; ++c) wt[size_t(o) * 2 * ci + c] = wt[size_t(o) * 2 * ci + ci + c] = src.w[size_t(o) * ci + c];
        const int kb = (2 * ci + 63) / 64;
        for (int kk = 0; kk < kb && kk < 64; ++kk)
            if (kk * 64 >= ci) u.lo_mask |= 1ull << kk;
    } else if (k == 3) {
        u.ntaps = 9; u.k_per_tap = 3 * ci;
        wt.resize(size_t(co) * 27 * ci);
        for (int o = 0; o < co; ++o)
            for (int c = 0; c < ci; ++c)
                for (int kt = 0; kt < 3; ++kt)
                    for (int kh = 0; kh < 3; ++kh)
                        for (int kw = 0; kw < 3; ++kw)
                            wt[(size_t(o) * 9 + kt * 3 + kh) * (3 * ci) + kw * ci + c] =
                                src.w[(((size_t(o) * ci + c) * 3 + kt) * 3 + kh) * 3 + kw];
    } else if (k == 7) {
        // stride-2 7x7x7 with TF-SAME padding (2 before, 3 after) == 4x4x4 stride-1 over the 8 phases:
        // filter index kk = 2*a + p for tap a in 0..3 (row offset a-1) and phase p in 0..1; kk == 7 does not exist.
        // The phase volume carries the 4 h-taps inside each row (slot b = source row h + b - 1, i3d_kernels.cu), so the
        // GEMM taps are the 4 t-taps, each a run of 4 w-positions x (4 slots x 8 phases x ci) channels.
        const int pc = 8 * ci;
        u.ntaps = 4; u.k_per_tap = 16 * pc;
        wt.assign(size_t(co) * 4 * 16 * pc, 0.f);
        for (int o = 0; o < co; ++o)
            for (int c = 0; c < ci; ++c)
                for (int a = 0; a < 4; ++a) for (int pt = 0; pt < 2; ++pt) {
                    const int kt = 2 * a + pt; if (kt > 6) continue;
                    for (int b = 0; b < 4; ++b) for (int ph = 0; ph < 2; ++ph) {
                        const int kh = 2 * b + ph; if (kh > 6) continue;
                        for (int cw = 0; cw < 4; ++cw) for (int pw = 0; pw < 2; ++pw) {
                            const int kw = 2 * cw + pw; if (kw > 6) continue;
                            wt[(size_t(o) * 4 + a) * (16 * pc) + cw * (4 * pc) + b * pc + ((pt * 2 + ph) * 2 + pw) * ci + c] =
                                src.w[(((size_t(o) * ci + c) * 7 + kt) * 7 + kh) * 7 + kw];
                        }
                    }
                }
    } else {
        return fail(VF_ERR_UNSUPPORTED, "i3d_create: unit %d has kernel size %d", idx, k);
    }
    if (u.k_per_tap % 8) return fail(VF_ERR_UNSUPPORTED, "i3d_create: unit %d: %d channels per tap", idx, u.k_per_tap);
    // Weight precision per layer: hi + lo fp16 pairs (two MMA passes per K step, ~22 mantissa bits) except where a CPU
    // emulation of the trained checkpoints shows single fp16 weights to be harmless (scripts/precision/
    // emulate_i3d_weights.py: rgb / flow, uniform-noise clips, 4 seeds): the stem and the four 3x3x3 convs of stage 3
    // (mixed_3b / 3c branch_1.1, branch_2.1 -- 61 of the 222 GFLOP) move the feature error from 1.6..3.7e-4 to 3.1..4.3e-4
    // rel-L2 (max-abs <= 6.0e-4); the 3x3x3 convs of stage 4 or conv3d_2c would take it to 5.4..6.8e-4 with max-abs at the
    // 1e-3 bar, so they stay split.  VF_I3D_SINGLE=none keeps every layer split, VF_I3D_FAST=1 makes every layer single.
    {
        const char* e = getenv("VF_I3D_SINGLE");
        const bool none = e && e[0] == 'n';
        const bool chosen = k == 7 || idx == 5 || idx == 7 || idx == 11 || idx == 13;
        u.nsplit = (h->nsplit == 2 && chosen && !none) ? 1 : h->nsplit;
        if (u.nsplit != 2) u.lo_mask = 0;
    }
    const size_t Kb = size_t(u.ntaps) * u.k_per_tap, Kt = Kb * u.nsplit;
    std::vector<__half> wh(size_t(co) * Kt);
    for (int o = 0; o < co; ++o)
        for (size_t j = 0; j < Kb; ++j) {
            const float v = wt[size_t(o) * Kb + j];
            const __half hi = __float2half_rn(v);
            wh[size_t(o) * Kt + j] = hi;
            if (u.nsplit == 2) wh[size_t(o) * Kt + Kb + j] = __float2half_rn(v - __half2float(hi));
        }
    std::vector<float> sc(co), bi(co);
    for (int o = 0; o < co; ++o) {
        const float s = src.bn_w[o] / sqrtf(src.bn_var[o] + 1e-5f);   // BatchNorm3d eval, eps 1e-5 (i3d_net.py:92)
        sc[o] = s;
        bi[o] = src.bn_b[o] - src.bn_mean[o] * s;
    }
    VF_TRY(ralloc(h, &u.w, wh.size()));
    VF_TRY(ralloc(h, &u.scale, size_t(co)));
    VF_TRY(ralloc(h, &u.bias, size_t(co)));
    VF_CUDA(cudaMemcpy(u.w, wh.data(), wh.size() * sizeof(__half), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(u.scale, sc.data(), co * sizeof(float), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(u.bias, bi.data(), co * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

// tap j's shift in (t, h, w) rows: 3x3x3 taps are (kt, kh) with the 3 kw positions inside the run; the stem's taps are
// its 4 t-taps (the h-taps live inside the row)
static void unit_tap(const ConvUnit& u, int j, int* dt, int* dh, int* dw) {
    *dt = 0; *dh = 0; *dw = 0;
    if (u.k == 3) { *dt = j / 3 - 1; *dh = j % 3 - 1; *dw = -1; }
    else if (u.k == 7) { *dt = j - 1; *dw = -1; }
}

// conv + BN + ReLU of one unit over a bordered volume; out rows keep the input's row indexing
// split_off > 0: the output is a pair tensor, hi at column n and lo at column split_off + n of the rows at `out`
static int run_unit(vf_i3d* h, const ConvUnit& u, const __half* X, int ldx_channels, const Vol& v, __half* out, int ldo,
                    cudaStream_t s, int split_off = 0) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.k_per_tap = u.k_per_tap;
    g.ntaps = u.ntaps;
    g.nsplit = u.nsplit;          // hi/lo weight passes share each A tile inside the kernel
    g.lo_mask = u.lo_mask;
    for (int j = 0; j < u.ntaps; ++j) {
        int dt, dh, dw;
        unit_tap(u, j, &dt, &dh, &dw);
        g.tap_off[j] = (dt * v.Hp + dh) * v.Wp + dw;
    }
    g.mask = 1;
    g.Tp = v.Tp; g.Hp = v.Hp; g.Wp = v.Wp;
    g.t0 = v.t0; g.t1 = v.t1; g.h0 = v.h0; g.h1 = v.h1; g.w0 = v.w0; g.w1 = v.w1;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.ldo = ldo; ep.out_f32 = 0; ep.bias = u.bias; ep.scale = u.scale; ep.act = VF_ACT_RELU;
    ep.split_off = split_off;
    h->launches += 1;
    return conv_gemm_f16(X, ldx_channels, v.rows(), u.w, u.cout, g, ep, s);
}

// x and out are pair tensors (rows [hi C | lo C]); the 1x1x1 reducers' outputs t1 / t2 feed 3x3x3 convs and are single fp16
static int mixed_block(vf_i3d* h, int m, const __half* x, const Vol& v, __half* out, cudaStream_t s) {
    const int* c = kMixed[m];
    const ConvUnit* u = &h->units[3 + 6 * m];
    const int cin = c[0], ctot = c[1] + c[3] + c[5] + c[6];
    VF_TRY(run_unit(h, u[0], x, 2 * cin, v, out, 2 * ctot, s, ctot));                              // branch_0
    VF_TRY(run_unit(h, u[1], x, 2 * cin, v, h->t1, c[2], s));                                      // branch_1.0
    VF_TRY(run_unit(h, u[2], h->t1, c[2], v, out + c[1], 2 * ctot, s, ctot));                      // branch_1.1 (3x3x3)
    VF_TRY(run_unit(h, u[3], x, 2 * cin, v, h->t2, c[4], s));                                      // branch_2.0
    VF_TRY(run_unit(h, u[4], h->t2, c[4], v, out + c[1] + c[3], 2 * ctot, s, ctot));               // branch_2.1 (3x3x3)
    VF_TRY(launch_maxpool3d(x, v, h->tp, v, cin, 3, 3, 3, 1, 1, 1, 1, 1, 1, s));                   // branch_3 pool (zero pad)
    h->launches += 1;
    VF_TRY(run_unit(h, u[5], h->tp, 2 * cin, v, out + c[1] + c[3] + c[5], 2 * ctot, s, ctot));     // branch_3.1
    return VF_OK;
}

static int ceil_div(int a, int b) { return (a + b - 1) / b; }

}  // namespace vf

extern "C" {

int vf_i3d_create(vf_i3d_t** out, const vf_i3d_weights* w, int in_channels, int device, int max_stacks, int max_T) {
    if (!out || !w) return fail(VF_ERR_INVALID, "i3d_create: null argument");
    *out = nullptr;
    if (in_channels != 3 && in_channels != 2) return fail(VF_ERR_INVALID, "i3d_create: in_channels must be 3 (rgb) or 2 (flow)");
    if (max_stacks <= 0) max_stacks = 4;
    if (max_T <= 0) max_T = 64;
    VF_TRY(check_device(device));
    vf_i3d* h = new vf_i3d();
    h->who = "i3d_create";
    h->device = device; h->cin = in_channels; h->max_stacks = max_stacks; h->max_T = max_T;
    {
        const char* e = getenv("VF_I3D_FAST");
        h->nsplit = (e && e[0] == '1') ? 1 : 2;
    }
    auto body = [&]() -> int {
        for (int i = 0; i < VF_I3D_UNITS; ++i) VF_TRY(prepare_unit(h, h->units[i], w->units[i], i));
        if (h->units[0].cin != in_channels || h->units[0].k != 7) return fail(VF_ERR_INVALID, "i3d_create: stem shape");
        const size_t n = size_t(max_stacks);
        const int T1 = max_T / 2, Tq = T1 + 3;       // stem: floor((T + 5 - 7) / 2) + 1 = T / 2
        const size_t rows0 = n * Tq * 115 * 115;
        VF_TRY(ralloc(h, &h->s0, rows0 * 32 * in_channels + 4096));
        VF_TRY(ralloc(h, &h->a1, rows0 * 128));          // pair tensors: 2 x channels
        const size_t rows1 = n * (T1 + 2) * 58 * 58;
        VF_TRY(ralloc(h, &h->p1, rows1 * 128));
        VF_TRY(ralloc(h, &h->c2b, rows1 * 64));
        VF_TRY(ralloc(h, &h->c2c, rows1 * 384));
        const size_t rows2 = n * (T1 + 2) * 30 * 30;    // largest Mixed stage
        VF_TRY(ralloc(h, &h->bufA, rows2 * 2048));
        VF_TRY(ralloc(h, &h->bufB, rows2 * 2048));
        VF_TRY(ralloc(h, &h->t1, rows2 * 192));
        VF_TRY(ralloc(h, &h->t2, rows2 * 64));
        VF_TRY(ralloc(h, &h->tp, rows2 * 1664));
        h->cap_rows2 = rows2;
        VF_TRY(ralloc(h, &h->feat, n * 1024));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_i3d_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_i3d_destroy(vf_i3d_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

}  // extern "C"

// geometry of the trunk for nb clips of T frames: the volumes after the stem, pool2a, pool3a, pool4a and pool5a, and
// where in bufA the mixed_4x and 5b outputs go
struct TrunkGeom { Vol v0, v1, v2, v3, v4; __half *a4, *a5; };
static TrunkGeom trunk_geom(const vf_i3d* h, int nb, int T) {
    TrunkGeom g;
    const int T1 = T / 2, Tq = T1 + 3;            // torch conv3d, pad (2,3), stride 2: floor((T-2)/2)+1
    const int T2 = ceil_div(T1, 2), T3 = ceil_div(T2, 2);
    g.v0 = Vol{nb, Tq, 115, 115, 1, 1 + T1, 1, 113, 1, 113};
    g.v1 = bordered(nb, T1, 56, 56);
    g.v2 = bordered(nb, T1, 28, 28);
    g.v3 = bordered(nb, T2, 14, 14);
    g.v4 = bordered(nb, T3, 7, 7);
    // bufA's later outputs go behind what stays readable for read_stage: mixed_3c (v2, 960 columns) at a4, mixed_4f
    // (v3, 1664 columns) at a5.  All three fit in bufA (its rows2 x 2048 holds rows2 x 1384 at T = 10, less beyond).
    g.a4 = h->bufA + size_t(g.v2.rows()) * 960;
    g.a5 = g.a4 + size_t(g.v3.rows()) * 1664;
    return g;
}

// the activations vf_i3d_read_stage reads after a forward of nb clips of T frames (graph replays included)
static void set_stages(vf_i3d* h, int nb, int T) {
    const TrunkGeom g = trunk_geom(h, nb, T);
    h->stages[0] = {h->a1, g.v0, 64};
    h->stages[1] = {h->c2c, g.v1, 192};
    h->stages[2] = {h->bufA, g.v2, 480};
    h->stages[3] = {g.a4, g.v3, 832};
    h->stages[4] = {h->bufB, g.v4, 1024};
}

// everything after the stem's phase volume h->s0 has been filled for nb clips of T frames
static int i3d_trunk(vf_i3d* h, int nb, int T, float* out, cudaStream_t s) {
    const TrunkGeom g = trunk_geom(h, nb, T);
    const Vol &v0 = g.v0, &v1 = g.v1, &v2 = g.v2, &v3 = g.v3, &v4 = g.v4;
    __half *a4 = g.a4, *a5 = g.a5;
    VF_TRY(run_unit(h, h->units[0], h->s0, 32 * h->cin, v0, h->a1, 128, s, 64));       // a1: pair tensor
    // ---- maxPool3d_2a (1,3,3)/(1,2,2), SAME pad (0,1) on H,W
    VF_TRY(launch_maxpool3d(h->a1, v0, h->p1, v1, 64, 1, 3, 3, 1, 2, 2, 0, 0, 0, s));
    VF_TRY(run_unit(h, h->units[1], h->p1, 128, v1, h->c2b, 64, s));                   // pair in, single out
    VF_TRY(run_unit(h, h->units[2], h->c2b, 64, v1, h->c2c, 384, s, 192));             // single in, pair out
    // ---- maxPool3d_3a
    VF_TRY(launch_maxpool3d(h->c2c, v1, h->bufA, v2, 192, 1, 3, 3, 1, 2, 2, 0, 0, 0, s));
    VF_TRY(mixed_block(h, 0, h->bufA, v2, h->bufB, s));     // 3b -> 256
    VF_TRY(mixed_block(h, 1, h->bufB, v2, h->bufA, s));     // 3c -> 480
    // ---- maxPool3d_4a 3x3x3 / 2, SAME pad (0,1)
    VF_TRY(launch_maxpool3d(h->bufA, v2, h->bufB, v3, 480, 3, 3, 3, 2, 2, 2, 0, 0, 0, s));
    VF_TRY(mixed_block(h, 2, h->bufB, v3, a4, s));          // 4b -> 512
    VF_TRY(mixed_block(h, 3, a4, v3, h->bufB, s));          // 4c
    VF_TRY(mixed_block(h, 4, h->bufB, v3, a4, s));          // 4d
    VF_TRY(mixed_block(h, 5, a4, v3, h->bufB, s));          // 4e -> 528
    VF_TRY(mixed_block(h, 6, h->bufB, v3, a4, s));          // 4f -> 832
    // ---- maxPool3d_5a 2x2x2 / 2, no padding, ceil mode
    if (v4.T() < 2) return fail(VF_ERR_INVALID, "i3d_forward: T=%d leaves %d temporal positions for the (2,7,7) pool", T, v4.T());
    VF_TRY(launch_maxpool3d(a4, v3, h->bufB, v4, 832, 2, 2, 2, 2, 2, 2, 0, 0, 0, s));
    VF_TRY(mixed_block(h, 7, h->bufB, v4, a5, s));          // 5b -> 832
    VF_TRY(mixed_block(h, 8, a5, v4, h->bufB, s));          // 5c -> 1024
    // ---- AvgPool3d((2,7,7),1) + mean over time
    VF_TRY(launch_i3d_head(h->bufB, v4, 1024, out, s));
    h->launches += 5;
    return VF_OK;
}

// the trunk, eagerly into out or through the graph of (clips, T), whose features land in h->feat and are copied out
static int i3d_trunk_graphed(vf_i3d* h, int nb, int T, float* out, cudaStream_t s) {
    if (!h->use_graph || gemm_profile_on()) {
        VF_TRY(i3d_trunk(h, nb, T, out, s));
    } else {
        VF_TRY(run_graphed(h, {nb, T, 0, 0}, [&] { return i3d_trunk(h, nb, T, h->feat, s); }));
        VF_CUDA(cudaMemcpyAsync(out, h->feat, size_t(nb) * 1024 * sizeof(float), cudaMemcpyDeviceToDevice, s));
        h->launches += 1;
    }
    set_stages(h, nb, T);
    return VF_OK;
}

static int i3d_check(vf_i3d* h, const void* in, int n, int T, const void* out, int need_cin) {
    if (!h || (n > 0 && (!in || !out))) return fail(VF_ERR_INVALID, "i3d_forward: null argument");
    if (T < 10 || T > h->max_T) return fail(VF_ERR_INVALID, "i3d_forward: T=%d outside [10, %d]", T, h->max_T);
    if (need_cin && h->cin != need_cin) return fail(VF_ERR_INVALID, "i3d_forward: handle was created for %d input channels", h->cin);
    return VF_OK;
}

extern "C" {

int vf_i3d_forward_f32(vf_i3d_t* h, const float* clips, int n, int T, float* out, void* stream) {
    VF_TRY(i3d_check(h, clips, n, T, out, 0));
    if (n <= 0) return VF_OK;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    for (int b0 = 0; b0 < n; b0 += h->max_stacks) {
        const int nb = (n - b0 < h->max_stacks) ? (n - b0) : h->max_stacks;
        VF_TRY(launch_i3d_phase_pack_f32(clips + size_t(b0) * h->cin * T * 224 * 224, nb, h->cin, T, h->s0, T / 2 + 3, s));
        h->launches += 1;
        VF_TRY(i3d_trunk_graphed(h, nb, T, out + size_t(b0) * 1024, s));
    }
    return leave(h, user);
}

int vf_i3d_forward_u8(vf_i3d_t* h, const uint8_t* frames, int n, int T, int Hr, int Wr, float* out, void* stream) {
    return vf_i3d_forward_u8_strided(h, frames, n, T, T, Hr, Wr, out, stream);
}

int vf_i3d_forward_u8_strided(vf_i3d_t* h, const uint8_t* frames, int n, int T, int64_t stack_stride, int Hr, int Wr,
                              float* out, void* stream) {
    VF_TRY(i3d_check(h, frames, n, T, out, 3));
    if (stack_stride < T) return fail(VF_ERR_INVALID, "i3d_forward_u8: stack stride %lld < T = %d", (long long)stack_stride, T);
    if (Hr < 224 || Wr < 224) return fail(VF_ERR_INVALID, "i3d_forward_u8: %dx%d frames are smaller than the 224 crop", Hr, Wr);
    if (n <= 0) return VF_OK;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    const int cy = (Hr - 224) / 2, cx = (Wr - 224) / 2;     // TensorCenterCrop: floor offsets (transforms.py:14-15)
    for (int b0 = 0; b0 < n; b0 += h->max_stacks) {
        const int nb = (n - b0 < h->max_stacks) ? (n - b0) : h->max_stacks;
        VF_TRY(launch_i3d_phase_pack_u8(frames + size_t(b0) * stack_stride * Hr * Wr * 3, nb, T, stack_stride, Hr, Wr, cy, cx,
                                        h->s0, T / 2 + 3, s));
        h->launches += 1;
        VF_TRY(i3d_trunk_graphed(h, nb, T, out + size_t(b0) * 1024, s));
    }
    return leave(h, user);
}

int vf_i3d_forward_flow(vf_i3d_t* h, const float* flow, int n, int T, int H, int W, float* out, void* stream) {
    VF_TRY(i3d_check(h, flow, n, T, out, 2));
    if (H < 224 || W < 224) return fail(VF_ERR_INVALID, "i3d_forward_flow: %dx%d flow is smaller than the 224 crop", H, W);
    if (n <= 0) return VF_OK;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    const int cy = (H - 224) / 2, cx = (W - 224) / 2;
    for (int b0 = 0; b0 < n; b0 += h->max_stacks) {
        const int nb = (n - b0 < h->max_stacks) ? (n - b0) : h->max_stacks;
        VF_TRY(launch_i3d_phase_pack_flow(flow + size_t(b0) * T * 2 * H * W, nb, T, H, W, cy, cx, h->s0, T / 2 + 3, s));
        h->launches += 1;
        VF_TRY(i3d_trunk_graphed(h, nb, T, out + size_t(b0) * 1024, s));
    }
    return leave(h, user);
}

int vf_i3d_read_stage(vf_i3d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream) {
    if (!h || stage < 0 || stage > 4 || !dims5) return fail(VF_ERR_INVALID, "i3d_read_stage: bad argument");
    const vf_i3d::StageRef& r = h->stages[stage];
    if (!r.p) return fail(VF_ERR_INVALID, "i3d_read_stage: no forward has run (since the last vf_i3d_debug_mixed)");
    dims5[0] = r.v.n; dims5[1] = r.C; dims5[2] = r.v.T(); dims5[3] = r.v.H(); dims5[4] = r.v.W();
    const int64_t need = int64_t(r.v.n) * r.C * r.v.T() * r.v.H() * r.v.W();
    if (!out) return VF_OK;
    if (capacity < need) return fail(VF_ERR_INVALID, "i3d_read_stage: capacity %lld < %lld", (long long)capacity, (long long)need);
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    VF_TRY(enter(h, user));
    VF_TRY(launch_unpack_ndhwc(r.p, r.v, r.C, 0, r.C, 2 * r.C, r.C, out, h->cs));      // retained stages are pair tensors
    return leave(h, user);
}

int vf_i3d_debug_mixed(vf_i3d_t* h, int block, const void* x_pairs, int n, int T, void* out_pairs, void* stream) {
    if (!h || !x_pairs || !out_pairs) return fail(VF_ERR_INVALID, "i3d_debug_mixed: null argument");
    if (block < 0 || block > 8 || n < 1 || T < 1)
        return fail(VF_ERR_INVALID, "i3d_debug_mixed: block %d, %d clips of %d frames", block, n, T);
    const int S = block < 2 ? 28 : block < 7 ? 14 : 7;
    const Vol v = bordered(n, T, S, S);
    // bufA / bufB (2048 columns), t1 (192), t2 (64) and tp (1664) hold cap_rows2 rows of any block's widest operand
    if (size_t(v.rows()) > h->cap_rows2)
        return fail(VF_ERR_INVALID, "i3d_debug_mixed: %d clips of %d frames exceed the workspace", n, T);
    const int* c = kMixed[block];
    const int cin = c[0], ctot = c[1] + c[3] + c[5] + c[6];
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    for (vf_i3d::StageRef& r : h->stages) r.p = nullptr;      // bufA / bufB no longer hold the last forward's stages
    VF_TRY(enter(h, user));
    VF_CUDA(cudaMemcpyAsync(h->bufA, x_pairs, size_t(v.rows()) * 2 * cin * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    VF_TRY(mixed_block(h, block, h->bufA, v, h->bufB, s));
    VF_CUDA(cudaMemcpyAsync(out_pairs, h->bufB, size_t(v.rows()) * 2 * ctot * sizeof(__half), cudaMemcpyDeviceToDevice, s));
    return leave(h, user);
}

int64_t vf_i3d_launch_count(const vf_i3d_t* h) { return h ? h->launches : 0; }

int vf_i3d_conv(const vf_i3d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "i3d_conv: null argument");
    if (index < 0 || index >= VF_I3D_UNITS)
        return fail(VF_ERR_INVALID, "i3d_conv: index %d outside the %d units", index, VF_I3D_UNITS);
    const ConvUnit& u = h->units[index];
    geom[0] = u.cout; geom[1] = u.ntaps; geom[2] = u.k_per_tap; geom[3] = u.nsplit;
    for (int j = 0; j < 64; ++j) {
        geom[4 + 3 * j] = geom[5 + 3 * j] = geom[6 + 3 * j] = 0;
        if (j < u.ntaps) unit_tap(u, j, &geom[4 + 3 * j], &geom[5 + 3 * j], &geom[6 + 3 * j]);
    }
    *lo_mask = u.lo_mask;
    VF_CUDA(cudaSetDevice(h->device));
    const size_t nw = size_t(u.cout) * u.nsplit * u.ntaps * u.k_per_tap;
    if (w) VF_CUDA(cudaMemcpy(w, u.w, nw * sizeof(__half), cudaMemcpyDeviceToDevice));
    if (scale) VF_CUDA(cudaMemcpy(scale, u.scale, size_t(u.cout) * sizeof(float), cudaMemcpyDeviceToDevice));
    if (bias) VF_CUDA(cudaMemcpy(bias, u.bias, size_t(u.cout) * sizeof(float), cudaMemcpyDeviceToDevice));
    return VF_OK;
}

}  // extern "C"
