// PWC-Net optical flow on the wgmma conv-GEMM.  Replaces `PWCNet()(first, second)` (reference:
// models/pwc/pwc_src/pwc_net.py:212-263 with correlation.py's CuPy cost volume; called at models/pwc/extract_pwc.py:97
// and models/i3d/extract_i3d.py:175).
//
// Layout: channels-last rows of zero-bordered 2-D volumes, every activation a split-fp16 pair [hi | lo] (RAFT's scheme,
// raft.cu): the consumer's weights are duplicated over both halves and uploaded as hi + lo passes, so every GEMM is
// emulated fp32 on the fp16 tensor cores.  Every 3x3 convolution is 9 taps of the shifted-row GEMM (dilated taps for
// the refiner); the extractor's stride-2 convs run on RAFT's phase repack.
// Decoder levels keep ONE row buffer per pair position, the dense concatenation
//     [c5 32 | c4 64 | c3 96 | c2 128 | c1 128 | vol 88 | f1 C | upflow 8 | upfeat 8]      (level 6: up to vol)
// in the reference's channel order (each new conv output is prepended, pwc_net.py:176-180), every slice holding its own
// [hi | lo] pair and widths padded to multiples of 8 with zero weight columns.  A decoder conv reads a suffix of that
// row, i.e. one contiguous column range, and writes its slice in place: no concatenation is ever copied.
// Weights: a power-of-two scale per output channel is folded into the weights before they are split, and its inverse
// into the epilogue's fp32 scale (both exact).  The checkpoint's level-6 weights (|w| <= 1e-36 .. 1e-3) would otherwise
// lose most of their bits to fp16's subnormal range.
// The extractor runs once per frame (interior frames belong to two pairs); the cost volume, warp, transposed-conv
// scatter and output upsample are fp32 CUDA-core kernels (pwc_kernels.cu).  Everything between the input pack and the
// output upsample is replayed as one CUDA graph per (frames, padded H, padded W).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <string>
#include <vector>

#include "internal.h"
#include "pwc_kernels.h"

namespace vf {

namespace {

struct PConv {              // a convolution prepared for conv_gemm_f16, weights W_hi | W_lo (nsplit = 2)
    int n_out = 0, ntaps = 0, k_per_tap = 0;
    std::vector<int> dh, dw;      // per tap: row and column shift in pixels
    unsigned long long lo_mask = 0;
    __half* w = nullptr;
    float *scale = nullptr, *bias = nullptr;
};

// host-side filter before the split: W[o][tap * k_per_tap + k] in fp32
struct HostConv {
    int n_out = 0, ntaps = 0, kpt = 0;
    std::vector<int> dh, dw;
    std::vector<float> W, bias;
    std::vector<char> hi;       // K columns that multiply a hi half
    void init(int n, int t, int k) {
        n_out = n; ntaps = t; kpt = k;
        W.assign(size_t(n) * t * k, 0.f);
        bias.assign(size_t(n), 0.f);
        hi.assign(size_t(t) * k, 0);
        dh.assign(size_t(t), 0);
        dw.assign(size_t(t), 0);
    }
    // weight w at the hi column khi and the lo column klo of tap `tap`
    void put(int o, int tap, int khi, int klo, float w) {
        const size_t base = (size_t(o) * ntaps + tap) * kpt;
        W[base + khi] = w;
        W[base + klo] = w;
        hi[size_t(tap) * kpt + khi] = 1;
    }
};

const int kFeatC[7] = {3, 16, 32, 64, 96, 128, 196};   // extractor channels per level (0: the image)
const char* const kLevelName[7] = {"", "One", "Two", "Thr", "Fou", "Fiv", "Six"};
const float kDbl[7] = {0.f, 0.f, 5.0f, 2.5f, 1.25f, 0.625f, 0.f};  // dblBackward of the decoder at each level
constexpr int kVolW = 88;          // 81 cost-volume channels padded
constexpr int kRefBorder = 16;     // the refiner's largest dilation

inline int r8(int c) { return (c + 7) / 8 * 8; }

// slices of a level's decoder row: 0..4 = c5..c1, 5 = vol, 6 = f1, 7 = upflow, 8 = upfeat
struct Layout {
    int n = 0, width[9] = {}, real[9] = {}, off[9] = {}, total = 0;
};
Layout layout(int l) {
    Layout L;
    const int w[9] = {32, 64, 96, 128, 128, kVolW, r8(kFeatC[l]), 8, 8};
    const int r[9] = {32, 64, 96, 128, 128, 81, kFeatC[l], 2, 2};
    L.n = l < 6 ? 9 : 6;
    for (int j = 0; j < L.n; ++j) {
        L.width[j] = w[j]; L.real[j] = r[j]; L.off[j] = L.total;
        L.total += 2 * w[j];
    }
    return L;
}
// reference channel c of the suffix that starts at slice s0 -> its hi and lo columns relative to the suffix start
void suffix_col(const Layout& L, int s0, int c, int* khi, int* klo) {
    for (int j = s0; j < L.n; ++j) {
        if (c < L.real[j]) {
            *khi = L.off[j] - L.off[s0] + c;
            *klo = *khi + L.width[j];
            return;
        }
        c -= L.real[j];
    }
    *khi = *klo = -1;
}
int suffix_channels(const Layout& L, int s0) {
    int c = 0;
    for (int j = s0; j < L.n; ++j) c += L.real[j];
    return c;
}

Vol2 feat_vol(int l, int n, int Hp, int Wp) {
    const int h = Hp >> l, w = Wp >> l;
    return Vol2{n, h + 2, w + 2, 1, 1 + h, 1, 1 + w};
}
Vol2 cat_vol(int l, int n, int Hp, int Wp) {
    const int h = Hp >> l, w = Wp >> l, B = l == 2 ? kRefBorder : 1;
    return Vol2{n, h + 2 * B, w + 2 * B, B, B + h, B, B + w};
}

}  // namespace

}  // namespace vf

using namespace vf;

struct vf_pwc : vf::EngineCore {
    int max_frames = 0, max_hp = 0, max_wp = 0;
    PConv ext[7][3];                  // extractor level 1..6, convs .0 .2 .4
    PConv upflow[7], upfeat[7];       // decoder levels 2..5
    PConv dec[7][6];                  // decoder levels 2..6, moduleOne .. moduleSix
    PConv ref[7];                     // refiner
    __half *in0 = nullptr, *ph = nullptr, *tA = nullptr, *tB = nullptr, *rA = nullptr, *rB = nullptr;
    __half *feat[7] = {}, *cat[7] = {}, *flow[7] = {};
    float *upA = nullptr, *upB = nullptr, *f2w = nullptr, *refine = nullptr, *mask[7] = {};
    int last_F = 0, last_hp = 0, last_wp = 0;     // geometry of the last call (debug reads)
};

namespace vf {

namespace {

struct TensorTable {
    const vf_named_tensor* t; int n;
    const float* get(const std::string& name, int64_t numel) const {
        for (int i = 0; i < n; ++i)
            if (name == t[i].name) return t[i].numel == numel ? t[i].data : nullptr;
        return nullptr;
    }
};

// Split and upload.  Output channel o is scaled by 2^e(o) before the split, e(o) putting its largest |w| in
// [2^14, 2^15) (at most 2^126, so that the epilogue's scale 2^-e stays a normal fp32), and the epilogue multiplies by
// 2^-e(o) before adding the unscaled bias.
int upload(vf_pwc* h, PConv& cw, const HostConv& hc) {
    const size_t Ktot = size_t(hc.ntaps) * hc.kpt;
    std::vector<__half> B(size_t(hc.n_out) * 2 * Ktot, __float2half_rn(0.f));
    std::vector<float> sc(size_t(hc.n_out)), bi(hc.bias);
    for (int o = 0; o < hc.n_out; ++o) {
        const float* row = hc.W.data() + size_t(o) * Ktot;
        float m = 0.f;
        for (size_t k = 0; k < Ktot; ++k) m = fmaxf(m, fabsf(row[k]));
        int e = 0;
        if (m > 0.f) {
            int ex = 0;
            frexpf(m, &ex);
            e = 15 - ex;
            if (e > 126) e = 126;
        }
        sc[o] = ldexpf(1.f, -e);
        for (size_t k = 0; k < Ktot; ++k) {
            if (row[k] == 0.f) continue;
            const float wf = float(ldexp(double(row[k]), e));
            const __half wv = __float2half_rn(wf);
            B[size_t(o) * 2 * Ktot + k] = wv;
            B[size_t(o) * 2 * Ktot + Ktot + k] = __float2half_rn(wf - __half2float(wv));
        }
    }
    cw.n_out = hc.n_out; cw.ntaps = hc.ntaps; cw.k_per_tap = hc.kpt; cw.dh = hc.dh; cw.dw = hc.dw;
    // a K block none of whose columns meets a hi half needs only the W_hi pass
    cw.lo_mask = 0;
    const int blocks = (hc.kpt + 63) / 64;
    if (blocks <= 64) {
        unsigned long long m = ~0ull;
        for (int t = 0; t < hc.ntaps; ++t)
            for (int kk = 0; kk < blocks; ++kk)
                for (int j = kk * 64; j < (kk + 1) * 64 && j < hc.kpt; ++j)
                    if (hc.hi[size_t(t) * hc.kpt + j]) m &= ~(1ull << kk);
        cw.lo_mask = blocks == 64 ? m : (m & ((1ull << blocks) - 1));
    }
    VF_TRY(ralloc(h, &cw.w, B.size()));
    VF_TRY(ralloc(h, &cw.scale, size_t(hc.n_out)));
    VF_TRY(ralloc(h, &cw.bias, size_t(hc.n_out)));
    VF_CUDA(cudaMemcpy(cw.w, B.data(), B.size() * sizeof(__half), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.scale, sc.data(), sc.size() * sizeof(float), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.bias, bi.data(), bi.size() * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

int get_conv(const TensorTable& T, const std::string& name, int co, int ci, int k, const float** w, const float** b) {
    *w = T.get(name + ".weight", int64_t(co) * ci * k * k);
    *b = T.get(name + ".bias", co);
    if (!*w || !*b) return fail(VF_ERR_INVALID, "pwc_create: missing or mis-shaped tensor '%s'", name.c_str());
    return VF_OK;
}

// 3x3 conv (dilation dil, padding dil) as 9 taps of k_per_tap columns; chan(c) gives input channel c's hi / lo columns
int prep_conv3(vf_pwc* h, PConv& cw, const TensorTable& T, const std::string& name, int co, int ci, int n_out, int kpt,
               int dil, const std::function<void(int, int*, int*)>& chan) {
    const float *w, *b;
    VF_TRY(get_conv(T, name, co, ci, 3, &w, &b));
    HostConv hc;
    hc.init(n_out, 9, kpt);
    for (int t = 0; t < 9; ++t) { hc.dh[t] = (t / 3 - 1) * dil; hc.dw[t] = (t % 3 - 1) * dil; }
    for (int c = 0; c < ci; ++c) {
        int khi, klo;
        chan(c, &khi, &klo);
        if (khi < 0 || klo < 0 || khi >= kpt || klo >= kpt) return fail(VF_ERR_INVALID, "pwc_create: column out of range in '%s'", name.c_str());
        for (int o = 0; o < co; ++o)
            for (int t = 0; t < 9; ++t) hc.put(o, t, khi, klo, w[((size_t(o) * ci + c) * 3 + t / 3) * 3 + t % 3]);
    }
    for (int o = 0; o < co; ++o) hc.bias[o] = b[o];
    return upload(h, cw, hc);
}

// stride-2 3x3 conv (padding 1) on the phase repack of a [hi C8 | lo C8] row: phase (ph, pw) at (ph*2+pw)*2*C8, two taps
// (raft.cu prep_stride2_conv with k = 3)
int prep_stride2(vf_pwc* h, PConv& cw, const TensorTable& T, const std::string& name, int co, int ci, int ci8, int n_out) {
    const float *w, *b;
    VF_TRY(get_conv(T, name, co, ci, 3, &w, &b));
    const int pitch = 8 * ci8, kpt = 2 * pitch;
    HostConv hc;
    hc.init(n_out, 2, kpt);
    for (int a = 0; a < 2; ++a) { hc.dh[a] = a - 1; hc.dw[a] = -1; }
    for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
            const int a = (kh + 1) / 2, ph = (kh + 1) % 2, bq = (kw + 1) / 2, pw = (kw + 1) % 2;
            for (int c = 0; c < ci; ++c) {
                const int k = bq * pitch + (ph * 2 + pw) * 2 * ci8 + c;
                for (int o = 0; o < co; ++o) hc.put(o, a, k, k + ci8, w[((size_t(o) * ci + c) * 3 + kh) * 3 + kw]);
            }
        }
    for (int o = 0; o < co; ++o) hc.bias[o] = b[o];
    return upload(h, cw, hc);
}

// ConvTranspose2d(ci, 2, 4, stride 2, padding 1) as one GEMM over the 3x3 input neighbourhood: column (py*2+px)*2 + oc
// is output phase (py, px) of channel oc, i.e. fine pixel (2m+py, 2n+px) from coarse pixels (m+di, n+dj), kernel tap
// (py+1-2di, px+1-2dj) where it lies in 0..3 (zero weights elsewhere).  Weight layout [ci][2][4][4].
int prep_deconv(vf_pwc* h, PConv& cw, const TensorTable& T, const std::string& name, int ci, int kpt,
                const std::function<void(int, int*, int*)>& chan) {
    const float* w = T.get(name + ".weight", int64_t(ci) * 2 * 16);
    const float* b = T.get(name + ".bias", 2);
    if (!w || !b) return fail(VF_ERR_INVALID, "pwc_create: missing or mis-shaped tensor '%s'", name.c_str());
    HostConv hc;
    hc.init(8, 9, kpt);
    for (int t = 0; t < 9; ++t) { hc.dh[t] = t / 3 - 1; hc.dw[t] = t % 3 - 1; }
    for (int c = 0; c < ci; ++c) {
        int khi, klo;
        chan(c, &khi, &klo);
        if (khi < 0 || klo < 0 || khi >= kpt || klo >= kpt) return fail(VF_ERR_INVALID, "pwc_create: column out of range in '%s'", name.c_str());
        for (int t = 0; t < 9; ++t) {
            const int di = t / 3 - 1, dj = t % 3 - 1;
            for (int py = 0; py < 2; ++py)
                for (int px = 0; px < 2; ++px) {
                    const int ky = py + 1 - 2 * di, kx = px + 1 - 2 * dj;
                    if (ky < 0 || ky > 3 || kx < 0 || kx > 3) continue;
                    for (int oc = 0; oc < 2; ++oc)
                        hc.put((py * 2 + px) * 2 + oc, t, khi, klo, w[((size_t(c) * 2 + oc) * 4 + ky) * 4 + kx]);
                }
        }
    }
    for (int n = 0; n < 8; ++n) hc.bias[n] = b[n % 2];
    return upload(h, cw, hc);
}

// out_f32: fp32 output; otherwise a split pair with the lo half split_off columns to the right
int run_conv(vf_pwc* h, const PConv& cw, const __half* X, int pitch, const Vol2& v, void* out, int ldo, bool out_f32,
             int act, int split_off, cudaStream_t s) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = cw.ntaps; g.k_per_tap = cw.k_per_tap; g.nsplit = 2; g.lo_mask = cw.lo_mask;
    for (int j = 0; j < cw.ntaps; ++j) g.tap_off[j] = cw.dh[j] * v.Wp + cw.dw[j];
    g.mask = 1; g.row0 = 0;
    g.Tp = 1; g.Hp = v.Hp; g.Wp = v.Wp; g.t0 = 0; g.t1 = 1; g.h0 = v.h0; g.h1 = v.h1; g.w0 = v.w0; g.w1 = v.w1;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.ldo = ldo; ep.out_f32 = out_f32 ? 1 : 0; ep.bias = cw.bias; ep.scale = cw.scale; ep.act = act;
    ep.split_off = out_f32 ? 0 : split_off;
    h->launches += 1;
    return conv_gemm_f16(X, pitch, v.rows(), cw.w, cw.n_out, g, ep, s);
}

// every conv in vf_pwc_conv's order
std::vector<const PConv*> conv_list(const vf_pwc* h) {
    std::vector<const PConv*> cs;
    for (int l = 1; l <= 6; ++l)
        for (int k = 0; k < 3; ++k) cs.push_back(&h->ext[l][k]);
    for (int l = 6; l >= 2; --l) {
        if (l < 6) { cs.push_back(&h->upflow[l]); cs.push_back(&h->upfeat[l]); }
        for (int k = 0; k < 6; ++k) cs.push_back(&h->dec[l][k]);
    }
    for (int k = 0; k < 7; ++k) cs.push_back(&h->ref[k]);
    return cs;
}

int prep_all(vf_pwc* h, const TensorTable& T) {
    // extractor
    for (int l = 1; l <= 6; ++l) {
        const std::string p = std::string("moduleExtractor.module") + kLevelName[l] + ".";
        const int ci = kFeatC[l - 1], ci8 = l == 1 ? 8 : r8(ci), co = kFeatC[l], co8 = r8(co);
        VF_TRY(prep_stride2(h, h->ext[l][0], T, p + "0", co, ci, ci8, co8));
        auto same = [=](int c, int* khi, int* klo) { *khi = c; *klo = co8 + c; };
        VF_TRY(prep_conv3(h, h->ext[l][1], T, p + "2", co, co, co8, 2 * co8, 1, same));
        VF_TRY(prep_conv3(h, h->ext[l][2], T, p + "4", co, co, co8, 2 * co8, 1, same));
    }
    // decoders
    for (int l = 6; l >= 2; --l) {
        const std::string p = std::string("module") + kLevelName[l] + ".";
        const Layout L = layout(l);
        if (l < 6) {
            const Layout Lc = layout(l + 1);
            VF_TRY(prep_deconv(h, h->upflow[l], T, p + "moduleUpflow", 2, 16,
                               [](int c, int* khi, int* klo) { *khi = c; *klo = 8 + c; }));
            VF_TRY(prep_deconv(h, h->upfeat[l], T, p + "moduleUpfeat", suffix_channels(Lc, 0), Lc.total,
                               [=](int c, int* khi, int* klo) { suffix_col(Lc, 0, c, khi, klo); }));
        }
        for (int k = 0; k < 6; ++k) {
            const int s0 = 5 - k;                       // moduleOne reads from the volume on, moduleSix the whole row
            const int co = k < 5 ? L.real[4 - k] : 2, n_out = k < 5 ? L.width[4 - k] : 8;
            VF_TRY(prep_conv3(h, h->dec[l][k], T, p + "module" + kLevelName[k + 1] + ".0", co, suffix_channels(L, s0),
                              n_out, L.total - L.off[s0], 1,
                              [=](int c, int* khi, int* klo) { suffix_col(L, s0, c, khi, klo); }));
        }
    }
    // refiner (pwc_net.py:189-210) on the level-2 row
    {
        const Layout L = layout(2);
        const int dil[7] = {1, 2, 4, 8, 16, 1, 1}, ch[8] = {0, 128, 128, 128, 96, 64, 32, 2};
        for (int k = 0; k < 7; ++k) {
            const std::string name = "moduleRefiner.moduleMain." + std::to_string(2 * k);
            const int co = ch[k + 1], n_out = r8(co);
            if (k == 0) {
                VF_TRY(prep_conv3(h, h->ref[0], T, name, co, suffix_channels(L, 0), n_out, L.total, 1,
                                  [=](int c, int* khi, int* klo) { suffix_col(L, 0, c, khi, klo); }));
            } else {
                const int ci = ch[k];
                VF_TRY(prep_conv3(h, h->ref[k], T, name, co, ci, n_out, 2 * ci, dil[k],
                                  [=](int c, int* khi, int* klo) { *khi = c; *klo = ci + c; }));
            }
        }
    }
    return VF_OK;
}

// extractor -> decoders 6..2 -> refiner on the input volume already in h->in0
int pwc_core(vf_pwc* h, int F, int Hp, int Wp, cudaStream_t s) {
    const int NP = F - 1;
    const __half* prev = h->in0;
    Vol2 vprev{F, Hp + 2, Wp + 2, 1, 1 + Hp, 1, 1 + Wp};
    int prev8 = 8;
    for (int l = 1; l <= 6; ++l) {
        const Vol2 v = feat_vol(l, F, Hp, Wp);
        const int c8 = r8(kFeatC[l]);
        VF_TRY(raft_phase_repack(prev, vprev, 2 * prev8, h->ph, v, s));
        h->launches += 1;
        VF_TRY(run_conv(h, h->ext[l][0], h->ph, 8 * prev8, v, h->tA, 2 * c8, false, VF_ACT_LEAKY, c8, s));
        VF_TRY(run_conv(h, h->ext[l][1], h->tA, 2 * c8, v, h->tB, 2 * c8, false, VF_ACT_LEAKY, c8, s));
        VF_TRY(run_conv(h, h->ext[l][2], h->tB, 2 * c8, v, h->feat[l], 2 * c8, false, VF_ACT_LEAKY, c8, s));
        prev = h->feat[l]; vprev = v; prev8 = c8;
    }
    for (int l = 6; l >= 2; --l) {
        const Layout L = layout(l);
        const Vol2 vc = cat_vol(l, NP, Hp, Wp), vf = feat_vol(l, F, Hp, Wp);
        const int C = kFeatC[l], C8 = r8(C), ldc = L.total;
        VF_CUDA(cudaMemsetAsync(h->cat[l], 0, size_t(vc.rows()) * ldc * sizeof(__half), s));
        if (l < 6) {
            const Layout Lc = layout(l + 1);
            const Vol2 vu = cat_vol(l + 1, NP, Hp, Wp);
            VF_TRY(run_conv(h, h->upflow[l], h->flow[l + 1], 16, vu, h->upA, 8, true, VF_ACT_NONE, 0, s));
            VF_TRY(run_conv(h, h->upfeat[l], h->cat[l + 1], Lc.total, vu, h->upB, 8, true, VF_ACT_NONE, 0, s));
            VF_TRY(pwc_up_scatter(h->upA, vu, h->cat[l], vc, ldc, L.off[7], s));
            VF_TRY(pwc_up_scatter(h->upB, vu, h->cat[l], vc, ldc, L.off[8], s));
            h->launches += 2;
        }
        const int h_l = Hp >> l, w_l = Wp >> l;
        VF_CUDA(cudaMemsetAsync(h->f2w, 0, size_t(NP) * (h_l + 8) * (w_l + 8) * C * sizeof(float), s));
        VF_TRY(pwc_warp(h->feat[l], vf, 2 * C8, C, C8, h->cat[l], vc, ldc, l < 6 ? L.off[7] : -1, kDbl[l], NP, h->f2w,
                        l < 6 ? h->mask[l] : nullptr, s));
        VF_TRY(pwc_correlation(h->feat[l], vf, 2 * C8, C, C8, h->f2w, h->cat[l], vc, ldc, L.off[5], l < 6 ? L.off[6] : -1,
                               NP, s));
        h->launches += 2;
        for (int k = 0; k < 5; ++k)
            VF_TRY(run_conv(h, h->dec[l][k], h->cat[l] + L.off[5 - k], ldc, vc, h->cat[l] + L.off[4 - k], ldc, false,
                            VF_ACT_LEAKY, L.width[4 - k], s));
        VF_TRY(run_conv(h, h->dec[l][5], h->cat[l], ldc, vc, h->flow[l], 16, false, VF_ACT_NONE, 8, s));
    }
    // refiner: the level-2 row -> 128, 128, 128, 96, 64, 32 channels in rA / rB ([hi C | lo C], pitch 256) -> fp32 flow
    const Vol2 v2 = cat_vol(2, NP, Hp, Wp);
    const int ch[8] = {0, 128, 128, 128, 96, 64, 32, 2};
    const __half* x = h->cat[2];
    int pitch = layout(2).total;
    for (int k = 0; k < 6; ++k) {
        __half* y = (k % 2 == 0) ? h->rA : h->rB;
        VF_TRY(run_conv(h, h->ref[k], x, pitch, v2, y, 256, false, VF_ACT_LEAKY, ch[k + 1], s));
        x = y; pitch = 256;
    }
    VF_TRY(run_conv(h, h->ref[6], x, 256, v2, h->refine, 8, true, VF_ACT_NONE, 0, s));
    return VF_OK;
}

}  // namespace

}  // namespace vf

extern "C" {

int vf_pwc_create(vf_pwc_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames, int max_h,
                  int max_w) {
    if (!out || !tensors || n_tensors <= 0) return fail(VF_ERR_INVALID, "pwc_create: null argument");
    *out = nullptr;
    if (max_frames < 2) max_frames = 2;
    if (max_h <= 0 || max_w <= 0) return fail(VF_ERR_INVALID, "pwc_create: max frame size required");
    VF_TRY(check_device(device));
    vf_pwc* h = new vf_pwc();
    h->who = "pwc_create";
    h->device = device; h->max_frames = max_frames;
    h->max_hp = (max_h + 63) / 64 * 64; h->max_wp = (max_w + 63) / 64 * 64;
    const TensorTable T{tensors, n_tensors};
    auto body = [&]() -> int {
        VF_TRY(prep_all(h, T));
        const size_t F = size_t(max_frames), NP = F - 1;
        const int Hp = h->max_hp, Wp = h->max_wp;
        VF_TRY(ralloc(h, &h->in0, F * (Hp + 2) * (Wp + 2) * 16));
        size_t ph = 0, tmp = 0, up = 0, f2w = 0;
        for (int l = 1; l <= 6; ++l) {
            const size_t rows = size_t(feat_vol(l, int(F), Hp, Wp).rows());
            const int c8 = r8(kFeatC[l]), p8 = l == 1 ? 8 : r8(kFeatC[l - 1]);
            ph = std::max(ph, rows * 8 * p8);
            tmp = std::max(tmp, rows * 2 * c8);
            VF_TRY(ralloc(h, &h->feat[l], rows * 2 * c8));
            if (l >= 2) {
                const size_t crows = size_t(cat_vol(l, int(NP), Hp, Wp).rows());
                VF_TRY(ralloc(h, &h->cat[l], crows * layout(l).total));
                VF_TRY(ralloc(h, &h->flow[l], crows * 16));
                if (l >= 3) up = std::max(up, crows * 8);
                if (l < 6) VF_TRY(ralloc(h, &h->mask[l], NP * size_t(Hp >> l) * (Wp >> l)));
                f2w = std::max(f2w, NP * size_t((Hp >> l) + 8) * ((Wp >> l) + 8) * kFeatC[l]);
            }
        }
        VF_TRY(ralloc(h, &h->ph, ph));
        VF_TRY(ralloc(h, &h->tA, tmp)); VF_TRY(ralloc(h, &h->tB, tmp));
        VF_TRY(ralloc(h, &h->upA, up)); VF_TRY(ralloc(h, &h->upB, up));
        VF_TRY(ralloc(h, &h->f2w, f2w));
        const size_t rows2 = size_t(cat_vol(2, int(NP), Hp, Wp).rows());
        VF_TRY(ralloc(h, &h->rA, rows2 * 256)); VF_TRY(ralloc(h, &h->rB, rows2 * 256));
        VF_TRY(ralloc(h, &h->refine, rows2 * 8));
        return open_stream(h);
    };
    const int st = body();
    if (st != VF_OK) { vf_pwc_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_pwc_destroy(vf_pwc_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_pwc_flow(vf_pwc_t* h, const void* frames, int is_u8, int chw_layout, int n_frames, int Hs, int Ws, float* out,
                void* stream) {
    if (!h || !frames || !out) return fail(VF_ERR_INVALID, "pwc_flow: null argument");
    if (n_frames < 2 || n_frames > h->max_frames)
        return fail(VF_ERR_INVALID, "pwc_flow: %d frames outside [2, %d]", n_frames, h->max_frames);
    if (Hs <= 0 || Ws <= 0) return fail(VF_ERR_INVALID, "pwc_flow: empty frame");
    const int Hp = (Hs + 63) / 64 * 64, Wp = (Ws + 63) / 64 * 64;        // pwc_net.py:241-242
    if (Hp > h->max_hp || Wp > h->max_wp)
        return fail(VF_ERR_INVALID, "pwc_flow: frame %dx%d outside the workspace (%dx%d)", Hs, Ws, h->max_hp, h->max_wp);
    const int F = n_frames, NP = F - 1;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_TRY(enter(h, user));
    VF_TRY(pwc_input_pack(frames, is_u8, chw_layout, F, Hs, Ws, h->in0, Vol2{F, Hp + 2, Wp + 2, 1, 1 + Hp, 1, 1 + Wp}, s));
    h->launches += 1;
    VF_TRY(run_graphed(h, {F, Hp, Wp, 0}, [&] { return pwc_core(h, F, Hp, Wp, s); }));
    h->last_F = F; h->last_hp = Hp; h->last_wp = Wp;
    VF_TRY(pwc_output(h->flow[2], h->refine, cat_vol(2, NP, Hp, Wp), NP, Hs, Ws, Hp, Wp, out, s));
    h->launches += 1;
    return leave(h, user);
}

int vf_pwc_debug_read(vf_pwc_t* h, int what, int level, float* out, int64_t capacity, int* dims4, void* stream) {
    if (!h || !dims4 || h->last_F <= 0) return fail(VF_ERR_INVALID, "pwc_debug_read: no forward has run");
    if (level < 1 || level > 6 || (what >= 1 && what != 5 && level < 2) || ((what == 2 || what == 3 || what == 6) && level > 5))
        return fail(VF_ERR_INVALID, "pwc_debug_read: tensor %d has no level %d", what, level);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    VF_CUDA(cudaStreamSynchronize(h->cs));     // diagnostics only: the engine stream has finished the last call
    const int F = h->last_F, NP = F - 1, Hp = h->last_hp, Wp = h->last_wp;
    const int l = what == 5 ? 2 : level, hl = Hp >> l, wl = Wp >> l;
    const int C = kFeatC[l], C8 = r8(C);
    dims4[0] = what == 0 ? F : NP; dims4[2] = hl; dims4[3] = wl;
    if (what == 0) dims4[1] = C;
    else if (what == 1) dims4[1] = 81;
    else if (what == 6) dims4[1] = 1;
    else if (what >= 2 && what <= 5) dims4[1] = 2;
    else return fail(VF_ERR_INVALID, "pwc_debug_read: unknown tensor id %d", what);
    const int64_t need = int64_t(dims4[0]) * dims4[1] * dims4[2] * dims4[3];
    if (!out) return VF_OK;
    if (capacity < need) return fail(VF_ERR_INVALID, "pwc_debug_read: capacity too small");
    const Layout L = layout(l);
    const Vol2 vc = cat_vol(l, NP, Hp, Wp);
    switch (what) {
        case 0: return raft_unpack2d(h->feat[l], feat_vol(l, F, Hp, Wp), 2 * C8, 0, C, C8, out, s);
        case 1: return raft_unpack2d(h->cat[l], vc, L.total, L.off[5], 81, kVolW, out, s);
        case 2: return raft_unpack2d(h->cat[l], vc, L.total, L.off[7], 2, 8, out, s);
        case 3: return raft_unpack2d(h->cat[l], vc, L.total, L.off[8], 2, 8, out, s);
        case 4: return raft_unpack2d(h->flow[l], vc, 16, 0, 2, 8, out, s);
        case 5: return raft_unpack2d_f32(h->refine, vc, 8, 0, 2, out, s);
        default:
            VF_CUDA(cudaMemcpyAsync(out, h->mask[l], size_t(need) * sizeof(float), cudaMemcpyDeviceToDevice, s));
            return VF_OK;
    }
}

int64_t vf_pwc_launch_count(const vf_pwc_t* h) { return h ? h->launches : 0; }

int vf_pwc_conv(const vf_pwc_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "pwc_conv: null argument");
    const std::vector<const PConv*> cs = conv_list(h);
    if (index < 0 || index >= int(cs.size()))
        return fail(VF_ERR_INVALID, "pwc_conv: index %d outside the %d convs", index, int(cs.size()));
    const PConv& c = *cs[index];
    geom[0] = c.n_out; geom[1] = c.ntaps; geom[2] = c.k_per_tap; geom[3] = 2;
    for (int j = 0; j < 64; ++j) {
        geom[4 + 3 * j] = 0;
        geom[5 + 3 * j] = j < c.ntaps ? c.dh[j] : 0;
        geom[6 + 3 * j] = j < c.ntaps ? c.dw[j] : 0;
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
