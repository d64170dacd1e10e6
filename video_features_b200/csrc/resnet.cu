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
#include <map>
#include <string>
#include <vector>

#include "internal.h"
#include "resnet_kernels.h"

namespace vf {

struct ResConv {
    int n_out = 0, ntaps = 0, k_per_tap = 0;
    int dh[4] = {0, 0, 0, 0}, dw[4] = {0, 0, 0, 0};   // per tap: shift in volume rows / columns
    unsigned long long lo_mask = 0;
    __half* w = nullptr;       // [n_out][2 * ntaps * k_per_tap]: hi pass | lo pass
    float *scale = nullptr, *bias = nullptr;
};

struct ResBlock {
    int cin = 0, width = 0, cout = 0, stride = 1;
    bool down = false;
    ResConv c1, c2, c3, dn;
};

}  // namespace vf

using namespace vf;

struct vf_resnet {
    int device = 0, depth = 0, max_frames = 0, out_dim = 0;
    bool bottleneck = false;
    int nblocks[4] = {0, 0, 0, 0}, cout[4] = {0, 0, 0, 0};
    std::vector<void*> allocs;
    ResConv stem;
    std::vector<ResBlock> blocks;
    // workspace: s0 = stem phase volume; stage outputs are kept for vf_resnet_read_stage
    __half *s0 = nullptr, *stem_out = nullptr, *pool_out = nullptr, *stage_out[4] = {nullptr, nullptr, nullptr, nullptr};
    __half *bufA = nullptr, *bufB = nullptr, *t1 = nullptr, *t2 = nullptr, *ds = nullptr, *ph1 = nullptr, *ph2 = nullptr;
    int64_t launches = 0;
    cudaStream_t cs = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    bool use_graph = true;
    std::map<int, std::pair<cudaGraphExec_t, int64_t>> graphs;     // frames -> (trunk graph, launches in it)
    int last_n = 0;
};

namespace vf {

static const int kStemQ = 115;                                  // stem phase / output volume side (112 + 3)
static const int kSide[4] = {56, 28, 14, 7};

static Vol2 stem_vol(int n) { return Vol2{n, kStemQ, kStemQ, 2, 114, 2, 114}; }
static Vol2 stage_vol(int n, int L) { return Vol2{n, kSide[L] + 2, kSide[L] + 2, 1, kSide[L] + 1, 1, kSide[L] + 1}; }

template <typename Tp>
static int ralloc(vf_resnet* h, Tp** p, size_t count) {
    // + 64 KB: the overlapping-row TMA view of a conv input extends up to (k_per_tap - C) elements past its last row;
    // zero-filled so that those elements are finite (they only feed masked border rows)
    void* q = nullptr;
    const size_t bytes = count * sizeof(Tp) + 65536;
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString(e));
    h->allocs.push_back(q);
    VF_CUDA(cudaMemset(q, 0, bytes));
    *p = static_cast<Tp*>(q);
    return VF_OK;
}

// torchvision state_dict lookup by key, with or without the "module." prefix of a DataParallel checkpoint
struct ResTensors {
    const vf_named_tensor* t; int n;
    int get(const std::string& name, int64_t numel, const float** out) const {
        for (int i = 0; i < n; ++i) {
            const char* k = t[i].name;
            if (!k || !(name == k || (strncmp(k, "module.", 7) == 0 && name == k + 7))) continue;
            if (!t[i].data || t[i].numel != numel)
                return fail(VF_ERR_INVALID, "resnet_create: tensor '%s' has %lld elements, expected %lld", name.c_str(),
                            (long long)t[i].numel, (long long)numel);
            *out = t[i].data;
            return VF_OK;
        }
        return fail(VF_ERR_INVALID, "resnet_create: missing tensor '%s'", name.c_str());
    }
};

// eval BatchNorm (eps 1e-5) as y = x * scale + shift, folded in double
static int bn_fold(const ResTensors& T, const std::string& p, int c, std::vector<float>& sc, std::vector<float>& sh) {
    const float *g, *b, *m, *v;
    VF_TRY(T.get(p + ".weight", c, &g)); VF_TRY(T.get(p + ".bias", c, &b));
    VF_TRY(T.get(p + ".running_mean", c, &m)); VF_TRY(T.get(p + ".running_var", c, &v));
    sc.resize(c); sh.resize(c);
    for (int i = 0; i < c; ++i) {
        const double s = double(g[i]) / sqrt(double(v[i]) + 1e-5);
        sc[i] = float(s);
        sh[i] = float(double(b[i]) - double(m[i]) * s);
    }
    return VF_OK;
}

// Uploads conv `name` (weight [co][ci][k][k], no bias) followed by BatchNorm `bn` as a hi + lo weight pair.
// col(kh, kw, c) -> K column of the activation's hi half; its lo half sits lo_off columns further and gets the same
// weight.  cw.ntaps / k_per_tap / dh / dw must be set.
static int upload_conv(vf_resnet* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                       int co, int ci, int k, int lo_off, const std::function<int(int, int, int)>& col) {
    const float* w;
    VF_TRY(T.get(name + ".weight", int64_t(co) * ci * k * k, &w));
    std::vector<float> sc, sh;
    VF_TRY(bn_fold(T, bn, co, sc, sh));
    const int Ktot = cw.ntaps * cw.k_per_tap;
    const size_t Kall = size_t(2) * Ktot;
    std::vector<__half> B(size_t(co) * Kall, __float2half_rn(0.f));
    std::vector<char> has_hi(size_t(Ktot), 0);
    for (int o = 0; o < co; ++o)
        for (int c = 0; c < ci; ++c)
            for (int a = 0; a < k; ++a)
                for (int d = 0; d < k; ++d) {
                    const int kc = col(a, d, c);
                    if (kc < 0 || kc + lo_off >= Ktot) return fail(VF_ERR_INVALID, "resnet_create: filter column out of range");
                    const float wf = w[((size_t(o) * ci + c) * k + a) * k + d];
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
        unsigned long long m = ~0ull;
        for (int t = 0; t < cw.ntaps; ++t)
            for (int kk = 0; kk < kpt_blocks; ++kk)
                for (int j = kk * 64; j < (kk + 1) * 64 && j < cw.k_per_tap; ++j)
                    if (has_hi[size_t(t) * cw.k_per_tap + j]) { m &= ~(1ull << kk); break; }
        cw.lo_mask = kpt_blocks == 64 ? m : (m & ((1ull << kpt_blocks) - 1));
    }
    VF_TRY(ralloc(h, &cw.w, B.size()));
    VF_TRY(ralloc(h, &cw.scale, size_t(co)));
    VF_TRY(ralloc(h, &cw.bias, size_t(co)));
    VF_CUDA(cudaMemcpy(cw.w, B.data(), B.size() * sizeof(__half), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.scale, sc.data(), co * sizeof(float), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.bias, sh.data(), co * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

// stride-1 k x k (k = 1 or 3, pad k/2) on split rows of 2*ci: one tap per kernel row of k * 2ci contiguous elements.
// Also the stride-2 1x1 downsample: one tap reading phase (0, 0) = the first 2*ci elements of a phase row.
static int prep_same(vf_resnet* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                     int co, int ci, int k) {
    cw.ntaps = k; cw.k_per_tap = k * 2 * ci;
    for (int a = 0; a < k; ++a) { cw.dh[a] = a - k / 2; cw.dw[a] = -(k / 2); }
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, name, bn, co, ci, k, ci, [=](int a, int d, int c) { return a * kpt + d * 2 * ci + c; });
}

// stride-2 3x3 (pad 1) on the phase repack of split rows of 2*ci: phase row q holds x[2(q-1)+p]; tap (a, b) reads
// phase row (q + a - 1, q' + b - 1), filter index kh = 2a + ph - 1 (likewise kw with b, pw).
static int prep_stride2(vf_resnet* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                        int co, int ci) {
    cw.ntaps = 4; cw.k_per_tap = 8 * ci;
    for (int t = 0; t < 4; ++t) { cw.dh[t] = t / 2 - 1; cw.dw[t] = t % 2 - 1; }
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, name, bn, co, ci, 3, ci, [=](int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return (a * 2 + b) * kpt + (ph * 2 + pw) * 2 * ci + c;
    });
}

// stem 7x7/2 pad 3 on the phase volume of the transform (rows [16 hi | 16 lo], 4 channels per phase, 3 used):
// phase row q holds x[2(q-2)+p]; 4 taps (kernel row pairs), each a run of 4 phase positions x 32 elements.
static int prep_stem(vf_resnet* h, ResConv& cw, const ResTensors& T) {
    cw.ntaps = 4; cw.k_per_tap = 128;
    for (int a = 0; a < 4; ++a) { cw.dh[a] = a - 2; cw.dw[a] = -2; }
    return upload_conv(h, cw, T, "conv1", "bn1", 64, 3, 7, 16, [](int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return a * 128 + b * 32 + (ph * 2 + pw) * 4 + c;
    });
}

// one conv over the volume v (rows of `pitch` elements in X) -> split rows of 2*n_out in `out`, rows outside the
// valid region zeroed
static int run_conv(vf_resnet* h, const ResConv& cw, const __half* X, int pitch, const Vol2& v, __half* out, bool relu,
                    cudaStream_t s) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = cw.ntaps; g.k_per_tap = cw.k_per_tap; g.nsplit = 2; g.lo_mask = cw.lo_mask;
    for (int j = 0; j < cw.ntaps; ++j) g.tap_off[j] = cw.dh[j] * v.Wp + cw.dw[j];
    g.mask = 1; g.row0 = 0;
    g.Tp = 1; g.Hp = v.Hp; g.Wp = v.Wp; g.t0 = 0; g.t1 = 1; g.h0 = v.h0; g.h1 = v.h1; g.w0 = v.w0; g.w1 = v.w1;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.ldo = 2 * cw.n_out; ep.out_f32 = 0; ep.bias = cw.bias; ep.scale = cw.scale;
    ep.act = relu ? VF_ACT_RELU : VF_ACT_NONE; ep.split_off = cw.n_out;
    h->launches += 1;
    return conv_gemm_f16(X, pitch, v.rows(), cw.w, cw.n_out, g, ep, s);
}

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
    VF_CUDA(cudaSetDevice(device));
    int major = 0, minor = 0;
    VF_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    VF_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    if (major != 9 || minor != 0)
        return fail(VF_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device, major, minor);
    vf_resnet* h = new vf_resnet();
    h->device = device; h->depth = depth; h->max_frames = max_frames; h->bottleneck = bottleneck;
    const ResTensors T{tensors, n_tensors};
    auto body = [&]() -> int {
        VF_TRY(prep_stem(h, h->stem, T));
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
                    if (B.stride == 2) VF_TRY(prep_stride2(h, B.c1, T, p + ".conv1", p + ".bn1", width, B.cin));
                    else               VF_TRY(prep_same(h, B.c1, T, p + ".conv1", p + ".bn1", width, B.cin, 3));
                    VF_TRY(prep_same(h, B.c2, T, p + ".conv2", p + ".bn2", width, width, 3));
                } else {
                    VF_TRY(prep_same(h, B.c1, T, p + ".conv1", p + ".bn1", width, B.cin, 1));
                    if (B.stride == 2) VF_TRY(prep_stride2(h, B.c2, T, p + ".conv2", p + ".bn2", width, width));
                    else               VF_TRY(prep_same(h, B.c2, T, p + ".conv2", p + ".bn2", width, width, 3));
                    VF_TRY(prep_same(h, B.c3, T, p + ".conv3", p + ".bn3", cout, width, 1));
                    e_act = std::max(e_act, rows(vi) * 2 * width);                  // c1 output at the input geometry
                    if (B.stride == 2) e_ph = std::max(e_ph, rows(vo) * 8 * width);
                }
                if (B.down) VF_TRY(prep_same(h, B.dn, T, p + ".downsample.0", p + ".downsample.1", cout, B.cin, 1));
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
        VF_CUDA(cudaStreamCreateWithFlags(&h->cs, cudaStreamNonBlocking));
        VF_CUDA(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
        VF_CUDA(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
        const char* e = getenv("VF_NO_GRAPH");
        h->use_graph = !(e && e[0] == '1');
        return VF_OK;
    };
    const int st = body();
    if (st != VF_OK) { vf_resnet_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_resnet_destroy(vf_resnet_t* h) {
    if (!h) return VF_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (void* p : h->allocs) cudaFree(p);
    for (auto& kv : h->graphs) cudaGraphExecDestroy(kv.second.first);
    if (h->cs) cudaStreamDestroy(h->cs);
    if (h->ev_in) cudaEventDestroy(h->ev_in);
    if (h->ev_out) cudaEventDestroy(h->ev_out);
    delete h;
    return VF_OK;
}

}  // extern "C"

namespace vf {

static int trunk_graph(vf_resnet* h, int m, cudaStream_t s) {
    if (!h->use_graph || gemm_profile_on()) return run_trunk(h, m, s);
    auto it = h->graphs.find(m);
    if (it == h->graphs.end()) {
        const int64_t before = h->launches;
        cudaGraph_t graph = nullptr;
        VF_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
        const int st = run_trunk(h, m, s);
        const cudaError_t ce = cudaStreamEndCapture(s, &graph);
        const int64_t n_launch = h->launches - before;
        h->launches = before;
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
        it = h->graphs.emplace(m, std::make_pair(exec, n_launch)).first;
    }
    VF_CUDA(cudaGraphLaunch(it->second.first, s));
    h->launches += it->second.second;
    return VF_OK;
}

static int resnet_forward(vf_resnet* h, const void* frames, int is_u8, int n, int Hr, int Wr, float* out, void* stream) {
    if (!h || !frames || !out) return fail(VF_ERR_INVALID, "resnet_forward: null argument");
    if (n < 0) return fail(VF_ERR_INVALID, "resnet_forward: %d frames", n);
    if (is_u8 && (Hr < 224 || Wr < 224))
        return fail(VF_ERR_INVALID, "resnet_forward: resized frame %dx%d is smaller than the 224 crop", Hr, Wr);
    if (n == 0) return VF_OK;
    const int cy = is_u8 ? center_crop_offset(Hr, 224) : 0, cx = is_u8 ? center_crop_offset(Wr, 224) : 0;
    const size_t frame_elems = is_u8 ? size_t(Hr) * Wr * 3 : size_t(3) * 224 * 224;
    cudaStream_t user = static_cast<cudaStream_t>(stream), s = h->cs;
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaEventRecord(h->ev_in, user));
    VF_CUDA(cudaStreamWaitEvent(s, h->ev_in, 0));
    for (int off = 0; off < n; off += h->max_frames) {      // calls beyond the workspace run in chunks
        const int m = std::min(h->max_frames, n - off);
        const void* src = is_u8 ? static_cast<const void*>(static_cast<const uint8_t*>(frames) + off * frame_elems)
                                : static_cast<const void*>(static_cast<const float*>(frames) + off * frame_elems);
        VF_TRY(resnet_input_pack(src, is_u8, m, Hr, Wr, cy, cx, h->s0, s));
        VF_TRY(trunk_graph(h, m, s));
        VF_TRY(resnet_avgpool(h->stage_out[3], stage_vol(m, 3), h->out_dim, out + size_t(off) * h->out_dim, s));
        h->launches += 2;
        h->last_n = m;
    }
    VF_CUDA(cudaEventRecord(h->ev_out, s));
    VF_CUDA(cudaStreamWaitEvent(user, h->ev_out, 0));
    return VF_OK;
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
    const ResConv& c = *cs[index];
    geom[0] = c.n_out; geom[1] = c.ntaps; geom[2] = c.k_per_tap;
    for (int j = 0; j < 4; ++j) { geom[3 + 3 * j] = 0; geom[4 + 3 * j] = c.dh[j]; geom[5 + 3 * j] = c.dw[j]; }
    *lo_mask = c.lo_mask;
    VF_CUDA(cudaSetDevice(h->device));
    const size_t nw = size_t(c.n_out) * 2 * c.ntaps * c.k_per_tap;
    if (w) VF_CUDA(cudaMemcpy(w, c.w, nw * sizeof(__half), cudaMemcpyDeviceToDevice));
    if (scale) VF_CUDA(cudaMemcpy(scale, c.scale, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    if (bias) VF_CUDA(cudaMemcpy(bias, c.bias, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    return VF_OK;
}

}  // extern "C"
