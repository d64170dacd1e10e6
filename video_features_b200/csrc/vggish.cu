// VGGish audio embeddings (torchvggish VGG, postprocess=False) on the wgmma conv-GEMM, with the reference's float64
// front end on the GPU.  Replaces models/vggish_torch: vggish_input.wavfile_to_examples (for PCM-16 samples already
// read) and VGG.forward.
//
// Front end (float64, vggish_kernels.cu): int16 samples -> mono mix / 32768 -> resampy 0.2.2 kaiser_best resample to
// 16 kHz (the time register as TimeSegs pieces) -> frames of 400 / hop 160 -> Hann -> |FFT 512| -> mel -> log(. + 0.01)
// -> fp32 examples [n][96][64].  The filter table, Hann window and mel matrix come from the caller (float64 numpy);
// the filter is scaled by the rate ratio on the host when downsampling, as resampy does.
// Trunk: every activation and weight a split-fp16 pair (scripts/precision/emulate_vggish.py); activations channels-last
// in zero-bordered volumes, rows [hi C | lo C] (raft_kernels.h Vol2).
//   conv1 (C = 1): a one-tap GEMM over im2col rows of 32 (vggish_im2col) on [n][98][66];
//   conv2..6: three taps (kernel rows) of 3 x 2C, as split_conv.h prep_same, bias in the epilogue, on
//     [n][50][34], [n][26][18] (conv3, conv4), [n][14][10] (conv5, conv6);
//   max-pools 2x2/2 (vggish_maxpool2) write the next conv's bordered volume; the last writes fc1's dense rows
//     [n][6 x 4 x (hi 512 | lo 512)], the reference's (H, W, C) flatten;
//   fc1, fc2: one-tap GEMMs with bias + ReLU to split rows; fc3 with bias + ReLU to fp32.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "internal.h"
#include "split_conv.h"
#include "vggish_kernels.h"

namespace vf {
constexpr int EX_FRAMES = 96, BANDS = 64, HOP = 160, WIN = 400, EX_SAMPLES = EX_FRAMES * HOP;
static const int kConvIdx[6] = {0, 3, 6, 8, 11, 13};
static const int kConvIn[6] = {1, 64, 128, 256, 256, 512};
static const int kConvOut[6] = {64, 128, 256, 256, 512, 512};
}  // namespace vf

using namespace vf;

struct vf_vggish : vf::EngineCore {
    int max_examples = 0, num_table = 0, nwin = 0, rate = 0;
    std::vector<double> base_win;                  // the unscaled filter table
    ResConv conv[6], fc[3];
    double *win = nullptr, *delta = nullptr, *hann = nullptr, *twiddle = nullptr, *mel = nullptr, *wave = nullptr;
    float *logmel = nullptr, *f3 = nullptr;
    __half *x1 = nullptr, *a = nullptr, *b = nullptr, *p[4] = {nullptr, nullptr, nullptr, nullptr};
    __half *f1 = nullptr, *f2 = nullptr;
    int last_n = 0;
    int64_t last_wave = 0;
};

namespace vf {

static Vol2 vol(int n, int L) {            // conv volume of level L: 96x64, 48x32, 24x16, 12x8 with a 1-position border
    const int H = 96 >> L, W = 64 >> L;
    return Vol2{n, H + 2, W + 2, 1, H + 1, 1, W + 1};
}

// 3x3 pad 1 conv + bias on split rows of 2*ci: prep_same's layout, scale 1
static int prep_conv3(vf_vggish* h, ResConv& cw, const float* w, const float* bias, int co, int ci) {
    cw.ntaps = 3; cw.k_per_tap = 3 * 2 * ci;
    for (int a = 0; a < 3; ++a) { cw.dh[a] = a - 1; cw.dw[a] = -1; }
    const int kpt = cw.k_per_tap;
    const std::vector<float> sc(size_t(co), 1.f), sh(bias, bias + co);
    return upload_weights(h, cw, w, {co, ci, 1, 3, 3}, ci, [=](int, int a, int d, int c) { return a * kpt + d * 2 * ci + c; },
                          sc, sh);
}

// one-tap GEMM over M rows of X (pitch elements) + bias + ReLU -> split rows of 2*n_out, or fp32 rows of n_out
static int run_fc(vf_vggish* h, const ResConv& cw, const __half* X, int pitch, int M, void* out, bool f32, cudaStream_t s) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = 1; g.k_per_tap = cw.k_per_tap; g.nsplit = 2; g.lo_mask = cw.lo_mask; g.mask = 0;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.bias = cw.bias; ep.scale = cw.scale; ep.act = VF_ACT_RELU;
    if (f32) { ep.ldo = cw.n_out; ep.out_f32 = 1; }
    else     { ep.ldo = 2 * cw.n_out; ep.split_off = cw.n_out; }
    h->launches += 1;
    return conv_gemm_f16(X, pitch, M, cw.w, cw.n_out, g, ep, s);
}

// conv1 .. fc3 on m examples whose log-mel is in h->logmel -> out[m][128] fp32
static int run_trunk(vf_vggish* h, int m, float* out, cudaStream_t s) {
    VF_TRY(vggish_im2col(h->logmel, m, h->x1, s));
    h->launches += 1;
    VF_TRY(run_conv(h, h->conv[0], h->x1, 32, vol(m, 0), h->a, true, s));
    VF_TRY(vggish_maxpool2(h->a, vol(m, 0), 64, h->p[0], vol(m, 1), 128, s));
    VF_TRY(run_conv(h, h->conv[1], h->p[0], 128, vol(m, 1), h->a, true, s));
    VF_TRY(vggish_maxpool2(h->a, vol(m, 1), 128, h->p[1], vol(m, 2), 256, s));
    VF_TRY(run_conv(h, h->conv[2], h->p[1], 256, vol(m, 2), h->a, true, s));
    VF_TRY(run_conv(h, h->conv[3], h->a, 512, vol(m, 2), h->b, true, s));
    VF_TRY(vggish_maxpool2(h->b, vol(m, 2), 256, h->p[2], vol(m, 3), 512, s));
    VF_TRY(run_conv(h, h->conv[4], h->p[2], 512, vol(m, 3), h->a, true, s));
    VF_TRY(run_conv(h, h->conv[5], h->a, 1024, vol(m, 3), h->b, true, s));
    VF_TRY(vggish_maxpool2(h->b, vol(m, 3), 512, h->p[3], Vol2{m, 6, 4, 0, 6, 0, 4}, 1024, s));
    h->launches += 4;
    VF_TRY(run_fc(h, h->fc[0], h->p[3], 24 * 1024, m, h->f1, false, s));
    VF_TRY(run_fc(h, h->fc[1], h->f1, 8192, m, h->f2, false, s));
    VF_TRY(run_fc(h, h->fc[2], h->f2, 8192, m, h->f3, true, s));
    VF_CUDA(cudaMemcpyAsync(out, h->f3, size_t(m) * 128 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    h->last_n = m;
    return VF_OK;
}

// the filter table for `rate` (scaled by the ratio when downsampling) and its forward difference, uploaded once per rate
static int set_rate(vf_vggish* h, int rate) {
    if (rate == h->rate) return VF_OK;
    const double ratio = 16000.0 / double(rate);
    std::vector<double> w(h->base_win), d(w.size(), 0.0);
    if (ratio < 1.0)
        for (double& v : w) v *= ratio;
    for (size_t i = 0; i + 1 < w.size(); ++i) d[i] = w[i + 1] - w[i];
    VF_CUDA(cudaMemcpy(h->win, w.data(), w.size() * sizeof(double), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(h->delta, d.data(), d.size() * sizeof(double), cudaMemcpyHostToDevice));
    h->rate = rate;
    return VF_OK;
}

}  // namespace vf

extern "C" {

int vf_vggish_destroy(vf_vggish_t* h) {
    if (!h) return VF_OK;
    release(h);
    delete h;
    return VF_OK;
}

int vf_vggish_create(vf_vggish_t** out, const vf_named_tensor* tensors, int n_tensors, const double* hann,
                     const double* mel, const double* interp_win, int n_win, int num_table, int device,
                     int max_examples) {
    if (!out || !tensors || n_tensors <= 0 || !hann || !mel || !interp_win)
        return fail(VF_ERR_INVALID, "vggish_create: null argument");
    if (n_win < 2 || num_table <= 0) return fail(VF_ERR_INVALID, "vggish_create: bad filter table (%d entries)", n_win);
    *out = nullptr;
    if (max_examples <= 0) max_examples = 64;
    VF_TRY(check_device(device));
    vf_vggish* h = new vf_vggish();
    h->who = "vggish_create";
    h->device = device; h->max_examples = max_examples; h->num_table = num_table; h->nwin = n_win;
    h->base_win.assign(interp_win, interp_win + n_win);
    const ResTensors T{tensors, n_tensors, "vggish_create"};
    auto body = [&]() -> int {
        for (int i = 0; i < 6; ++i) {
            const std::string p = "features." + std::to_string(kConvIdx[i]);
            const int co = kConvOut[i], ci = kConvIn[i];
            const float *w, *b;
            VF_TRY(T.get(p + ".weight", int64_t(co) * ci * 9, &w));
            VF_TRY(T.get(p + ".bias", co, &b));
            if (i == 0) {             // one tap over the im2col rows: hi at kh * 3 + kw, lo 16 columns further
                ResConv& c = h->conv[0];
                c.ntaps = 1; c.k_per_tap = 32;
                const std::vector<float> sc(size_t(co), 1.f), sh(b, b + co);
                VF_TRY(upload_weights(h, c, w, {co, 1, 1, 3, 3}, 16, [](int, int a, int d, int) { return a * 3 + d; }, sc, sh));
            } else {
                VF_TRY(prep_conv3(h, h->conv[i], w, b, co, ci));
            }
        }
        const int fin[3] = {12288, 4096, 4096}, fout[3] = {4096, 4096, 128};
        for (int i = 0; i < 3; ++i) {
            const std::string p = "embeddings." + std::to_string(2 * i);
            const float *w, *b;
            VF_TRY(T.get(p + ".weight", int64_t(fout[i]) * fin[i], &w));
            VF_TRY(T.get(p + ".bias", fout[i], &b));
            ResConv& c = h->fc[i];
            c.ntaps = 1; c.k_per_tap = 2 * fin[i];
            const std::vector<float> sc(size_t(fout[i]), 1.f), sh(b, b + fout[i]);
            if (i == 0)               // input feature (h * 4 + w) * 512 + c sits in position block h * 4 + w of 1024
                VF_TRY(upload_weights(h, c, w, {fout[i], fin[i], 1, 1, 1}, 512,
                                      [](int, int, int, int c) { return (c / 512) * 1024 + c % 512; }, sc, sh));
            else
                VF_TRY(upload_weights(h, c, w, {fout[i], fin[i], 1, 1, 1}, fin[i], [](int, int, int, int c) { return c; }, sc,
                                      sh));
        }
        const size_t E = size_t(max_examples);
        VF_TRY(ralloc(h, &h->win, size_t(n_win)));
        VF_TRY(ralloc(h, &h->delta, size_t(n_win)));
        VF_TRY(ralloc(h, &h->hann, size_t(WIN)));
        VF_TRY(ralloc(h, &h->twiddle, size_t(512)));
        VF_TRY(ralloc(h, &h->mel, size_t(257) * BANDS));
        VF_TRY(ralloc(h, &h->wave, E * EX_SAMPLES + (WIN - HOP)));
        VF_TRY(ralloc(h, &h->logmel, E * EX_FRAMES * BANDS));
        VF_TRY(ralloc(h, &h->x1, E * vol(1, 0).rows() * 32));
        VF_TRY(ralloc(h, &h->a, E * vol(1, 0).rows() * 128));
        VF_TRY(ralloc(h, &h->b, E * vol(1, 2).rows() * 512));
        for (int L = 0; L < 3; ++L) VF_TRY(ralloc(h, &h->p[L], E * vol(1, L + 1).rows() * (256 << L)));
        VF_TRY(ralloc(h, &h->p[3], E * 24 * 1024));
        VF_TRY(ralloc(h, &h->f1, E * 8192));
        VF_TRY(ralloc(h, &h->f2, E * 8192));
        VF_TRY(ralloc(h, &h->f3, E * 128));
        double tw[512];
        for (int k = 0; k < 256; ++k) { tw[k] = cos(2.0 * M_PI * k / 512.0); tw[256 + k] = sin(2.0 * M_PI * k / 512.0); }
        VF_CUDA(cudaMemcpy(h->twiddle, tw, sizeof(tw), cudaMemcpyHostToDevice));
        VF_CUDA(cudaMemcpy(h->hann, hann, WIN * sizeof(double), cudaMemcpyHostToDevice));
        VF_CUDA(cudaMemcpy(h->mel, mel, size_t(257) * BANDS * sizeof(double), cudaMemcpyHostToDevice));
        return VF_OK;
    };
    const int st = body();
    if (st != VF_OK) { vf_vggish_destroy(h); return st; }
    *out = h;
    return VF_OK;
}

int vf_vggish_forward_pcm16(vf_vggish_t* h, const int16_t* samples, int64_t n_samples, int channels, int sample_rate,
                            float* out, int64_t capacity, int64_t* n_out, void* stream) {
    if (!h || !n_out || (n_samples > 0 && !samples)) return fail(VF_ERR_INVALID, "vggish_forward_pcm16: null argument");
    if (n_samples < 0 || channels <= 0 || sample_rate <= 0)
        return fail(VF_ERR_INVALID, "vggish_forward_pcm16: %lld samples x %d channels at %d Hz", (long long)n_samples,
                    channels, sample_rate);
    const bool resample = sample_rate != 16000;
    const double ratio = 16000.0 / double(sample_rate);
    const int64_t n16 = resample ? int64_t(double(n_samples) * ratio) : n_samples;
    const int64_t frames = n16 >= WIN ? 1 + (n16 - WIN) / HOP : 0, n_ex = frames / EX_FRAMES;
    *n_out = n_ex;
    if (n_ex == 0) return VF_OK;
    if (!out || capacity < n_ex * 128)
        return fail(VF_ERR_INVALID, "vggish_forward_pcm16: %lld examples need %lld output floats, capacity %lld",
                    (long long)n_ex, (long long)(n_ex * 128), (long long)capacity);
    VF_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    TimeSegs segs;
    segs.n = 0;
    if (resample) {
        VF_TRY(set_rate(h, sample_rate));
        VF_TRY(vggish_time_segs(1.0 / ratio, n16, &segs));
    }
    for (int64_t e0 = 0; e0 < n_ex; e0 += h->max_examples) {    // features do not depend on the split
        const int m = int(std::min<int64_t>(h->max_examples, n_ex - e0));
        const int64_t count = int64_t(m) * EX_SAMPLES + (WIN - HOP);
        VF_TRY(vggish_resample(samples, n_samples, channels, resample ? h->win : nullptr, h->delta, h->nwin,
                               h->num_table, ratio, segs, e0 * EX_SAMPLES, count, h->wave, s));
        VF_TRY(vggish_logmel(h->wave, int64_t(m) * EX_FRAMES, h->hann, h->twiddle, h->mel, h->logmel, s));
        h->launches += 2;
        h->last_wave = count;
        VF_TRY(run_trunk(h, m, out + e0 * 128, s));
    }
    return VF_OK;
}

int vf_vggish_forward_logmel_f32(vf_vggish_t* h, const float* examples, int n, float* out, void* stream) {
    if (!h || (n > 0 && (!examples || !out))) return fail(VF_ERR_INVALID, "vggish_forward_logmel_f32: null argument");
    if (n < 0) return fail(VF_ERR_INVALID, "vggish_forward_logmel_f32: %d examples", n);
    VF_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    for (int e0 = 0; e0 < n; e0 += h->max_examples) {
        const int m = std::min(h->max_examples, n - e0);
        VF_CUDA(cudaMemcpyAsync(h->logmel, examples + size_t(e0) * EX_FRAMES * BANDS,
                                size_t(m) * EX_FRAMES * BANDS * sizeof(float), cudaMemcpyDeviceToDevice, s));
        h->last_wave = 0;
        VF_TRY(run_trunk(h, m, out + size_t(e0) * 128, s));
    }
    return VF_OK;
}

int vf_vggish_read_stage(vf_vggish_t* h, int stage, void* out, int64_t capacity, int* dims4, void* stream) {
    if (!h || !dims4 || h->last_n <= 0) return fail(VF_ERR_INVALID, "vggish_read_stage: no forward has run");
    if (stage < 0 || stage > 8) return fail(VF_ERR_INVALID, "vggish_read_stage: unknown stage %d", stage);
    if (stage == 0 && h->last_wave <= 0)
        return fail(VF_ERR_INVALID, "vggish_read_stage: the last call started from log-mel examples");
    const int n = h->last_n;
    int64_t numel;
    if (stage == 0) { dims4[0] = int(h->last_wave); dims4[1] = dims4[2] = dims4[3] = 1; }
    else if (stage == 1) { dims4[0] = n; dims4[1] = 1; dims4[2] = EX_FRAMES; dims4[3] = BANDS; }
    else if (stage <= 5) {          // pool 1..4: 64 x 48 x 32, 128 x 24 x 16, 256 x 12 x 8, 512 x 6 x 4
        const int L = stage - 2;
        dims4[0] = n; dims4[1] = 64 << L; dims4[2] = 48 >> L; dims4[3] = 32 >> L;
    } else { dims4[0] = n; dims4[1] = stage == 8 ? 128 : 4096; dims4[2] = dims4[3] = 1; }
    numel = int64_t(dims4[0]) * dims4[1] * dims4[2] * dims4[3];
    if (!out) return VF_OK;
    if (capacity < numel) return fail(VF_ERR_INVALID, "vggish_read_stage: capacity too small");
    VF_CUDA(cudaSetDevice(h->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    float* o = static_cast<float*>(out);
    switch (stage) {
        case 0: VF_CUDA(cudaMemcpyAsync(out, h->wave, size_t(numel) * sizeof(double), cudaMemcpyDeviceToDevice, s)); break;
        case 1: VF_CUDA(cudaMemcpyAsync(out, h->logmel, size_t(numel) * sizeof(float), cudaMemcpyDeviceToDevice, s)); break;
        case 2: case 3: case 4:
            return raft_unpack2d(h->p[stage - 2], vol(n, stage - 1), 2 * dims4[1], 0, dims4[1], dims4[1], o, s);
        // pool 4: fc1's dense rows
        case 5: return raft_unpack2d(h->p[3], Vol2{n, 6, 4, 0, 6, 0, 4}, 1024, 0, 512, 512, o, s);
        case 6: return raft_unpack2d(h->f1, Vol2{n, 1, 1, 0, 1, 0, 1}, 8192, 0, 4096, 4096, o, s);
        case 7: return raft_unpack2d(h->f2, Vol2{n, 1, 1, 0, 1, 0, 1}, 8192, 0, 4096, 4096, o, s);
        default: VF_CUDA(cudaMemcpyAsync(out, h->f3, size_t(numel) * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    return VF_OK;
}

int64_t vf_vggish_launch_count(const vf_vggish_t* h) { return h ? h->launches : 0; }

int vf_vggish_conv(const vf_vggish_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    if (!h || !geom || !lo_mask) return fail(VF_ERR_INVALID, "vggish_conv: null argument");
    if (index < 0 || index >= 9) return fail(VF_ERR_INVALID, "vggish_conv: index %d outside the 9 convs", index);
    return read_back_conv(h->device, index < 6 ? h->conv[index] : h->fc[index - 6], geom, lo_mask, w, scale, bias);
}

int vf_vggish_time_register(int sample_rate, int64_t t0, int64_t count, double* out) {
    if (sample_rate <= 0 || t0 < 0 || count < 0 || (count > 0 && !out))
        return fail(VF_ERR_INVALID, "vggish_time_register: bad argument");
    TimeSegs S;
    VF_TRY(vggish_time_segs(1.0 / (16000.0 / double(sample_rate)), t0 + count, &S));
    int s = 0;
    for (int64_t t = t0; t < t0 + count; ++t) {
        while (s + 1 < S.n && S.t[s + 1] <= t) ++s;
        out[t - t0] = S.r[s] + double(t - S.t[s]) * S.d[s];
    }
    return VF_OK;
}

}  // extern "C"
