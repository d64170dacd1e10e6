// Split-fp16 conv plumbing shared by resnet.cu and clip_resnet.cu (split_conv.h).
#include <math.h>
#include <string.h>

#include "split_conv.h"

namespace vf {

int conv_alloc_bytes(ConvHost* h, void** p, size_t bytes) {
    void* q = nullptr;
    bytes += 65536;
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "%s: cudaMalloc(%zu bytes): %s", h->who, bytes, cudaGetErrorString(e));
    h->allocs.push_back(q);
    VF_CUDA(cudaMemset(q, 0, bytes));
    *p = q;
    return VF_OK;
}

int ResTensors::get(const std::string& name, int64_t numel, const float** out) const {
    for (int i = 0; i < n; ++i) {
        const char* k = t[i].name;
        if (!k || !(name == k || (strncmp(k, "module.", 7) == 0 && name == k + 7))) continue;
        if (!t[i].data || t[i].numel != numel)
            return fail(VF_ERR_INVALID, "%s: tensor '%s' has %lld elements, expected %lld", who, name.c_str(),
                        (long long)t[i].numel, (long long)numel);
        *out = t[i].data;
        return VF_OK;
    }
    return fail(VF_ERR_INVALID, "%s: missing tensor '%s'", who, name.c_str());
}

int bn_fold(const ResTensors& T, const std::string& p, int c, std::vector<float>& sc, std::vector<float>& sh) {
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

int upload_weights(ConvHost* h, ResConv& cw, const float* w, int co, int ci, int k, int lo_off,
                   const std::function<int(int, int, int)>& col, const std::vector<float>& sc,
                   const std::vector<float>& sh, int reps, int rep_stride) {
    const int Ktot = cw.ntaps * cw.k_per_tap;
    const size_t Kall = size_t(2) * Ktot;
    std::vector<__half> B(size_t(co) * Kall, __float2half_rn(0.f));
    std::vector<char> has_hi(size_t(Ktot), 0);
    for (int o = 0; o < co; ++o)
        for (int c = 0; c < ci; ++c)
            for (int a = 0; a < k; ++a)
                for (int d = 0; d < k; ++d) {
                    const float wf = w[((size_t(o) * ci + c) * k + a) * k + d];
                    const __half wh = __float2half_rn(wf), wl = __float2half_rn(wf - __half2float(wh));
                    for (int r = 0; r < reps; ++r) {
                        const int kc = col(a, d, c) + r * rep_stride;
                        if (kc < 0 || kc + lo_off >= Ktot) return fail(VF_ERR_INVALID, "%s: filter column out of range", h->who);
                        for (int kk : {kc, kc + lo_off}) {
                            B[size_t(o) * Kall + kk] = wh;
                            B[size_t(o) * Kall + Ktot + kk] = wl;
                        }
                        has_hi[kc] = 1;
                    }
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

int upload_conv(ConvHost* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn, int co,
                int ci, int k, int lo_off, const std::function<int(int, int, int)>& col, int reps, int rep_stride,
                float scale_mul) {
    const float* w;
    VF_TRY(T.get(name + ".weight", int64_t(co) * ci * k * k, &w));
    std::vector<float> sc, sh;
    VF_TRY(bn_fold(T, bn, co, sc, sh));
    for (float& s : sc) s *= scale_mul;
    return upload_weights(h, cw, w, co, ci, k, lo_off, col, sc, sh, reps, rep_stride);
}

int prep_same(ConvHost* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn, int co,
              int ci, int k) {
    cw.ntaps = k; cw.k_per_tap = k * 2 * ci;
    for (int a = 0; a < k; ++a) { cw.dh[a] = a - k / 2; cw.dw[a] = -(k / 2); }
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, name, bn, co, ci, k, ci, [=](int a, int d, int c) { return a * kpt + d * 2 * ci + c; });
}

int prep_stride2(ConvHost* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn, int co,
                 int ci) {
    cw.ntaps = 4; cw.k_per_tap = 8 * ci;
    for (int t = 0; t < 4; ++t) { cw.dh[t] = t / 2 - 1; cw.dw[t] = t % 2 - 1; }
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, name, bn, co, ci, 3, ci, [=](int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return (a * 2 + b) * kpt + (ph * 2 + pw) * 2 * ci + c;
    });
}

int run_conv(ConvHost* h, const ResConv& cw, const __half* X, int pitch, const Vol2& v, __half* out, bool relu,
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

int read_back_conv(int device, const ResConv& c, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    geom[0] = c.n_out; geom[1] = c.ntaps; geom[2] = c.k_per_tap;
    for (int j = 0; j < 4; ++j) { geom[3 + 3 * j] = 0; geom[4 + 3 * j] = c.dh[j]; geom[5 + 3 * j] = c.dw[j]; }
    *lo_mask = c.lo_mask;
    VF_CUDA(cudaSetDevice(device));
    const size_t nw = size_t(c.n_out) * 2 * c.ntaps * c.k_per_tap;
    if (w) VF_CUDA(cudaMemcpy(w, c.w, nw * sizeof(__half), cudaMemcpyDeviceToDevice));
    if (scale) VF_CUDA(cudaMemcpy(scale, c.scale, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    if (bias) VF_CUDA(cudaMemcpy(bias, c.bias, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    return VF_OK;
}

}  // namespace vf
