// Split-fp16 conv plumbing shared by the conv-engine drivers (split_conv.h).
#include <math.h>
#include <string.h>

#include <algorithm>

#include "split_conv.h"

namespace vf {

const vf_named_tensor* ResTensors::find(const std::string& name) const {
    for (int i = 0; i < n; ++i) {
        const char* k = t[i].name;
        if (k && (name == k || (strncmp(k, "module.", 7) == 0 && name == k + 7))) return &t[i];
    }
    return nullptr;
}

int ResTensors::get(const std::string& name, int64_t numel, const float** out) const {
    const vf_named_tensor* e = find(name);
    if (!e) return fail(VF_ERR_INVALID, "%s: missing tensor '%s'", who, name.c_str());
    if (!e->data || e->numel != numel)
        return fail(VF_ERR_INVALID, "%s: tensor '%s' has %lld elements, expected %lld", who, name.c_str(),
                    (long long)e->numel, (long long)numel);
    *out = e->data;
    return VF_OK;
}

int ResTensors::spatial_width(const std::string& name, int ci, int* co) const {
    const vf_named_tensor* e = find(name);
    if (!e) return fail(VF_ERR_INVALID, "%s: missing tensor '%s'", who, name.c_str());
    if (e->numel <= 0 || e->numel % (int64_t(9) * ci) != 0 || e->numel / (int64_t(9) * ci) > 65536)
        return fail(VF_ERR_INVALID, "%s: tensor '%s' has %lld elements, not a (co, %d, 1, 3, 3) weight", who,
                    name.c_str(), (long long)e->numel, ci);
    *co = int(e->numel / (int64_t(9) * ci));
    return VF_OK;
}

int bn_fold(const ResTensors& T, const std::string& p, int c, double eps, std::vector<float>& sc, std::vector<float>& sh) {
    const float *g, *b, *m, *v;
    VF_TRY(T.get(p + ".weight", c, &g)); VF_TRY(T.get(p + ".bias", c, &b));
    VF_TRY(T.get(p + ".running_mean", c, &m)); VF_TRY(T.get(p + ".running_var", c, &v));
    sc.resize(c); sh.resize(c);
    for (int i = 0; i < c; ++i) {
        const double s = double(g[i]) / sqrt(double(v[i]) + eps);
        sc[i] = float(s);
        sh[i] = float(double(b[i]) - double(m[i]) * s);
    }
    return VF_OK;
}

int upload_weights(EngineCore* h, ResConv& cw, const float* w, const Filter& f, int lo_off, const FilterCol& col,
                   const std::vector<float>& sc, const std::vector<float>& sh, int reps, int rep_stride) {
    const int n_out = int(sc.size());
    const int Ktot = cw.ntaps * cw.k_per_tap;
    const size_t Kall = size_t(2) * Ktot;
    std::vector<__half> B(size_t(n_out) * Kall, __float2half_rn(0.f));
    std::vector<char> has_hi(size_t(Ktot), 0);
    for (int o = 0; o < f.co; ++o)
        for (int c = 0; c < f.ci; ++c)
            for (int a = 0; a < f.kt; ++a)
                for (int y = 0; y < f.kh; ++y)
                    for (int x = 0; x < f.kw; ++x) {
                        const float wf = w[(((size_t(o) * f.ci + c) * f.kt + a) * f.kh + y) * f.kw + x];
                        const __half wh = __float2half_rn(wf), wl = __float2half_rn(wf - __half2float(wh));
                        for (int r = 0; r < reps; ++r) {
                            const int kc = col(a, y, x, c) + r * rep_stride;
                            if (kc < 0 || kc + lo_off >= Ktot) return fail(VF_ERR_INVALID, "%s: filter column out of range", h->who);
                            for (int kk : {kc, kc + lo_off}) {
                                B[size_t(o) * Kall + kk] = wh;
                                B[size_t(o) * Kall + Ktot + kk] = wl;
                            }
                            has_hi[kc] = 1;
                        }
                    }
    cw.n_out = n_out;
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
    VF_TRY(ralloc(h, &cw.scale, size_t(n_out)));
    VF_TRY(ralloc(h, &cw.bias, size_t(n_out)));
    VF_CUDA(cudaMemcpy(cw.w, B.data(), B.size() * sizeof(__half), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.scale, sc.data(), n_out * sizeof(float), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(cw.bias, sh.data(), n_out * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

int upload_conv(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                double eps, const Filter& f, int lo_off, const FilterCol& col, int co_pad, int reps, int rep_stride,
                float scale_mul) {
    const float* w;
    VF_TRY(T.get(name + ".weight", int64_t(f.co) * f.ci * f.kt * f.kh * f.kw, &w));
    std::vector<float> sc, sh;
    VF_TRY(bn_fold(T, bn, f.co, eps, sc, sh));
    for (float& s : sc) s *= scale_mul;
    sc.resize(std::max(f.co, co_pad), 0.f);
    sh.resize(std::max(f.co, co_pad), 0.f);
    return upload_weights(h, cw, w, f, lo_off, col, sc, sh, reps, rep_stride);
}

int prep_same(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
              double eps, int co, int ci, int k, int ci_p, int co_pad) {
    if (ci_p == 0) ci_p = ci;
    cw.ntaps = k; cw.k_per_tap = k * 2 * ci_p;
    for (int a = 0; a < k; ++a) { cw.dh[a] = a - k / 2; cw.dw[a] = -(k / 2); }
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, name, bn, eps, {co, ci, 1, k, k}, ci_p,
                       [=](int, int a, int d, int c) { return a * kpt + d * 2 * ci_p + c; }, co_pad);
}

int prep_stride2(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                 double eps, int co, int ci, int co_pad) {
    cw.ntaps = 4; cw.k_per_tap = 8 * ci;
    for (int t = 0; t < 4; ++t) { cw.dh[t] = t / 2 - 1; cw.dw[t] = t % 2 - 1; }
    const int kpt = cw.k_per_tap;
    return upload_conv(h, cw, T, name, bn, eps, {co, ci, 1, 3, 3}, ci, [=](int, int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return (a * 2 + b) * kpt + (ph * 2 + pw) * 2 * ci + c;
    }, co_pad);
}

int prep_temporal(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                  double eps, int co, int ci, int ci_p, int co_pad) {
    if (ci_p == 0) ci_p = ci;
    cw.ntaps = 3; cw.k_per_tap = 2 * ci_p;
    for (int a = 0; a < 3; ++a) cw.dt[a] = a - 1;
    return upload_conv(h, cw, T, name, bn, eps, {co, ci, 3, 1, 1}, ci_p,
                       [=](int kt, int, int, int c) { return kt * 2 * ci_p + c; }, co_pad);
}

int prep_stem(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
              double eps, int co, int co_pad) {
    cw.ntaps = 4; cw.k_per_tap = 128;
    for (int a = 0; a < 4; ++a) { cw.dh[a] = a - 2; cw.dw[a] = -2; }
    return upload_conv(h, cw, T, name, bn, eps, {co, 3, 1, 7, 7}, 16, [](int, int kh, int kw, int c) {
        const int a = (kh + 1) / 2, ph = (kh + 1) % 2, b = (kw + 1) / 2, pw = (kw + 1) % 2;
        return a * 128 + b * 32 + (ph * 2 + pw) * 4 + c;
    }, co_pad);
}

int run_conv(EngineCore* h, const ResConv& cw, const __half* X, int pitch, const Vol3& v, __half* out, bool relu,
             cudaStream_t s, int ldo) {
    if (ldo == 0) ldo = 2 * cw.n_out;
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = cw.ntaps; g.k_per_tap = cw.k_per_tap; g.nsplit = 2; g.lo_mask = cw.lo_mask;
    for (int j = 0; j < cw.ntaps; ++j) g.tap_off[j] = (cw.dt[j] * v.Hp + cw.dh[j]) * v.Wp + cw.dw[j];
    g.mask = 1; g.row0 = 0;
    g.Tp = v.Tp; g.Hp = v.Hp; g.Wp = v.Wp;
    g.t0 = v.t0; g.t1 = v.t1; g.h0 = v.h0; g.h1 = v.h1; g.w0 = v.w0; g.w1 = v.w1;
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = out; ep.ldo = ldo; ep.out_f32 = 0; ep.bias = cw.bias; ep.scale = cw.scale;
    ep.act = relu ? VF_ACT_RELU : VF_ACT_NONE; ep.split_off = ldo / 2;
    h->launches += 1;
    return conv_gemm_f16(X, pitch, v.rows(), cw.w, cw.n_out, g, ep, s);
}

int run_conv(EngineCore* h, const ResConv& cw, const __half* X, int pitch, const Vol2& v, __half* out, bool relu,
             cudaStream_t s) {
    return run_conv(h, cw, X, pitch, Vol3{v.n, 1, v.Hp, v.Wp, 0, 1, v.h0, v.h1, v.w0, v.w1}, out, relu, s);
}

int read_back_conv(int device, const ResConv& c, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias) {
    geom[0] = c.n_out; geom[1] = c.ntaps; geom[2] = c.k_per_tap;
    for (int j = 0; j < 4; ++j) { geom[3 + 3 * j] = c.dt[j]; geom[4 + 3 * j] = c.dh[j]; geom[5 + 3 * j] = c.dw[j]; }
    *lo_mask = c.lo_mask;
    VF_CUDA(cudaSetDevice(device));
    const size_t nw = size_t(c.n_out) * 2 * c.ntaps * c.k_per_tap;
    if (w) VF_CUDA(cudaMemcpy(w, c.w, nw * sizeof(__half), cudaMemcpyDeviceToDevice));
    if (scale) VF_CUDA(cudaMemcpy(scale, c.scale, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    if (bias) VF_CUDA(cudaMemcpy(bias, c.bias, size_t(c.n_out) * sizeof(float), cudaMemcpyDeviceToDevice));
    return VF_OK;
}

int clip_window(const char* who, const int* starts, int n, int T, int per_chunk, int slots, int* m, int* lo, int* hi,
                R21DStarts* st) {
    // the chunk's frames [lo, hi) are transformed once each, so they must fit the per-frame buffer
    int k = 0, l = starts[0], u = starts[0] + T;
    while (k < n && k < per_chunk) {
        const int l2 = std::min(l, starts[k]), u2 = std::max(u, starts[k] + T);
        if (k > 0 && u2 - l2 > slots) break;
        l = l2; u = u2; ++k;
    }
    if (u - l > slots) return fail(VF_ERR_INVALID, "%s: clip exceeds the frame workspace", who);
    for (int b = 0; b < k; ++b) st->first[b] = starts[b] - l;
    *m = k; *lo = l; *hi = u;
    return VF_OK;
}

int upload_vec(EngineCore* h, const ResTensors& T, const std::string& name, int64_t n, float** dst) {
    const float* a;
    VF_TRY(T.get(name, n, &a));
    VF_TRY(ralloc(h, dst, size_t(n)));
    VF_CUDA(cudaMemcpy(*dst, a, size_t(n) * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

int upload_split_mat(EngineCore* h, const ResTensors& T, const std::string& name, int64_t rows, int64_t cols,
                     __half** dst, int64_t cols_pad) {
    const float* a;
    VF_TRY(T.get(name, rows * cols, &a));
    const int64_t kp = cols_pad > 0 ? cols_pad : cols;
    std::vector<__half> tmp(size_t(rows * kp * 2), __float2half_rn(0.f));
    for (int64_t r = 0; r < rows; ++r)
        for (int64_t c = 0; c < cols; ++c) {
            const __half hi = __float2half_rn(a[r * cols + c]);
            tmp[size_t(r * 2 * kp + c)] = hi;
            tmp[size_t(r * 2 * kp + kp + c)] = __float2half_rn(a[r * cols + c] - __half2float(hi));
        }
    VF_TRY(ralloc(h, dst, tmp.size()));
    VF_CUDA(cudaMemcpy(*dst, tmp.data(), tmp.size() * sizeof(__half), cudaMemcpyHostToDevice));
    return VF_OK;
}

GemmEpi linear_epi(void* out, int ldo, int out_f32, const float* bias, int act, int accumulate) {
    GemmEpi e;
    memset(&e, 0, sizeof(e));
    e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.bias = bias; e.act = act; e.accumulate = accumulate;
    return e;
}

int split_linear(const __half* A, int M, int N, int K, const __half* W2, const GemmEpi& ep, cudaStream_t s) {
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = 1; g.k_per_tap = K; g.nsplit = 2; g.lo_mask = 0; g.mask = 0;
    return conv_gemm_f16(A, K, M, W2, N, g, ep, s);
}

}  // namespace vf
