// Host-side pieces of libvfeat.so that are not kernels: error text, the frame sampler and shard arithmetic,
// Pillow coefficient tables, resize / transform entry points, and the handle core every engine driver embeds.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "internal.h"

namespace vf {

static thread_local char g_err[1024] = {0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

// ---- Pillow precompute_coeffs + normalize_coeffs_8bpc (third-party Pillow libImaging/Resample.c; the reference
// reaches it through torchvision Resize in the CLIP transform and models/i3d/transforms/transforms.py:121,125).
static double filter_bicubic(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}
static double filter_bilinear(double x) {
    if (x < 0.0) x = -x;
    if (x < 1.0) return 1.0 - x;
    return 0.0;
}

struct CoefTable {
    int ksize = 0;
    std::vector<int> bounds;   // [out*2]: first source index, tap count
    std::vector<int> coefs;    // [out*ksize] fixed point, 22 fractional bits
};

static bool build_coeffs(int in_size, int out_size, int filter, CoefTable* t) {
    double (*f)(double);
    double fsupport;
    if (filter == VF_FILTER_BICUBIC) { f = filter_bicubic; fsupport = 2.0; }
    else if (filter == VF_FILTER_BILINEAR) { f = filter_bilinear; fsupport = 1.0; }
    else return false;
    const double scale = double(in_size) / double(out_size);
    double filterscale = scale;
    if (filterscale < 1.0) filterscale = 1.0;
    const double support = fsupport * filterscale;
    const int ksize = int(ceil(support)) * 2 + 1;
    t->ksize = ksize;
    t->bounds.assign(size_t(out_size) * 2, 0);
    t->coefs.assign(size_t(out_size) * ksize, 0);
    std::vector<double> k(ksize);
    const double ss = 1.0 / filterscale;
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        double ww = 0.0;
        int xmin = int(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = int(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        for (int x = 0; x < xmax; ++x) {
            const double w = f((x + xmin - center + 0.5) * ss);
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x) {
            if (ww != 0.0) k[x] /= ww;
        }
        for (int x = 0; x < xmax; ++x) {
            const double v = k[x];
            t->coefs[size_t(xx) * ksize + x] = v < 0 ? int(-0.5 + v * double(1 << 22)) : int(0.5 + v * double(1 << 22));
        }
        t->bounds[2 * xx] = xmin;
        t->bounds[2 * xx + 1] = xmax;
    }
    return true;
}

// device-resident coefficient tables, cached per (device, in, out, filter)
struct DevCoefs {
    int ksize = 0;
    int* bounds = nullptr;
    int* coefs = nullptr;
};
static std::mutex g_coef_mu;
static std::map<std::tuple<int, int, int, int>, DevCoefs> g_coef_cache;

static int get_dev_coefs(int in_size, int out_size, int filter, cudaStream_t s, DevCoefs* out) {
    int dev = 0;
    VF_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_coef_mu);
    auto key = std::make_tuple(dev, in_size, out_size, filter);
    auto it = g_coef_cache.find(key);
    if (it != g_coef_cache.end()) { *out = it->second; return VF_OK; }
    CoefTable t;
    if (!build_coeffs(in_size, out_size, filter, &t)) return fail(VF_ERR_INVALID, "resize: unknown filter %d", filter);
    DevCoefs d;
    d.ksize = t.ksize;
    VF_CUDA(cudaMalloc(&d.bounds, t.bounds.size() * sizeof(int)));
    VF_CUDA(cudaMalloc(&d.coefs, t.coefs.size() * sizeof(int)));
    // synchronous copies: the host vectors die at scope exit; tables are built once per geometry
    VF_CUDA(cudaMemcpy(d.bounds, t.bounds.data(), t.bounds.size() * sizeof(int), cudaMemcpyHostToDevice));
    VF_CUDA(cudaMemcpy(d.coefs, t.coefs.data(), t.coefs.size() * sizeof(int), cudaMemcpyHostToDevice));
    (void)s;
    g_coef_cache[key] = d;
    *out = d;
    return VF_OK;
}

int resize_u8(const uint8_t* src, int n, int in_h, int in_w, uint8_t* dst, int out_h, int out_w, int filter,
              uint8_t* tmp, cudaStream_t s) {
    if (n <= 0) return VF_OK;
    if (in_h <= 0 || in_w <= 0 || out_h <= 0 || out_w <= 0) return fail(VF_ERR_INVALID, "resize: bad geometry");
    DevCoefs kh, kv;
    VF_TRY(get_dev_coefs(in_w, out_w, filter, s, &kh));
    VF_TRY(get_dev_coefs(in_h, out_h, filter, s, &kv));
    if (out_w != in_w && out_h != in_h && tmp == nullptr) return fail(VF_ERR_INVALID, "resize: tmp scratch required");
    return launch_resample(src, n, in_h, in_w, tmp, dst, out_h, out_w, kh.bounds, kh.coefs, kh.ksize, kv.bounds,
                           kv.coefs, kv.ksize, s);
}

// torchvision CenterCrop offset: int(round((dim - crop) / 2.0)) with Python's round-half-to-even
int center_crop_offset(int dim, int crop) {
    const int d = dim - crop;
    if (d >= 0) {
        if ((d & 1) == 0) return d / 2;
        const int q = d / 2;   // value is q + 0.5
        return (q & 1) ? q + 1 : q;
    }
    const int e = -d;          // negative: -(e/2) or -(q+0.5)
    if ((e & 1) == 0) return -(e / 2);
    const int q = e / 2;
    return -((q & 1) ? q + 1 : q);
}

// ---- engine handles
int check_device(int device) {
    VF_CUDA(cudaSetDevice(device));
    int major = 0, minor = 0;
    VF_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    VF_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
    if (major != 9 || minor != 0)
        return fail(VF_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device, major, minor);
    return VF_OK;
}

bool graphs_enabled() {
    const char* e = getenv("VF_NO_GRAPH");
    return !(e && e[0] == '1');
}

bool graph_trace() {
    const char* e = getenv("VF_GRAPH_TRACE");
    return e && e[0] == '1';
}

int engine_alloc(EngineCore* h, void** p, size_t bytes) {
    void* q = nullptr;
    bytes += 65536;
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "%s: cudaMalloc(%zu bytes): %s", h->who, bytes, cudaGetErrorString(e));
    h->allocs.push_back(q);
    VF_CUDA(cudaMemset(q, 0, bytes));
    *p = q;
    return VF_OK;
}

int open_stream(EngineCore* h) {
    VF_CUDA(cudaStreamCreateWithFlags(&h->cs, cudaStreamNonBlocking));
    VF_CUDA(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
    VF_CUDA(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
    return VF_OK;
}

int enter(EngineCore* h, cudaStream_t user) {
    VF_CUDA(cudaSetDevice(h->device));
    VF_CUDA(cudaEventRecord(h->ev_in, user));
    VF_CUDA(cudaStreamWaitEvent(h->cs, h->ev_in, 0));
    return VF_OK;
}

int leave(EngineCore* h, cudaStream_t user) {
    VF_CUDA(cudaEventRecord(h->ev_out, h->cs));
    VF_CUDA(cudaStreamWaitEvent(user, h->ev_out, 0));
    return VF_OK;
}

void release(EngineCore* h) {
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (void* p : h->allocs) cudaFree(p);
    for (auto& kv : h->graphs) cudaGraphExecDestroy(kv.second.exec);
    cudaFree(h->resized);
    cudaFree(h->resize_tmp);
    if (h->cs) cudaStreamDestroy(h->cs);
    if (h->ev_in) cudaEventDestroy(h->ev_in);
    if (h->ev_out) cudaEventDestroy(h->ev_out);
}

int grow(EngineCore* h, uint8_t** p, size_t* cap, size_t need) {
    if (need <= *cap) return VF_OK;
    if (*p) {
        VF_CUDA(cudaStreamSynchronize(h->cs));
        VF_CUDA(cudaFree(*p));
        *p = nullptr; *cap = 0;
    }
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, need);
    if (e != cudaSuccess) return fail(VF_ERR_NOMEM, "%s: cudaMalloc(%zu bytes): %s", h->who, need, cudaGetErrorString(e));
    *p = static_cast<uint8_t*>(q);
    *cap = need;
    return VF_OK;
}

int upload_f32(EngineCore* h, float** dst, const float* src, size_t count) {
    if (!src) return fail(VF_ERR_INVALID, "%s: missing weight tensor", h->who);
    VF_TRY(ralloc(h, dst, count));
    VF_CUDA(cudaMemcpy(*dst, src, count * sizeof(float), cudaMemcpyHostToDevice));
    return VF_OK;
}

int upload_f16(EngineCore* h, __half** dst, const float* src, size_t rows, size_t cols, size_t ld, bool transpose) {
    if (!src) return fail(VF_ERR_INVALID, "%s: missing weight tensor", h->who);
    if (ld == 0) ld = cols;
    std::vector<__half> tmp(rows * ld, __float2half_rn(0.f));
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) tmp[r * ld + c] = __float2half_rn(transpose ? src[c * rows + r] : src[r * cols + c]);
    VF_TRY(ralloc(h, dst, rows * ld));
    VF_CUDA(cudaMemcpy(*dst, tmp.data(), tmp.size() * sizeof(__half), cudaMemcpyHostToDevice));
    return VF_OK;
}

int capture_graph(EngineCore* h, cudaStream_t s, const std::function<int()>& run, CachedGraph* g) {
    const int64_t before = h->launches;
    cudaGraph_t graph = nullptr;
    VF_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
    const int st = run();
    const cudaError_t ce = cudaStreamEndCapture(s, &graph);
    g->launches = h->launches - before;
    h->launches = before;
    if (st != VF_OK) { if (graph) cudaGraphDestroy(graph); return st; }
    if (ce != cudaSuccess) return fail(VF_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(ce));
    const cudaError_t ie = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) return fail(VF_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ie));
    return VF_OK;
}

int run_graphed(EngineCore* h, const GraphKey& key, const std::function<int()>& run) {
    if (!h->use_graph || gemm_profile_on()) return run();
    auto it = h->graphs.find(key);
    if (it == h->graphs.end()) {
        // bounded cache: ragged last chunks of many videos, or videos of many resolutions, must not pile up executable
        // graphs; an evicted graph that is still running is freed by the runtime when it completes
        const bool full = h->graphs.size() >= h->max_graphs;
        if (h->seen.size() > 4096) h->seen.clear();
        if (++h->seen[key] < h->capture_after || (full && !h->evict_when_full)) return run();
        CachedGraph g;
        VF_TRY(capture_graph(h, h->cs, run, &g));
        if (full) {
            cudaGraphExecDestroy(h->graphs.begin()->second.exec);
            h->graphs.erase(h->graphs.begin());
        }
        it = h->graphs.emplace(key, g).first;
        if (h->trace_graphs)
            fprintf(stderr, "[vf] %s: graph captured for key (%d, %d, %d, %d), %zu cached\n", h->who, key[0], key[1], key[2],
                    key[3], h->graphs.size());
    }
    VF_CUDA(cudaGraphLaunch(it->second.exec, h->cs));
    h->launches += it->second.launches;
    return VF_OK;
}

int frame_geometry(const char* who, int H, int W, int resize_to, int crop, FrameGeom* g) {
    if (H <= 0 || W <= 0) return fail(VF_ERR_INVALID, "%s: bad frame geometry %dx%d", who, H, W);
    VF_TRY(vf_resize_geometry(H, W, resize_to, 1, &g->rh, &g->rw));
    if (g->rh < crop || g->rw < crop)
        return fail(VF_ERR_INVALID, "%s: a %dx%d frame resizes to %dx%d, smaller than the %d crop", who, H, W, g->rh,
                    g->rw, crop);
    g->resize = g->rh != H || g->rw != W;
    g->cy = center_crop_offset(g->rh, crop);
    g->cx = center_crop_offset(g->rw, crop);
    return VF_OK;
}

int resize_frames(EngineCore* h, const uint8_t* frames, int n, int H, int W, const FrameGeom& g, int max_frames,
                  cudaStream_t s, const uint8_t** src) {
    *src = frames;
    if (!g.resize) return VF_OK;
    VF_TRY(grow(h, &h->resized, &h->resized_cap, size_t(max_frames) * g.rh * g.rw * 3));
    VF_TRY(grow(h, &h->resize_tmp, &h->tmp_cap, size_t(max_frames) * H * g.rw * 3));
    VF_TRY(resize_u8(frames, n, H, W, h->resized, g.rh, g.rw, g.filter, h->resize_tmp, s));
    h->launches += (g.rh != H) + (g.rw != W);
    *src = h->resized;
    return VF_OK;
}

int balanced_step(int n, int max_frames) {
    const int nchunks = (n + max_frames - 1) / max_frames;
    return nchunks > 0 ? (n + nchunks - 1) / nchunks : max_frames;
}

int debug_frames(const EngineCore* h, const void* a, const void* b, int n, int limit, const char* limit_name,
                 const char* what) {
    if (!h || !a || !b) return fail(VF_ERR_INVALID, "%s: null argument", what);
    if (n <= 0 || n > limit)
        return fail(VF_ERR_INVALID, "%s: %d frames (1 .. %d, the handle's %s)", what, n, limit, limit_name);
    VF_CUDA(cudaSetDevice(h->device));
    return VF_OK;
}

GemmEpi linear_epi(void* out, int ldo, int out_f32, const float* bias, int act, int accumulate) {
    GemmEpi e;
    memset(&e, 0, sizeof(e));
    e.out = out; e.ldo = ldo; e.out_f32 = out_f32; e.bias = bias; e.act = act; e.accumulate = accumulate;
    return e;
}

}  // namespace vf

using namespace vf;

extern "C" {

int vf_version(void) { return 2; }
const char* vf_last_error(void) { return g_err; }

int vf_sample_indices(const char* method, int param, int64_t frame_cnt, double fps, int64_t* out_idx, int64_t cap,
                      int64_t* out_n) {
    if (!method || !out_n) return fail(VF_ERR_INVALID, "sample_indices: null argument");
    int64_t n;
    if (strcmp(method, "uni") == 0) {
        n = param;                                                     // utils/utils.py:323
    } else if (strcmp(method, "fix") == 0) {
        volatile double t = double(frame_cnt) / fps;                   // utils/utils.py:315
        volatile double u = t * double(param);
        n = int64_t(u);
    } else {
        return fail(VF_ERR_UNSUPPORTED, "%s are not supported", method);   // utils/utils.py:333
    }
    if (n < 0) return fail(VF_ERR_INVALID, "Number of samples, %lld, must be non-negative.", (long long)n);
    *out_n = n;
    if (n == 0 || out_idx == nullptr) return VF_OK;   // null out_idx: size query
    if (cap < n) return fail(VF_ERR_INVALID, "sample_indices: output capacity %lld < %lld",
                                         (long long)cap, (long long)n);
    // np.linspace(1, frame_cnt - 2, n).astype(int): y[i] = i*step + start in float64 (two roundings), last = stop
    const double start = 1.0, stop = double(frame_cnt - 2);
    if (n == 1) { out_idx[0] = int64_t(start); return VF_OK; }
    const double delta = stop - start;
    const double step = delta / double(n - 1);
    for (int64_t i = 0; i < n; ++i) {
        volatile double prod = (step == 0.0) ? (double(i) / double(n - 1)) * delta : double(i) * step;
        volatile double y = prod + start;
        out_idx[i] = int64_t(y);
    }
    out_idx[n - 1] = int64_t(stop);
    return VF_OK;
}

int vf_shard_range(int64_t n_items, int n_parts, int part, int64_t* begin, int64_t* end) {
    if (n_parts <= 0 || part < 0 || part >= n_parts || !begin || !end || n_items < 0)
        return fail(VF_ERR_INVALID, "shard_range: bad arguments");
    // main.py:49-53: device_ids[:len(indices)] then torch.chunk -> chunk size ceil(n/k)
    int64_t k = n_parts < n_items ? n_parts : n_items;
    if (k <= 0) { *begin = *end = 0; return VF_OK; }
    const int64_t cs = (n_items + k - 1) / k;
    int64_t b = int64_t(part) * cs, e = b + cs;
    if (b > n_items) b = n_items;
    if (e > n_items) e = n_items;
    *begin = b;
    *end = e;
    return VF_OK;
}

int vf_resize_geometry(int in_h, int in_w, int size, int to_smaller_edge, int* out_h, int* out_w) {
    if (in_h <= 0 || in_w <= 0 || size <= 0 || !out_h || !out_w) return fail(VF_ERR_INVALID, "resize_geometry");
    // models/i3d/transforms/transforms.py:114-125 (== torchvision Resize(int) for to_smaller_edge)
    const int w = in_w, h = in_h;
    if ((w <= h && w == size) || (h <= w && h == size)) { *out_h = h; *out_w = w; return VF_OK; }
    if ((w < h) == (to_smaller_edge != 0)) { *out_w = size; *out_h = int(double(int64_t(size) * h) / double(w)); }
    else                                   { *out_h = size; *out_w = int(double(int64_t(size) * w) / double(h)); }
    return VF_OK;
}

int vf_resize_u8(const uint8_t* src, int n, int in_h, int in_w, uint8_t* dst, int out_h, int out_w, int filter,
                 uint8_t* tmp, void* stream) {
    if (!src || !dst) return fail(VF_ERR_INVALID, "resize: null buffer");
    return resize_u8(src, n, in_h, in_w, dst, out_h, out_w, filter, tmp, static_cast<cudaStream_t>(stream));
}

int vf_clip_normalize_u8(const uint8_t* src, int n, int src_h, int src_w, float* dst, void* stream) {
    if (!src || !dst) return fail(VF_ERR_INVALID, "clip_normalize: null buffer");
    if (src_h < 224 || src_w < 224) return fail(VF_ERR_INVALID, "clip_normalize: %dx%d smaller than the crop", src_h, src_w);
    if (n <= 0) return VF_OK;
    return launch_clip_normalize_f32(src, n, src_h, src_w, center_crop_offset(src_h, 224),
                                     center_crop_offset(src_w, 224), dst, static_cast<cudaStream_t>(stream));
}

int vf_gemm_profile(int enable) { return gemm_profile(enable); }
int vf_gemm_profile_read(double* ms, int64_t* launches, double* executed_flops) {
    return gemm_profile_read(ms, launches, executed_flops);
}

int vf_gemm_f16(const void* A, int lda, const void* B, int ldb, int M, int N, int K, void* D, int ldd, int out_f32,
                const float* bias, const float* scale, int act, void* stream) {
    if (!A || !B || !D) return fail(VF_ERR_INVALID, "gemm: null buffer");
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = D; ep.ldo = ldd; ep.out_f32 = out_f32; ep.bias = bias; ep.scale = scale; ep.act = act;
    return gemm_f16(static_cast<const __half*>(A), lda, static_cast<const __half*>(B), ldb, M, N, K, ep,
                    static_cast<cudaStream_t>(stream));
}

int vf_gemm_f16_accumulate(const void* A, int lda, const void* B, int ldb, int M, int N, int K, float* D, int ldd,
                           const float* bias, const float* scale, int act, void* stream) {
    if (!A || !B || !D) return fail(VF_ERR_INVALID, "gemm: null buffer");
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = D; ep.ldo = ldd; ep.out_f32 = 1; ep.bias = bias; ep.scale = scale; ep.act = act; ep.accumulate = 1;
    return gemm_f16(static_cast<const __half*>(A), lda, static_cast<const __half*>(B), ldb, M, N, K, ep,
                    static_cast<cudaStream_t>(stream));
}

int vf_gemm_f16_split(const void* A, int lda, const void* B, int ldb, int M, int N, int K, void* D, int ldd, int split_off,
                      const float* bias, const float* scale, int act, void* stream) {
    if (!A || !B || !D) return fail(VF_ERR_INVALID, "gemm: null buffer");
    if (split_off < N || ldd < split_off + N) return fail(VF_ERR_INVALID, "gemm: split output needs ldd >= split_off + N, split_off >= N");
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = D; ep.ldo = ldd; ep.out_f32 = 0; ep.bias = bias; ep.scale = scale; ep.act = act; ep.split_off = split_off;
    return gemm_f16(static_cast<const __half*>(A), lda, static_cast<const __half*>(B), ldb, M, N, K, ep,
                    static_cast<cudaStream_t>(stream));
}

int vf_conv_gemm_f16(const void* X, int C, int64_t P, const void* Wt, int N, int ntaps, int k_per_tap, const int* tap_off,
                     int nsplit, uint64_t lo_mask, int row0, const int* region, void* D, int ldd, int out_f32, int split_off,
                     const float* bias, const float* scale, int act, void* stream) {
    if (!X || !Wt || !D || !tap_off) return fail(VF_ERR_INVALID, "conv_gemm: null buffer");
    if (ntaps < 1 || ntaps > 64) return fail(VF_ERR_INVALID, "conv_gemm: %d taps (1..64)", ntaps);
    if (split_off > 0 && ldd < split_off + N)
        return fail(VF_ERR_INVALID, "conv_gemm: split output needs ldd >= split_off + N");
    ConvGeom g;
    memset(&g, 0, sizeof(g));
    g.ntaps = ntaps; g.k_per_tap = k_per_tap; g.nsplit = nsplit; g.lo_mask = lo_mask; g.row0 = row0;
    memcpy(g.tap_off, tap_off, sizeof(int) * size_t(ntaps));
    if (region) {
        g.mask = 1;
        g.Tp = region[0]; g.Hp = region[1]; g.Wp = region[2];
        g.t0 = region[3]; g.t1 = region[4]; g.h0 = region[5]; g.h1 = region[6]; g.w0 = region[7]; g.w1 = region[8];
    }
    GemmEpi ep;
    memset(&ep, 0, sizeof(ep));
    ep.out = D; ep.ldo = ldd; ep.out_f32 = out_f32; ep.bias = bias; ep.scale = scale; ep.act = act; ep.split_off = split_off;
    return conv_gemm_f16(static_cast<const __half*>(X), C, P, static_cast<const __half*>(Wt), N, g, ep,
                         static_cast<cudaStream_t>(stream));
}

}  // extern "C"
