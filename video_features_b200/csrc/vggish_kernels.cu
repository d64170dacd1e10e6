// VGGish audio front end (float64, as the reference's numpy / numba code) and the trunk's 2x2 max-pool (vggish.cu).
#include <math.h>

#include "internal.h"
#include "vggish_kernels.h"

namespace vf {

int vggish_time_segs(double inc, int64_t n_out, TimeSegs* S) {
    S->n = 0;
    auto push = [&](int64_t t, double r, double d) -> int {
        if (S->n >= VGGISH_MAX_SEGS) return fail(VF_ERR_INVALID, "vggish: %lld outputs need too many time segments", (long long)n_out);
        S->t[S->n] = t; S->r[S->n] = r; S->d[S->n] = d; ++S->n;
        return VF_OK;
    };
    VF_TRY(push(0, 0.0, 0.0));
    volatile double vinc = inc;           // every sum below is one rounded float64 add, as in the sequential loop
    int64_t t = 1;
    double r = 0.0 + vinc;
    while (t < n_out) {
        const double r1 = r + vinc, r2 = r1 + vinc, d = r1 - r;
        if (r2 - r1 != d) {               // the first step's rounding differs from the next one's: r stands alone
            VF_TRY(push(t, r, 0.0));
            r = r1; t += 1;
            continue;
        }
        // r = m u with u = ulp of r's binade [2^(e-1), 2^e); r + j d stays a multiple of u below 2^e, where every
        // sequential add rounds to the same step d (r's last bit is settled after one step, so no tie alternates)
        int e;
        frexp(r, &e);
        const double u = ldexp(1.0, e - 53);
        const int64_t gap = int64_t((ldexp(1.0, e) - r) / u), q = int64_t(d / u);
        int64_t cnt = (gap - 1) / q + 1;
        if (cnt > n_out - t) cnt = n_out - t;
        VF_TRY(push(t, r, d));
        r = r + double(cnt - 1) * d;      // exact: a multiple of u below 2^e
        t += cnt;
        r = r + vinc;
    }
    return VF_OK;
}

namespace {

inline unsigned nb(int64_t total, int threads) { return unsigned((total + threads - 1) / threads); }

__device__ __forceinline__ double mono_at(const int16_t* __restrict__ pcm, int64_t j, int ch) {
    int s = 0;
    for (int c = 0; c < ch; ++c) s += __ldg(pcm + j * ch + c);
    const double v = __dmul_rn(double(s), 1.0 / 32768.0);          // the channel sum of exact v / 32768 is exact
    return ch == 1 ? v : __ddiv_rn(v, double(ch));
}

__global__ void resample_kernel(const int16_t* __restrict__ pcm, int64_t n_in, int ch, const double* __restrict__ win,
                                const double* __restrict__ delta, int nwin, int num_table, double ratio, TimeSegs segs,
                                int64_t t0, int64_t count, double* __restrict__ out) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= count) return;
    const int64_t t = t0 + idx;
    if (!win) { out[idx] = mono_at(pcm, t, ch); return; }
    int s = 0;
    while (s + 1 < segs.n && segs.t[s + 1] <= t) ++s;
    const double reg = __dadd_rn(segs.r[s], __dmul_rn(double(t - segs.t[s]), segs.d[s]));
    const double scale = ratio < 1.0 ? ratio : 1.0;
    const int step = int(__dmul_rn(scale, double(num_table)));
    const int64_t n = int64_t(reg);
    double frac = __dmul_rn(scale, __dsub_rn(reg, double(n)));
    double index_frac = __dmul_rn(frac, double(num_table));
    int offset = int(index_frac);
    double eta = __dsub_rn(index_frac, double(offset));
    double y = 0.0;
    const int64_t i_max = min(n + 1, int64_t((nwin - offset) / step));
    for (int64_t i = 0; i < i_max; ++i) {
        const int o = offset + int(i) * step;
        const double w = __dadd_rn(__ldg(win + o), __dmul_rn(eta, __ldg(delta + o)));
        y = __dadd_rn(y, __dmul_rn(w, mono_at(pcm, n - i, ch)));
    }
    frac = __dsub_rn(scale, frac);
    index_frac = __dmul_rn(frac, double(num_table));
    offset = int(index_frac);
    eta = __dsub_rn(index_frac, double(offset));
    const int64_t k_max = min(n_in - n - 1, int64_t((nwin - offset) / step));
    for (int64_t k = 0; k < k_max; ++k) {
        const int o = offset + int(k) * step;
        const double w = __dadd_rn(__ldg(win + o), __dmul_rn(eta, __ldg(delta + o)));
        y = __dadd_rn(y, __dmul_rn(w, mono_at(pcm, n + k + 1, ch)));
    }
    out[idx] = y;
}

// one block of 256 threads per frame: radix-2 decimation-in-time FFT of the 512 zero-padded windowed samples in shared
// memory (bit-reversed load, nine butterfly stages), |X_k| by hypot, the mel dot in four partial sums of 65 bins
__global__ void __launch_bounds__(256) logmel_kernel(const double* __restrict__ x, const double* __restrict__ hann,
                                                     const double* __restrict__ twiddle, const double* __restrict__ mel,
                                                     float* __restrict__ out) {
    __shared__ double re[512], im[512], mag[260], part[4][64];
    const int tid = threadIdx.x;
    const int64_t f = blockIdx.x;
    const double* src = x + f * 160;
    for (int j = tid; j < 512; j += 256) {
        const int r = __brev(unsigned(j)) >> 23;
        re[r] = j < 400 ? __dmul_rn(__ldg(src + j), __ldg(hann + j)) : 0.0;
        im[r] = 0.0;
    }
    __syncthreads();
    for (int half = 1; half < 512; half <<= 1) {
        const int k = tid & (half - 1), i = ((tid - k) << 1) + k, j = i + half;
        const int tw = k * (256 / half);
        const double c = __ldg(twiddle + tw), sn = -__ldg(twiddle + 256 + tw);    // e^{-2 pi i tw / 512}
        const double tr = c * re[j] - sn * im[j], ti = c * im[j] + sn * re[j];
        const double ar = re[i], ai = im[i];
        re[j] = ar - tr; im[j] = ai - ti;
        re[i] = ar + tr; im[i] = ai + ti;
        __syncthreads();
    }
    for (int k = tid; k < 257; k += 256) mag[k] = hypot(re[k], im[k]);
    __syncthreads();
    const int band = tid & 63, q = tid >> 6;
    double acc = 0.0;
    for (int k = q * 65; k < min(257, (q + 1) * 65); ++k) acc += mag[k] * __ldg(mel + k * 64 + band);
    part[q][band] = acc;
    __syncthreads();
    if (tid < 64) {
        const double m = (part[0][band] + part[1][band]) + (part[2][band] + part[3][band]);
        out[f * 64 + band] = float(log(m + 0.01));
    }
}

__global__ void im2col_kernel(const float* __restrict__ lm, int n, __half* __restrict__ X) {
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(n) * 98 * 66) return;
    const int xq = int(idx % 66), yq = int((idx / 66) % 98), b = int(idx / (98 * 66));
    __align__(16) __half v[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = __float2half_rn(0.f);
    if (yq >= 1 && yq <= 96 && xq >= 1 && xq <= 64) {
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int y = yq - 2 + a, x = xq - 2 + d;
                if (y < 0 || y >= 96 || x < 0 || x >= 64) continue;
                const float f = __ldg(lm + (int64_t(b) * 96 + y) * 64 + x);
                const __half hi = __float2half_rn(f);
                v[a * 3 + d] = hi;
                v[16 + a * 3 + d] = __float2half_rn(f - __half2float(hi));
            }
    }
    uint4* o = reinterpret_cast<uint4*>(X + idx * 32);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = reinterpret_cast<const uint4*>(v)[i];
}

__global__ void maxpool2_kernel(const __half* __restrict__ in, Vol2 vi, int C, __half* __restrict__ out, Vol2 vo, int ld) {
    const int cg = C >> 3;
    const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= int64_t(vo.n) * vo.Hp * vo.Wp * cg) return;
    const int c8 = int(idx % cg);
    const int64_t pos = idx / cg;
    const int wq = int(pos % vo.Wp), hq = int((pos / vo.Wp) % vo.Hp), b = int(pos / (int64_t(vo.Wp) * vo.Hp));
    __half* o = out + pos * ld + c8 * 8;
    if (hq < vo.h0 || hq >= vo.h1 || wq < vo.w0 || wq >= vo.w1) {
        *reinterpret_cast<uint4*>(o) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(o + C) = make_uint4(0, 0, 0, 0);
        return;
    }
    const int i = hq - vo.h0, j = wq - vo.w0;
    float best[8];
    __align__(16) __half bh[8], bl[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) best[k] = -INFINITY;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const __half* p = in + ((int64_t(b) * vi.Hp + 2 * i + dy + vi.h0) * vi.Wp + 2 * j + dx + vi.w0) * (2 * C) + c8 * 8;
            const uint4 h4 = __ldg(reinterpret_cast<const uint4*>(p)), l4 = __ldg(reinterpret_cast<const uint4*>(p + C));
            const __half *ph = reinterpret_cast<const __half*>(&h4), *pl = reinterpret_cast<const __half*>(&l4);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float v = __half2float(ph[k]) + __half2float(pl[k]);
                if (v > best[k]) { best[k] = v; bh[k] = ph[k]; bl[k] = pl[k]; }
            }
        }
    *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(bh);
    *reinterpret_cast<uint4*>(o + C) = *reinterpret_cast<const uint4*>(bl);
}

}  // namespace

#define LAUNCH_CHECK() do { VF_CUDA(cudaGetLastError()); return VF_OK; } while (0)

int vggish_resample(const int16_t* pcm, int64_t n_in, int ch, const double* win, const double* delta, int nwin,
                    int num_table, double ratio, const TimeSegs& segs, int64_t t0, int64_t count, double* out,
                    cudaStream_t s) {
    if (count <= 0) return VF_OK;
    resample_kernel<<<nb(count, 128), 128, 0, s>>>(pcm, n_in, ch, win, delta, nwin, num_table, ratio, segs, t0, count, out);
    LAUNCH_CHECK();
}
int vggish_logmel(const double* x, int64_t n_frames, const double* hann, const double* twiddle, const double* mel,
                  float* out, cudaStream_t s) {
    if (n_frames <= 0) return VF_OK;
    logmel_kernel<<<unsigned(n_frames), 256, 0, s>>>(x, hann, twiddle, mel, out);
    LAUNCH_CHECK();
}
int vggish_im2col(const float* logmel, int n, __half* X, cudaStream_t s) {
    const int64_t total = int64_t(n) * 98 * 66;
    im2col_kernel<<<nb(total, 256), 256, 0, s>>>(logmel, n, X);
    LAUNCH_CHECK();
}
int vggish_maxpool2(const __half* in, const Vol2& vi, int C, __half* out, const Vol2& vo, int ld, cudaStream_t s) {
    const int64_t total = vo.rows() * (C / 8);
    maxpool2_kernel<<<nb(total, 256), 256, 0, s>>>(in, vi, C, out, vo, ld);
    LAUNCH_CHECK();
}

}  // namespace vf
