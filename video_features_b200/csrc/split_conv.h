// Split-fp16 conv plumbing shared by the ResNet, CLIP ResNet, VGGish, R(2+1)D and S3D drivers: one uploaded conv
// (weights as a hi + lo fp16 pair with eval BatchNorm folded into the epilogue), state-dict lookup, the layouts the
// drivers share and the launch of one conv on a zero-bordered volume of split rows [hi C | lo C] (r21d_kernels.h Vol3;
// a raft_kernels.h Vol2 is its one-frame case).
#pragma once
#include <functional>
#include <string>
#include <vector>

#include "internal.h"
#include "r21d_kernels.h"
#include "raft_kernels.h"

namespace vf {

struct ResConv {
    int n_out = 0, ntaps = 0, k_per_tap = 0;
    int dt[4] = {0, 0, 0, 0}, dh[4] = {0, 0, 0, 0}, dw[4] = {0, 0, 0, 0};   // per tap: shift in frames / rows / columns
    unsigned long long lo_mask = 0;
    __half* w = nullptr;       // [n_out][2 * ntaps * k_per_tap]: hi pass | lo pass
    float *scale = nullptr, *bias = nullptr;
};

// state_dict lookup by key, with or without the "module." prefix of a DataParallel checkpoint; a missing key or a
// wrong element count fails naming the key
struct ResTensors {
    const vf_named_tensor* t; int n; const char* who;
    const vf_named_tensor* find(const std::string& name) const;     // null when absent
    int get(const std::string& name, int64_t numel, const float** out) const;
    // output channels of the (1,3,3) conv `name` over ci input channels: its weight is [co][ci][1][3][3]
    int spatial_width(const std::string& name, int ci, int* co) const;
};

// eval BatchNorm as y = x * scale + shift, folded in double
int bn_fold(const ResTensors& T, const std::string& p, int c, double eps, std::vector<float>& sc, std::vector<float>& sh);

// conv weight [co][ci][kt][kh][kw]; col(kt, kh, kw, c) -> K column of the activation's hi half
struct Filter { int co, ci, kt, kh, kw; };
using FilterCol = std::function<int(int, int, int, int)>;

// Uploads weight w as a hi + lo pair of sc.size() >= f.co output rows (rows from f.co on get zero weights; their sc / sh
// must be zero) with epilogue scale sc / bias sh.  The lo half of column col(...) sits lo_off columns further and gets
// the same weight.  reps > 1 writes every weight again at rep_stride, 2 * rep_stride, ... columns further (the four
// phase slots of a pooled 1x1 conv).  cw.ntaps / k_per_tap and the tap shifts must be set.
int upload_weights(EngineCore* h, ResConv& cw, const float* w, const Filter& f, int lo_off, const FilterCol& col,
                   const std::vector<float>& sc, const std::vector<float>& sh, int reps = 1, int rep_stride = 0);
// conv `name` (no bias) followed by BatchNorm `bn` (eps): upload_weights with the folded BatchNorm, its scale times
// `scale_mul` (a power of two: exact), output rows zero-padded to co_pad (0: none)
int upload_conv(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                double eps, const Filter& f, int lo_off, const FilterCol& col, int co_pad = 0, int reps = 1,
                int rep_stride = 0, float scale_mul = 1.f);

// stride-1 (1,k,k) (k = 1 or 3, pad k/2) on split rows of 2*ci_p (the ci filter channels, zero-padded to ci_p): one tap
// per kernel row of k * 2ci_p contiguous elements.  Also the stride-2 1x1 downsample on the phase repack: one tap
// reading phase (0, 0) = the first 2*ci elements of a phase row.
int prep_same(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
              double eps, int co, int ci, int k, int ci_p = 0, int co_pad = 0);
// stride-(1,2,2) (1,3,3) (pad 1) on the phase repack of split rows of 2*ci: phase row q holds x[2(q-1)+p]; tap (a, b)
// reads phase row (q + a - 1, q' + b - 1), filter index kh = 2a + ph - 1 (likewise kw with b, pw).
int prep_stride2(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                 double eps, int co, int ci, int co_pad = 0);
// (3,1,1) stride 1 pad 1 on split rows of 2*ci_p: 3 taps one frame apart
int prep_temporal(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
                  double eps, int co, int ci, int ci_p = 0, int co_pad = 0);
// stem (1,7,7) stride (1,2,2) pad (0,3,3) on the phase volume the transform kernels write (rows [16 hi | 16 lo],
// 4 channels per phase, 3 used): phase row q holds x[2(q-2)+p]; 4 taps (kernel row pairs), each a run of 4 phase
// positions x 32 elements
int prep_stem(EngineCore* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn,
              double eps, int co, int co_pad = 0);

// one conv over the volume v (rows of `pitch` elements in X) -> split rows [hi n_out | lo n_out] at column 0 of rows of
// ldo elements (0: 2 * n_out; split_off = ldo / 2, so a channel slice of concat rows takes ldo = 2 * concat width), rows
// outside the valid region zeroed
int run_conv(EngineCore* h, const ResConv& cw, const __half* X, int pitch, const Vol3& v, __half* out, bool relu,
             cudaStream_t s, int ldo = 0);
int run_conv(EngineCore* h, const ResConv& cw, const __half* X, int pitch, const Vol2& v, __half* out, bool relu,
             cudaStream_t s);

// ---- split-fp16 linears of the video transformers (swin3d.cu, mvit.cu)
// fp32 vector `name` of n elements -> device copy
int upload_vec(EngineCore* h, const ResTensors& T, const std::string& name, int64_t n, float** dst);
// weight [rows][cols] -> split-fp16 pair rows [hi kp | lo kp] (kp = cols_pad, 0: cols; columns from cols on zero),
// lo = fp16(w - hi), round-to-nearest-even
int upload_split_mat(EngineCore* h, const ResTensors& T, const std::string& name, int64_t rows, int64_t cols,
                     __half** dst, int64_t cols_pad = 0);
GemmEpi linear_epi(void* out, int ldo, int out_f32, const float* bias, int act, int accumulate = 0);
// out = A[M, K] . (W_hi + W_lo)^T with the epilogue `ep`: a 1-tap split-weight linear on the conv-mode GEMM (A rows of
// pitch K, no row mask), as clip_resnet.cu's linears
int split_linear(const __half* A, int M, int N, int K, const __half* W2, const GemmEpi& ep, cudaStream_t s);

// vf_*_conv read-back: geometry, lo_mask and (when the pointers are set) the uploaded weights / scale / bias
int read_back_conv(int device, const ResConv& c, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);

// the next chunk of a u8 clip entry: up to per_chunk of the n clips (first frames starts[0..n), T frames each) whose
// frames [lo, hi) fit the `slots` frames of the per-frame buffer; st gets each clip's first frame relative to lo
int clip_window(const char* who, const int* starts, int n, int T, int per_chunk, int slots, int* m, int* lo, int* hi,
                R21DStarts* st);

}  // namespace vf
