// Split-fp16 conv plumbing shared by the ResNet (resnet.cu) and CLIP ResNet (clip_resnet.cu) drivers: one uploaded
// conv (weights as a hi + lo fp16 pair with eval BatchNorm folded into the epilogue), state-dict lookup, workspace
// allocation and the launch of one conv on a zero-bordered volume of split rows [hi C | lo C] (raft_kernels.h Vol2).
#pragma once
#include <functional>
#include <string>
#include <vector>

#include "internal.h"
#include "raft_kernels.h"

namespace vf {

struct ResConv {
    int n_out = 0, ntaps = 0, k_per_tap = 0;
    int dh[4] = {0, 0, 0, 0}, dw[4] = {0, 0, 0, 0};   // per tap: shift in volume rows / columns
    unsigned long long lo_mask = 0;
    __half* w = nullptr;       // [n_out][2 * ntaps * k_per_tap]: hi pass | lo pass
    float *scale = nullptr, *bias = nullptr;
};

// What a driver handle keeps for the plumbing: `who` prefixes error messages ("resnet_create", ...), every device
// allocation is freed by the driver's destroy, and every kernel launch is counted.
struct ConvHost {
    const char* who = "";
    std::vector<void*> allocs;
    int64_t launches = 0;
};

// cudaMalloc'd, zeroed, + 64 KB: the overlapping-row TMA view of a conv input extends up to (k_per_tap - C) elements
// past its last row; zero-filled so that those elements are finite (they only feed masked border rows)
int conv_alloc_bytes(ConvHost* h, void** p, size_t bytes);
template <typename Tp>
int ralloc(ConvHost* h, Tp** p, size_t count) {
    void* q = nullptr;
    VF_TRY(conv_alloc_bytes(h, &q, count * sizeof(Tp)));
    *p = static_cast<Tp*>(q);
    return VF_OK;
}

// state_dict lookup by key, with or without the "module." prefix of a DataParallel checkpoint; a missing key or a
// wrong element count fails naming the key
struct ResTensors {
    const vf_named_tensor* t; int n; const char* who;
    int get(const std::string& name, int64_t numel, const float** out) const;
};

// eval BatchNorm (eps 1e-5) as y = x * scale + shift, folded in double
int bn_fold(const ResTensors& T, const std::string& p, int c, std::vector<float>& sc, std::vector<float>& sh);

// Uploads weight w [co][ci][k][k] as a hi + lo pair with epilogue scale sc / bias sh.  col(kh, kw, c) -> K column of
// the activation's hi half; its lo half sits lo_off columns further and gets the same weight.  reps > 1 writes every
// weight again at rep_stride, 2 * rep_stride, ... columns further (the four phase slots of a pooled 1x1 conv).
// cw.ntaps / k_per_tap / dh / dw must be set.
int upload_weights(ConvHost* h, ResConv& cw, const float* w, int co, int ci, int k, int lo_off,
                   const std::function<int(int, int, int)>& col, const std::vector<float>& sc,
                   const std::vector<float>& sh, int reps = 1, int rep_stride = 0);
// conv `name` (weight [co][ci][k][k], no bias) followed by BatchNorm `bn`: upload_weights with the folded BatchNorm,
// its scale times `scale_mul` (a power of two: exact)
int upload_conv(ConvHost* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn, int co,
                int ci, int k, int lo_off, const std::function<int(int, int, int)>& col, int reps = 1, int rep_stride = 0,
                float scale_mul = 1.f);

// stride-1 k x k (k = 1 or 3, pad k/2) on split rows of 2*ci: one tap per kernel row of k * 2ci contiguous elements.
// Also the stride-2 1x1 downsample: one tap reading phase (0, 0) = the first 2*ci elements of a phase row.
int prep_same(ConvHost* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn, int co,
              int ci, int k);
// stride-2 3x3 (pad 1) on the phase repack of split rows of 2*ci: phase row q holds x[2(q-1)+p]; tap (a, b) reads
// phase row (q + a - 1, q' + b - 1), filter index kh = 2a + ph - 1 (likewise kw with b, pw).
int prep_stride2(ConvHost* h, ResConv& cw, const ResTensors& T, const std::string& name, const std::string& bn, int co,
                 int ci);

// one conv over the volume v (rows of `pitch` elements in X) -> split rows of 2*n_out in `out`, rows outside the
// valid region zeroed
int run_conv(ConvHost* h, const ResConv& cw, const __half* X, int pitch, const Vol2& v, __half* out, bool relu,
             cudaStream_t s);

// vf_*_conv read-back: geometry, lo_mask and (when the pointers are set) the uploaded weights / scale / bias
int read_back_conv(int device, const ResConv& c, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);

}  // namespace vf
