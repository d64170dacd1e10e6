// Launchers of the VGGish audio front end and pooling kernels (vggish_kernels.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "raft_kernels.h"

namespace vf {

// resampy's time register, piecewise: outputs t in [t[s], t[s+1]) have register r[s] + (t - t[s]) * d[s], exactly the
// sequential float64 sum of 1 / ratio (inside one binade the sum advances by one fixed rounded step; a step whose
// rounding differs -- leaving a binade, or a round-half-even tie -- starts a new piece).  Passed by value.
constexpr int VGGISH_MAX_SEGS = 128;
struct TimeSegs {
    int n;
    long long t[VGGISH_MAX_SEGS];
    double r[VGGISH_MAX_SEGS], d[VGGISH_MAX_SEGS];
};
// the pieces for n_out outputs at time increment inc; VF_ERR_INVALID past VGGISH_MAX_SEGS
int vggish_time_segs(double inc, int64_t n_out, TimeSegs* S);

// Resampled mono waveform, float64, outputs [t0, t0 + count) -> out[0, count).  pcm: n_in x ch interleaved int16; the
// mono mix is (sum of the channels) / 32768 / ch.  win / delta null: 16 kHz input, out = the mono mix itself.
// Otherwise resampy 0.2.2 resample_f: scale = min(1, ratio), index_step = int(scale * num_table), left then right
// wing, every operation a separately rounded float64 op.
int vggish_resample(const int16_t* pcm, int64_t n_in, int ch, const double* win, const double* delta, int nwin,
                    int num_table, double ratio, const TimeSegs& segs, int64_t t0, int64_t count, double* out,
                    cudaStream_t s);
// frames f < n_frames of the 16 kHz waveform x (frame f = x[160 f .. 160 f + 400)): periodic Hann (hann[400]), 512-point
// FFT, magnitude, mel (mel[257][64]), log(. + 0.01), rounded to fp32 -> out[f][64].  twiddle: cos | sin of 2 pi k / 512,
// k < 256.
int vggish_logmel(const double* x, int64_t n_frames, const double* hann, const double* twiddle, const double* mel,
                  float* out, cudaStream_t s);
// conv1's input as one-tap im2col rows: logmel [n][96][64] fp32 -> X rows of the zero-bordered volume [n][98][66] of
// 32 fp16: [hi of the 3x3 neighbourhood (kh * 3 + kw), 7 zeros | lo likewise]; border rows zero.
int vggish_im2col(const float* logmel, int n, __half* X, cudaStream_t s);
// 2x2/2 max-pool of split rows [hi C | lo C] over vi's valid region -> vo (rows of ld elements, border rows zeroed).
// The winning hi / lo pair is copied; the input is post-ReLU, so there is nothing to pad.
int vggish_maxpool2(const __half* in, const Vol2& vi, int C, __half* out, const Vol2& vo, int ld, cudaStream_t s);

}  // namespace vf
