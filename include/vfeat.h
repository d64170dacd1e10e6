/* libvfeat.so -- C ABI of the H100-native video-feature engine.
 *
 * Every entry point is `extern "C"`, takes plain pointers and sizes, returns an int status
 * (VF_OK == 0) and never throws.  Device buffers are raw CUDA device pointers owned by the
 * caller; `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Handles
 * are opaque, own their device weights + workspace, and are not shared between threads.
 *
 * Each function names the reference interface it replaces
 * (Kamino666/video_features @ dc9df59e, paths relative to the reference root).
 */
#ifndef VFEAT_H_
#define VFEAT_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VF_OK 0
#define VF_ERR_INVALID 1   /* bad argument */
#define VF_ERR_CUDA 2      /* a CUDA runtime / driver call failed */
#define VF_ERR_NOMEM 3
#define VF_ERR_UNSUPPORTED 4

#define VF_ACT_NONE 0
#define VF_ACT_QUICKGELU 1 /* x * sigmoid(1.702 x) */
#define VF_ACT_RELU 2
#define VF_ACT_SIGMOID 3
#define VF_ACT_TANH 4
#define VF_ACT_LEAKY 5     /* LeakyReLU(0.1): built for the conv mode with split weights (nsplit = 2) only */
#define VF_ACT_GELU 6      /* exact GELU, 0.5 x (1 + erf(x / sqrt 2)): built for the plain GEMM (vf_gemm_f16) and the
                              conv mode with split weights (nsplit = 2), without split output, only */

#define VF_FILTER_BILINEAR 2 /* PIL.Image.BILINEAR */
#define VF_FILTER_BICUBIC 3  /* PIL.Image.BICUBIC  */

/* ABI version; bumped on any signature change. */
int vf_version(void);
/* Text of the last error raised on the calling thread ("" if none). */
const char* vf_last_error(void);

/* ---- sampler: utils/utils.py:297-333 `extract_frames` index arithmetic -------------------------
 * method "uni": n = param; "fix": n = (int)(frame_cnt / fps * param).  Writes
 * np.linspace(1, frame_cnt-2, n).astype(int) into out_idx (capacity cap) and n into *out_n;
 * out_idx == NULL only queries n. */
int vf_sample_indices(const char* method, int param, int64_t frame_cnt, double fps, int64_t* out_idx, int64_t cap,
                      int64_t* out_n);
/* contiguous chunk shard of `n_items` over `n_parts` as torch.chunk does (main.py:49-53):
 * part p gets [*begin, *end); parts beyond the last non-empty chunk get begin == end. */
int vf_shard_range(int64_t n_items, int n_parts, int part, int64_t* begin, int64_t* end);

/* ---- PIL-compatible resample: Pillow Image.resize as used by torchvision Resize in the CLIP
 * transform (models/CLIP/extract_clip.py:112) and models/i3d/transforms/transforms.py:121,125.
 * src: n frames HWC uint8 (3 channels) on the device; dst: n x out_h x out_w x 3 uint8.
 * tmp: device scratch of n*in_h*out_w*3 bytes (horizontal pass output); byte-exact with Pillow. */
int vf_resize_u8(const uint8_t* src, int n, int in_h, int in_w, uint8_t* dst, int out_h, int out_w, int filter,
                 uint8_t* tmp, void* stream);
/* output geometry of "short side -> size" (torchvision Resize(int) / ResizeImproved). */
int vf_resize_geometry(int in_h, int in_w, int size, int to_smaller_edge, int* out_h, int* out_w);

/* ---- CLIP transform: ToTensor + Normalize + CenterCrop(224) (clip.clip._transform as invoked at
 * models/CLIP/extract_clip.py:107-113,125-126).  src: n x src_h x src_w x 3 uint8 (already
 * resized); dst: n x 3 x 224 x 224 fp32, bit-exact with torchvision's fp32 arithmetic. */
int vf_clip_normalize_u8(const uint8_t* src, int n, int src_h, int src_w, float* dst, void* stream);

/* ---- tensor-core GEMM (exported for the parity tests): D = act(A . B^T * scale + bias)
 * A: M x K fp16 (row pitch lda elements), B: N x K fp16 (torch Linear weight layout),
 * D: fp16 or fp32 (out_f32, row pitch ldd elements, 16-byte aligned rows), bias/scale: fp32 [N] or NULL. */
int vf_gemm_f16(const void* A, int lda, const void* B, int ldb, int M, int N, int K, void* D, int ldd, int out_f32,
                const float* bias, const float* scale, int act, void* stream);
/* D += act(A . B^T * scale + bias), D fp32: added by fp32 global reductions from the GEMM epilogue, each element exactly once -- the
 * residual-stream update `x = x + attn(...)` / `x = x + mlp(...)` of clip/model.py ResidualAttentionBlock.forward. */
int vf_gemm_f16_accumulate(const void* A, int lda, const void* B, int ldb, int M, int N, int K, float* D, int ldd,
                           const float* bias, const float* scale, int act, void* stream);
/* Same GEMM with the result written as a split-fp16 pair: D[m][n] = fp16(v) and D[m][split_off + n] = fp16(v - fp16(v))
 * (split_off >= N, multiple of 8, ldd >= split_off + N).  RAFT's GEMM -> GEMM activations are carried this way: the
 * consumer's weights are duplicated over both halves, which restores ~22 mantissa bits on the activation operand. */
int vf_gemm_f16_split(const void* A, int lda, const void* B, int ldb, int M, int N, int K, void* D, int ldd, int split_off,
                      const float* bias, const float* scale, int act, void* stream);
/* The same GEMM in its shifted-row convolution mode, the one every I3D / RAFT convolution runs (exported for the parity
 * tests).  X holds channels-last rows of C elements (fp16, row pitch C); row p of the A operand of tap j is the
 * k_per_tap contiguous elements starting at element (p + tap_off[j]) * C, so X must be readable for (P-1)*C + k_per_tap
 * elements, and rows that fall before 0 or at / past P read as zeros.  Wt: N x (nsplit*ntaps*k_per_tap) fp16, row-major,
 * tap j at columns j*k_per_tap; nsplit = 2 appends the lo halves of a hi+lo weight pair after all the hi columns.
 * lo_mask (nsplit = 2): bit kk skips the W_lo pass on K block kk (64 columns) of every tap; bits must name existing
 * blocks of a tap of at most 64 blocks.  region: NULL (no mask) or {Tp, Hp, Wp, t0, t1, h0, h1, w0, w1}: output row m
 * is volume position m - row0 of [n][Tp][Hp][Wp] and is written as 0 outside [t0,t1) x [h0,h1) x [w0,w1) and for
 * m < row0.  D: P rows of pitch ldd, fp16 or fp32 (out_f32); split_off > 0 writes a split-fp16 pair as vf_gemm_f16_split
 * does.  1 <= ntaps <= 64, C and k_per_tap multiples of 8, N a multiple of 8. */
int vf_conv_gemm_f16(const void* X, int C, int64_t P, const void* Wt, int N, int ntaps, int k_per_tap, const int* tap_off,
                     int nsplit, uint64_t lo_mask, int row0, const int* region, void* D, int ldd, int out_f32, int split_off,
                     const float* bias, const float* scale, int act, void* stream);

/* Roofline instrumentation (bench.py): while enabled on the calling thread, every wgmma GEMM launch of any handle
 * is bracketed by CUDA events on its stream.  _read synchronises the device and returns the summed device time (ms),
 * the launch count and the EXECUTED flops (2*M*N*K including zero-padded K blocks and hi/lo weight passes). */
int vf_gemm_profile(int enable);
int vf_gemm_profile_read(double* ms, int64_t* launches, double* executed_flops);

/* ---- CLIP ViT-B/32 image tower: replaces `clip.load(...)` + `model.encode_image(frames)`
 * (models/CLIP/extract_clip.py:47,128).  Weight pointers are HOST fp32 arrays in openai layout. */
typedef struct vf_clip_layer_weights {
    const float *ln_1_w, *ln_1_b;           /* [768] */
    const float *in_proj_w, *in_proj_b;     /* [2304,768], [2304] */
    const float *out_proj_w, *out_proj_b;   /* [768,768], [768] */
    const float *ln_2_w, *ln_2_b;           /* [768] */
    const float *c_fc_w, *c_fc_b;           /* [3072,768], [3072] */
    const float *c_proj_w, *c_proj_b;       /* [768,3072], [768] */
} vf_clip_layer_weights;

typedef struct vf_clip_weights {
    const float* conv1_w;                   /* [768,3,32,32] */
    const float* class_embedding;           /* [768] */
    const float* positional_embedding;      /* [50,768] */
    const float *ln_pre_w, *ln_pre_b, *ln_post_w, *ln_post_b; /* [768] */
    const float* proj;                      /* [768,512] */
    vf_clip_layer_weights layers[12];
} vf_clip_weights;

typedef struct vf_clip vf_clip_t;

/* Uploads weights to `device` (fp16 GEMM operands, fp32 vectors) and allocates workspace for
 * chunks of `chunk_frames` frames (0 = default). */
int vf_clip_create(vf_clip_t** out, const vf_clip_weights* w, int device, int chunk_frames);
/* Same for the reference's other ViT-B feature type: patch_size 32 ('CLIP-ViT-B/32', identical to vf_clip_create) or 16
 * ('CLIP-ViT-B/16': conv1_w is [768,3,16,16], positional_embedding [197,768]; same width, depth, heads and output size).
 * Reference: models/CLIP/extract_clip.py:42-47 (clip.load(feature_type) for either name). */
int vf_clip_create_vit(vf_clip_t** out, const vf_clip_weights* w, int device, int chunk_frames, int patch_size);
int vf_clip_destroy(vf_clip_t* h);
/* encode_image on n already-transformed frames: frames n x 3 x 224 x 224 fp32 (device) -> out n x 512 fp32. */
int vf_clip_encode_f32(vf_clip_t* h, const float* frames, int n, float* out, void* stream);
/* Fused transform + encode_image: frames n x src_h x src_w x 3 uint8 (device, as the decoder delivers
 * them, channel order untouched) -> Resize(224,bicubic) -> CenterCrop(224) -> normalise -> tower. */
int vf_clip_encode_u8(vf_clip_t* h, const uint8_t* frames, int n, int src_h, int src_w, float* out, void* stream);
/* Same with HOST buffers: stages H2D copies of the frames and the D2H copy of the features on
 * `stream` and synchronises it before returning (the call ExtractCLIP.extract makes per video). */
int vf_clip_encode_u8_host(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_host,
                           void* stream);
/* Host frames in, features left ON THE DEVICE in out_dev (n x 512 fp32, ordered on `stream`) -- what a rank hands to the
 * all-gather of main.py's --device_ids dispatch (main.py:49-53) -- and, when out_host is not NULL, copied to the host as
 * well.  Returns once the host frames have been consumed (and out_host, if given, is complete). */
int vf_clip_encode_u8_host_dev(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_dev,
                               float* out_host, void* stream);

/* Asynchronous form of the two calls above: returns once the copies and kernels are enqueued.  `frames_host` and `out_host`
 * must be pinned and stay untouched until vf_clip_wait(h, *ticket) returns; out_dev (may be NULL) is ordered on `stream`
 * like any other device output.  Calls in flight share the handle's staging slots under event ordering, so the H2D copy
 * of call k+1 overlaps the tower of call k -- the pattern of a list of videos (reference: the per-video loop of
 * models/CLIP/extract_clip.py:70-88, where nothing overlaps).  At most 4 calls are in flight; a fifth blocks on the
 * oldest.  One enqueuing host thread per handle; vf_clip_wait may be called from another thread. */
int vf_clip_encode_u8_host_async(vf_clip_t* h, const uint8_t* frames_host, int n, int src_h, int src_w, float* out_dev,
                                 float* out_host, void* stream, int64_t* ticket);
int vf_clip_wait(vf_clip_t* h, int64_t ticket);
/* Diagnostics / parity tests: the attention half of resblock `layer` alone -- x: n_frames*50 x 768 fp16 (the ln_1 output),
 * out: n_frames*50 x 768 fp16 = concat_heads(softmax(q k^T / 8) v) BEFORE the out-projection (third-party clip
 * ResidualAttentionBlock.attention / nn.MultiheadAttention).  fused = 1: the QKV-projection + attention kernel the tower
 * runs; fused = 0: QKV GEMM, then the stand-alone attention kernel. */
int vf_clip_block_attention(vf_clip_t* h, int layer, const void* x, int n_frames, void* out, int fused, void* stream);
/* Diagnostics / parity tests: the three pieces the tower consists of, one at a time.  They run the functions the encode
 * calls run (eagerly, on the caller's stream, on the handle's first workspace; no CUDA graph is captured or replayed), take
 * 1 <= n <= the handle's chunk_frames frames (VF_ERR_INVALID otherwise, before any launch), and must not overlap an
 * asynchronous call in flight.  T = tokens per frame (50 / 197); all buffers are on the device.
 *   embed:  patchify, the patch-embedding GEMM, class / positional embedding + ln_pre -> x_out, the fp32 residual stream
 *           n*T x 768.  _f32 takes frames n x 3 x 224 x 224 as vf_clip_encode_f32 does, _u8 frames n x src_h x src_w x 3
 *           as vf_clip_encode_u8 does.
 *   blocks: resblocks [layer_begin, layer_end) of 0 .. 12 on the residual stream x (n_frames*T x 768 fp32, in place), by
 *           the handle's configured path (fused or split attention; VF_CLIP_RESID=acc|y|mix).  When layer_end == 12 the
 *           last block runs on the class-token rows only, as in the tower: afterwards only rows frame*T of x are defined.
 *           In the y forms the MLP increment of block layer_end - 1, which the tower would add in the next LayerNorm
 *           pass, is added to x (fp32) before returning, by the same add + LayerNorm kernel with its LayerNorm output
 *           dropped: x holds the same fp32 values the next pass would have normalised.
 *   head:   ln_post on rows frame*T of x (row pitch T*768) and the 768 -> 512 projection -> out, n_frames x 512 fp32.
 * embed -> blocks(0, 12) -> head gives the bits of vf_clip_encode_f32 / _u8. */
int vf_clip_debug_embed_f32(vf_clip_t* h, const float* frames, int n, float* x_out, void* stream);
int vf_clip_debug_embed_u8(vf_clip_t* h, const uint8_t* frames, int n, int src_h, int src_w, float* x_out, void* stream);
int vf_clip_debug_blocks(vf_clip_t* h, float* x, int n_frames, int layer_begin, int layer_end, void* stream);
int vf_clip_debug_head(vf_clip_t* h, const float* x, int n_frames, float* out, void* stream);
/* number of kernels this library has launched on behalf of `h` so far (diagnostics / bench). */
int64_t vf_clip_launch_count(const vf_clip_t* h);
/* Roofline instrumentation for bench.py: while enabled, every tensor-core GEMM launch of `h` is bracketed by a
 * pair of CUDA events recorded on the launching stream.  vf_clip_profile_read synchronises the device, returns the
 * summed GEMM device time (ms), the number of GEMM launches and their algorithmic FLOPs (2*M*N*K), and resets. */
int vf_clip_profile(vf_clip_t* h, int enable);
int vf_clip_profile_read(vf_clip_t* h, double* gemm_ms, int64_t* gemm_launches, double* gemm_flops);
/* device ms per kernel category of the last vf_clip_profile_read window: [0] GEMM, [1] LayerNorm, [2] attention,
 * [3] frame transform (resize / normalise / patchify). */
int vf_clip_profile_categories(const vf_clip_t* h, double* ms4);

/* ---- I3D (Inception-3D) feature extractor: replaces `I3D(400, modality)(x, features=True)`
 * (models/i3d/i3d_src/i3d_net.py:238-264, called at models/i3d/extract_i3d.py:186).
 * One conv unit = Conv3d (no bias) + BatchNorm3d (eval) + ReLU (Unit3Dpy, i3d_net.py:37-105); weights are HOST fp32
 * in the checkpoint's own layout.  Unit order: conv3d_1a_7x7, conv3d_2b_1x1, conv3d_2c_3x3, then for each of
 * mixed_3b,3c,4b,4c,4d,4e,4f,5b,5c: branch_0, branch_1.0, branch_1.1, branch_2.0, branch_2.1, branch_3.1. */
#define VF_I3D_UNITS 57
typedef struct vf_conv_unit {
    const float* w;                               /* [cout, cin, k, k, k] */
    const float *bn_w, *bn_b, *bn_mean, *bn_var;  /* [cout] */
    int cout, cin, k;
} vf_conv_unit;
typedef struct vf_i3d_weights {
    vf_conv_unit units[VF_I3D_UNITS];
} vf_i3d_weights;
typedef struct vf_i3d vf_i3d_t;

/* in_channels: 3 (rgb stream) or 2 (flow stream).  Workspace is sized for max_stacks clips of max_T frames. */
int vf_i3d_create(vf_i3d_t** out, const vf_i3d_weights* w, int in_channels, int device, int max_stacks, int max_T);
int vf_i3d_destroy(vf_i3d_t* h);
/* clips: n x C x T x 224 x 224 fp32 on the device (the tensor the reference passes to I3D) -> out n x 1024 fp32. */
int vf_i3d_forward_f32(vf_i3d_t* h, const float* clips, int n, int T, float* out, void* stream);
/* rgb stream with the T2 transform fused (extract_i3d.py:62-66): frames n x T x Hr x Wr x 3 uint8 on the device,
 * already resized (vf_resize_u8, bilinear, short side 256) -> TensorCenterCrop(224) -> 2x/255-1 -> I3D. */
int vf_i3d_forward_u8(vf_i3d_t* h, const uint8_t* frames, int n, int T, int Hr, int Wr, float* out, void* stream);
/* same, stack b = frames [b * stack_stride, b * stack_stride + T) of the buffer (stack_stride >= T, in frames): the rgb
 * stream of the reference is `stack[:-1]` of the 65-frame stacks the flow stream also reads (extract_i3d.py:150-158). */
int vf_i3d_forward_u8_strided(vf_i3d_t* h, const uint8_t* frames, int n, int T, int64_t stack_stride, int Hr, int Wr,
                              float* out, void* stream);
/* flow stream with the T3 transform fused (extract_i3d.py:67-73): flow n x T x 2 x H x W fp32 on the device (the RAFT
 * output, still padded) -> crop 224 -> clamp(+-20) -> 128+255/40 f -> round -> 2x/255-1 -> I3D. */
int vf_i3d_forward_flow(vf_i3d_t* h, const float* flow, int n, int T, int H, int W, float* out, void* stream);
/* Diagnostics: copy a retained internal activation (0: conv3d_1a, 1: conv3d_2c, 2: mixed_3c, 3: mixed_4f, 4: mixed_5c)
 * of the last forward (of its last chunk of max_stacks clips) to fp32 NCTHW; dims5 receives (n, C, T, H, W); out == NULL
 * only queries the shape. */
int vf_i3d_read_stage(vf_i3d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream);
int64_t vf_i3d_launch_count(const vf_i3d_t* h);
/* Diagnostics: unit `index` (0 .. VF_I3D_UNITS - 1, the order of vf_i3d_weights) as uploaded.  geom receives 196 ints:
 * n_out, ntaps, k_per_tap, nsplit (2: W_hi | W_lo along K, 1: single fp16 weights), then (dt, dh, dw) of taps 0..63 (the
 * row shift of tap j on a volume of Tp x Hp x Wp rows is (dt Hp + dh) Wp + dw); lo_mask its K blocks without a W_lo
 * pass.  w (n_out x nsplit ntaps k_per_tap fp16), scale and bias (n_out fp32, the folded BatchNorm) are DEVICE buffers
 * filled when not NULL.  An index past the last unit is VF_ERR_INVALID. */
int vf_i3d_conv(const vf_i3d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);
/* Diagnostics: Mixed block `block` (0 .. 8: mixed_3b .. mixed_5c) once, on the engine's uploaded weights, buffers and
 * kernels.  x_pairs: DEVICE fp16 pair volume [n][T+2][S+2][S+2][2 cin] (rows [hi cin | lo cin], border 1, zero border)
 * with S = 28 (blocks 0, 1), 14 (2 .. 6), 7 (7, 8); out_pairs receives the concat pair volume [n][T+2][S+2][S+2]
 * [2 ctot] (rows [hi ctot | lo ctot], branches in order, border rows included).  The volume goes through the engine's
 * own activation buffers: more rows than the workspace holds is VF_ERR_INVALID before any launch, and afterwards
 * vf_i3d_read_stage is VF_ERR_INVALID until the next forward. */
int vf_i3d_debug_mixed(vf_i3d_t* h, int block, const void* x_pairs, int n, int T, void* out_pairs, void* stream);

/* ---- RAFT optical flow: replaces `RAFT()(image1, image2, iters=20, test_mode=True)` + InputPadder
 * (models/raft/raft_src/raft.py:27-44,115-174; called at models/raft/extract_raft.py:94-104 and
 * models/i3d/extract_i3d.py:172).  Weights: the checkpoint's tensors by name (keys of raft-sintel.pth without the
 * "module." prefix), HOST fp32. */
typedef struct vf_named_tensor {
    const char* name;
    const float* data;
    int64_t numel;
} vf_named_tensor;
typedef struct vf_raft vf_raft_t;

/* Workspace is sized for windows of max_frames frames of at most max_h x max_w pixels (before /8 padding). */
int vf_raft_create(vf_raft_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames, int max_h,
                   int max_w);
int vf_raft_destroy(vf_raft_t* h);
/* Flow between consecutive frames of a window: frames n_frames x (Hs x Ws x 3 if !chw_layout else 3 x Hs x Ws), uint8
 * or fp32 in [0,255] on the device, RGB order as given; == model(pad(frames)[:-1], pad(frames)[1:]).
 * out: (n_frames-1) x 2 x Ho x Wo fp32 with (Ho,Wo) = (Hs,Ws) if unpad (extract_raft.py:101) else the /8-padded size
 * (extract_i3d.py:172 never unpads; query it with vf_raft_padded_size). */
int vf_raft_flow(vf_raft_t* h, const void* frames, int is_u8, int chw_layout, int n_frames, int Hs, int Ws, int iters,
                 int unpad, float* out, void* stream);
int vf_raft_padded_size(int Hs, int Ws, int* H, int* W);
/* Diagnostics: internal tensors of the last call as fp32 NCHW at 1/8 resolution.  what: 0 fnet features (all
 * frames), 1 cnet output (raw), 2 GRU hidden state, 3 low-res flow, 4 last correlation lookup (324 ch),
 * 5 the correlation pyramid rows (n, H8*W8, 1, row pitch): level l at cumulative offset of the level sizes. */
int vf_raft_debug_read(vf_raft_t* h, int what, float* out, int64_t capacity, int* dims4, void* stream);
int64_t vf_raft_launch_count(const vf_raft_t* h);
/* Diagnostics: conv `index` as uploaded, as vf_i3d_conv (dt is 0).  Order: per encoder (fnet, then cnet) conv1,
 * layer1's four convs, layer2's conv1, downsample, three convs, the same for layer3, conv2 (16 each); then the update
 * block's convc1, convc2, convf1, convf2, conv, the stacked convz1|convr1, convq1, convz2|convr2, convq2, the flow head's
 * conv1, conv2 and the mask head's mask.0, mask.2 (45 in all).  n_out is the GEMM width (padded rows included). */
int vf_raft_conv(const vf_raft_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);

/* ---- PWC-Net optical flow: replaces `PWCNet()(first, second)` (models/pwc/pwc_src/pwc_net.py:212-263, with
 * correlation.py's cost volume; called at models/pwc/extract_pwc.py:97 and models/i3d/extract_i3d.py:175).  Weights: the
 * checkpoint's tensors by name (keys of pwc_net_sintel.pt), HOST fp32. */
typedef struct vf_pwc vf_pwc_t;

/* Workspace is sized for calls of max_frames frames of at most max_h x max_w pixels (each rounded up to 64). */
int vf_pwc_create(vf_pwc_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames, int max_h,
                  int max_w);
int vf_pwc_destroy(vf_pwc_t* h);
/* Flow between consecutive frames: frames n_frames x (Hs x Ws x 3 if !chw_layout else 3 x Hs x Ws), uint8 or fp32 in
 * [0,255] on the device, passed as the reference's caller passes them (the model swaps channels 0 and 2 itself);
 * == model(frames[:-1], frames[1:]).  out: (n_frames-1) x 2 x Hs x Ws fp32. */
int vf_pwc_flow(vf_pwc_t* h, const void* frames, int is_u8, int chw_layout, int n_frames, int Hs, int Ws, float* out,
                void* stream);
/* Diagnostics: tensors of the last call as fp32 NCHW at pyramid level `level` (1..6: 1/2 .. 1/64 of the size rounded up
 * to 64).  what: 0 extractor features (all frames), 1 cost volume after the LeakyReLU (81 ch), 2 upsampled flow
 * (moduleUpflow, levels 2..5), 3 upsampled feature (moduleUpfeat, levels 2..5), 4 decoder flow, 5 refiner output (level
 * 2; `level` ignored), 6 warp mask (levels 2..5).  dims4 receives the shape; out == NULL only queries it. */
int vf_pwc_debug_read(vf_pwc_t* h, int what, int level, float* out, int64_t capacity, int* dims4, void* stream);
int64_t vf_pwc_launch_count(const vf_pwc_t* h);
/* Diagnostics: conv `index` as uploaded, as vf_raft_conv.  Order: the extractor's three convs per level 1..6; per decoder
 * level 6, 5, 4, 3, 2: moduleUpflow, moduleUpfeat (not at level 6; ConvTranspose2d as 9 taps x 8 columns (py*2+px)*2 +
 * oc), moduleOne .. moduleSix; the refiner's seven convs (63 in all).  Weights carry a power-of-two scale 2^e per output
 * row (largest |w| in [2^14, 2^15), e <= 126) and scale holds 2^-e. */
int vf_pwc_conv(const vf_pwc_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);

/* ---- ResNet-18/34/50/101/152 frame features: replaces torchvision `models.resnetXX(pretrained=True)` with
 * `fc = Identity()` in eval mode, and its per-frame transform Resize(256) -> CenterCrop(224) -> ToTensor -> Normalize
 * (models/resnet/extract_resnet.py:32-38,52-72,108).  Weights: the torchvision state_dict by key (optionally with the
 * "module." prefix), HOST fp32; fc.* is ignored.  An unknown depth, or a missing / mis-sized tensor, is VF_ERR_INVALID. */
typedef struct vf_resnet vf_resnet_t;

/* depth: 18, 34, 50, 101 or 152.  Workspace holds max_frames frames (0 = 64); larger calls run in chunks of that size. */
int vf_resnet_create(vf_resnet_t** out, const vf_named_tensor* tensors, int n_tensors, int depth, int device, int max_frames);
int vf_resnet_destroy(vf_resnet_t* h);
/* frames: n x 3 x 224 x 224 fp32 on the device, already transformed (the tensor the reference passes to the model)
 * -> out: n x D fp32 (D = 512 for depths 18 / 34, 2048 otherwise). */
int vf_resnet_forward_f32(vf_resnet_t* h, const float* frames, int n, float* out, void* stream);
/* transform fused: frames n x Hr x Wr x 3 uint8 BGR on the device (the decoder's order), already resized to short side
 * 256 (vf_resize_u8, bilinear) -> BGR->RGB, CenterCrop(224), ToTensor, Normalize -> network.  Hr, Wr >= 224. */
int vf_resnet_forward_u8(vf_resnet_t* h, const uint8_t* frames, int n, int Hr, int Wr, float* out, void* stream);
/* Diagnostics: an activation of the last chunk of the last call as fp32 NCHW: stage 0 stem (conv1 + bn1 + relu),
 * 1 maxpool, 2..5 layer1..layer4.  dims4 receives (n, C, H, W); out == NULL only queries the shape. */
int vf_resnet_read_stage(vf_resnet_t* h, int stage, float* out, int64_t capacity, int* dims4, void* stream);
int64_t vf_resnet_launch_count(const vf_resnet_t* h);
/* Diagnostics: conv `index` of the trunk as uploaded, in execution order (the stem, then per block conv1, conv2, conv3
 * of a bottleneck, the downsample if any).  geom receives 15 ints: n_out, ntaps, k_per_tap, then (dt, dh, dw) of taps
 * 0..3 (the row shift of tap j on a volume of Hp x Wp rows is (dt Hp + dh) Wp + dw); lo_mask its K blocks without a
 * W_lo pass.  w (n_out x 2 ntaps k_per_tap fp16: W_hi | W_lo), scale and bias (n_out fp32, the folded BatchNorm) are
 * DEVICE buffers filled when not NULL.  An index past the last conv is VF_ERR_INVALID. */
int vf_resnet_conv(const vf_resnet_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);

/* ---- R(2+1)D clip features: replaces torchvision `r2plus1d_18(pretrained=True)` with `fc = Identity()` in eval mode
 * (and the IG65M R(2+1)D-34 models, vf_r21d_create2), and its clip transform ToFloatTensorInZeroOne -> Resize((128, 171)) -> Normalize -> CenterCrop(112)
 * (models/r21d/extract_r21d.py).  Weights: the torchvision state_dict by key (optionally with the "module." prefix),
 * HOST fp32; fc.* is ignored.  A missing / mis-sized tensor is VF_ERR_INVALID. */
typedef struct vf_r21d vf_r21d_t;

/* Workspace holds max_clips clips of max_T frames (0 = 4 and 16); a call of T-frame clips runs in chunks of
 * max_clips * (max_T + 2) / (T + 2) clips (at most 256), so any T up to that holds with bounded device memory. */
int vf_r21d_create(vf_r21d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips, int max_T);
/* The same with BatchNorm eps bn_eps (vf_r21d_create: 1e-5, torchvision's; the IG65M R(2+1)D-34 models: 1e-3).  The
 * network's depth comes from the state dict: blocks per stage (the layerL.B.conv1.0.0.weight keys), each
 * Conv2Plus1D's mid width (conv{1,2}.0.0.weight, which may differ between conv1 and conv2 of a block) and the
 * downsamples (required where a block changes stride or width, refused elsewhere). */
int vf_r21d_create2(vf_r21d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips, int max_T,
                    double bn_eps);
int vf_r21d_destroy(vf_r21d_t* h);
/* clips: n x 3 x T x 112 x 112 fp32 on the device, already transformed (the tensor the reference passes to the model)
 * -> out: n x 512 fp32. */
int vf_r21d_forward_f32(vf_r21d_t* h, const float* clips, int n, int T, float* out, void* stream);
/* transform fused: frames n_frames x H x W x 3 uint8 BGR on the device (the decoder's order, any size); clip i is
 * frames starts[i] .. starts[i] + T - 1 (starts: HOST array of n ints) -> BGR->RGB, /255, bilinear Resize((128, 171))
 * of the 112 x 112 CenterCrop window, Normalize -> network -> out: n x 512 fp32.  A frame that several clips of one
 * chunk share is transformed once. */
int vf_r21d_forward_u8(vf_r21d_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n, int T,
                       float* out, void* stream);
/* Diagnostics: an activation of the last chunk of the last call as fp32 NCTHW: stage 0 stem (after the temporal
 * conv), 1..4 the output of the last block of layer1..layer4.  dims5 receives (n, C, T, H, W); out == NULL only queries the shape. */
int vf_r21d_read_stage(vf_r21d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream);
int64_t vf_r21d_launch_count(const vf_r21d_t* h);
/* Diagnostics: conv `index` as uploaded, in execution order (the stem's spatial and temporal convs, then per block
 * conv1's spatial and temporal convs, conv2's, the downsample if any); the rest as vf_resnet_conv.  n_out is the width
 * padded to a multiple of 8. */
int vf_r21d_conv(const vf_r21d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);

/* ---- CLIP ResNet image towers (openai/CLIP ModifiedResNet: RN50, RN101, RN50x4, RN50x16): replaces
 * `clip.load("RN50" | ...)` and `model.encode_image(preprocess(frame))` (models/CLIP/extract_clip.py:45-64) with its
 * transform Resize(n_px, bicubic) -> CenterCrop(n_px) -> ToTensor -> Normalize.  Weights: openai's `visual.*` keys,
 * HOST fp32 (other keys are ignored).  Width, stage depths, resolution n_px, heads and output width are inferred from
 * the sizes as clip.model.build_model does; a missing / mis-sized tensor is VF_ERR_INVALID naming the key. */
typedef struct vf_clip_rn vf_clip_rn_t;

/* Workspace holds max_frames frames (0 = 64 at n_px 224, 32 at 288, 16 above); larger calls run in chunks. */
int vf_clip_rn_create(vf_clip_rn_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames);
int vf_clip_rn_destroy(vf_clip_rn_t* h);
/* info receives 11 ints: out_dim, n_px, width, embed dim, heads, tokens (HW + 1), max_frames, blocks of layer1..4. */
int vf_clip_rn_info(const vf_clip_rn_t* h, int* info);
/* frames: n x 3 x n_px x n_px fp32 on the device, already transformed -> out: n x out_dim fp32 on the device. */
int vf_clip_rn_encode_f32(vf_clip_rn_t* h, const float* frames, int n, float* out, void* stream);
/* transform fused: frames n x H x W x 3 uint8 on the device, any size, channel order untouched (the reference feeds the
 * decoder's BGR frame as it is) -> Pillow-exact bicubic resize of the short side to n_px, CenterCrop(n_px), ToTensor,
 * Normalize -> tower.  Bit-identical to vf_clip_rn_encode_f32 on the same transformed frames. */
int vf_clip_rn_encode_u8(vf_clip_rn_t* h, const uint8_t* frames, int n, int H, int W, float* out, void* stream);
/* Diagnostics: an activation of the last chunk of the last call as fp32 NCHW: stage 0 stem (conv3 + bn3 + relu, before
 * the pool), 1..4 layer1..layer4, 5 the attention-pool tokens (n, E, T, 1: mean first, positional embedding added),
 * 6 the attention output before c_proj (n, E, 1, 1).  dims4 receives the shape; out == NULL only queries it. */
int vf_clip_rn_read_stage(vf_clip_rn_t* h, int stage, float* out, int64_t capacity, int* dims4, void* stream);
int64_t vf_clip_rn_launch_count(const vf_clip_rn_t* h);
/* Diagnostics: stage 0 .. 4 of vf_clip_rn_read_stage as the engine holds it, the raw zero-bordered pair volume
 * (n, S+2, S+2, 2C) fp16 with its border rows; capacity: halves of out. */
int vf_clip_rn_read_pairs(vf_clip_rn_t* h, int stage, void* out, int64_t capacity, void* stream);
/* Diagnostics: conv `index` as uploaded, in execution order: the stem's conv1, conv2, conv3, then per block conv1,
 * conv2, conv3, the downsample if any, then the attention pool's q_proj, k|v (one projection of 2E outputs) and c_proj
 * (linears: one tap, scale 1, the bias).  Same contract as vf_resnet_conv; a pooled 1x1 conv carries its weight in all
 * four phase slots and 1/4 in its scale. */
int vf_clip_rn_conv(const vf_clip_rn_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);
/* Diagnostics: Bottleneck `block` (0 .. sum of the layers - 1, execution order) once, through the trunk's own kernels
 * and buffers, on n (1 .. max_frames) frames.  x_pairs: zero-bordered channels-last pair volume (n, S_in+2, S_in+2,
 * 2 cin) on the device -- block 0 takes the UNPOOLED stem output (S_in = n_px/2; layer1.0's AvgPool2d(2) is fused into
 * its convs), the first block of layer L > 1 layer L-1's output, every other block its own layer's.  out_pairs: the
 * block output (n, S_out+2, S_out+2, 2 cout), border rows included; branch_out: bn3's output before the residual add,
 * shortcut_out (NULL to skip; untouched by a block without a downsample): the downsample's output, both pair volumes of
 * the output's geometry.  Afterwards vf_clip_rn_read_stage is VF_ERR_INVALID until the next encode. */
int vf_clip_rn_debug_block(vf_clip_rn_t* h, int block, const void* x_pairs, int n, void* out_pairs, void* branch_out,
                           void* shortcut_out, void* stream);
/* Diagnostics: AttentionPool2d as the encode runs it (tokens -> K|V -> Q -> attention -> c_proj) on a layer4 pair
 * volume x_pairs (n, S4+2, S4+2, 2E), n = 1 .. max_frames -> features n x out_dim fp32.  Then read_stage is
 * VF_ERR_INVALID until the next encode, and vf_clip_rn_debug_attnpool_read returns the intermediates. */
int vf_clip_rn_debug_attnpool(vf_clip_rn_t* h, const void* x_pairs, int n, float* features, void* stream);
/* An intermediate of the last vf_clip_rn_debug_attnpool (until the next encode or debug call), copied raw: what 0 the
 * tokens (n T rows of [hi E | lo E] fp16), 1 K|V (n T rows of [k E | v E] fp32, biases added), 2 Q (n rows of E fp32,
 * bias added, unscaled), 3 the attention output (n rows of [hi E | lo E] fp16).  capacity: elements of out. */
int vf_clip_rn_debug_attnpool_read(vf_clip_rn_t* h, int what, void* out, int64_t capacity, void* stream);
/* Diagnostics, stateless: the towers' attention kernel on caller-supplied fp32 K|V (n T rows of [k E | v E]) and Q (n
 * rows of E) -> out_pairs (n rows of [hi E | lo E] fp16): per (frame, head of 64) softmax((q / 8) . k) v.  E must be a
 * multiple of 64, and the T scores must fit the kernel's dynamic shared memory (VF_ERR_INVALID otherwise). */
int vf_debug_clip_rn_attention(const float* kv, const float* q, int n, int T, int E, void* out_pairs, void* stream);

/* ---- CLIP ViT-L/14 image towers (224 px, 257 tokens; 336 px, 577 tokens): replace `clip.load("ViT-L/14" |
 * "ViT-L/14@336px")` and `model.encode_image(preprocess(frame))` with its transform Resize(n_px, bicubic) ->
 * CenterCrop(n_px) -> ToTensor -> Normalize.  Weights: openai's `visual.*` keys, HOST fp32 (other keys are ignored).
 * Width, patch, depth, heads, n_px and output width are inferred from the sizes as clip.model.build_model does; exactly
 * (1024, 14, 24, 16, 224 | 336, 768) is accepted, anything else is refused naming the key. */
typedef struct vf_clip_vitl vf_clip_vitl_t;

/* Workspace holds max_frames frames (0 = 352 at 224 px, 160 at 336 px: about 2.5 GB); larger calls run in chunks. */
int vf_clip_vitl_create(vf_clip_vitl_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames);
int vf_clip_vitl_destroy(vf_clip_vitl_t* h);
/* info receives 8 ints: out_dim (768), n_px, width, layers, heads, patch, tokens, max_frames. */
int vf_clip_vitl_info(const vf_clip_vitl_t* h, int* info);
/* frames: n x 3 x n_px x n_px fp32 on the device, already transformed -> out: n x 768 fp32 on the device. */
int vf_clip_vitl_encode_f32(vf_clip_vitl_t* h, const float* frames, int n, float* out, void* stream);
/* transform fused: frames n x H x W x 3 uint8 on the device, any size, channel order untouched -> Pillow-exact bicubic
 * resize of the short side to n_px, CenterCrop(n_px), ToTensor, Normalize -> tower.  Bit-identical to
 * vf_clip_vitl_encode_f32 on the same transformed frames. */
int vf_clip_vitl_encode_u8(vf_clip_vitl_t* h, const uint8_t* frames, int n, int H, int W, float* out, void* stream);
/* Diagnostics, eager, n <= max_frames, on `stream`: the embedding (patch GEMM, tokens, ln_pre) -> x_out n x tokens x
 * 1024 fp32; resblocks [layer_begin, layer_end) in place on x (block 23 updates the class rows only); ln_post + proj
 * on the class rows of x -> out n x 768. */
int vf_clip_vitl_debug_embed_f32(vf_clip_vitl_t* h, const float* frames, int n, float* x_out, void* stream);
int vf_clip_vitl_debug_embed_u8(vf_clip_vitl_t* h, const uint8_t* frames, int n, int H, int W, float* x_out,
                                void* stream);
int vf_clip_vitl_debug_blocks(vf_clip_vitl_t* h, float* x, int n, int layer_begin, int layer_end, void* stream);
int vf_clip_vitl_debug_head(vf_clip_vitl_t* h, const float* x, int n, float* out, void* stream);
/* The tower's attention on caller rows: qkv n_frames x tokens x 3072 fp16 (q | k | v after the bias, 16 heads of 64)
 * -> out n_frames x tokens x 1024 fp16; 1 <= tokens <= 577. */
int vf_clip_vitl_attention(vf_clip_vitl_t* h, const void* qkv, int n_frames, int tokens, void* out, void* stream);
int64_t vf_clip_vitl_launch_count(const vf_clip_vitl_t* h);

/* ---- VGGish audio embeddings (torchvggish VGG, postprocess=False): replaces models/vggish_torch's
 * vggish_input.wavfile_to_examples + VGG.forward for PCM-16 samples.  Weights: torchvggish keys features.{0,3,6,8,11,13}
 * and embeddings.{0,2,4} (.weight / .bias), HOST fp32.  The front end's float64 tables come from the caller: hann[400]
 * (periodic Hann), mel[257][64] (HTK mel matrix, DC row zero) and resampy's kaiser_best interp_win[n_win] with
 * num_table entries per zero crossing. */
typedef struct vf_vggish vf_vggish_t;

/* Workspace holds max_examples examples of 0.96 s (0 = 64); longer inputs run in chunks with the same features. */
int vf_vggish_create(vf_vggish_t** out, const vf_named_tensor* tensors, int n_tensors, const double* hann,
                     const double* mel, const double* interp_win, int n_win, int num_table, int device,
                     int max_examples);
int vf_vggish_destroy(vf_vggish_t* h);
/* samples: n_samples x channels interleaved int16 on the device, at sample_rate -> *n_out examples (complete 96-frame
 * examples of the 16 kHz log-mel; 0 when the audio is shorter than 15600 samples at 16 kHz, and nothing is written) ->
 * out: n_out x 128 fp32 on the device (capacity in floats).  Mono mix and /32768 in float64, resampy 0.2.2
 * kaiser_best to 16 kHz unless sample_rate is 16000, log-mel in float64, rounded to fp32 once. */
int vf_vggish_forward_pcm16(vf_vggish_t* h, const int16_t* samples, int64_t n_samples, int channels, int sample_rate,
                            float* out, int64_t capacity, int64_t* n_out, void* stream);
/* examples: n x 96 x 64 fp32 log-mel on the device (the network input) -> out: n x 128 fp32 on the device. */
int vf_vggish_forward_logmel_f32(vf_vggish_t* h, const float* examples, int n, float* out, void* stream);
/* Diagnostics, of the last chunk of the last call: stage 0 the resampled 16 kHz waveform the chunk's frames read
 * (float64, dims (count, 1, 1, 1); only after vf_vggish_forward_pcm16), 1 the log-mel (n, 1, 96, 64), 2..5 the
 * outputs of max-pools 1..4 as NCHW, 6..8 fc1..fc3 after their ReLU (n, D, 1, 1); fp32 except stage 0.  out == NULL
 * only queries dims4; capacity in elements. */
int vf_vggish_read_stage(vf_vggish_t* h, int stage, void* out, int64_t capacity, int* dims4, void* stream);
int64_t vf_vggish_launch_count(const vf_vggish_t* h);
/* Diagnostics: conv `index` as uploaded: 0..5 conv1..conv6, 6..8 fc1..fc3.  Same contract as vf_resnet_conv; scale 1,
 * bias the layer's.  conv1 is one tap of 32 over im2col rows (hi at kh * 3 + kw, lo 16 further); fc1 reads the
 * position-major split rows of pool 4 (input feature (h * 4 + w) * 512 + c at column (h * 4 + w) * 1024 + c). */
int vf_vggish_conv(const vf_vggish_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);
/* Host only: resampy's time register (the sequential float64 sum of sample_rate / 16000) of outputs [t0, t0 + count),
 * as the resampling kernel evaluates it. */
int vf_vggish_time_register(int sample_rate, int64_t t0, int64_t count, double* out);

/* ---- S3D clip features: torchvision `s3d()` in eval mode, the 1024-d `avgpool(features(x)).mean((2, 3, 4))`, and the
 * S3D_Weights.KINETICS400_V1 clip transform.  Weights: the torchvision state_dict by key (optionally with the "module."
 * prefix), HOST fp32; classifier.* is ignored.  A missing / mis-sized tensor is VF_ERR_INVALID. */
typedef struct vf_s3d vf_s3d_t;

/* Workspace holds max_clips clips of max_T frames (0 = 2 and 64; max_T >= 13); a call runs in chunks of as many clips
 * of its T as the workspace holds (at most 256), so device memory does not grow with the call. */
int vf_s3d_create(vf_s3d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips, int max_T);
int vf_s3d_destroy(vf_s3d_t* h);
/* clips: n x 3 x T x 224 x 224 fp32 on the device, already transformed; T >= 13 (the smallest clip whose (2,7,7)
 * average pool has a position) -> out: n x 1024 fp32. */
int vf_s3d_forward_f32(vf_s3d_t* h, const float* clips, int n, int T, float* out, void* stream);
/* transform fused: frames n_frames x H x W x 3 uint8 BGR on the device (the decoder's order, any size); clip i is
 * frames starts[i] .. starts[i] + T - 1 (starts: HOST array of n ints) -> BGR->RGB, bilinear Resize((256, 256)) on
 * uint8 of the 224 x 224 CenterCrop window, /255, Normalize -> network -> out: n x 1024 fp32.  A frame that several
 * clips of one chunk share is transformed once. */
int vf_s3d_forward_u8(vf_s3d_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n, int T,
                      float* out, void* stream);
/* Diagnostics: an activation of the last chunk of the last call as fp32 NCTHW: stage 0 stem (after the temporal conv),
 * 1 features.3 (the separable conv before the second pool), 2 Mixed 3c, 3 Mixed 4f, 4 Mixed 5c.  dims5 receives
 * (n, C, T, H, W); out == NULL only queries the shape. */
int vf_s3d_read_stage(vf_s3d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream);
int64_t vf_s3d_launch_count(const vf_s3d_t* h);
/* Diagnostics: conv `index` as uploaded, in execution order (the stem's spatial and temporal convs, features.2,
 * features.3's spatial and temporal convs, then per Mixed block branch0, branch1's 1x1x1, spatial and temporal convs,
 * branch2's likewise, branch3's 1x1x1); the rest as vf_r21d_conv. */
int vf_s3d_conv(const vf_s3d_t* h, int index, int* geom, uint64_t* lo_mask, void* w, float* scale, float* bias);
/* Diagnostics: Mixed block `block` (0 .. 8: features.5, 6, 8 .. 12, 14, 15) once, as vf_i3d_debug_mixed (same volume
 * layout, S and rules; afterwards vf_s3d_read_stage is VF_ERR_INVALID until the next forward). */
int vf_s3d_debug_mixed(vf_s3d_t* h, int block, const void* x_pairs, int n, int T, void* out_pairs, void* stream);

/* ---- diagnostics of the pool and head kernels I3D and S3D share.  A volume is 10 ints: n, Tp, Hp, Wp (the padded
 * extents of a channels-last volume of pair rows [hi C | lo C]), then t0, t1, h0, h1, w0, w1 (its valid region). */
#define VF_POOL_GENERAL 0   /* bounds-checked kernel, any window */
#define VF_POOL_FAST 1      /* fixed windows 1x3x3/1x2x2, 3x3x3/2, 2x2x2/2 with no leading padding, every window
                               inside the input's padded extent */
#define VF_POOL_SAME3 2     /* 3x3x3 / 1 pad 1 onto the input's own geometry, border >= 1: the rolling-max kernel */
/* Max pool of the valid region with zero padding (k, s, p: kt kh kw, st sh sw, pt ph pw), pair rows in and out, border
 * rows of the output written as zeros; path receives the VF_POOL_* kernel that ran.  C must be a multiple of 8. */
int vf_debug_maxpool3d(const void* in, const int* vol_in, void* out, const int* vol_out, int C, const int* k,
                       const int* s, const int* p, int* path, void* stream);
/* AvgPool3d((2,7,7), 1) of a T3 (>= 2) x 7 x 7 valid region, then the mean over time: out n x C fp32. */
int vf_debug_i3d_head(const void* in, const int* vol, int C, float* out, void* stream);

/* ---- Swin3D clip features: torchvision `swin3d_t` / `swin3d_s` / `swin3d_b` in eval mode, the feature
 * `flatten(avgpool(norm(features(patch_embed(x)))))` (768-d for t / s, 1024-d for b), and the
 * Swin3D_*_Weights.KINETICS400_V1 clip transform.  Weights: the torchvision state_dict by key (optionally with the
 * "module." prefix), HOST fp32; head.* and relative_position_index are ignored (the index is computed).  The shape is
 * inferred from the weights: embed dim from patch_embed.proj, depths from the features.{0,2,4,6}.* block keys, heads =
 * dim / 32; patch (2,4,4) and window (8,7,7) are checked against the conv weight and the bias-table size.  Exactly the
 * t / s / b shapes are accepted (VF_ERR_UNSUPPORTED naming the key otherwise). */
typedef struct vf_swin3d vf_swin3d_t;

/* Workspace holds max_clips clips of max_T frames (0 = 4 and 32); a call runs in chunks of as many clips of its T as the
 * workspace holds (at most 256). */
int vf_swin3d_create(vf_swin3d_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips,
                     int max_T);
int vf_swin3d_destroy(vf_swin3d_t* h);
/* info receives 8 ints: out_dim, embed dim, the 4 depths, max_clips, max_T. */
int vf_swin3d_info(const vf_swin3d_t* h, int* info);
/* clips: n x 3 x T x 224 x 224 fp32 on the device, already transformed; T >= 1 (an odd T gets PatchEmbed3d's zero
 * frame) -> out: n x out_dim fp32. */
int vf_swin3d_forward_f32(vf_swin3d_t* h, const float* clips, int n, int T, float* out, void* stream);
/* transform fused: frames n_frames x H x W x 3 uint8 BGR on the device, any size; clip i is frames starts[i] ..
 * starts[i] + T - 1 (starts on the HOST) -> BGR->RGB, Resize([256]) bilinear without antialias on uint8, CenterCrop(224),
 * /255, Normalize -> network.  Bit-identical to vf_swin3d_forward_f32 on the same transformed clips. */
int vf_swin3d_forward_u8(vf_swin3d_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n,
                         int T, float* out, void* stream);
/* Diagnostics, the last chunk of the last forward, fp32 channels-last: stage 0 patch_embed (conv + norm), 1..4 the output
 * of features.0 / 2 / 4 / 6, 5 the final norm.  dims5 receives (n, T', H', W', C); out == NULL only queries the shape. */
int vf_swin3d_read_stage(vf_swin3d_t* h, int stage, float* out, int64_t capacity, int* dims5, void* stream);
/* The window attention alone on caller rows: qkv n x Tq x H x W x 3C fp16 (q | k | v after the bias, heads of 32),
 * bias_qkv the 3C fp32 qkv bias and table the (2535, C / 32) fp32 relative_position_bias_table, both on the device ->
 * out n x Tq x H x W x C fp16.  Window (8,7,7), shift (4,3,3) if `shifted`, both clamped as torchvision's
 * _get_window_and_shift_size does. */
int vf_swin3d_attention(const void* qkv, const float* bias_qkv, const float* table, int n, int Tq, int H, int W, int C,
                        int shifted, void* out, void* stream);
int64_t vf_swin3d_launch_count(const vf_swin3d_t* h);

/* ---- MViT clip features: torchvision `mvit_v1_b` / `mvit_v2_s` in eval mode, the feature `norm(x)[:, 0]` (the class
 * token after the final norm, 768-d), and the MViT_*_Weights.KINETICS400_V1 clip transform (16 frames, Resize([256]),
 * CenterCrop(224), Normalize(0.45, 0.225)).  Weights: the torchvision state_dict by key (optionally with the "module."
 * prefix), HOST fp32; head.* is ignored.  v2 is inferred from blocks.0.attn.rel_pos_h, v1 from
 * pos_encoding.spatial_pos; every other key must have the size torchvision gives it (VF_ERR_INVALID /
 * VF_ERR_UNSUPPORTED naming the key otherwise). */
typedef struct vf_mvit vf_mvit_t;

/* Workspace holds max_clips clips (0 = 4), about 190 MB each; a call runs in chunks of as many clips (at most 256). */
int vf_mvit_create(vf_mvit_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_clips);
int vf_mvit_destroy(vf_mvit_t* h);
/* info receives 4 ints: out_dim (768), version (1 or 2), T (16), max_clips. */
int vf_mvit_info(const vf_mvit_t* h, int* info);
/* clips: n x 3 x 16 x 224 x 224 fp32 on the device, already transformed; T must be 16 -> out: n x 768 fp32. */
int vf_mvit_forward_f32(vf_mvit_t* h, const float* clips, int n, int T, float* out, void* stream);
/* transform fused: frames n_frames x H x W x 3 uint8 BGR on the device, any size; clip i is frames starts[i] ..
 * starts[i] + 15 (starts on the HOST) -> BGR->RGB, Resize([256]) bilinear without antialias on uint8, CenterCrop(224),
 * /255, Normalize -> network.  Bit-identical to vf_mvit_forward_f32 on the same transformed clips. */
int vf_mvit_forward_u8(vf_mvit_t* h, const uint8_t* frames, int n_frames, int H, int W, const int* starts, int n, int T,
                       float* out, void* stream);
/* Diagnostics, the last chunk of the last forward, fp32 token rows [class | T' x H' x W' tokens]: stage 0 the patch
 * embedding with class token and positions, 1..4 the output of blocks 0 / 2 / 13 / 15 (the blocks before each q stride
 * and the last), 5 the final norm on every row.  dims3 receives (n, tokens, C); out == NULL only queries the shape. */
int vf_mvit_read_stage(vf_mvit_t* h, int stage, float* out, int64_t capacity, int* dims3, void* stream);
/* The pooling attention alone: q n x (1 + prod(q_thw)) rows of pitch ldq, k / v n x (1 + prod(k_thw)) x heads*96 fp16
 * (heads of 96 channels) -> out n x (1 + prod(q_thw)) x heads*96 fp16.  rel: the decomposed rel-pos bias from rel_h /
 * rel_w (2 max(q_h, k_h) - 1 rows of 96) and rel_t (2 max(q_t, k_t) - 1 rows), fp32 on the device; resid: + q on the
 * token rows.  k_thw[0] + k_thw[1] + k_thw[2] <= 48. */
int vf_mvit_attention(const void* q, int ldq, const void* k, const void* v, const float* rel_h, const float* rel_w,
                      const float* rel_t, int n, int heads, const int* q_thw, const int* k_thw, int rel, int resid,
                      void* out, void* stream);
/* The head pooling alone: src n x (1 + T H W) rows of pitch ld_src fp16 -> depthwise 3x3x3 conv, stride
 * (1, stride, stride), pad 1 (weight 96 x 27 fp32) per head of 96 on the tokens, class row passed through, then
 * LayerNorm(96, eps 1e-6) (gamma, beta) on every row -> dst n x (1 + T Ho Wo) x heads*96 fp16. */
int vf_mvit_head_pool(const void* src, int ld_src, int n, int heads, int T, int H, int W, int stride,
                      const float* weight, const float* gamma, const float* beta, void* dst, void* stream);
/* The skip max-pool alone: MaxPool3d((1,3,3), (1,2,2), (0,1,1)) of x n x (1 + T H W) x C fp32 tokens, class row
 * copied -> y n x (1 + T Ho Wo) x C. */
int vf_mvit_skip_pool(const float* x, int n, int C, int T, int H, int W, float* y, void* stream);
int64_t vf_mvit_launch_count(const vf_mvit_t* h);

/* ---- CLIP text tower (zero-shot --show_pred of the CLIP feature types): openai/CLIP's `CLIP.encode_text` followed by
 * L2 normalisation.  Weights: the checkpoint's non-visual tensors by key (token_embedding.weight, positional_embedding,
 * transformer.resblocks.*, ln_final.*, text_projection), HOST fp32.  The geometry is read from them as
 * clip.build_model reads it; 12 blocks at width 512 (8 heads), 640 (10) or 768 (12) are built, anything else is
 * refused (VF_ERR_UNSUPPORTED). */
typedef struct vf_clip_text vf_clip_text_t;

/* Workspace of max_rows token rows (0 = 8192); a call runs in chunks of max_rows / L prompts. */
int vf_clip_text_create(vf_clip_text_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_rows);
int vf_clip_text_destroy(vf_clip_text_t* h);
/* info receives 7 ints: width, heads, layers, context, embed, vocabulary size, max_rows. */
int vf_clip_text_info(const vf_clip_text_t* h, int* info);
/* tokens: n x context int32 on the HOST (clip.tokenize rows) -> out: n x embed fp32 on the device, each row
 * encode_text / ||encode_text||.  The EOT row of a prompt is its argmax id; the tower runs on L = 1 + the largest EOT
 * position of the call rows per prompt.  An id outside the vocabulary is refused. */
int vf_clip_text_encode(vf_clip_text_t* h, const int32_t* tokens, int n, float* out, void* stream);
/* Diagnostics: blocks first .. first + count - 1 in place on the residual stream x, n x L x width fp32 on the device. */
int vf_clip_text_blocks(vf_clip_text_t* h, float* x, int n, int L, int first, int count, void* stream);
/* The causal attention alone: qkv n x L rows [q | k | v] of 3 x heads*64 fp16 -> out n x L x heads*64 fp16; L <= 77.
 * Row i reads rows 0..i only, in an order fixed by i: its bits do not depend on L. */
int vf_clip_text_attention(const void* qkv, int n, int L, int heads, void* out, void* stream);
/* out[r] = x[r] / ||x[r]||_2, n rows of C fp32 on the device (out == x allowed). */
int vf_l2_normalize_rows(const float* x, int n, int C, float* out, void* stream);
int64_t vf_clip_text_launch_count(const vf_clip_text_t* h);

/* ---- DINOv2 frame features: `torch.hub.load('facebookresearch/dinov2', name)(x)` at 224 px, the class token after the
 * final norm, for dinov2_vit{s,b,l,g}14 and their _reg variants.  Weights: the hub checkpoint's tensors by key, HOST
 * fp32, plus "pos_embed_224", the (257, D) positional table the hub interpolates for a 224-px input
 * (video_features_b200/dinov2_engine.py pos_table_224 computes it).  The shape is read from the weights: width from cls_token, depth from the blocks.{i} keys,
 * heads = width / 64, SwiGLU when blocks.0.mlp.w12.weight is present, registers when register_tokens is.  Exactly
 * (384, 12), (768, 12), (1024, 24) and (1536, 40, SwiGLU) are built; anything else is refused naming the key. */
typedef struct vf_dinov2 vf_dinov2_t;

/* Workspace of max_frames frames (0 = a default that keeps it near 2.5 GB); a call runs in chunks. */
int vf_dinov2_create(vf_dinov2_t** out, const vf_named_tensor* tensors, int n_tensors, int device, int max_frames);
int vf_dinov2_destroy(vf_dinov2_t* h);
/* info receives 7 ints: width D, depth, heads, tokens (257 or 261), registers, FFN kind (0 GELU MLP, 1 SwiGLU),
 * max_frames. */
int vf_dinov2_info(const vf_dinov2_t* h, int* info);
/* frames: n x 3 x 224 x 224 fp32 on the device, already transformed -> out: n x D fp32. */
int vf_dinov2_encode_f32(vf_dinov2_t* h, const float* frames, int n, float* out, void* stream);
/* transform fused: frames n x H x W x 3 uint8 BGR on the device, any size -> Resize(256, bicubic, Pillow-exact),
 * CenterCrop(224), BGR->RGB, ToTensor, Normalize (ImageNet) -> network.  Bit-identical to vf_dinov2_encode_f32 on the
 * same transformed frames. */
int vf_dinov2_encode_u8(vf_dinov2_t* h, const uint8_t* frames, int n, int H, int W, float* out, void* stream);
/* Diagnostics, eagerly on the caller's stream, n <= max_frames: the embedding (token assembly) -> x_out n x tokens x D
 * fp32; blocks [layer_begin, layer_end) in place on x (the last block updates the class rows only); the final norm of
 * the class rows of x -> out n x D. */
int vf_dinov2_debug_embed_f32(vf_dinov2_t* h, const float* frames, int n, float* x_out, void* stream);
int vf_dinov2_debug_embed_u8(vf_dinov2_t* h, const uint8_t* frames, int n, int H, int W, float* x_out, void* stream);
int vf_dinov2_debug_blocks(vf_dinov2_t* h, float* x, int n, int layer_begin, int layer_end, void* stream);
int vf_dinov2_debug_head(vf_dinov2_t* h, const float* x, int n, float* out, void* stream);
/* The SwiGLU kernel alone: ab rows x 2 hidden fp32 ([a | b], the w12 output) -> out rows x hidden fp16,
 * silu(a) * b in fp32 rounded once. */
int vf_dinov2_swiglu(const float* ab, int rows, int hidden, void* out, void* stream);
/* The attention the blocks use alone: qkv n x S rows [q | k | v] of 3 x heads*64 fp16 -> out n x S x heads*64 fp16,
 * scale 1/8, no mask, S <= 577. */
int vf_dinov2_attention(const void* qkv, int n, int S, int heads, void* out, void* stream);
int64_t vf_dinov2_launch_count(const vf_dinov2_t* h);

/* ---- classifier head (--show_pred): replaces `model.fc(feats)` of models/resnet/extract_resnet.py:105-114 and
 * models/r21d/extract_r21d.py:113-121, I3D's conv3d_0c_1x1 + mean over time (models/i3d/i3d_src/i3d_net.py:266-274),
 * and the softmax + sort of utils/utils.py:19-47.  weight: n_classes x n_features, bias: n_classes, HOST fp32. */
typedef struct vf_head vf_head_t;

int vf_head_create(vf_head_t** out, const float* weight, const float* bias, int n_classes, int n_features, int device);
int vf_head_destroy(vf_head_t* h);
int vf_head_info(const vf_head_t* h, int* n_classes, int* n_features);
/* feats: n x n_features fp32 on the device (n_features must equal the head's) -> logits, probs: n x n_classes fp32;
 * top_idx (int32), top_logit, top_prob: n x k, 1 <= k <= min(8, n_classes); all on the device, on `stream`.
 * Each logit is one sequential fp32 FMA chain over the features, plus the bias.  probs = expf(l - max) / sum, as torch's
 * softmax.  Top-k order: probability descending, equal probabilities by the lower class index.  Two launches; n == 0
 * writes nothing. */
int vf_head_forward(vf_head_t* h, const float* feats, int n, int n_features, float* logits, float* probs, int k,
                    int32_t* top_idx, float* top_logit, float* top_prob, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VFEAT_H_ */
