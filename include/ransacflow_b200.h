/*
 * ransacflow_b200 - C ABI of the H100 (sm_90a) implementation of RANSAC-Flow's
 * per-pair inference hot path.
 *
 * The reference (XiSHEN0220/RANSAC-Flow) is pure Python on PyTorch: it has no
 * FFI.  Its drop-in boundary is a set of Python modules (`outil`, `model`,
 * `coarseAlignFeatMatch`, `kornia.geometry`; SURVEY.md section 8b).  The Python
 * mirror of those modules (package `ransac-flow_b200/`) is a thin layer over
 * THIS library; every entry point below names the reference code it replaces
 * (paths relative to the reference checkout).
 *
 * Conventions
 *   - plain pointers and sizes only; all data pointers are DEVICE pointers
 *     unless the parameter name ends in `_host`;
 *   - `stream` is a `cudaStream_t` passed as `void*` (NULL = default stream);
 *     every call is asynchronous on that stream unless stated otherwise;
 *   - return value 0 = OK, non-zero = error (message: rf_last_error_string());
 *   - no allocation inside: scratch memory comes from the caller (`ws`), sized
 *     by the matching `*_workspace()` query;
 *   - activations are NHWC fp32, "ragged batch": `nimg` images of different
 *     (H, W) packed back to back in one buffer (`hw_host[2*i] = H_i`,
 *     `hw_host[2*i+1] = W_i`); outputs are packed the same way;
 *   - there is NO CPU fallback anywhere in this library.
 */
#ifndef RANSACFLOW_B200_H
#define RANSACFLOW_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RF_MAX_IMGS 16

/* status written by rf_ransac_homography to *status_out (device int) */
#define RF_RANSAC_OK 0          /* H_out / nbInlier_out / mask_out valid                          */
#define RF_RANSAC_NONE 1        /* reference returns (None, 0, [], []): utils/outil.py:145-146      */
#define RF_RANSAC_NO_MODEL 2    /* reference raises TypeError at utils/outil.py:162 (bestParams None) */
#define RF_RANSAC_TOO_FEW 3     /* fewer than 4 matches (callers return None before calling)      */

int rf_version(void);
/* sha256 of the sources (csrc/, this header, compiler flags) the library was built from; the Python binding refuses a library
 * whose digest differs from the sources next to it */
const char* rf_source_digest(void);
const char* rf_last_error_string(void);
/* number of kernel launches issued through this library since load (bench.py's gpu_launches) */
uint64_t rf_launch_count(void);

/* ---------------------------------------------------------------- matching --
 * utils/outil.py:32-45 mutualMatching, fused: the NA x NB score matrix is never
 * written.  featA [NA][C], featB [NB][C] (K-major rows = one feature vector).
 * Outputs: idx1/idx2 (int64, capacity >= min(NA,NB)) sorted by idx1, *count.
 * precision: 0 = exact fp32 FMA (SIMT); 1 = 3xTF32 on wgmma tensor cores (hi*hi + lo*hi + hi*lo, C % 32 == 0);
 * 2 = fp16 split on wgmma (x = hi + lo * 2^-11 in fp16, cross terms in a second accumulator, C % 64 == 0): the
 * same 22 significand bits with half the MMAs per channel.
 * Every precision ends in the same mutual test + compaction launch on the row / column arg-max keys.  Before the
 * correlation, precision 0 zeroes the keys with a memset, precision 1 adds two split launches, precision 2 splits both
 * operands and zeroes the keys in one launch.  rf_corr_mutual_nn_launches() (host only) returns the number of launches
 * of a call with this precision: 3, 5 or 3. */
size_t rf_corr_mutual_nn_workspace(int NA, int NB, int C, int precision);
int rf_corr_mutual_nn_launches(int precision);
int rf_corr_mutual_nn(const float* featA, int NA, const float* featB, int NB, int C,
                      int64_t* idx1_out, int64_t* idx2_out, int* count_out,
                      void* ws, size_t ws_bytes, int precision, void* stream);

/* The same with operands their producer already split (rf_l2norm_split_nhwc writes the normalised rows as fp16 hi / lo * 2^11
 * planes): no split pass.  A_hi / A_lo [NA][C], B_hi / B_lo [NB][C] fp16, C % 64 == 0.  Three graph nodes: memset of the
 * arg-max keys, the fp16-split wgmma kernel (precision 2 of rf_corr_mutual_nn, identical arithmetic), the
 * mutual test + compaction. */
size_t rf_corr_mutual_nn_presplit_workspace(int NA, int NB);
int rf_corr_mutual_nn_presplit(const void* A_hi, const void* A_lo, int NA, const void* B_hi, const void* B_lo, int NB, int C,
                               int64_t* idx1_out, int64_t* idx2_out, int* count_out, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ RANSAC --
 * utils/outil.py:117-164 RANSAC + :102-113 ScoreRANSAC + :68-87 Homography +
 * :97-100 Prediction as ONE persistent kernel.  `samples` is the (nbIter,4)
 * int64 tensor `torch.randint` returned at utils/outil.py:120 (the draw stays
 * on the host side so the generator stream is the reference's).
 * match1/match2 [M][3] fp32 (x, y, 1).  `M_dev` (nullable) overrides M with a
 * device-side count (<= M) so no host sync is needed after matching.
 * Outputs: H_out[9] fp32, nbInlier_out int64, mask_out[M] u8, status_out int. */
/* `sample_mode`: how `samples` (nbIter x 4 int64) becomes match indices.
 *   RF_SAMPLES_INDEX    the tensor torch.randint(M, (nbIter, 4)) returned (utils/outil.py:120), used as is;
 *   RF_SAMPLES_MOD      arbitrary non-negative integers, reduced `% M` on the device (M = *M_dev);
 *   RF_SAMPLES_PHILOX64 full-range 64-bit generator words (`Tensor.random_(-2**63, None)` on CUDA = (x << 32) | y of one
 *                       curand4 call per element): index = x % M, which IS what torch.randint(M, (nbIter, 4), device='cuda')
 *                       returns from the same generator state (ATen random_from_to_kernel, range < 2^28, nbIter * 4 <=
 *                       256 * SMs * blocks-per-SM so that every element has its own Philox subsequence) - the reference's
 *                       seeded sample stream without knowing M on the host, usable inside a CUDA graph. */
#define RF_SAMPLES_INDEX 0
#define RF_SAMPLES_MOD 1
#define RF_SAMPLES_PHILOX64 2
size_t rf_ransac_workspace(int nbIter);
int rf_ransac_homography(const float* match1, const float* match2, int M, const int* M_dev,
                         const int64_t* samples, int sample_mode, int nbIter, float tolerance, int chunk,
                         float* H_out, int64_t* nbInlier_out, uint8_t* mask_out, int* status_out,
                         void* ws, size_t ws_bytes, void* stream);
/* rf_ransac_homography on the table a device slot chain picks: `tables` holds n_tables (nbIter x 4) tables back to back
 * (table j = the j-th draw the reference would make), the kernel reads table *slot_in (clamped to n_tables - 1) and writes
 * *slot_out = *slot_in + (M >= 4), M = min(*M_dev, M): a call that does not draw (the reference returns None before
 * torch.randint) passes its table on to the next call.  slot_in and slot_out are two different int32 device scalars;
 * chaining calls through slots[i] -> slots[i + 1] makes each call read the table the reference's draw sequence gives it. */
int rf_ransac_homography_drawn(const float* match1, const float* match2, int M, const int* M_dev,
                               const int64_t* tables, int n_tables, int sample_mode, int nbIter, float tolerance, int chunk,
                               const int* slot_in, int* slot_out, float* H_out, int64_t* nbInlier_out, uint8_t* mask_out,
                               int* status_out, void* ws, size_t ws_bytes, void* stream);
/* evaluation/evalYFCC/evaluation.py:195-212 on the device, one CTA: the four rotations' RANSAC statuses (RF_RANSAC_*),
 * match counts (read as min(*count[k], cap[k])) and inlier masks (u8, cap[k] entries) -> one int32 record of
 * RF_YFCC_REC_WORDS words: the winner (first maximum of the scores), the four scores (popcount of mask[:M] for a rotation
 * that drew, M >= nbPoint, and returned a model; 0 otherwise), the number of rotations that drew, an error flag (a rotation
 * that drew returned RF_RANSAC_NO_MODEL: utils/outil.py:162 raises TypeError) and the winner's orientation class
 * (winner & 1: 0 / 180 degrees share the resized target's shape, 90 / 270 the transposed one).  `status`, `count`, `mask`
 * and `cap` are host arrays of 4 (a mask may be null where its cap is 0).  No atomics: deterministic, graph-capturable. */
#define RF_YFCC_REC_WINNER 0
#define RF_YFCC_REC_SCORES 1
#define RF_YFCC_REC_DRAWN 5
#define RF_YFCC_REC_ERROR 6
#define RF_YFCC_REC_CLASS 7
#define RF_YFCC_REC_WORDS 8
int rf_yfcc_rotation_select(const int* const* status, const int* const* count, const uint8_t* const* mask, const int* cap,
                            int nbPoint, int* rec_out, void* stream);
/* dst[0:bytes] <- src[*sel][0:bytes] (src: a host array of nsrc <= 4 device pointers, null entries copy nothing), with the
 * index read on the device: a graph copies the buffers of a rotation chosen by an earlier kernel. */
int rf_select_copy(const void* const* src, int nsrc, const int* sel, void* dst, size_t bytes, void* stream);
/* utils/outil.py:68-87 Homography alone: X,Y [N][4][3] -> H [N][9] (for tests). */
int rf_homography_dlt(const float* X, const float* Y, int N, float* H_out, void* stream);
/* utils/outil.py:97-100 Prediction: err [N][M]. */
int rf_prediction(const float* match1, const float* match2, int M, const float* H, int N, float* err_out, void* stream);
/* coarseAlignFeatMatch.py (variant A :158-168, variant C :146-155): gather the
 * matched cell-centre coordinates into match1/match2 [M][3] = (x=H, y=W, 1).
 * valid16 (nullable, u8 [NB]) drops matches whose target cell is masked; the
 * surviving count goes to *count_out, order preserved. */
int rf_build_matches(const int64_t* idx1, const int64_t* idx2, const int* count_in,
                     const float* W1, const float* H1, const float* W2, const float* H2,
                     const uint8_t* valid16, float* match1_out, float* match2_out,
                     int64_t* idx2_kept_out, int* count_out, int capacity, void* stream);

/* ---------------------------------------------------------------- networks --
 * conv + folded BatchNorm (eval) + optional residual add + optional ReLU:
 * model/model.py:27-56,59-125,167-322; torchvision ResNet-50 bottlenecks.
 * x: ragged NHWC [sum HW][Cin]; w: [R*S*Cin][Cout] (tap-major, Cout contiguous);
 * bias [Cout] (nullable); residual: packed like y (nullable).
 * engine: 0 = fp32 SIMT implicit GEMM everywhere; 1 = TF32 wgmma implicit GEMM for the layers it
 * supports (stride 1, Cin % 32 == 0, 1x1 / 3x3; w_tc = same weights as [Cout][R*S*Cin]), the exact-fp32
 * SIMT kernel for the rest (3-channel stems, stride-2 convs);
 * 2 = fp16 wgmma implicit GEMM: x, residual, y and w_tc ([Cout][R*S*Cin]) hold IEEE fp16 elements behind the
 * same pointers (10-bit mantissa like TF32, half the HBM bytes, twice the tensor rate), fp32 accumulation and fp32
 * bias, outputs saturated to +-65504; needs Cin % 64 == 0, Cout % 8 == 0, 1x1 / 3x3, stride 1 / 2 and fails otherwise
 * (no fallback).  Used for the ResNet-50 conv4 trunk. */
#define RF_ENGINE_FP32 0
#define RF_ENGINE_TF32 1
#define RF_ENGINE_F16 2
#define RF_ENGINE_F16_OUT32 3   /* engine 2 operands, fp32 output rounded to TF32 after ReLU (3x3 / stride 1 / no residual):
                                   the layer that hands over from fp16 activations to a TF32 layer */
/* 4 = fp32-GRADE wgmma implicit GEMM ("f16x3"): every activation / weight element is carried as two fp16 values,
 * v = hi + lo * 2^-11 (hi = fp16(v), lo = fp16((v - hi) * 2^11): 22 significand bits), and every MAC is three kind::f16 MMAs
 * (hi*hi | hi*lo + lo*hi in a second accumulator).  x, residual and y are SPLIT tensors behind the same pointers:
 * [2][sum HW][C] fp16, plane 0 = hi, plane 1 = lo * 2^11 (4 bytes per element like fp32); w_tc = [2][Cout][R*S*Cin] fp16,
 * split the same way.  fp32 accumulation, bias, residual add and ReLU; needs Cin % 64 == 0, Cout % 8 == 0, 1x1 / 3x3,
 * stride 1 / 2 (no fallback).  This is the engine whose features reproduce the reference's fp32 arg-max (match set).
 * 5 = engine 4 operands with a plain fp32 [sum HoWo][Cout] output (any Cout, no residual): the heads' 49- / 1-channel layers. */
#define RF_ENGINE_SPLIT 4
#define RF_ENGINE_SPLIT_OUT32 5
int rf_conv2d_nhwc(const float* x, int nimg, const int* hw_host, int Cin,
                   const float* w, const float* w_tc, const float* bias, const float* residual,
                   int Cout, int R, int S, int stride, int pad, int relu, int engine,
                   float* y, void* stream);
/* Engine 4 only: a 1x1 convolution over TWO inputs whose channels are concatenated along K,
 *   y = act(W[:, :Cin1] x1 + W[:, Cin1:] x2[::stride2, ::stride2] + bias),
 * i.e. a ResNet bottleneck's conv3 + bn3 and its down-sampling branch (downsample.0 + downsample.1 of torchvision's Bottleneck,
 * which quick_start/coarseAlignFeatMatch.py:31-38 runs up to layer3) + the residual add + ReLU as ONE GEMM: the branch's output
 * never goes to HBM.  x1 / x2 / y split tensors; hw1 = sizes of x1 and y, hw2 = sizes of x2 ((h2 - 1) / stride2 + 1 == h1);
 * w_split = [2][Cout][Cin1 + Cin2] fp16; Cin1 % 64 == Cin2 % 64 == 0, Cout % 8 == 0, stride2 1 or 2. */
int rf_conv1x1_dual_split(const void* x1, const void* x2, int nimg, const int* hw1_host, const int* hw2_host, int Cin1, int Cin2,
                          int stride2, const void* w_split, const float* bias, int Cout, int relu, void* y, void* stream);
/* A whole network in one call: `layers_host[n]` executed in order over a ragged batch.  Buffers are numbered
 * "slots" (`slots_host[i]` = device pointer, caller-allocated); slot `layers[0].src` holds the input images
 * (`hw_host` = their sizes) and every layer's output sizes follow from its input's.  This is what the Python
 * mirrors of FeatureExtractor / NetFlowCoarse / NetMatchability / ResNet-50 conv4 call (one host call per
 * network instead of one per layer). */
#define RF_OP_CONV 0      /* conv + bias (+ residual slot) (+ ReLU) */
#define RF_OP_MAXPOOL 1   /* k, stride, pad */
#define RF_OP_BLUR 2      /* model/downsample.py: reflect-pad 1 + [1 2 1]^2/16, stride */
#define RF_OP_IM2COL 3    /* k x k x Cin patches (r, s, c order) zero-padded to Cout floats per output pixel: few-channel stems */
#define RF_OP_POOLBLUR 4  /* MaxPool2d(2, stride 1) + blur stride 2 fused (model/model.py:71-72) */
#define RF_OP_STEM7 5     /* engines 2 / 4 only: a direct stem on the 3-channel fp32 image + bias + ReLU -> fp16 / split, 64 channels,
                             without the im2col matrix: k 7 / stride 2 / pad 3 (ResNet-50) or k 3 / stride 1 / pad 1 (FeatureExtractor);
                             w_f16 = [64][Kpad] ([2][64][Kpad] for engine 4) in (r, s, c) order, zero padded to Kpad = 192 / 64 */
#define RF_OP_CONV_DUAL 6  /* engine 4 only: rf_conv1x1_dual_split; src = x1 (Cin channels), src2 = x2 (Cin2 channels, stride2), w_f16 = [2][Cout][Cin + Cin2] */
#define RF_OP_STEM3 7      /* engine 4 only: the first conv of segNet's deep stem (segNet/segModel.py:64,108) fused: 3x3 / stride 2 / pad 1 on the
                             3-channel fp32 input slot + bias + ReLU -> split, 64 channels, exact fp32 FMA; w = [27][64] ((r, s, c) rows) */
#define RF_MAX_SLOTS 32
typedef struct rf_layer {
    int op;
    int src, dst, res;              /* slot indices; res < 0 = none */
    int Cin, Cout, k, stride, pad, relu;
    const float* w;                 /* [k*k*Cin][Cout] */
    const float* w_tc;              /* [Cout][k*k*Cin] */
    const float* bias;              /* [Cout] or NULL */
    const void* w_f16;              /* engine 2: [Cout][k*k*Cin] fp16; engine 4: [2][Cout][k*k*Cin] fp16 hi / lo planes (NULL otherwise) */
    int flags;                      /* engines 2 / 4: RF_LAYER_* */
    int src2, Cin2, stride2;        /* RF_OP_CONV_DUAL: second input slot, its channels and sampling stride (ignored otherwise) */
    int dil;                        /* RF_OP_CONV dilation: 0 or 1 = none; > 1 only for 3x3 / stride 1 layers on engine 4.  Output size
                                       (h + 2 pad - dil (k - 1) - 1) / stride + 1; out-of-image taps read zeros */
} rf_layer_t;
#define RF_LAYER_OUT_F32 1          /* conv: fp16 operands, fp32 output (RF_ENGINE_F16_OUT32; engine 4: RF_ENGINE_SPLIT_OUT32) */
#define RF_LAYER_TF32 2             /* conv: fp32 input and output on the TF32 engine (e.g. a 49-channel head after an OUT_F32 layer) */
#define RF_LAYER_STEM_POOL 4        /* 7x7 RF_OP_STEM7 whose output only feeds the next layer, a 3x3 / stride 2 / pad 1 RF_OP_MAXPOOL: both run
                                       as one kernel that writes the max-pool's dst slot; the stem's own dst slot is never written */
/* engine 2: slots hold fp16 except the input of an RF_OP_IM2COL (the fp32 image; row length = Cout % 64 == 0), the
 * output of an RF_LAYER_OUT_F32 conv and the input / output of an RF_LAYER_TF32 conv; pooling and blur run in fp16. */
/* engine 4: slots hold split tensors ([2][P][C] fp16) except the fp32 input image of an RF_OP_IM2COL / RF_OP_STEM7 and the fp32
 * output of an RF_LAYER_OUT_F32 conv; pooling and blur rebuild the fp32 values and split their results again. */
int rf_run_layers(const rf_layer_t* layers_host, int n, void* const* slots_host, int nimg, const int* hw_host,
                  int engine, void* stream);
/* max pooling k x k / stride / zero-free padding: nn.MaxPool2d (model/model.py:71; torchvision resnet maxpool) */
int rf_maxpool2d_nhwc(const float* x, int nimg, const int* hw_host, int C, int k, int stride, int pad,
                      float* y, void* stream);
/* model/downsample.py:12-46: reflect-pad 1 + depthwise [1 2 1]x[1 2 1]/16, stride */
int rf_blur_downsample_nhwc(const float* x, int nimg, const int* hw_host, int C, int stride, float* y, void* stream);
/* F.normalize(x, dim=1): y = x / max(||x||_2, 1e-12) per pixel over C (P = total pixels).
 * mask (nullable, u8 [P]): masked pixels are written as zeros (quick_start/coarseAlignFeatMatch.py:143). */
int rf_l2norm_nhwc(const float* x, long long P, int C, const uint8_t* mask, float* y, void* stream);
/* same with a split input (engine 4: [2][P][C] fp16), fp32 output y (nullable); y_hi / y_lo (nullable, together): write the
 * normalised rows as fp16 hi / lo * 2^11 planes [P][C] - the operands of rf_corr_mutual_nn_presplit; C % 8 == 0 */
int rf_l2norm_split_nhwc(const void* x_split, long long P, int C, const uint8_t* mask, float* y, void* y_hi, void* y_lo, void* stream);
/* same with fp16 input (the engine-2 trunk's output), fp32 output; C % 8 == 0 */
int rf_l2norm_f16_nhwc(const void* x_f16, long long P, int C, const uint8_t* mask, float* y, void* stream);
/* model/model.py:129-160 CorrNeigh: x,y NHWC [N][h][w][C] -> out NHWC [N][h][w][ldo], channels >= k*k are
 * written as zeros (ldo = 64 makes the 49-channel volume a 128-byte-aligned operand for the conv engines);
 * round_tf32_out = 1 stores the values rounded to nearest TF32 (operand of the tensor-core heads);
 * round_tf32_out = 2 stores fp16 (out then holds N*h*w*ldo halves: the operand of the engine-2 heads) */
int rf_corr_neigh_nhwc(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, int round_tf32_out,
                       float* out, void* stream);
/* CorrNeigh(x, y) -> out_xy AND CorrNeigh(y, x) -> out_yx in one launch: the two volumes every PredFlowMask computes
 * (evaluation/evalHpatch/evaluation.py:29-30; evalCorr/evaluation.py:36-37) hold the same dot products,
 * out_yx[p][d] = out_xy[p+d][-d], so each product is computed once and stored twice (bit-identical to two
 * rf_corr_neigh_nhwc calls). */
int rf_corr_neigh_pair_nhwc(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, int round_tf32_out,
                            float* out_xy, float* out_yx, void* stream);
/* engine 4 form of the pair call: split outputs (fp16 hi / lo * 2^11 planes).  out12_split = CorrNeigh(x, y) as [2][P][ldo] (the
 * flow head's input), both_split = the two-image tensor [2][2P][ldo] = [CorrNeigh(x, y) ; CorrNeigh(y, x)] the matchability head
 * runs on (P = N*h*w; also usable with both_split = NULL for a single volume). */
int rf_corr_neigh_pair_split(const float* x, const float* y, int N, int h, int w, int C, int k, int ldo, void* out12_split, void* both_split,
                             void* stream);
/* model/model.py:226-233: softmax over k*k logits + expected offset -> flow NCHW [N][2][h][w] */
int rf_softmax_flow(const float* logits, int N, int h, int w, int k, float* flow_nchw, void* stream);
/* model/model.py:306: sigmoid, NHWC [P][1] -> [P] */
int rf_sigmoid(const float* x, long long n, float* y, void* stream);
/* ToTensor (+ Normalize): u8 HWC -> fp32 NHWC, (v/255 - mean)/std, exact torchvision op order.
 * normalize = 0 gives plain ToTensor.  (coarseAlignFeatMatch.py:63-66,106) */
int rf_preproc_u8(const uint8_t* img, long long npix, int normalize, float* out_nhwc, void* stream);
/* PIL ImagingResample (LANCZOS, 8bpc fixed point) on device: one pass.
 * coefficients come from rf_lanczos_coeffs_host (exact PIL arithmetic). */
int rf_resample_u8(const uint8_t* in, int in_h, int in_w, int channels, int horizontal,
                   const int* bounds, const int* kk, int ksize, int out_size, uint8_t* out, void* stream);
int rf_lanczos_coeffs_host(int in_size, int out_size, int* bounds_host, int* kk_host, int kk_capacity, int* ksize_out);
/* The same tables for PIL's BILINEAR filter (triangle, support 1): Image.resize(size, BILINEAR) through rf_resample_u8, the
 * resize of segNet/segData.py:7-17,71 (called from :53-76 getImg). */
int rf_bilinear_coeffs_host(int in_size, int out_size, int* bounds_host, int* kk_host, int kk_capacity, int* ksize_out);
/* The byte-scaling step of SciPy 1.2's imresize on a float32 map, as the drivers' `imresize(It_bg, (h, w)) < 128` runs it
 * (evaluation/evalHpatch/evaluation.py:180, evalCorr:187, evalYFCC:200/212, evalKITTI:248), after np.rot90 of the map:
 * out (uint8, [W][H] for odd rot, else [H][W]) = scipy.misc.bytescale(np.rot90(map [H][W], rot)), i.e. in fp32
 * clip((x - cmin) * (255 / span), 0, 255) + 0.5 truncated, span = cmax - cmin or 1 when the map is constant.  cmin / cmax are
 * reduced on the device (two launches, no host read, graph-capturable, deterministic); NaN-free maps.  The PIL BILINEAR
 * resize that follows is rf_resample_u8 with channels = 1 and the rf_bilinear_coeffs_host tables. */
size_t rf_bytescale_mask_u8_workspace(int H, int W);
int rf_bytescale_mask_u8(const float* map, int H, int W, int rot, uint8_t* out, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------ segNet --
 * The decoder of the ADE20K scene-parsing network (segNet/segModel.py:218-264 PPMDeepsup, inference) and the multi-scale vote of
 * segNet/segEval.py:23-43 getSky, on engine-4 split tensors.  The encoder (segModel.py:156-216 ResnetDilated) is an
 * rf_run_layers program with dilated 3x3 convolutions (rf_layer_t.dil).
 *
 * rf_adaptive_avgpool_split: nn.AdaptiveAvgPool2d(b) (segModel.py:227) of every image of the split batch x [2][sum HW][C] for every
 * bin count bins_host[j], in one launch.  y_host[j] (device pointer) receives the split tensor [2][nimg * b * b][C] of the b x b maps,
 * image after image.  Bin i of n rows spans [floor(i n / b), ceil((i + 1) n / b)): bins overlap or repeat when n < b.  C % 8 == 0,
 * nbins <= 8. */
int rf_adaptive_avgpool_split(const void* x, int nimg, const int* hw_host, int C, const int* bins_host, int nbins, void* const* y_host,
                              void* stream);
/* The input of PPMDeepsup.conv_last (segModel.py:249-256) in one pass: y [2][sum HW][C5 + nbins * Cb] split, channels [0, C5) a copy
 * of conv5 [2][sum HW][C5], channel block j the bilinear (align_corners=False) upsampling of branch j (y_host[j] of
 * rf_adaptive_avgpool_split after its 1x1 conv: [2][nimg * b_j * b_j][Cb]) to each image's size.  C5 % 8 == Cb % 8 == 0. */
int rf_ppm_concat_split(const void* conv5, int nimg, const int* hw_host, int C5, void* const* branches_host, const int* bins_host, int nbins,
                        int Cb, void* y, void* stream);
/* segEval.py:28-43 for one image.  logits fp32 [sum h_j w_j][ncls] of the distinct scales (hw_host = their sizes; the output of
 * conv_last's final 1x1 conv on RF_ENGINE_SPLIT_OUT32); order_host[k] (k < norder) = the scale each of the reference's passes used, with
 * repeats.  Per pixel of the H x W output: bilinear (align_corners=False) upsampling of each pass's logits, softmax over the ncls
 * classes, scores += p / 5 in pass order (segEval.py:36), arg-max with the lowest index on ties, mask_out[p] = (pred == segId) as
 * float (1 - that when segFg).  class_out (int32 [H][W]) and scores_out (fp32 [H][W][ncls]) are nullable debug outputs.
 * ncls <= 160, norder <= 8. */
int rf_seg_vote(const float* logits, int nimg, const int* hw_host, int ncls, const int* order_host, int norder, int H, int W, int segId,
                int segFg, float* mask_out, int* class_out, float* scores_out, void* stream);

/* -------------------------------------------------------------------- warp --
 * kornia 0.1.4 HomographyWarper.warp_grid: H [N][9] -> grid [N][h][w][2] */
int rf_warp_grid(const float* H, int N, int h, int w, float* grid_out, void* stream);
/* F.grid_sample(bilinear, zeros).  Generic element strides so NCHW and NHWC both work.
 * in: (N,C,Hin,Win) with strides in_s[4] (N,C,H,W); grid [N][Hout][Wout][2]; out strides out_s[4]. */
int rf_grid_sample(const float* in, int N, int C, int Hin, int Win, const long long* in_s_host,
                   const float* grid, int Hout, int Wout, int align_corners,
                   float* out, const long long* out_s_host, void* stream);
/* train/generate_coarse_aligned_pair.ipynb cells 13 + ToPILImage in one pass: out [h][w][3] uint8 = (uint8)(255 * grid_sample(
 * ToTensor(src), warp_grid(H, h, w))), truncated, with rf_warp_grid's, rf_grid_sample's and rf_preproc_u8's arithmetic (bit for bit
 * the composition of the three and the quantisation).  H: 9 floats in DEVICE memory (a non-finite H samples nothing: zeros);
 * src [Hin][Win][3] uint8. */
int rf_warp_sample_u8(const float* H, const uint8_t* src, int Hin, int Win, int h, int w, int align_corners, uint8_t* out, void* stream);
/* train/validation.py:80,98-99 in one pass: out_nhwc [h][w][3] fp32 = F.grid_sample(ToTensor(src), F.affine_grid(theta, (1, 3, h, w)))
 * (bilinear, zeros, align_corners=False), written where the FeatureExtractor's input row of the image goes.  theta: 6 floats
 * (2 x 3, row-major) in DEVICE memory (a non-finite theta samples zeros); src [Hin][Win][3] uint8. */
int rf_affine_sample_u8(const float* theta, const uint8_t* src, int Hin, int Win, int h, int w, float* out_nhwc, void* stream);
/* train/validation.py:93-107 + alignmentError (:33-53) at the keypoints only, from flowDown8 = softmax_flow's (2, h8, w8) on the
 * H x W target: kpts [capacity][4] int32 (xa, ya, xb, yb), *count (DEVICE) of them used; theta 6 floats in DEVICE memory; wA, hA
 * the resized source's size.  counts [T + 1] uint64 (DEVICE) accumulate, per threshold, the keypoints whose fp64 distance is
 * strictly below it, and the keypoints scored; an index outside torch's [-n, n) range sets *err = min(*err, pair).
 * dist_out [capacity] fp64 and flow_out [capacity][4] fp32 (16-byte aligned: the clamped fine flow at (yb, xb), then the composed
 * flow, i.e. the affine grid sampled there) are optional (NULL). */
int rf_val_keypoints(const float* flowDown8, int h8, int w8, const float* theta, int H, int W, int wA, int hA, const int* kpts,
                     const int* count, int capacity, int pair, const double* thresholds_host, int T, unsigned long long* counts,
                     int* err, double* dist_out, float* flow_out, void* stream);
/* evaluation/evalCorr/getResults.py:78-134 (getFlow, or getFlow_Coarse with onlyCoarse) + :220-227 + alignmentError (:15-38) at
 * the keypoints only, for one pair: flowDown8 / matchDown8 [nH][2][h8][w8] and H [nH][9] fp32 in DEVICE memory (the flows
 * and matchabilities may be NULL with onlyCoarse), composed at 8h8 x 8w8; kpts [capacity][4] int32 (xa, ya, xb, yb), *count
 * (DEVICE) of them used; Ith x Itw the target's size, wA x hA the source's.  th: the merge threshold (float32), multiH: merge
 * all hypotheses, else hypothesis 0 alone.  thresholds_host [T] pixel thresholds (<=); mth_host [J] the matchability thresholds
 * th_j in order and slot_host [J] their accumulator rows.  counts [rows][T + 1] uint64 (DEVICE) accumulate, per row, the
 * keypoints within each pixel threshold and the keypoints scored; an index outside numpy's [-n, n) range sets
 * *err = min(*err, pair).  Optional (NULL) per-keypoint outputs: flow_out [capacity][2] and match_out [capacity] the merged flow
 * and matchability at (yb, xb), hyp_out [capacity] the winning hypothesis, dist_out [capacity][J] the fp64 distance per th_j
 * (NaN where the keypoint is not selected).  For th_j > 0 the map must be square (see DESIGN.md section 12). */
int rf_corr_keypoints(const float* flowDown8, const float* matchDown8, const float* H, int nH, int h8, int w8, int Ith, int Itw,
                      int wA, int hA, const int* kpts, const int* count, int capacity, int pair, float th, int multiH, int onlyCoarse,
                      const double* thresholds_host, int T, const double* mth_host, const int* slot_host, int J,
                      unsigned long long* counts, int* err, float* flow_out, float* match_out, int* hyp_out, double* dist_out,
                      void* stream);
/* F.interpolate(mode='bilinear', align_corners=False): NCHW [NC][h][w] -> [NC][H][W] */
int rf_upsample_bilinear(const float* in, int NC, int h, int w, int H, int W, float* out, void* stream);
/* PredFlowMask tail, evaluation/evalHpatch/evaluation.py:37-51 fused:
 * flowUp = clamp(interp(flowDown8) + grid); flow12 = grid_sample(coarse, flowUp);
 * match = interp(match12) [* grid_sample(interp(match21), flowUp)] * inside(flow12).
 * flowDown8 NCHW [2][h8][w8]; match12/match21 [h8][w8] (match21 nullable);
 * coarse [H][W][2]; outputs flow12 [H][W][2], match [H][W] (nullable), flowUp [H][W][2] (nullable). */
int rf_compose_fine(const float* flowDown8, const float* match12, const float* match21, int h8, int w8,
                    const float* coarse, int H, int W, int clamp, int align_corners,
                    float* flow12_out, float* match_out, float* flowUp_out, void* stream);
/* The same with a coarse grid of its own size, coarse [Hc][Wc][2] sampled at the (H, W) output positions: the second
 * level of the KITTI flow (evaluation/evalKITTI/evaluation.py:296-302: PredFlowMask with the resized image's flow and
 * the original image's grid) and the two-level recomposition of evaluation/evalKITTI/getResults.py:104-113. */
int rf_compose_fine_ex(const float* flowDown8, const float* match12, const float* match21, int h8, int w8,
                       const float* coarse, int Hc, int Wc, int H, int W, int clamp, int align_corners,
                       float* flow12_out, float* match_out, float* flowUp_out, void* stream);
/* remove_small_cc, evaluation/evalKITTI/evaluation.py:85-100 and evalKITTI/getResults.py:66-83, in place on
 * match [N][H][W]: every 8-connected component (skimage.measure.label's default for 2-D) of (match > match_th) whose
 * area fraction count / (H*W) is <= cc_th gets its matchability zeroed; cc_th == 0 leaves the map untouched. */
size_t rf_remove_small_cc_workspace(int H, int W);
int rf_remove_small_cc(float* match, int N, int H, int W, float match_th, double cc_th, void* ws, size_t ws_bytes, void* stream);
/* One hypothesis of evalKITTI's loop after remove_small_cc (evaluation/evalKITTI/evaluation.py:316-326), with the host's
 * decisions kept on the device.  match, bg [H][W] fp32 (bg: 1 = kept); Mask, fgMask [H][W] fp32 {0, 1}, in / out; status
 * (int32, RF_RANSAC_*) and alive (int32 flag, in / out) are device scalars.
 *   count = #{p : match[p] > 0.9999f && fgMask[p] == 0}      (exact: both factors of the reference's product are 0 / 1)
 *   alive = alive && status == 0 && (first || count >= cmin)
 * and where alive holds, in fp32 as numpy evaluates it: Mask = ((Mask + match * (1 - fgMask)) > 0.9999f), then
 * fgMask = ((Mask + (1 - bg)) > 0.5f).  Where it does not, Mask and fgMask are left untouched.  cmin is the smallest count the
 * reference's float32 test `mean > maskRegionTh` accepts for an H*W map (found on the host).  rec (nullable, int32 [2]) receives
 * {alive, count}.  Two launches (per-CTA partial counts, then a fixed-order reduction in every CTA + the update), no host read,
 * no atomics: graph-capturable and deterministic. */
size_t rf_kitti_region_step_workspace(int H, int W);
int rf_kitti_region_step(const float* match, float* Mask, const float* bg, float* fgMask, int H, int W, const int* status, int* alive,
                         int first, int cmin, int* rec, void* ws, size_t ws_bytes, void* stream);

/* interpolate_flow_match, evaluation/evalKITTI/getResults.py:87-93: flow_out[p] = flow[nearest matched pixel of p]
 * (exact Euclidean distance; a matched pixel keeps its own flow).  flow / flow_out [H][W][2] (distinct buffers), matched
 * u8 [H][W] (non-zero = matched), index_out (nullable) int32 [H][W][2] = (row, col) of the chosen pixel.  Between
 * equidistant matched pixels the choice is this library's (documented at the kernel), not scipy's. */
size_t rf_fill_nearest_matched_workspace(int H, int W);
int rf_fill_nearest_matched(const float* flow, const uint8_t* matched, int H, int W, float* flow_out, int* index_out,
                            void* ws, size_t ws_bytes, void* stream);

/* -------------------------------------------------------------- YFCC pose --
 * The relative-pose metric of evaluation/evalYFCC/getResults.py:53-111 (matches_from_flow, norm_kp, opencv_decompose) in
 * fp64 on the device.  The point count stays on the device; the three calls share one record the host reads at the end. */
#define RF_POSE_OK 0          /* E (and, after rf_recover_pose, R / t) valid                                     */
#define RF_POSE_TOO_FEW 1     /* fewer than 5 matches: the driver's pts1.shape[0] >= 5 test fails (no model)     */
#define RF_POSE_NO_MODEL 2    /* findEssentialMat finds no E with 5 or more inliers; findFundamentalMat no F     */
#define RF_POSE_NO_POSE 3     /* every recoverPose count is 0: the driver's loop keeps no (R, t)                 */
typedef struct rf_pose_record {
    int status;                     /* RF_POSE_* */
    int n_points;                   /* N */
    int niters;                     /* RANSAC iteration budget at the end (RANSACUpdateNumIters); 0 from rf_fundamental_8point */
    int best_iter, best_cand;       /* (iteration, candidate) of the best E; -1 when none, and from rf_fundamental_8point */
    int ransac_count;               /* its inlier count; -1 from rf_fundamental_8point (its mask is all ones) */
    int n_E;                        /* stacked candidates in E: 1, or every solution of the single minimal problem when N == 5
                                       (rf_essential_ransac) or N == 7 (rf_fundamental_8point: 1..3) */
    int pose_count;                 /* the driver's num_inlier */
    int pose_cand, pose_index;      /* the winning candidate and its pose (0..3: (R1, t), (R2, t), (R1, -t), (R2, -t)) */
    int pose_counts[40];            /* [candidate][pose] cheirality counts */
    double E[90];                   /* [n_E][3][3] row-major: E with unit Frobenius norm (rf_essential_ransac), or F as
                                       cv2.findFundamentalMat returns it, F22 = 1 unless |F22| <= FLT_EPSILON (rf_fundamental_8point) */
    double poses[480];              /* [candidate][pose][3][4] = [R | t] of decomposeEssentialMat */
    double R[9], t[3];
} rf_pose_record_t;
/* matches_from_flow (:53-71) + norm_kp (:29-50): flow [H][W][2] fp32 (flowGlobal), mask [H][W] u8 (non-zero = matched), the target
 * grid np.rot90(meshgrid(arange(wB), arange(hB)), k) (H x W after the rotation, else an error), (wA, hA) the source size,
 * norm1_host / norm2_host = (cx, cy, fx, fy) of each image.  pts1 = ((f + 1) * (wA - 1) / 2 in fp32 - c) / f_ in fp64,
 * pts2 = (grid - c) / f_ in fp64, [H*W][2] capacity, in numpy's boolean-index (row-major) order; the count goes to *N_out. */
size_t rf_yfcc_matches_workspace(int H, int W);
int rf_yfcc_matches(const float* flow, const uint8_t* mask, int H, int W, int k, int wB, int hB, int wA, int hA,
                    const double* norm1_host, const double* norm2_host, double* pts1_out, double* pts2_out, int* N_out,
                    void* ws, size_t ws_bytes, void* stream);
/* cv2.findEssentialMat(pts1, pts2, method=RANSAC, threshold) (focal 1, pp (0, 0), prob 0.999, maxIters 1000): cv::RNG((uint64)-1)
 * subsets, every real five-point solution of each (ascending root), OpenCV's Sampson error cast to fp32 against (float)(t * t),
 * and RANSACPointSetRegistrator::run's sequential best / iteration-budget update, scored 64 iterations per launch (a launch past
 * the budget exits at once: a fixed launch sequence, graph-capturable).  pts [capacity][2], N = *N_dev <= capacity.
 * Writes rec (status, E, counts) and mask_out[N] (the best E's inliers; all ones when N == 5).
 * ws holds four segments, each starting at a multiple of 256 bytes after the one before it: idx [1000][5] int32 (the subset
 * table; untouched when N < 5, row 0 only when N == 5), candE [1000][10][9] fp64 (the solutions of each subset), ncand [1000]
 * int32 (their count), counts [1000][10] int32 (Sampson inlier counts; zero for launches past the budget). */
size_t rf_essential_ransac_workspace(int capacity);
int rf_essential_ransac(const double* pts1, const double* pts2, int capacity, const int* N_dev, double threshold,
                        rf_pose_record_t* rec, uint8_t* mask_out, void* ws, size_t ws_bytes, void* stream);
/* cv2.recoverPose(E, pts1, pts2, mask=mask_in) for each stacked E of rec (distance threshold 50), with the driver's loop
 * (:96-104): cv2 writes each call's mask into mask_in, so candidate c + 1 starts from candidate c's output, and the first
 * candidate with the strictly largest count wins.  Writes rec (R, t, pose_count, status) and mask_out[N] whatever the status:
 * the winner's mask, or zeros when no candidate wins (RF_POSE_NO_POSE) or rec holds no E (RF_POSE_TOO_FEW, RF_POSE_NO_MODEL).
 * The first 8 * capacity bytes of ws hold the per-point cheirality bits: bit 4 c + p = pose p of candidate c passes. */
size_t rf_recover_pose_workspace(int capacity);
int rf_recover_pose(const double* pts1, const double* pts2, int capacity, const uint8_t* mask_in, rf_pose_record_t* rec,
                    uint8_t* mask_out, void* ws, size_t ws_bytes, void* stream);
/* The stages of rf_essential_ransac alone (for tests): the [1000][5] int32 subset table of N = *N_dev points; the five-point
 * solutions E_out [nsamples][10][9] / nsol_out [nsamples] of the subsets idx [nsamples][5]; the Sampson inlier counts of nmodels
 * (<= 640) models E [nmodels][9] over N points, with the fp32 errors in err_out [nmodels][N] (nullable). */
int rf_essential_samples(const int* N_dev, int* idx_out, void* stream);
int rf_essential_five_point(const double* pts1, const double* pts2, const int* idx, int nsamples, double* E_out, int* nsol_out,
                            void* stream);
int rf_essential_score(const double* pts1, const double* pts2, int N, const double* E, int nmodels, double threshold,
                       int* counts_out, float* err_out, void* stream);
/* cv2.findFundamentalMat(pts1, pts2, method=FM_8POINT), the driver's non-RANSAC branch (:84-87), with the points cast to fp32
 * first as cv2 does: N < 5 RF_POSE_TOO_FEW; 5 <= N < 7 RF_POSE_NO_MODEL; N == 7 the seven-point solver (n_E = 1..3 stacked
 * candidates in cv2's order); N >= 8 the eight-point solver (n_E = 1); a degenerate normalisation or eigen-spectrum, or no real
 * root, RF_POSE_NO_MODEL.  mask_out[N] is all ones whenever N >= 7.  Three grid-wide fp64 reductions (centroids, mean
 * distances, the 45 moments of A = sum r r^T) write per-CTA partials that are summed in a fixed order (no atomics: the same
 * bits on every run), then one warp solves the 9 x 9 eigenproblem.  A fixed launch sequence sized from capacity, N = *N_dev
 * <= capacity on the device: graph-capturable.  rf_recover_pose then runs on rec as it does after rf_essential_ransac. */
size_t rf_fundamental_8point_workspace(int capacity);
int rf_fundamental_8point(const double* pts1, const double* pts2, int capacity, const int* N_dev, rf_pose_record_t* rec,
                          uint8_t* mask_out, void* ws, size_t ws_bytes, void* stream);
/* The reductions of rf_fundamental_8point alone (for tests), N = *N_dev >= 1: out[51] = (m1c.x, m1c.y, m2c.x, m2c.y, scale1,
 * scale2, A[45]) with scale = sqrt(2) / mean distance and A's upper triangle row by row (A00, A01, ..., A08, A11, ..., A88).
 * ws as rf_fundamental_8point_workspace(capacity). */
int rf_fundamental_moments(const double* pts1, const double* pts2, int capacity, const int* N_dev, double* out, void* ws,
                           size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
