/*
 * b200seg.h -- C ABI of the H100-native (sm_90a) segmentation hot path.
 *
 * The reference (junqiangchen/PytorchDeepLearing) has NO native code and NO FFI: its "plugin
 * boundary" is the Python nn.Module protocol used by model/modelVNet.py:490-497,546-548,580-593
 * and model/modelUnet.py:46,270,490,793 (SURVEY.md section 8b).  The Python drop-in
 * (pytorchdeeplearing_b200/) keeps that protocol and binds the entry points below through ctypes
 * (pytorchdeeplearing_b200/_abi.py).  Each entry point replaces the ATen call sites cited next to
 * it (file:line relative to the reference root).
 *
 * Conventions
 *   - returns 0 on success, a negative B200SEG_E* code otherwise (b200seg_last_error() has text);
 *   - never allocates, frees or synchronises: caller owns every buffer (torch caching allocator),
 *     every launch goes to the cudaStream_t passed in, on CUDA device `device`;
 *   - re-entrant and thread-safe (autograd runs backward on its own thread);
 *   - activations are channels-last tensors (N, D, H, W, C) with a channel pitch `ld >= C`
 *     (elements) so that a producer can write into a slice of a skip-concat buffer; 2-D networks
 *     use D == 1 and `dims == 2`.
 */
#ifndef B200SEG_H
#define B200SEG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SEG_VERSION 200

#define B200SEG_OK 0
#define B200SEG_EINVAL (-1)   /* bad argument / unsupported combination */
#define B200SEG_ECUDA (-2)    /* CUDA runtime error (text in b200seg_last_error) */

#define B200SEG_F32 0
#define B200SEG_BF16 1
#define B200SEG_BF16_TC 2 /* weights only: bf16 packed [tap][N][K] (K-major) for the wgmma/TMA conv path */
#define B200SEG_BF16_HALO 3 /* weights only: bf16 packed [tap][K/8][N][8] (smem image of the halo-staged 3x3x3 path) */
#define B200SEG_BF16_HALO_WS 4 /* weights only: bf16 packed [N/NT][tap][K/8][NT][8], NT = b200seg_conv_halo_ws_ntile():
                                  per-group tap blocks streamed by the 64/128-channel halo-staged 3x3x3 path */

#define B200SEG_I64 16 /* labels only: int64 class indices (model/dataset.py:114); B200SEG_F32 = soft binary targets */
#define B200SEG_U8 17  /* masks only: one byte per voxel (bool or uint8) */
#define B200SEG_I32 18 /* masks only: int32 */
#define B200SEG_I16 19 /* resampled volumes only: int16 */

/* intensity steps of b200seg_resample_linear / b200seg_normalize */
#define B200SEG_NORM_NONE 0    /* resample only */
#define B200SEG_NORM_MEANSTD 1 /* truncate to [lower, upper], then (x - mean) / sigma (N - 1) */
#define B200SEG_NORM_PCTL 2    /* dataprocess/utils.py normalize(): 5/95 percentile clip, z-score of the nonzero voxels */

/* conv kinds */
#define B200SEG_K3 0    /* 3x3x3 (dims==3) or 1x3x3 (dims==2), stride 1, zero pad 1 */
#define B200SEG_K1 1    /* 1x1x1 */
#define B200SEG_DOWN 2  /* k=2, s=2 convolution (space-to-depth GEMM) */
#define B200SEG_UP 3    /* k=2, s=2 transposed convolution (GEMM + depth-to-space) */

/* kernel families b200seg_conv chooses from (b200seg_conv_path) */
#define B200SEG_CONV_PW_MMA 0    /* pw_mma.cu: register-level mma.sync 1x1x1 / transposed conv, >= 65536 voxels */
#define B200SEG_CONV_TC 1        /* conv_tc.cu: wgmma + TMA implicit GEMM */
#define B200SEG_CONV_HALO2D 2    /* conv_halo.cu: halo-staged 3x3, 16/32 channels */
#define B200SEG_CONV_HALO3 3     /* conv_halo.cu: halo-staged 3x3x3, 16/32 channels */
#define B200SEG_CONV_HALO_WS 4   /* conv_halo_ws.cu: weight-streaming halo-staged 3x3x3, 64/128 input channels */
#define B200SEG_CONV_STEM_MMA 5  /* stem_mma.cu: one input channel on mma.sync */
#define B200SEG_CONV_STEM 6      /* stem.cu: one input channel on CUDA cores */
#define B200SEG_CONV_SMALLCIN 7  /* small_channels.cu: <= 4 input channels */
#define B200SEG_CONV_GENERIC 8   /* conv_generic.cu: any shape */
/* kernel families b200seg_wgrad chooses from (b200seg_wgrad_path) */
#define B200SEG_WGRAD_HALO_MMA 0 /* wgrad_halo_mma.cu: 3x3x3, 16/32 channels, >= 32768 voxels */
#define B200SEG_WGRAD_TC 1       /* wgrad_tc.cu: wgmma + TMA */
#define B200SEG_WGRAD_STEM_MMA 2 /* stem_mma.cu */
#define B200SEG_WGRAD_STEM 3     /* stem.cu */
#define B200SEG_WGRAD_SMALLCIN 4 /* small_channels.cu */
#define B200SEG_WGRAD_GENERIC 5  /* wgrad_generic.cu */

/* loss terms (bitmask) */
#define B200SEG_LOSS_DICE 1
#define B200SEG_LOSS_CE 2
#define B200SEG_LOSS_FOCAL 4
/* one of these alone (not combined with each other or with the three above) */
#define B200SEG_LOSS_JACCARD 8    /* BinaryJaccardLoss, model/losses.py:19-30 */
#define B200SEG_LOSS_ELDICE 16    /* BinaryELDiceLoss (C == 1) losses.py:66-74, MutilELDiceLoss (C > 1) :358-382 */
#define B200SEG_LOSS_TVERSKY 32   /* BinaryTverskyLoss, losses.py:113-126 */
#define B200SEG_LOSS_SS 64        /* BinarySSLoss, losses.py:87-99 (partials: b200seg_loss_partials_ss) */
#define B200SEG_LOSS_EXT_MASK (B200SEG_LOSS_JACCARD | B200SEG_LOSS_ELDICE | B200SEG_LOSS_TVERSKY | B200SEG_LOSS_SS)

typedef struct b200seg_tensor {
  void* ptr;       /* device pointer to element (0,0,0,0,0) */
  int32_t n, d, h, w, c;
  int64_t ld;      /* channel pitch in elements: element (n,d,h,w,c) is at (((n*d_+d)*h_+h)*w_+w)*ld + c */
  int32_t dtype;   /* B200SEG_F32 | B200SEG_BF16 */
} b200seg_tensor;

typedef void* b200seg_stream; /* cudaStream_t */
struct b200seg_gn;

int b200seg_version(void);
const char* b200seg_last_error(void);
/* one-time per-process/per-device setup (opt-in shared memory sizes); safe to call repeatedly */
int b200seg_init(int device);

/* ---- weights --------------------------------------------------------------------------------
 * out[t][k][n2][n1] = w[tmap(t)*st + k*sk + n2*sn2 + n1*sn1], tmap(t) = flip ? T-1-t : t.
 * Turns nn.Conv3d (Co,Ci,k,k,k) / nn.ConvTranspose3d (Ci,Co,k,k,k) parameters
 * (networks/VNet3d.py:8,28,29,49,65,70,88; Unet3d.py:26-34,67-81) into the [tap][K][N] operand
 * layouts of b200seg_conv (forward and data-gradient forms). */
int b200seg_pack_weight(const float* w, void* out, int out_dtype, int T, int K, int N2, int N1, int64_t st,
                        int64_t sk, int64_t sn2, int64_t sn1, int flip, int device, b200seg_stream stream);
/* grad[t*st + k*sk + n*sn] = dwp[t][k][n]  (inverse permutation, fp32 -> parameter .grad layout) */
int b200seg_unpack_wgrad(const float* dwp, float* grad, int T, int K, int N, int64_t st, int64_t sk, int64_t sn,
                         int device, b200seg_stream stream);

/* Multi-tensor forms of the two calls above: ONE launch for every conv operand of a network.  `table` is a DEVICE
 * array of `count` descriptors; descriptor i owns thread blocks [block_start, block_start + nblocks) and
 * total_blocks = sum of nblocks.  pack: dst[t][k][n2][n1] (out_dtype) = src[tmap(t)*st + k*sk + n2*sn2 + n1*sn1];
 * unpack: dst[t*st + k*sk + n*sn2] = src[(t*K + k)*N2 + n] (fp32, N1 ignored). */
typedef struct b200seg_pack_desc {
  const float* src;
  void* dst;
  int64_t st, sk, sn2, sn1;
  int32_t out_dtype, T, K, N2, N1, flip;
  int32_t block_start, nblocks;
} b200seg_pack_desc;
int b200seg_pack_weights_multi(const b200seg_pack_desc* table, int count, int total_blocks, int device,
                               b200seg_stream stream);
/* Copy a small host array (descriptor table; bytes % 16 == 0, 16-byte aligned destination) to device memory through
 * KERNEL ARGUMENTS instead of a memcpy: inside a captured step this keeps the copy engines free for the caller's own
 * input prefetch (a memcpy node would queue behind it and stall the graph).  The host array is read during the call. */
int b200seg_upload_table(const void* host_table, int64_t bytes, void* device_dst, int device, b200seg_stream stream);
int b200seg_unpack_wgrads_multi(const b200seg_pack_desc* table, int count, int total_blocks, int device,
                                b200seg_stream stream);

/* ---- convolution family (replaces F.conv3d / F.conv_transpose3d / F.conv2d, call sites above;
 * the data-gradient half of aten::convolution_backward runs through the same entry with
 * dgrad-packed weights).
 *   y = conv_kind(x, wpk) [+ bias] [+ addend];   stats[n][c] += {sum, sum of squares} of (conv + bias)
 * x: F32|T, wpk: T (dtype w_dtype), y: T|F32, addend: same dtype as y or NULL, bias fp32 or NULL,
 * stats: double [N][Cout][2] or NULL (GroupNorm statistics fused into the epilogue: nn.GroupNorm,
 * VNet3d.py:9,30,50,66; Unet3d.py:73,82). */
int b200seg_conv(int kind, int dims, const b200seg_tensor* x, const void* wpk, int w_dtype, const float* bias,
                 const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device,
                 b200seg_stream stream);
/* the B200SEG_CONV_* kernel family b200seg_conv would run for these arguments (host only, launches nothing), or
 * B200SEG_EINVAL where b200seg_conv would refuse them */
int b200seg_conv_path(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                      const b200seg_tensor* addend);

/* Data-gradient convolution that ALSO accumulates the GroupNorm-backward sums of the layer behind its output:
 * g = conv_kind(x, wpk) [+ addend] is dL/d(activation) of the layer whose raw conv output is `yfwd` and whose
 * GroupNorm / dropout coefficients follow from `gn` (its forward statistics); with m = [yfwd*A + B > 0]
 *   sums[n][c][0] += sum g*m,   sums[n][c][1] += sum g*m*yfwd        (double [N][C][3], caller zero-fills; [2] untouched)
 * i.e. what b200seg_gn_bwd_reduce_gn would compute in a separate pass over g and yfwd (native_group_norm_backward +
 * threshold_backward, VNet3d.py:9-15).  Follow with b200seg_gn_bwd_apply_gn(..., sum_y_from_stats = 1).  Only the
 * 3-D halo-staged 16/32-channel 3x3x3 kernel has this epilogue: ask b200seg_conv_bwdstats_supported first. */
int b200seg_conv_bwdstats_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                                    const b200seg_tensor* addend, const b200seg_tensor* yfwd);
int b200seg_conv_bwdstats(int kind, int dims, const b200seg_tensor* x, const void* wpk, int w_dtype,
                          const b200seg_tensor* y, const b200seg_tensor* addend, const b200seg_tensor* yfwd,
                          const struct b200seg_gn* gn, double* sums, int device, b200seg_stream stream);

/* 1 if b200seg_conv runs (kind, Cin -> Cout) on the wgmma + TMA path when given bf16 activations and
 * B200SEG_BF16_TC weights ([tap][Cout][Cin] for the forward form, [tap'][Cin][Cout], taps flipped, for the
 * data-gradient form); 0 -> pack [tap][K][N] and use the CUDA-core path. */
int b200seg_conv_tc_eligible(int kind, int cin, int cout);
/* 1 if (kind, Cin -> Cout) can run on the halo-staged wgmma kernel (3x3x3 / 3x3, 16/32 channels) given
 * B200SEG_BF16_HALO weights; meant for the full-resolution layers (each input voxel is staged once in shared
 * memory instead of once per tap). */
int b200seg_conv_halo_eligible(int kind, int cin, int cout);
/* columns per weight group (NT) if (kind, Cin -> Cout) can run on the weight-streaming halo-staged wgmma kernel
 * (3x3x3, 64/128 input channels: the 24^3 / 12^3 pyramid levels) given B200SEG_BF16_HALO_WS weights, else 0. */
int b200seg_conv_halo_ws_ntile(int kind, int cin, int cout);

/* weight-gradient half of aten::convolution_backward:
 *   dwp[t][ka][kb] += sum_{n,o} a[n, o*s + t - p, ka] * b[n, o, kb]      (fp32, caller zero-fills)
 * kind in {K3, K1, DOWN}; for the transposed conv call with kind = DOWN, a = dy (fine), b = x. */
int b200seg_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                  b200seg_stream stream);
/* the B200SEG_WGRAD_* kernel family b200seg_wgrad would run for these arguments (host only), or B200SEG_EINVAL */
int b200seg_wgrad_path(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b);

/* ---- GroupNorm(8) + Dropout(p) + ReLU tail (nn.GroupNorm / nn.Dropout3d / nn.ReLU, VNet3d.py:9-11,14;
 * Unet3d.py:73-75) split into statistics (conv epilogue) -> finalize -> apply (SURVEY.md App. G) */
int b200seg_gn_finalize(const double* stats, const float* gamma, const float* beta, const float* scale, int N, int C,
                        int groups, int64_t vox, float eps, float* coef /*[N][C][2]*/, float* mr /*[N][G][2]*/,
                        int device, b200seg_stream stream);
/* out = relu(y1*A1+B1) [+ relu(y2*A2+B2)] [+ res]   (torch.add residuals VNet3d.py:41,58,79) */
int b200seg_apply(const b200seg_tensor* y1, const float* coef1, const b200seg_tensor* y2, const float* coef2,
                  const b200seg_tensor* res, const b200seg_tensor* out, int device, b200seg_stream stream);
/* Fused-coefficient forms: the kernels derive A, B (and the backward P, Q, R, d gamma, d beta, d bias) for their
 * own channels from the fp64 statistics, so no finalize launches are needed.  `b200seg_gn` names one GroupNorm
 * application: statistics [N][C][2] written by b200seg_conv, affine parameters, optional dropout scale [N][C]. */
typedef struct b200seg_gn {
  const double* stats;
  const float* gamma;
  const float* beta;
  const float* scale;
  int32_t groups;
  int64_t vox;     /* voxels per sample of the normalised tensor */
  float eps;
} b200seg_gn;
int b200seg_apply_gn(const b200seg_tensor* y1, const b200seg_gn* gn1, const b200seg_tensor* y2, const b200seg_gn* gn2,
                     const b200seg_tensor* res, const b200seg_tensor* out, int device, b200seg_stream stream);
int b200seg_gn_bwd_reduce_gn(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, double* sums,
                             int device, b200seg_stream stream);
/* dy as b200seg_gn_bwd_apply; additionally dgamma[c] +=, dbeta[c] +=, dbias[c] += (dbias may be NULL; fp32 atomics
 * over the samples: the caller zero-fills the gradient bucket) */
int b200seg_gn_bwd_apply_gn(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, const double* sums,
                            const b200seg_tensor* dy, float* dgamma, float* dbeta, float* dbias,
                            int sum_y_from_stats /* 1: sums[..][2] is not filled, sum y = gn->stats[..][0] */, int device,
                            b200seg_stream stream);

/* b200seg_gn_bwd_reduce_gn + b200seg_gn_bwd_apply_gn in ONE launch for small tensors (the 24^3 level and below: the
 * two passes are separated by a grid-wide barrier and the tensors stay in L2).  `sums` [N][C][3] and the barrier
 * word `counter` must be zero on entry; every CTA of the launch has to be resident, so ask
 * b200seg_gn_bwd_fused_supported (size, layout, N <= #SMs) first and fall back to the two-launch form. */
int b200seg_gn_bwd_fused_supported(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_tensor* dy, int device);
int b200seg_gn_bwd_fused_gn(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, double* sums,
                            unsigned int* counter, const b200seg_tensor* dy, float* dgamma, float* dbeta,
                            float* dbias, int device, b200seg_stream stream);

/* native_group_norm_backward + threshold_backward + dropout backward:
 *   sums[n][c] += { sum g*m, sum g*m*y, sum y },  m = [y*A+B > 0] */
int b200seg_gn_bwd_reduce(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, double* sums,
                          int device, b200seg_stream stream);
int b200seg_gn_bwd_finalize(const double* sums, const float* mr, const float* gamma, const float* scale, int N, int C,
                            int groups, int64_t vox, float* coef3 /*[N][C][3]*/, float* dgamma /* += */,
                            float* dbeta /* += */, float* dbias /* = or NULL */, int device, b200seg_stream stream);
/* dy = (y*A+B > 0 ? g*P : 0) + y*Q + R */
int b200seg_gn_bwd_apply(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, const float* coef3,
                         const b200seg_tensor* dy, int device, b200seg_stream stream);
/* out[c] = sum_{n,d,h,w} dy[...,c]   (bias gradient of convs without GroupNorm) */
int b200seg_colsum(const b200seg_tensor* dy, float* out, int device, b200seg_stream stream);

/* ---- fused input block (VNet3d.py:25-43 / ResNet3d.py:24-41): conv1 3x3x3 and conv2 1x1x1 of a one-channel fp32
 * image x, 16 channels each, ONE GroupNorm(8, 16) applied to each branch with its own statistics, dropout, ReLU and
 * the sum of the branches.  No pass stores the raw stem outputs: each recomputes them from x with the arithmetic of
 * b200seg_conv's stem kernels, so the results equal b200seg_conv (stats) -> b200seg_apply_gn(y_a, y_b) on the
 * forward side and b200seg_gn_bwd_reduce_gn -> b200seg_gn_bwd_apply_gn -> b200seg_wgrad per branch on the backward
 * side.  w3 / w1: the bf16 forward operands (b200seg_pack_weight, [27][16] / [1][16]); gn3 / gn1: the GroupNorm
 * reference of each branch (8 groups, vox = D*H*W); stats [N][16][2], sums [N][16][3] fp64, zero on entry where
 * written.  Ask b200seg_stem_gn_supported first (3-D, fp32 x, H % 8 == 0, W a multiple of 16, 16 channels). */
int b200seg_stem_gn_supported(const b200seg_tensor* x, int cout, int dims);
/* per-(n, c) sum y, sum y^2 of both branches (what b200seg_conv writes into its stats argument) */
int b200seg_stem_gn_stats(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                          double* stats3, double* stats1, int device, b200seg_stream stream);
/* out = relu(y3*A3+B3) + relu(y1*A1+B1); out: bf16, 16 channels, any pitch */
int b200seg_stem_gn_apply(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                          const b200seg_gn* gn3, const b200seg_gn* gn1, const b200seg_tensor* out, int device,
                          b200seg_stream stream);
/* sums3 / sums1 [N][16][3] += {sum g*m, sum g*m*y, sum y} of each branch (b200seg_gn_bwd_reduce_gn's layout) */
int b200seg_stem_gn_bwd_sums(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                             const b200seg_gn* gn3, const b200seg_gn* gn1, const b200seg_tensor* g, double* sums3,
                             double* sums1, int device, b200seg_stream stream);
/* dw3 [27][16] +=, dw1 [16] +=, dgamma, dbeta [16] += (both branches), db3, db1 [16] += (may be NULL): the weight
 * gradients of both stems with the GroupNorm backward folded in; dy itself never leaves the chip */
int b200seg_stem_gn_bwd(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                        const b200seg_gn* gn3, const b200seg_gn* gn1, const b200seg_tensor* g, const double* sums3,
                        const double* sums1, float* dw3, float* dw1, float* dgamma, float* dbeta, float* db3,
                        float* db1, int device, b200seg_stream stream);

/* ---- nn.MaxPool3d/2d(2,2) (Unet3d.py:18-24) */
int b200seg_pool_fwd(const b200seg_tensor* x, const b200seg_tensor* out, int dims, int device, b200seg_stream stream);
int b200seg_pool_bwd(const b200seg_tensor* x, const b200seg_tensor* g_out, const b200seg_tensor* addend,
                     const b200seg_tensor* g_x, int dims, int device, b200seg_stream stream);

/* ---- fused head (OutputTransition3d, VNet3d.py:90-99; Unet3d.py:56-61): 1x1 conv to `nc` <= 8 classes + bias,
 * then sigmoid (nc == 1) or softmax over classes.  w: the nn.Conv parameter itself, fp32 [nc][Cin]; logits and
 * probs: fp32 channels-last [voxels][nc]; probs may be NULL (logits only). */
int b200seg_head_fwd(const b200seg_tensor* x, const float* w, const float* bias, float* logits, float* probs, int nc,
                     int device, b200seg_stream stream);
/* backward of the head conv in one pass: dx = dlogits * W (same dtype as x), dw[nc][Cin] += dlogits^T x,
 * db[nc] += sum dlogits.  Returns B200SEG_EINVAL for shapes outside the fused path (nc > 4, Cin not 16/32):
 * query with b200seg_head_bwd_supported and use b200seg_conv / b200seg_wgrad / b200seg_colsum instead. */
int b200seg_head_bwd_supported(int cin, int nc);
int b200seg_head_bwd(const b200seg_tensor* x, const float* dlogits, const float* w, const b200seg_tensor* dx,
                     float* dw, float* db, int nc, int device, b200seg_stream stream);

/* ---- head activation: torch.sigmoid / torch.softmax(dim=1) (VNet3d.py:95-98; Unet3d.py:58-61) */
int b200seg_head_probs(const float* logits, float* probs, int64_t nvox, int C, int device, b200seg_stream stream);

/* ---- losses (model/losses.py:33-53,129-197,247-342), logits fp32 channels-last [N][vox][C]; labels [N][vox] int64
 * (B200SEG_I64) or, for the binary losses only, fp32 soft targets (B200SEG_F32: ``y_true.float()`` losses.py:47,144).
 * part (double, += ): C>1: I_c[C], P_c[C], Cnt_c[C], sum_nll, sum_focal, V, BAD ; C==1: I, P, T, sum_bce, sum_focal,
 * V, BAD -- BAD counts labels outside [0, C) (the reference raises in F.one_hot / F.cross_entropy, losses.py:254,311:
 * such voxels are skipped, b200seg_loss_finalize turns the loss into NaN and the host binding raises).
 * metric (double [N][C][3], += , or NULL): per sample and class {sum [p_c>.5][t==c], sum [p_c>.5], sum [t==c]} -- the
 * sums of the per-step accuracy (dice_coeff / multiclass_dice_coeff, model/metric.py:146-181, called every step at
 * model/modelVNet.py:582) from the SAME read of logits + labels (SURVEY 8f-2). */
int b200seg_loss_partials(const float* logits, const void* labels, int label_dtype, int N, int64_t vox_per_sample,
                          int C, float gamma, float alpha_f, double* part, double* metric, int device,
                          b200seg_stream stream);
/* lcoef (fp32): C>1: a_c[C], b_c[C], ce_scale, focal_scale, gamma ; C==1: a, b, bce_scale, focal_scale, gamma
 * terms JACCARD / ELDICE / TVERSKY (losses.py:19-30,66-74,113-126,358-382) write the same layout (a, b only), so
 * b200seg_loss_bwd takes their gradient; TVERSKY reads alpha from alpha_f and beta from gamma.  SS (losses.py:87-99)
 * reads r from alpha_f and the sums of b200seg_loss_partials_ss, writes lcoef = {r/(s+T), (1-r)/(s+V-T), 0, 0, 0}
 * for b200seg_loss_bwd_ss. */
int b200seg_loss_finalize(const double* part, int C, int terms, const float* alpha, float gamma, float alpha_f,
                          float* loss, float* lcoef, int device, b200seg_stream stream);
int b200seg_loss_bwd(const float* logits, const void* labels, int label_dtype, int64_t nvox, int C,
                     const float* lcoef, const float* gscale, float* dlogits, int device, b200seg_stream stream);
/* BinarySSLoss (losses.py:87-99), C == 1: part (double [7], += ) = {I, P, T, sum (p-t)^2 t, sum (p-t)^2 (1-t), V, 0};
 * metric as b200seg_loss_partials.  Backward: dlogits = gscale 2 (p-t) (lcoef[0] t + lcoef[1] (1-t)) p (1-p). */
int b200seg_loss_partials_ss(const float* logits, const void* labels, int label_dtype, int N, int64_t vox_per_sample,
                             double* part, double* metric, int device, b200seg_stream stream);
int b200seg_loss_bwd_ss(const float* logits, const void* labels, int label_dtype, int64_t nvox, const float* lcoef,
                        const float* gscale, float* dlogits, int device, b200seg_stream stream);

/* ---- stable segmented LSD radix sort of (uint32 key, int32 value) pairs, ascending by key, ties in input order:
 * nseg segments of seg_len pairs each, segment s at [s*seg_len, (s+1)*seg_len).  Inputs are not modified;
 * `workspace` of b200seg_radix_sort_workspace(nseg, seg_len) bytes.  seg_len < 2^31. */
int64_t b200seg_radix_sort_workspace(int nseg, int64_t seg_len);
int b200seg_radix_sort_pairs(const uint32_t* keys_in, const int32_t* vals_in, uint32_t* keys_out, int32_t* vals_out,
                             int nseg, int64_t seg_len, void* workspace, int64_t workspace_bytes, int device,
                             b200seg_stream stream);

/* ---- Lovasz-Softmax (LovaszLoss, model/losses.py:462-473 -> model/lovasz.py:90-138), C >= 2.  The logits are the
 * "probabilities", as LovaszLoss.forward passes them (lovasz.py:133).  Per class c over the flattened P = n*vox + v
 * (lovasz.py:141-158; per_image: per sample n), skipping voxels labelled `ignore` (if has_ignore): e = |[t==c] - z_c|
 * sorted descending (stable: ties in ascending P), grad = Lovasz gradient of the sorted [t==c] (lovasz.py:21-32);
 * class loss = dot(e_sorted, grad); classes with no voxel of the class are skipped (lovasz.py:125); loss = mean over
 * the rest (0 if none; per_image: the mean over samples of those means).  Labels outside [0, C) are background for
 * every class.  logits fp32 channels-last [N][vox][C], labels int64 [N][vox].
 * b200seg_lovasz_fwd writes loss, coef [N][vox][C] (the Lovasz gradient of every voxel and class, 0 where ignored)
 * and seg_scale [S] (S = C, or N*C with per_image: the weight of each class segment in the mean).
 * b200seg_lovasz_bwd: dlogits = gscale * coef * sgn(z_c - [t==c]) * seg_scale.  Segments must hold < 2^31 voxels. */
int64_t b200seg_lovasz_workspace(int N, int64_t vox_per_sample, int C, int per_image);
int b200seg_lovasz_fwd(const float* logits, const int64_t* labels, int N, int64_t vox_per_sample, int C, int per_image,
                       int has_ignore, int64_t ignore, void* workspace, int64_t workspace_bytes, float* loss,
                       float* coef, float* seg_scale, int device, b200seg_stream stream);
int b200seg_lovasz_bwd(const float* logits, const int64_t* labels, int N, int64_t vox_per_sample, int C, int per_image,
                       const float* coef, const float* seg_scale, const float* gscale, float* dlogits, int device,
                       b200seg_stream stream);

/* ---- per-step accuracy (model/metric.py:146-181).  b200seg_metric_partials: the sums above from MATERIALISED
 * probabilities (fp32 channels-last [N][vox][C], threshold 0.5 in the reference); b200seg_metric_finalize:
 * out[0] = dice_coeff (C == 1) / multiclass_dice_coeff (mean over classes 1..C-1), out[1] = the iou_coeff analogue. */
int b200seg_metric_partials(const float* probs, const void* labels, int label_dtype, int N, int64_t vox_per_sample,
                            int C, float threshold, double* metric, int device, b200seg_stream stream);
int b200seg_metric_finalize(const double* metric, int N, int C, float* out /*[2]*/, int device, b200seg_stream stream);

/* ---- 3-D segmentation metrics of Seg_Metirc3d (model/metric.py:11-142; scipy binary_erosion + cKDTree there) for N
 * volumes of (D, H, W) voxels.  real / pred: dense [N][D][H][W] masks of dtype B200SEG_U8 (bool, uint8), B200SEG_I32
 * or B200SEG_I64; nonzero is foreground.  spacing_zyx: DEVICE fp64 [N][3] (z, y, x) in mm, the reversed SimpleITK
 * spacing (metric.py:47).  A surface voxel is a foreground voxel with background in its 18-neighbourhood (faces and
 * edges; outside the volume is background: metric.py:41-42).  Distances are exact Euclidean distances in mm from each
 * surface voxel to the nearest surface voxel of the other mask (metric.py:49-65), from a separable exact distance
 * transform in fp64.
 * b200seg_segmetric3d writes counts int64 [N][6] = {R, P, I, U, S_r, S_p} (foreground, intersection, union and surface
 * voxel counts), metrics fp64 [N][9] = {dice 2I/(R+P), jaccard I/U, VOE 1 - I/U, RVD (P-R)/R, FNR (R-I)/U,
 * FPR (P-I)/U, ASSD, RMSD, MSD} (metric.py:68-142; distance metrics NaN where a mask is empty) and flags int32 [N]
 * (1 where a mask holds a value outside {0, 1}).  Every reduction has a fixed order: reruns are bit-identical.
 * b200seg_segmetric3d_points writes, for each surface in C order over all volumes (volume n's points follow those of
 * volumes < n, counts from b200seg_segmetric3d), the linear voxel index within the volume (metric.py:43-44) and the
 * distance to the other surface (real2pred_nn / pred2real_nn, metric.py:58-65); at most cap_r / cap_p points are
 * written.  Both take a workspace of b200seg_segmetric3d_workspace(N, D, H, W) bytes (about 65 bytes per voxel). */
int64_t b200seg_segmetric3d_workspace(int N, int D, int H, int W);
int b200seg_segmetric3d(const void* real, int real_dtype, const void* pred, int pred_dtype, int N, int D, int H, int W,
                        const double* spacing_zyx, void* workspace, int64_t workspace_bytes, int64_t* counts,
                        double* metrics, int32_t* flags, int device, b200seg_stream stream);
int b200seg_segmetric3d_points(const void* real, int real_dtype, const void* pred, int pred_dtype, int N, int D, int H,
                               int W, const double* spacing_zyx, void* workspace, int64_t workspace_bytes,
                               int64_t cap_r, int64_t cap_p, int64_t* real_idx, int64_t* pred_idx, double* real2pred,
                               double* pred2real, int device, b200seg_stream stream);

/* ---- SSIM / SSIM3D (model/lossesSSIM.py:49-93: five depthwise F.conv2d / F.conv3d with a dense Gaussian window
 * there).  img1, img2: fp32 (N, C, H, W) (dims == 2; pass D = 1) or (N, C, D, H, W) with element strides
 * {n, c, d, h, w} (host int64 [5], read during the call; NCDHW-contiguous and channels-last views alike).  taps: the
 * window_size (1..31) 1-D Gaussian taps of lossesSSIM.py:28-30 (host fp32, read during the call), applied separably
 * along H, W (and D) with zero padding P = window_size / 2, so each map axis has length L + 2P - window_size + 1.
 * The map S (lossesSSIM.py:52-64, 73-88) is formed per voxel in fp64.
 * b200seg_ssim_fwd writes fp64 partial sums of S into `workspace` (b200seg_ssim_workspace bytes) and, when coef is
 * not NULL, the four backward coefficients fp64 [4][N][C][D'][H'][W'] = {dS/dmu1, dS/dmu2, dS/dm11 = dS/dm22, dS/dm12}.
 * b200seg_ssim_finalize sums the partials in a fixed order (reduce != 0) into acc: size_average: acc[2] = {sum S,
 * count}, value[1] = S.mean(); otherwise per sample, dims == 2: acc[N], value[N] = S.mean(1).mean(1).mean(1); dims ==
 * 3: acc[N][W'], value[N][W'] (the reference's three means run over C, D and H only).  With reduce == 0 it only
 * recomputes value from acc (after a data-parallel all-reduce of acc).
 * b200seg_ssim_bwd: grad1 / grad2 (fp32 NCDHW-contiguous, either may be NULL) = d loss / d img from gout (fp32, the
 * shape of value) and the forward's coef and acc (the mean's count is read from acc[1]). */
int64_t b200seg_ssim_workspace(int dims, int N, int C, int D, int H, int W, int window_size);
int b200seg_ssim_fwd(int dims, const float* img1, const int64_t* strides1, const float* img2, const int64_t* strides2,
                     int N, int C, int D, int H, int W, int window_size, const float* taps, double* coef,
                     void* workspace, int64_t workspace_bytes, int device, b200seg_stream stream);
int b200seg_ssim_finalize(int dims, int N, int C, int D, int H, int W, int window_size, int size_average, int reduce,
                          const void* workspace, int64_t workspace_bytes, double* acc, float* value, int device,
                          b200seg_stream stream);
int b200seg_ssim_bwd(int dims, const float* img1, const int64_t* strides1, const float* img2, const int64_t* strides2,
                     int N, int C, int D, int H, int W, int window_size, const float* taps, const double* coef,
                     int size_average, const float* gout, const double* acc, float* grad1, float* grad2, int device,
                     b200seg_stream stream);

/* ---- fused optimizer step over FLAT fp32 buffers (torch.optim.AdamW(lr) model/modelVNet.py:548, weight_decay 0.01,
 * decoupled = 1; torch.optim.Adam model/modelUnet.py:849, decoupled = 0): ONE launch for all parameters instead of
 * ~6 foreach launches over 128 tensors.  state (fp32 [4], device): [0] step count t, [1] lr/(1-b1^t), [2]
 * sqrt(1-b2^t); tick != 0 advances t first (one extra 1-thread launch) so a captured step replays correctly.
 * gscale: optional device scalar multiplied into the gradient (e.g. 1/world for an averaged all-reduce) or NULL. */
int b200seg_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float* state,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int decoupled,
                      const float* gscale, int tick, int device, b200seg_stream stream);

/* ---- ALL dropout channel masks of one forward in one launch (nn.Dropout3d/2d(p), VNet3d.py:11,31,51,67;
 * Unet3d.py:74,83): out[first_k + i] = keep(k, j0_k + i) ? 1/(1-p) : 0 for i < count_k, where keep(k, j) is exactly
 * element j of what the k-th ``x.new_empty((N,C_k,1,..)).bernoulli_(1-p)`` of a forward draws from a CUDA generator
 * at {seed, offset} = rng[0], rng[1] (device memory; Philox4_32_10, the k-th call sees offset + 4k).  The caller
 * advances its generator by 4*nmasks.  table: device int32 [nmasks][3] = {first_k, count_k, j0_k}; j0_k != 0 lets a
 * data-parallel rank take its slice of the global-batch draw (SURVEY.md 8e). */
int b200seg_dropout_masks(const int64_t* rng, const int32_t* table, int nmasks, int total, double p_drop, float* out,
                          int device, b200seg_stream stream);

/* ---- forward-only head for inference (predict, model/modelVNet.py:655-676): 1x1 conv to nc <= 8 classes, then
 * mask = (sigmoid > threshold) * 255 (nc == 1) or argmax over classes (first maximum, as np.argmax) -> uint8
 * [voxels]; neither logits nor probs are written.  b200seg_mask_logits: the same from fp32 channels-last logits. */
int b200seg_head_mask(const b200seg_tensor* x, const float* w, const float* bias, uint8_t* mask, int nc,
                      float threshold, int device, b200seg_stream stream);
int b200seg_mask_logits(const float* logits, int64_t nvox, int C, float threshold, uint8_t* mask, int device,
                        b200seg_stream stream);

/* ---- classifier head of ResNet2d / ResNet3d (networks/ResNet3d.py:61-118): GlobalAveragePooling -> Linear(C, Hd)
 * -> ReLU -> Linear(Hd, K).  x: the last encoder activation (N, D, H, W, C), F32 or BF16, with channel pitch.
 * w1 [Hd][C], b1 [Hd], w2 [K][Hd], b2 [K]: fp32 in nn.Linear layout.  C, Hd, K in [1, 1024].  Two launches each way,
 * fixed-order sums without atomics (reruns are bit-identical), no allocation, no host synchronisation.
 *   fwd: pooled [N][C] = mean over voxels, hidden [N][Hd] = relu(w1 pooled + b1), logits [N][K] = w2 hidden + b2 (fp32)
 *   bwd: dlogits [N][K] -> dw1, db1, dw2, db2 (written, not accumulated) and the dense activation gradient
 *        dx (N, D, H, W, C) = (w1^T ((w2^T dlogits) * [hidden > 0])) / (D*H*W) broadcast over the voxels (dx's dtype);
 *        work: fp32 scratch of N*(Hd + C) elements. */
int b200seg_cls_head_fwd(const b200seg_tensor* x, const float* w1, const float* b1, const float* w2, const float* b2,
                         int hidden_width, int ncls, float* pooled, float* hidden, float* logits, int device,
                         b200seg_stream stream);
int b200seg_cls_head_bwd(const float* dlogits, const float* pooled, const float* hidden, const float* w1,
                         const float* w2, int hidden_width, int ncls, float* work, const b200seg_tensor* dx, float* dw1,
                         float* db1, float* dw2, float* db2, int device, b200seg_stream stream);

/* ---- device-side input staging (SURVEY.md 8f-4): the per-sample host work of the reference's datasets, from the raw
 * 8-bit images.  datasetModelSegwithopencv.__getitem__ (model/dataset.py:138-142): image = (image - image.mean()) /
 * image.std() in float64 with the population std, then .float(); labels .long() (dataset.py:150-157) with the trainer's
 * y[y != 0] = 1 (model/modelUnet.py:130) when `binarize`.
 *   b200seg_stage_u8_sums      sums[n][2] (ZEROED by the caller) += { sum x, sum x*x } of sample n, exact integers
 *   b200seg_stage_u8_normalize out[n][i] = (float)(((double)x - mean_n) / std_n), fp32 or bf16 (out_dtype); a constant
 *                              image gives NaN, as numpy's 0/0 does
 *   b200seg_stage_labels_u8    out[i] = binarize ? (lab[i] != 0) : lab[i], int64
 * img: [n][per_sample] uint8, densely packed. */
int b200seg_stage_u8_sums(const uint8_t* img, int n, int64_t per_sample, uint64_t* sums, int device,
                          b200seg_stream stream);
int b200seg_stage_u8_normalize(const uint8_t* img, int n, int64_t per_sample, const uint64_t* sums, void* out,
                               int out_dtype, int device, b200seg_stream stream);
int b200seg_stage_labels_u8(const uint8_t* lab, int64_t count, int binarize, int64_t* out, int device,
                            b200seg_stream stream);

/* ---- whole-volume 3-D inference (XModel.inference / inference_patch, model/modelVNet.py:678-698,
 * model/modelUnet.py:684-763): SimpleITK's resamples and the intensity normalisations around the network.  Volumes
 * are dense [D][H][W]; ratio_zyx (host fp64 [3], read during the call) is the input-index step per output index
 * along D, H, W (S_in / S_out, or new spacing / old spacing).  A sample exists where -0.5 <= i * r < S_in - 0.5 on
 * every axis (ITK's inside-buffer rule), else the output is 0.
 * b200seg_resample_linear: trilinear sample in fp64 (lerps along W, H, then D), cast to the input's pixel type
 * (src_dtype B200SEG_U8, B200SEG_I16, B200SEG_I32: clamped to the type's range, truncated toward zero; B200SEG_F32:
 * rounded), then written as fp32 to out [oD][oH][oW].  norm_mode B200SEG_NORM_MEANSTD also truncates to [lower,
 * upper] and writes per-block fp64 sums to the workspace; B200SEG_NORM_PCTL writes the sort keys there
 * (B200SEG_NORM_NONE needs no workspace).
 * b200seg_normalize: x (the resample's output, same norm_mode and workspace) -> out, a separate buffer.  The workspace's
 * first 64 bytes hold fp64 stats {mean, sigma, p5, p95, unchanged flag, count}: MEANSTD uses the N - 1 deviation of
 * all voxels; PCTL the numpy 'linear' 5th / 95th percentiles, then the mean and population deviation of the nonzero
 * clipped voxels, and the flag is 1 where normalize() returns the clipped volume unchanged (a std of 0).
 * b200seg_resample_nearest_u8: out [oD][oH][oW] uint8; voxels with an index >= (vD, vH, vW) on any axis are 0,
 * the rest take src at floor(i * r + 0.5).
 * Sizes >= 1; the PCTL network grid holds < 2^31 voxels.  Every reduction has a fixed order. */
int64_t b200seg_resample_workspace(int norm_mode, int oD, int oH, int oW);
int b200seg_resample_linear(const void* src, int src_dtype, int D, int H, int W, const double* ratio_zyx, int oD,
                            int oH, int oW, int norm_mode, float lower, float upper, float* out, void* workspace,
                            int64_t workspace_bytes, int device, b200seg_stream stream);
int b200seg_normalize(int norm_mode, const float* x, int oD, int oH, int oW, void* workspace, int64_t workspace_bytes,
                      float* out, int device, b200seg_stream stream);
int b200seg_resample_nearest_u8(const uint8_t* src, int D, int H, int W, const double* ratio_zyx, int vD, int vH,
                                int vW, int oD, int oH, int oW, uint8_t* out, int device, b200seg_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SEG_H */
