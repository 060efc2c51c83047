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

#define B200SEG_VERSION 201

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
/* output tile geometries of B200SEG_CONV_HALO_WS (b200seg_conv_halo_ws_geometry) */
#define B200SEG_WS_GEOM_COLUMN 0 /* 8 wide x 16 high tiles of the H x W plane */
#define B200SEG_WS_GEOM_FLAT 1   /* 128 consecutive anchors h * (W + 2) + w of the padded plane */
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
/* the B200SEG_WS_GEOM_* output tile geometry b200seg_conv / b200seg_conv_bwdstats would use for these arguments on
 * the B200SEG_CONV_HALO_WS path (chosen by the plane's shape; host only), or B200SEG_EINVAL if they take another path */
int b200seg_conv_halo_ws_geometry(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
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
/* activation after the norm and dropout (b200seg_gn.act) */
#define B200SEG_ACT_RELU 0   /* nn.ReLU */
#define B200SEG_ACT_LEAKY 1  /* nn.LeakyReLU(0.01): v > 0 ? v : v * 0.01f; backward g > 0 ? g : g * 0.01f by the sign of
                                the pre-activation (leaky_relu_backward).  Only the elementwise GroupNorm entry points
                                (b200seg_apply_gn, b200seg_gn_bwd_reduce_gn, b200seg_gn_bwd_apply_gn,
                                b200seg_gn_bwd_fused_gn) take it; the fused families (b200seg_conv_bwdstats,
                                b200seg_stem_gn_*, b200seg_up_gn_*) return B200SEG_EINVAL for act != RELU. */
typedef struct b200seg_gn {
  const double* stats;
  const float* gamma;
  const float* beta;
  const float* scale;
  int32_t groups;  /* 8 for nn.GroupNorm(8, C); C for nn.InstanceNorm3d(C, affine=True) (C <= 512) */
  int64_t vox;     /* voxels per sample of the normalised tensor */
  float eps;
  int32_t act;     /* B200SEG_ACT_*: fills the padding after eps, sizeof is unchanged */
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

/* ---- fused first layer of VNet3d's up_tr32 (VNet3d.py:62-72): up_conv, a 2x2x2 stride-2 transposed convolution of a
 * bf16 32-channel input x to 16 channels at twice the resolution, then GroupNorm(8, 16), dropout and ReLU.  No pass
 * stores the raw output y: each recomputes it from x with the arithmetic of b200seg_conv's pointwise mma.sync kernel,
 * so the results equal b200seg_conv (stats) -> b200seg_apply_gn on the forward side and b200seg_gn_bwd_reduce_gn ->
 * b200seg_gn_bwd_apply_gn -> b200seg_wgrad + the data-gradient b200seg_conv on the backward side.  w: the bf16 forward
 * operand (b200seg_pack_weight, [8][16][32]); gn: the layer's GroupNorm reference (8 groups, vox = the fine grid's
 * D*H*W); stats [N][16][2], sums [N][16][3] fp64, zero on entry where written.  Ask b200seg_up_gn_supported first. */
int b200seg_up_gn_supported(const b200seg_tensor* x, int cout, int dims);
/* per-(n, c) sum y, sum y^2 (what b200seg_conv writes into its stats argument) */
int b200seg_up_gn_stats(const b200seg_tensor* x, const void* w, const float* bias, double* stats, int device,
                        b200seg_stream stream);
/* out = relu(y*A+B); out: bf16, 16 channels, the fine grid, 16-byte aligned rows (pitch a multiple of 8) */
int b200seg_up_gn_apply(const b200seg_tensor* x, const void* w, const float* bias, const b200seg_gn* gn,
                        const b200seg_tensor* out, int device, b200seg_stream stream);
/* sums [N][16][3] += {sum g*m, sum g*m*y, sum y} (b200seg_gn_bwd_reduce_gn's layout) */
int b200seg_up_gn_bwd_sums(const b200seg_tensor* x, const void* w, const float* bias, const b200seg_gn* gn,
                           const b200seg_tensor* g, double* sums, int device, b200seg_stream stream);
/* dw [8][16][32] += (b200seg_wgrad's layout for this layer), dx = the data gradient (bf16, 32 channels, the coarse
 * grid), dgamma, dbeta [16] +=, dbias [16] += (may be NULL); dy itself never leaves the chip */
int b200seg_up_gn_bwd(const b200seg_tensor* x, const void* w, const float* bias, const b200seg_gn* gn,
                      const b200seg_tensor* g, const double* sums, float* dw, const b200seg_tensor* dx, float* dgamma,
                      float* dbeta, float* dbias, int device, b200seg_stream stream);

/* ---- nn.MaxPool3d/2d(2,2) (Unet3d.py:18-24) */
int b200seg_pool_fwd(const b200seg_tensor* x, const b200seg_tensor* out, int dims, int device, b200seg_stream stream);
int b200seg_pool_bwd(const b200seg_tensor* x, const b200seg_tensor* g_out, const b200seg_tensor* addend,
                     const b200seg_tensor* g_x, int dims, int device, b200seg_stream stream);

/* ---- UNet3dthin's decoder join (Unet3dthin.py:40-54): nn.Upsample(scale_factor=2, mode='trilinear') + torch.add.
 * S (N, 2d, 2h, 2w, C) = up2(a) + e for a (N, d, h, w, C); e has S's shape.  up2 is torch's upsample_trilinear3d with
 * align_corners=False: per axis fine 2k reads coarse (k-1, k) with (1/4, 3/4), fine 2k+1 reads (k, k+1) with (3/4, 1/4),
 * and the edges clamp (fine 0 and fine 2n-1 take coarse 0 and n-1 with weight 1).  Sums in fp32, one rounding to the
 * storage type.  The backward writes ga = up2^T(gS), a fixed-order gather (no atomics); the skip's gradient is gS
 * itself.  All tensors share one dtype (F32 or BF16); C and every pitch are multiples of 8, every pointer 16-byte
 * aligned; any coarse extent >= 1. */
int b200seg_upsample2_add(const b200seg_tensor* a, const b200seg_tensor* e, const b200seg_tensor* s, int device,
                          b200seg_stream stream);
int b200seg_upsample2_bwd(const b200seg_tensor* g_s, const b200seg_tensor* g_a, int device, b200seg_stream stream);

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

/* ---- binary Lovasz hinge (BinaryLovaszLoss, model/losses.py:235-242 -> model/lovasz.py:35-84), one logit channel.
 * Over the flattened P = n*vox + v (per_image: per sample n), skipping voxels labelled `ignore` (if has_ignore):
 * e = 1 - z (t == 1) or 1 + z (t == 0) in fp32, sorted descending (stable: ties in ascending P), grad = Lovasz
 * gradient of the sorted t (lovasz.py:21-32; no present-class skip: with no foreground grad = (1, 0, ...)), segment
 * loss = dot(relu(e_sorted), grad), loss = the segment loss, or with per_image the mean over the N samples (a sample
 * with every voxel ignored adds 0).  Exact integer counts, fp64 Jaccard terms and fixed-order fp64 sums.
 * logits fp32 [N][vox], labels int64 [N][vox] with values 0, 1 or `ignore`.
 * b200seg_lovasz_hinge_fwd writes loss, coef [N][vox] = d loss / d logits (0 where ignored or e <= 0) and, if bad is
 * not null, bad[0] = the number of labels other than 0, 1 and `ignore` (such labels are taken as background).
 * b200seg_lovasz_hinge_bwd: dlogits = gscale * coef over nvox = N*vox values.  Segments must hold < 2^31 voxels. */
int64_t b200seg_lovasz_hinge_workspace(int N, int64_t vox_per_sample, int per_image);
int b200seg_lovasz_hinge_fwd(const float* logits, const int64_t* labels, int N, int64_t vox_per_sample, int per_image,
                             int has_ignore, int64_t ignore, void* workspace, int64_t workspace_bytes, float* loss,
                             float* coef, int64_t* bad, int device, b200seg_stream stream);
int b200seg_lovasz_hinge_bwd(const float* coef, int64_t nvox, const float* gscale, float* dlogits, int device,
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

/* ---- soft-clDice (model/lossescldice.py, with its four defects repaired: DESIGN.md section 2).  Shapes are (N, C, D,
 * H, W) (2-D: pass D = 1).  A field is fp32 with element strides {n, c, d, h, w} (host int64 [5], read during the call;
 * NCDHW and channels-last views alike), or, where a *_labels pointer is given instead, the one-hot of dense int64
 * labels [N][D][H][W] (value 1 where label == c).  One skeleton round is, in fp32 and bit-identical to torch:
 * m = minpool(x), M = maxpool(m), x' = relu(x - relu(M - m)), 3x3x3 pools (3x3 when D = 1), stride 1, padding 1.
 * b200seg_cldice_skeleton runs `rounds` (1..64) rounds; round r writes fields + (r % nfields) * N*C*D*H*W (dense
 * NCDHW; nfields >= min(rounds, 2); nfields = rounds keeps every round for the backward).  With `other` (or
 * other_labels) the last round also writes per-CTA fp64 sums {sum x' * other, sum x'} into half `pass` (0: pred's
 * skeleton against the target, 1: the target's against pred) of `workspace` (b200seg_cldice_workspace bytes); a labels
 * pass also counts labels outside [0, C).
 * b200seg_cldice_finalize: stats fp64 [N*C*8 + 3*G + 1] = per (n, c) {sum sk(p) t, sum sk(p), sum sk(t) p, sum sk(t),
 * iflat, tflat, d loss / d iflat, d loss / d tflat}, then the G group sums {sum iflat * tflat, sum iflat, sum tflat}
 * (G = C with per_class, else 1), then the count of bad labels (labels != 0).  loss fp32 [1]: binary
 * 1 - (2 I + smooth) / max(sum iflat + sum tflat + smooth, eps), or per class with alpha (device fp32 [C]) weights,
 * summed and divided by C.  reduce == 0 starts from the group sums (after a data-parallel all-reduce of them).
 * b200seg_cldice_bwd: grad (dense fp32 (N, C, D, H, W)) = d / d x of the `rounds` rounds run on x, from fields
 * [rounds][N*C*D*H*W] of the skeleton pass (nfields = rounds) and scratch (one dense field; both unused when rounds = 1).
 * The seed is grad_skeleton (dense fp32), or, when that is NULL, the loss: gout (device fp32 [1]) times d loss / d
 * sk(pred) from the target and stats, plus the direct tflat term from target_skeleton.  Fixed-order gathers, no atomics.
 * b200seg_cldice_norm: out fp32 [N*C] = (sum cl * vessel + 1) / (sum cl + 1) and sums fp64 [N*C][2] = {sum cl *
 * vessel, sum cl}; b200seg_cldice_norm_bwd: grad_cl / grad_vessel (dense fp32, either may be NULL) from gout
 * (fp32 [N*C]) and sums. */
int64_t b200seg_cldice_workspace(int N, int C, int D, int H, int W);
int b200seg_cldice_skeleton(const float* x, const int64_t* x_strides, const int64_t* x_labels, int N, int C, int D,
                            int H, int W, int rounds, float* fields, int nfields, const float* other,
                            const int64_t* other_strides, const int64_t* other_labels, int pass, void* workspace,
                            int64_t workspace_bytes, int device, b200seg_stream stream);
int b200seg_cldice_finalize(int N, int C, int D, int H, int W, int per_class, int labels, const float* alpha,
                            double smooth, double eps, int reduce, const void* workspace, int64_t workspace_bytes,
                            double* stats, float* loss, int device, b200seg_stream stream);
int b200seg_cldice_bwd(const float* x, const int64_t* x_strides, int N, int C, int D, int H, int W, int rounds,
                       const float* fields, const float* grad_skeleton, const float* target,
                       const int64_t* target_strides, const int64_t* target_labels, const float* target_skeleton,
                       const double* stats, const float* gout, float* grad, float* scratch, int device,
                       b200seg_stream stream);
int b200seg_cldice_norm(const float* cl, const int64_t* cl_strides, const float* vessel, const int64_t* vessel_strides,
                        int N, int C, int D, int H, int W, double* sums, float* out, int device,
                        b200seg_stream stream);
int b200seg_cldice_norm_bwd(const float* cl, const int64_t* cl_strides, const float* vessel,
                            const int64_t* vessel_strides, int N, int C, int D, int H, int W, const double* sums,
                            const float* gout, float* grad_cl, float* grad_vessel, int device, b200seg_stream stream);

/* ---- fused optimizer step over FLAT fp32 buffers (torch.optim.AdamW(lr) model/modelVNet.py:548, weight_decay 0.01,
 * decoupled = 1; torch.optim.Adam model/modelUnet.py:849, decoupled = 0): ONE launch for all parameters instead of
 * ~6 foreach launches over 128 tensors.  state (fp32 [4], device): [0] step count t, [1] lr/(1-b1^t), [2]
 * sqrt(1-b2^t); tick != 0 advances t first (one extra 1-thread launch) so a captured step replays correctly.
 * gscale: optional device scalar multiplied into the gradient (e.g. 1/world for an averaged all-reduce) or NULL.
 * lr, the betas and weight_decay are the Python (double) values: as in torch.optim, 1 - beta1, 1 - beta2,
 * 1 - lr*weight_decay, beta^t and lr/(1-beta1^t) are computed in double and rounded to fp32 once; beta2,
 * weight_decay and eps enter the elementwise update as their fp32 roundings. */
int b200seg_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float* state,
                      double lr, double beta1, double beta2, float eps, double weight_decay, int decoupled,
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

/* ---- 2-D image resize: OpenCV's uint8 cv2.resize(img, (oW, oH)) with the default INTER_LINEAR, as the reference's 2-D
 * datasets (model/dataset.py:63,140,154: before the z-score; the segmentation label too) and 2-D inference methods
 * (model/modelVNet.py:231-242,450-461, model/modelUnet.py:231-242,450-461, model/modelResNet.py:212-221,428-437: the
 * image before "/ 255." and the uint8 mask back to image.shape) call it on the host.  Per axis (source size s,
 * destination size d, destination index i): scale = 1.0 / ((double)d / s) in fp64; f = (float)((i + 0.5) * scale -
 * 0.5) with the fp64 multiply and subtract rounded separately; k = floor(f), f -= k (fp32).  Along x, k < 0 gives
 * k = 0, f = 0 and k >= s - 1 gives k = s - 1, f = 0, taps k and min(k + 1, s - 1); along y f is not clamped and the
 * taps are clamp(k, 0, s - 1), clamp(k + 1, 0, s - 1).  c0 = rint((1 - f) * 2048), c1 = rint(f * 2048) (half to
 * even).  Horizontal r = src[k] c0 + src[k + 1] c1 (int32); vertical, with b0, b1 the y coefficients and r0, r1 the
 * two rows: v = (((b0 (r0 >> 4)) >> 16) + ((b1 (r1 >> 4)) >> 16) + 2) >> 2 (OpenCV's SIMD form, not the textbook
 * (r0 b0 + r1 b1 + 2^21) >> 22), saturated to [0, 255].
 * One launch resizes a ragged batch: desc (device memory, n entries) gives each sample's byte offset into src and its
 * (h, w) >= 1, dense rows of w bytes.  out: dense [n][oH][oW], out_mode B200SEG_U8 (the cv2 bytes) or B200SEG_F32
 * ((float)((double)v / 255.0): the inference methods' "/ 255." and .float()).  n <= 65535, sizes >= 1. */
typedef struct b200seg_resize_src {
  int64_t offset; /* byte offset of the sample's pixel (0, 0) in src */
  int32_t h, w;   /* its height and width */
} b200seg_resize_src;
int b200seg_resize_linear_u8(const uint8_t* src, const b200seg_resize_src* desc, int n, int oH, int oW, void* out,
                             int out_mode, int device, b200seg_stream stream);

/* ---- 3-D augmentation warp: ImageDataGenerator3D.random_transform + standardize
 * (dataprocess/Augmentation/images_masks_3dtransform.py, driven by DataAug3D, ImageAugmentation.py:26-75), i.e.
 * scipy.ndimage.affine_transform(v, M, off, order=0, mode, cval) of every channel and of the label, then the channel
 * shift, the flips and "x *= rescale".  Per output voxel (d, h, w) of sample s: the flipped axes are un-flipped
 * (i_a = len_a - 1 - i_a where bit a of param.flip is set); per input axis a of length n,
 * cc = off[a]; cc += m[3a] i0; cc += m[3a + 1] i1; cc += m[3a + 2] i2 (fp64, each product and sum rounded on its own,
 * no FMA); cc outside [0, n - 1] is mapped by the mode (NEAREST clamps, CONSTANT fills the whole voxel with cval,
 * REFLECT / MIRROR / WRAP fold it as scipy's map_coordinate: periods 2n, 2n - 2, n - 1); k = floor(cc + 0.5), an index
 * one past the edge folded back (REFLECT repeats the edge voxel, MIRROR reflects about it).  The gathered image value
 * (fp32 cval outside) goes through, in this order: with shift != 0, clip(v + shift[c], min, max) in fp32, min / max
 * over every channel of the warped sample (numpy's clip: NaN propagates); B200SEG_RESCALE_F32: v * (float)rescale;
 * B200SEG_RESCALE_F64: (float)((double)v * rescale).  The label (scipy's cval cast outside: fp32 cval, or for uint8
 * (cval > 0 ? cval + 0.5 : 0) saturated at 255 and truncated) is written as y_dtype, or as int64 (label_out ==
 * B200SEG_I64: uint8 widened, fp32 truncated toward zero), or with binarize as int64 (y != 0) (model/modelVNet.py:576).
 * x, x_out: dense [n][D][H][W][C] fp32, C in {1, 3, 4}; y, y_out: dense [n][D][H][W]; y_dtype B200SEG_U8 or
 * B200SEG_F32; params: device memory, n entries.  With shift a first pass writes per-block min / max partials into ws
 * (b200seg_augment3d_workspace bytes); min and max do not depend on order, so reruns are bit-identical.
 * D * H * W < 2^31, n <= 65535; x_out must not alias x. */
#define B200SEG_AUG_NEAREST 0
#define B200SEG_AUG_CONSTANT 1
#define B200SEG_AUG_REFLECT 2
#define B200SEG_AUG_WRAP 3
#define B200SEG_AUG_MIRROR 4
#define B200SEG_RESCALE_NONE 0
#define B200SEG_RESCALE_F32 1 /* rescale was a Python number: numpy multiplies in fp32 by (float)rescale */
#define B200SEG_RESCALE_F64 2 /* rescale was a numpy float64: fp64 multiply, rounded once to fp32 */
typedef struct b200seg_aug3d_param {
  double m[9];    /* the centred matrix's 3x3 block, row-major */
  double off[3];  /* its last column */
  float shift[4]; /* (float) of the channel-shift draw u_c, read when shift != 0 */
  int32_t flip;   /* bit a set: flip array axis a (0: vertical_flip, 1: horizontal_flip, 2: depth_flip) */
  int32_t pad;
} b200seg_aug3d_param; /* 120 bytes */
int64_t b200seg_augment3d_workspace(int n, int D, int H, int W);
int b200seg_augment3d(const float* x, const void* y, int y_dtype, int n, int D, int H, int W, int C,
                      const b200seg_aug3d_param* params, int fill_mode, double cval, int shift, double rescale,
                      int rescale_mode, float* x_out, void* y_out, int label_out, int binarize, void* ws,
                      int64_t ws_bytes, int device, b200seg_stream stream);

/* ---- 2-D augmentation: Segmenation_Aug (dataprocess/AugData.py), albumentations' HorizontalFlip, VerticalFlip,
 * OneOf(MotionBlur, MedianBlur, Blur), ShiftScaleRotate and RandomBrightnessContrast, byte for byte OpenCV 4.13's
 * uint8 cv2.flip, cv2.filter2D, cv2.medianBlur(3), cv2.blur((3, 3)), cv2.warpAffine (INTER_LINEAR for images,
 * INTER_NEAREST for masks, BORDER_REFLECT_101) and cv2.LUT.  One entry per image (device memory, n entries): its
 * source at byte offset src of src, dense (h, w, c) rows with c in {1, 3} interleaved; its output at byte offset dst
 * of out, same layout; optionally a (h, w) mask at mask_src of msrc (mask_src < 0: none) written at mask_dst of mout.
 * Stages, in this order, each applied when its bit of flags is set:
 *   HFLIP / VFLIP: image and mask;
 *   BLUR: blur = MOTION: filter2D over the ntaps taps (tap_dy, tap_dx offsets from the centre, tap_w weights, in the
 *     kernel's row-major order), reflect-101, fp32, s = fma(v, w, s) for the row elements x * filter_cn + ch below
 *     (w * filter_cn) & ~3 and s + v * w (rounded separately) above, cvRound (OpenCV's AVX2 body and scalar tail;
 *     filter_cn is the channel count of the row cv2 filtered, c itself or 3 for a gray image read back from the
 *     reference's BGR files); MEDIAN: the 3x3 median, replicated border; BOX: rint(3x3 sum / 9), reflect-101;
 *   WARP: minv the inverse 2x3 matrix (cv2.invertAffineTransform, fp64); OpenCV's fixed-point map
 *     adelta = rint(minv[0] x 1024), X0 = rint((minv[1] y + minv[2]) 1024) + 16, X = (X0 + adelta) >> 5 (fp64
 *     products and sums rounded one by one), tap x = X >> 5, fraction X & 31 (likewise y with minv[3..5]); taps
 *     reflected (101); v = (sum of taps x 32 (32 - f)(32 - f') products + 2^14) >> 15.  The mask: (X0 + 512 +
 *     adelta) >> 10, reflected;
 *   LUT: v = lut[v] (image only).
 * The blur writes the blurred image into ws at the entry's dst offset (ws_bytes >= out_bytes =
 * b200seg_augment2d_workspace(out_bytes)); stages is the OR of every entry's flags: without BLUR the blur launch is
 * skipped and ws may be null.  max_hw >= every entry's h * w.  h, w in [1, 8192], n <= 65535; outputs must not alias
 * inputs.  No reductions: reruns are bit-identical. */
#define B200SEG_AUG2D_HFLIP 1
#define B200SEG_AUG2D_VFLIP 2
#define B200SEG_AUG2D_BLUR 4
#define B200SEG_AUG2D_WARP 8
#define B200SEG_AUG2D_LUT 16
#define B200SEG_AUG2D_MOTION 1
#define B200SEG_AUG2D_MEDIAN 2
#define B200SEG_AUG2D_BOX 3
#define B200SEG_AUG2D_MAX_TAPS 8
#define B200SEG_AUG2D_MAX_SIDE 8192
typedef struct b200seg_aug2d_param {
  int64_t src, dst;           /* byte offsets of the image in src and of its output in out (and ws) */
  int64_t mask_src, mask_dst; /* byte offsets of the mask in msrc and mout; mask_src < 0: no mask */
  double minv[6];             /* inverse warp matrix, row-major 2x3 */
  float tap_w[8];             /* motion kernel weights of the nonzero taps */
  int8_t tap_dy[8], tap_dx[8];
  int32_t h, w, c, flags, blur, ntaps, filter_cn, pad;
  uint8_t lut[256];
} b200seg_aug2d_param; /* 416 bytes */
int64_t b200seg_augment2d_workspace(int64_t out_bytes);
int b200seg_augment2d(const uint8_t* src, const uint8_t* msrc, const b200seg_aug2d_param* params, int n,
                      int64_t max_hw, int stages, uint8_t* out, int64_t out_bytes, uint8_t* mout, void* ws,
                      int64_t ws_bytes, int device, b200seg_stream stream);

/* ---- mask post-processing (dataprocess/utils.py:7-66; SimpleITK on the CPU there).  One dense mask of (D, H, W)
 * voxels, a 2-D mask as D = 1, D * H * W < 2^31; mask dtypes B200SEG_U8 (bool, uint8), B200SEG_I16, B200SEG_I32,
 * B200SEG_I64, and for the morphology B200SEG_F32 too (NaN is nonzero).  Every result is an integer: reruns are
 * bit-identical.
 *
 * b200seg_largest_component replaces GetLargestConnectedCompont (utils.py:19-44: sitk.ConnectedComponent with its
 * default face connectivity, LabelIntensityStatisticsImageFilter and the loop over GetPhysicalSize): union-find
 * labelling of the nonzero voxels over 6 (D > 1) or 4 face neighbours, each component labelled by its first voxel in
 * C order.  out: uint8 [D][H][W], 1 on the component with the most voxels (ties: the earlier first voxel, ITK's
 * raster-order labels) and 0 elsewhere, all 0 without foreground.  stats: int64 [2] = {number of components, voxels
 * of the largest}.  Workspace: b200seg_components_workspace(D, H, W) bytes (8 per voxel).
 *
 * b200seg_morphology replaces MorphologicalOperation (utils.py:47-66: BinaryMorphologicalOpening / Closing,
 * BinaryDilate, BinaryErode of mask != 0 with the default sitkBall of radius r).  The ball is {d : |d|^2 <= r^2 + r}
 * over `dims` axes (ITK's FlatStructuringElement::Ball with axes 2r + 1).  DILATE: outside the image is background;
 * ERODE: outside is foreground (BoundaryToForeground); OPEN: erode, then dilate; CLOSE: on the image padded by r on
 * each of the `dims` axes with background (SafeBorder), dilate, erode, crop.  dims 2 needs D == 1; dims 3 with D == 1
 * is a one-slice 3-D image.  out: uint8 0/1 [D][H][W].  0 <= radius <= B200SEG_MORPH_MAX_RADIUS; for CLOSE the
 * padded grid must stay below 2^31 voxels.  Workspace: b200seg_morphology_workspace(...) bytes (4 per voxel of the
 * grid, 5 for OPEN and CLOSE).
 *
 * b200seg_label_bbox replaces GetLargestConnectedCompontBoundingbox (utils.py:7-16:
 * LabelShapeStatisticsImageFilter.GetBoundingBox(1) of the input itself, not of its largest component).  box: int64
 * [2 dims + 1] = {x0, y0, [z0,] size x, size y, [size z,] voxels equal to 1}, all zero when no voxel equals 1 (ITK
 * raises there).  Workspace: b200seg_label_bbox_workspace() bytes. */
#define B200SEG_MORPH_DILATE 0
#define B200SEG_MORPH_ERODE 1
#define B200SEG_MORPH_OPEN 2
#define B200SEG_MORPH_CLOSE 3
#define B200SEG_MORPH_MAX_RADIUS 64
int64_t b200seg_components_workspace(int D, int H, int W);
int b200seg_largest_component(const void* mask, int mask_dtype, int D, int H, int W, void* workspace,
                              int64_t workspace_bytes, uint8_t* out, int64_t* stats, int device,
                              b200seg_stream stream);
int64_t b200seg_morphology_workspace(int dims, int D, int H, int W, int radius, int op);
int b200seg_morphology(const void* mask, int mask_dtype, int dims, int D, int H, int W, int radius, int op,
                       void* workspace, int64_t workspace_bytes, uint8_t* out, int device, b200seg_stream stream);
int64_t b200seg_label_bbox_workspace(void);
int b200seg_label_bbox(const void* mask, int mask_dtype, int dims, int D, int H, int W, void* workspace,
                       int64_t workspace_bytes, int64_t* box, int device, b200seg_stream stream);

/* ---- Grad-CAM of ResNet2d (model/visualization.py:112-224, GradCAM; model/modelResNet.py:419-426,
 * Grad_CAM_Visual).  One call per target stage, in forward order, then one final scale; the map is fp32 [N][H][W].
 * act / grad: one stage's output and d(sum_i logit[i, t_i]) / d output, (N, 1, h, w, C), F32 or BF16, channel pitch,
 * C <= 1024, N <= 65535.  Stage `layer` of `nlayers`:
 *   w[n][c] = mean over the h*w pixels of grad (fp64 fixed-order sums), cam = max(sum_c w[c] act[..., c], 0),
 *   s = (cam - min) / (1e-7 + (max - min)) per image in fp32, then OpenCV's INTER_LINEAR resize to (H, W) in fp32:
 *   fx = (float)((d + 0.5) / (D / S) - 0.5), s0 = floor(fx), weights (1 - (fx - s0), fx - s0), clamped at the borders,
 *   the horizontal pass first, every product rounded before the sum (a stage at (H, W) is copied).
 *   out = s (layer 0) or out + s; the last stage divides by nlayers (np.mean over the stages).
 * b200seg_gradcam_scale: out = (out - min) / (1e-7 + (max - min)) per image, in place.
 * The workspace (b200seg_gradcam_workspace bytes, the largest over the stages of one map) carries the per-image min / max
 * from the stage calls to the scale call.  Min and max go through atomics (exact, order-free), sums have a fixed
 * order: reruns are bit-identical.  No allocation, no host synchronisation.
 * b200seg_gradcam_target: dlogits [N][K] = one-hot of t_i (target >= 0: t_i = target; target < 0: the arg-max of
 * logits row i, the first of equal maxima) and category [N] = t_i. */
int64_t b200seg_gradcam_workspace(int n, int h, int w, int c);
int b200seg_gradcam_layer(const b200seg_tensor* act, const b200seg_tensor* grad, int H, int W, int layer, int nlayers,
                          void* workspace, int64_t workspace_bytes, float* out, int device, b200seg_stream stream);
int b200seg_gradcam_scale(float* out, int n, int H, int W, void* workspace, int64_t workspace_bytes, int device,
                          b200seg_stream stream);

/* ---- voxelmorph's SpatialTransformer as VNet3dRegistration uses it (networks/VNet3dregistration.py:6-45,171-206):
 * F.grid_sample(src, new_locs, align_corners=True, padding_mode='zeros') at new_locs built from the displacement
 * field.  ddf: fp32 channels-last [N][D][H][W][3] (channel i displaces axis i: 0 = D, 1 = H, 2 = W), as the head
 * writes it.  Per voxel (d, h, w) and axis i with grid g = (d, h, w) and s_i = (D, H, W)[i] > 1, in fp32 in this order
 * and without FMA contraction:
 *   loc = g_i + ddf_i,   nrm = 2 * (loc / (s_i - 1) - 0.5),   u_i = ((nrm + 1) / 2) * (s_i - 1)
 * (the reference's normalisation, then grid_sample's align-corners unnormalisation; the channel reversal
 * [..., [2, 1, 0]] makes u_2 the x coordinate over W and u_0 the z coordinate over D).
 * b200seg_warp3d writes, for every channel, moved_image = trilinear sample of image at u (torch's floor cell and
 * weights, the eight corners in grid_sample's order, out-of-volume corners read 0) and moved_label = label at
 * nearbyint(u) (round half to even; 0 outside the volume).  image / moved_image: fp32 NCDHW-contiguous [N][Ci][D][H][W],
 * label / moved_label: fp32 [N][Cl][D][H][W]; either pair may be NULL (Ci or Cl = 0).
 * b200seg_warp3d_bwd: gddf [N][D][H][W][3] = d loss / d ddf from gmoved (d loss / d moved_image, NCDHW) through the
 * trilinear path (grid_sample's grid gradient: the one-sided derivative of the floor cell, summed over the channels in
 * order, times (s_i - 1) / 2, then the normalisation's 2 / (s_i - 1)), plus addend (same layout, or NULL).  The label
 * path passes no gradient, and there is none to image or label.  One thread per voxel: no atomics, reruns are
 * bit-identical.  D, H, W >= 2; N * D * H * W < 2^31. */
int b200seg_warp3d(const float* ddf, const float* image, int ci, const float* label, int cl, int N, int D, int H, int W,
                   float* moved_image, float* moved_label, int device, b200seg_stream stream);
int b200seg_warp3d_bwd(const float* ddf, const float* image, int ci, const float* gmoved, const float* addend, int N,
                       int D, int H, int W, float* gddf, int device, b200seg_stream stream);
int b200seg_gradcam_target(const float* logits, int n, int k, int target, float* dlogits, int64_t* category,
                           int device, b200seg_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SEG_H */
