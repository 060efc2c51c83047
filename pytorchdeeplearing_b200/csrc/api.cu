// extern "C" surface of libb200seg.so (see include/b200seg.h for the contract).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace b200seg {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// implemented in the other translation units
int conv_generic(int kind, int dims, const b200seg_tensor* x, const void* wpk, int w_dtype, const float* bias,
                 const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, cudaStream_t st);
int conv_tc_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                      const b200seg_tensor* addend);
int conv_tc(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias, const b200seg_tensor* y,
            double* stats, const b200seg_tensor* addend, int device, cudaStream_t st);
int conv_tc_init(int device);
int conv_halo_channels_ok(int kind, int cin, int cout);
int conv_halo_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                        const b200seg_tensor* addend);
int conv_halo(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias, const b200seg_tensor* y,
              double* stats, const b200seg_tensor* addend, int device, cudaStream_t st,
              const b200seg_tensor* yfwd = nullptr, const b200seg_gn* gn = nullptr, double* sums = nullptr);
int pw_mma_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                     const b200seg_tensor* addend);
int pw_mma_conv(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device, cudaStream_t st);
int conv_halows_ntile(int kind, int cin, int cout);
int conv_halows_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                          const b200seg_tensor* addend);
int conv_halows(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias,
                const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device, cudaStream_t st,
                const b200seg_tensor* yfwd = nullptr, const b200seg_gn* gn = nullptr, double* sums = nullptr);
int conv_tc_channels_ok(int kind, int cin, int cout);
int smallcin_conv_supported(int kind, const b200seg_tensor* x, const b200seg_tensor* y, const b200seg_tensor* addend);
int smallcin_conv(int kind, int dims, const b200seg_tensor* x, const void* w, int w_dtype, const float* bias,
                  const b200seg_tensor* y, double* stats, int device, cudaStream_t st);
int smallcin_wgrad_supported(int kind, const b200seg_tensor* a, const b200seg_tensor* b);
int smallcin_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st);
int stem_mma_conv_supported(int kind, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                            const b200seg_tensor* addend);
int stem_mma_conv(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                  const b200seg_tensor* y, double* stats, int device, cudaStream_t st);
int stem_mma_wgrad_supported(int kind, const b200seg_tensor* a, const b200seg_tensor* b);
int stem_mma_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st);
int stem_gn_supported(const b200seg_tensor* x, int cout, int dims);
int stem_gn(int mode, const b200seg_tensor* x, const void* wa, const float* ba, const void* wb, const float* bb,
            const b200seg_gn* gna, const b200seg_gn* gnb, double* stats_a, double* stats_b,
            const b200seg_tensor* out, const b200seg_tensor* gr, double* sums_a, double* sums_b, float* dwa,
            float* dwb, float* dgamma, float* dbeta, float* dba, float* dbb, int device, cudaStream_t st);
int stem_conv_supported(int kind, const b200seg_tensor* x, const b200seg_tensor* y, const b200seg_tensor* addend);
int stem_conv(int kind, int dims, const b200seg_tensor* x, const void* w, int w_dtype, const float* bias,
              const b200seg_tensor* y, double* stats, int device, cudaStream_t st);
int stem_wgrad_supported(int kind, const b200seg_tensor* a, const b200seg_tensor* b);
int stem_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
               cudaStream_t st);
int head_fwd(const b200seg_tensor* x, const float* w, const float* bias, float* logits, float* probs, int nc,
             int device, cudaStream_t st);
int head_bwd_supported(const b200seg_tensor* x, int nc);
int head_bwd(const b200seg_tensor* x, const float* dl, const float* w, const b200seg_tensor* dx, float* dw, float* db,
             int nc, int device, cudaStream_t st);
int wgrad_halo_mma_supported(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b);
int wgrad_halo_mma(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st);
int wgrad_tc_supported(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b);
int wgrad_tc(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
             cudaStream_t st);
int wgrad_generic(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                  cudaStream_t st);
int ew_pack_weight(const float* w, void* out, int out_dtype, int T, int K, int N2, int N1, long long st,
                   long long sk, long long sn2, long long sn1, int flip, cudaStream_t s);
int ew_unpack_wgrad(const float* dwp, float* grad, int T, int K, int N, long long st, long long sk, long long sn,
                    cudaStream_t s);
int ew_pack_multi(const void* table_dev, int count, int total_blocks, int unpack, cudaStream_t s);
int ew_upload_table(const void* host, long long bytes, void* dev_dst, cudaStream_t s);
int ew_gn_finalize(const double* stats, const float* gamma, const float* beta, const float* scale, int N, int C,
                   int groups, long long vox, float eps, float* coef, float* mr, cudaStream_t s);
int ew_apply(const b200seg_tensor* y1, const float* c1, const b200seg_gn* g1, const b200seg_tensor* y2,
             const float* c2, const b200seg_gn* g2, const b200seg_tensor* res, const b200seg_tensor* out, int device,
             cudaStream_t s);
int ew_gn_bwd_reduce(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, const b200seg_gn* gn,
                     double* sums, int device, cudaStream_t s);
int ew_gn_bwd_finalize(const double* sums, const float* mr, const float* gamma, const float* scale, int N, int C,
                       int groups, long long vox, float* coef3, float* dgamma, float* dbeta, float* dbias,
                       cudaStream_t s);
int ew_gn_bwd_fused_supported(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_tensor* dy);
int ew_gn_bwd_fused(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, double* sums,
                    unsigned int* counter, float* dgamma, float* dbeta, float* dbias, const b200seg_tensor* dy,
                    int device, cudaStream_t s);
int ew_gn_bwd_apply(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, const float* coef3,
                    const b200seg_gn* gn, const double* sums, float* dgamma, float* dbeta, float* dbias,
                    const b200seg_tensor* dy, int device, cudaStream_t s, int sum_y_from_stats = 0);
int ew_colsum(const b200seg_tensor* dy, float* out, int device, cudaStream_t s);
int ew_pool_fwd(const b200seg_tensor* x, const b200seg_tensor* out, int dims, int device, cudaStream_t s);
int ew_pool_bwd(const b200seg_tensor* x, const b200seg_tensor* go, const b200seg_tensor* addend,
                const b200seg_tensor* gx, int dims, int device, cudaStream_t s);
int ew_head_probs(const float* logits, float* probs, long long nvox_, int C, int device, cudaStream_t s);
int loss_partials(const float* logits, const void* labels, int label_dtype, int N, long long vox, int C, float gamma,
                  float alpha_f, double* part, double* metric, int device, cudaStream_t s);
int metric_partials(const float* probs, const void* labels, int label_dtype, int N, long long vox, int C, float thr,
                    double* metric, int device, cudaStream_t s);
int metric_finalize(const double* metric, int N, int C, float* out, cudaStream_t s);
int adam_step(float* p, const float* g, float* m, float* v, long long n, float* state, float lr, float beta1,
              float beta2, float eps, float wd, int decoupled, const float* gscale, int tick, int device,
              cudaStream_t s);
int dropout_masks(const long long* rng, const int* table, int nmasks, int total, double p_drop, float* out,
                  cudaStream_t s);
int head_mask(const b200seg_tensor* x, const float* w, const float* bias, unsigned char* mask, int nc, float thr,
              int device, cudaStream_t st);
int mask_logits(const float* logits, long long nv, int C, float thr, unsigned char* mask, int device, cudaStream_t st);
int stage_u8_sums(const unsigned char* img, int n, long long per, unsigned long long* sums, int device, cudaStream_t st);
int stage_u8_normalize(const unsigned char* img, int n, long long per, const unsigned long long* sums, void* out,
                       int out_dtype, int device, cudaStream_t st);
int stage_labels_u8(const unsigned char* lab, long long count, int binarize, long long* out, int device, cudaStream_t st);
int loss_finalize(const double* part, int C, int terms, const float* alpha, float gamma, float alpha_f, float* loss,
                  float* lcoef, cudaStream_t s);
int loss_bwd(const float* logits, const void* labels, int label_dtype, long long nvox_, int C, const float* lcoef,
             const float* gscale, float* dlogits, int device, cudaStream_t s);
int loss_partials_ss(const float* logits, const void* labels, int label_dtype, int N, long long vox, double* part,
                     double* metric, int device, cudaStream_t s);
int loss_bwd_ss(const float* logits, const void* labels, int label_dtype, long long nvox_, const float* lcoef,
                const float* gscale, float* dlogits, int device, cudaStream_t s);
int64_t radix_sort_workspace(int nseg, long long len);
int radix_sort_pairs(const uint32_t* kin, const int32_t* vin, uint32_t* kout, int32_t* vout, int nseg, long long len,
                     void* ws, long long ws_bytes, cudaStream_t s);
int64_t lovasz_workspace(int N, long long vox, int C, int per_image);
int lovasz_fwd(const float* z, const long long* t, int N, long long vox, int C, int per_image, int has_ignore,
               long long ignore, void* ws, long long ws_bytes, float* loss, float* coef, float* seg_scale, int device,
               cudaStream_t s);
int lovasz_bwd(const float* z, const long long* t, int N, long long vox, int C, int per_image, const float* coef,
               const float* seg_scale, const float* gscale, float* dz, int device, cudaStream_t s);
int64_t segmetric3d_workspace(int N, int D, int H, int W);
int segmetric3d(const void* real, int rdt, const void* pred, int pdt, int N, int D, int H, int W,
                const double* spacing, void* ws, long long ws_bytes, long long* counts, double* metrics, int* flags,
                int device, cudaStream_t s);
int segmetric3d_points(const void* real, int rdt, const void* pred, int pdt, int N, int D, int H, int W,
                       const double* spacing, void* ws, long long ws_bytes, long long cap_r, long long cap_p,
                       long long* real_idx, long long* pred_idx, double* real_nn, double* pred_nn, int device,
                       cudaStream_t s);
int64_t ssim_workspace(int dims, int N, int C, int D, int H, int W, int k);
int ssim_fwd(int dims, const float* x, const int64_t* xs, const float* y, const int64_t* ys, int N, int C, int D,
             int H, int W, int k, const float* taps, double* coef, void* ws, long long ws_bytes, int device,
             cudaStream_t st);
int ssim_finalize(int dims, int N, int C, int D, int H, int W, int k, int size_average, int reduce, const void* ws,
                  long long ws_bytes, double* acc, float* value, cudaStream_t st);
int ssim_bwd(int dims, const float* x, const int64_t* xs, const float* y, const int64_t* ys, int N, int C, int D,
             int H, int W, int k, const float* taps, const double* coef, int size_average, const float* gout,
             const double* acc, float* dx, float* dy, int device, cudaStream_t st);
int cls_head_fwd(const b200seg_tensor* x, const float* w1, const float* b1, const float* w2, const float* b2, int Hd,
                 int K, float* pooled, float* hidden, float* logits, cudaStream_t st);
int cls_head_bwd(const float* dlogits, const float* pooled, const float* hidden, const float* w1, const float* w2,
                 int Hd, int K, float* work, const b200seg_tensor* dx, float* dw1, float* db1, float* dw2, float* db2,
                 int device, cudaStream_t st);

int64_t resample_workspace(int mode, long long nvox);
int resample_linear(const void* src, int dtype, int D, int H, int W, const double* ratio, int oD, int oH, int oW,
                    int mode, float lower, float upper, float* out, void* ws, long long ws_bytes, cudaStream_t st);
int normalize_volume(int mode, const float* x, long long nvox, void* ws, long long ws_bytes, float* out, int device,
                     cudaStream_t st);
int resample_nearest_u8(const uint8_t* src, int D, int H, int W, const double* ratio, int vD, int vH, int vW, int oD,
                        int oH, int oW, uint8_t* out, int device, cudaStream_t st);

static bool valid_tensor(const b200seg_tensor* t) {
  return t && t->ptr && t->n > 0 && t->d > 0 && t->h > 0 && t->w > 0 && t->c > 0 && t->ld >= t->c &&
         (t->dtype == B200SEG_F32 || t->dtype == B200SEG_BF16);
}

}  // namespace b200seg

using namespace b200seg;

#define ST(s) static_cast<cudaStream_t>(s)
#define REQ_TENSOR(t, what) B200_CHECK_ARG(valid_tensor(t), "%s: invalid tensor descriptor '%s'", __func__, what)
#define OPT_TENSOR(t, what) B200_CHECK_ARG((t) == nullptr || valid_tensor(t), "%s: invalid tensor descriptor '%s'", __func__, what)

extern "C" {

int b200seg_version(void) { return B200SEG_VERSION; }

const char* b200seg_last_error(void) { return g_err; }

int b200seg_init(int device) {
  B200_DEVICE(device);
  return conv_tc_init(device);
}

int b200seg_pack_weight(const float* w, void* out, int out_dtype, int T, int K, int N2, int N1, int64_t st, int64_t sk,
                        int64_t sn2, int64_t sn1, int flip, int device, b200seg_stream stream) {
  B200_CHECK_ARG(w && out && T > 0 && K > 0 && N2 > 0 && N1 > 0, "b200seg_pack_weight: bad argument");
  B200_CHECK_ARG(out_dtype == B200SEG_F32 || out_dtype == B200SEG_BF16, "b200seg_pack_weight: bad dtype");
  B200_DEVICE(device);
  return ew_pack_weight(w, out, out_dtype, T, K, N2, N1, st, sk, sn2, sn1, flip, ST(stream));
}

int b200seg_unpack_wgrad(const float* dwp, float* grad, int T, int K, int N, int64_t st, int64_t sk, int64_t sn,
                         int device, b200seg_stream stream) {
  B200_CHECK_ARG(dwp && grad && T > 0 && K > 0 && N > 0, "b200seg_unpack_wgrad: bad argument");
  B200_DEVICE(device);
  return ew_unpack_wgrad(dwp, grad, T, K, N, st, sk, sn, ST(stream));
}

int b200seg_pack_weights_multi(const b200seg_pack_desc* table, int count, int total_blocks, int device,
                               b200seg_stream stream) {
  B200_CHECK_ARG(table != nullptr && count >= 0 && total_blocks >= 0, "b200seg_pack_weights_multi: bad argument");
  B200_DEVICE(device);
  return ew_pack_multi(table, count, total_blocks, 0, ST(stream));
}

int b200seg_upload_table(const void* host_table, int64_t bytes, void* device_dst, int device, b200seg_stream stream) {
  B200_CHECK_ARG(host_table != nullptr && device_dst != nullptr && bytes > 0, "b200seg_upload_table: bad argument");
  B200_DEVICE(device);
  return ew_upload_table(host_table, bytes, device_dst, ST(stream));
}

int b200seg_unpack_wgrads_multi(const b200seg_pack_desc* table, int count, int total_blocks, int device,
                                b200seg_stream stream) {
  B200_CHECK_ARG(table != nullptr && count >= 0 && total_blocks >= 0, "b200seg_unpack_wgrads_multi: bad argument");
  B200_DEVICE(device);
  return ew_pack_multi(table, count, total_blocks, 1, ST(stream));
}

// The kernel family b200seg_conv runs, from the arguments alone (x, y, addend already validated).  b200seg_conv
// switches on this value, so the query and the launch cannot disagree.
static int conv_path(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                     const b200seg_tensor* addend) {
  if (pw_mma_supported(kind, dims, x, w_dtype, y, addend)) return B200SEG_CONV_PW_MMA;
  if (conv_tc_supported(kind, dims, x, w_dtype, y, addend)) return B200SEG_CONV_TC;
  if (conv_halo_supported(kind, dims, x, w_dtype, y, addend))
    return dims == 3 ? B200SEG_CONV_HALO3 : B200SEG_CONV_HALO2D;
  if (conv_halows_supported(kind, dims, x, w_dtype, y, addend)) return B200SEG_CONV_HALO_WS;
  if (w_dtype == B200SEG_BF16_TC || w_dtype == B200SEG_BF16_HALO || w_dtype == B200SEG_BF16_HALO_WS)
    return B200SEG_EINVAL;
  const bool small_types =
      w_dtype == B200SEG_F32 ? (x->dtype == B200SEG_F32 && y->dtype == B200SEG_F32) : y->dtype == B200SEG_BF16;
  if (stem_mma_conv_supported(kind, x, w_dtype, y, addend)) return B200SEG_CONV_STEM_MMA;
  if (small_types && stem_conv_supported(kind, x, y, addend)) return B200SEG_CONV_STEM;
  if (small_types && smallcin_conv_supported(kind, x, y, addend)) return B200SEG_CONV_SMALLCIN;
  return B200SEG_CONV_GENERIC;
}

int b200seg_conv_path(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                      const b200seg_tensor* addend) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(y, "y");
  OPT_TENSOR(addend, "addend");
  B200_CHECK_ARG(dims == 2 || dims == 3, "b200seg_conv_path: dims must be 2 or 3");
  B200_CHECK_ARG(dims == 3 || (x->d == 1 && y->d == 1), "b200seg_conv_path: 2-D tensors must have d == 1");
  const int path = conv_path(kind, dims, x, w_dtype, y, addend);
  B200_CHECK_ARG(path >= 0, "b200seg_conv_path: packed tensor-core weights need bf16, 16-byte aligned activations of "
                 "a supported shape");
  return path;
}

int b200seg_conv(int kind, int dims, const b200seg_tensor* x, const void* wpk, int w_dtype, const float* bias,
                 const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device,
                 b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(y, "y");
  OPT_TENSOR(addend, "addend");
  B200_CHECK_ARG(wpk != nullptr, "b200seg_conv: null weights");
  B200_CHECK_ARG(dims == 2 || dims == 3, "b200seg_conv: dims must be 2 or 3");
  B200_CHECK_ARG(dims == 3 || (x->d == 1 && y->d == 1), "b200seg_conv: 2-D tensors must have d == 1");
  B200_DEVICE(device);
  switch (conv_path(kind, dims, x, w_dtype, y, addend)) {
    case B200SEG_CONV_PW_MMA:
      return pw_mma_conv(kind, dims, x, wpk, bias, y, stats, addend, device, ST(stream));
    case B200SEG_CONV_TC:
      return conv_tc(kind, dims, x, wpk, bias, y, stats, addend, device, ST(stream));
    case B200SEG_CONV_HALO2D:
    case B200SEG_CONV_HALO3:
      if (conv_tc_init(device) != B200SEG_OK) return B200SEG_ECUDA;
      return conv_halo(kind, dims, x, wpk, bias, y, stats, addend, device, ST(stream));
    case B200SEG_CONV_HALO_WS:
      if (conv_tc_init(device) != B200SEG_OK) return B200SEG_ECUDA;
      return conv_halows(kind, dims, x, wpk, bias, y, stats, addend, device, ST(stream));
    case B200SEG_CONV_STEM_MMA:
      return stem_mma_conv(kind, dims, x, wpk, bias, y, stats, device, ST(stream));
    case B200SEG_CONV_STEM:
      return stem_conv(kind, dims, x, wpk, w_dtype, bias, y, stats, device, ST(stream));
    case B200SEG_CONV_SMALLCIN:
      return smallcin_conv(kind, dims, x, wpk, w_dtype, bias, y, stats, device, ST(stream));
    case B200SEG_CONV_GENERIC:
      return conv_generic(kind, dims, x, wpk, w_dtype, bias, y, stats, addend, ST(stream));
  }
  set_error("b200seg_conv: B200SEG_BF16_TC weights need bf16, 16-byte aligned activations of a supported shape");
  return B200SEG_EINVAL;
}

int b200seg_conv_bwdstats_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                                    const b200seg_tensor* addend, const b200seg_tensor* yfwd) {
  if (x == nullptr || y == nullptr || yfwd == nullptr) return 0;
  // only where b200seg_conv itself takes a kernel with the backward-sums epilogue
  const int path = conv_path(kind, dims, x, w_dtype, y, addend);
  if (path != B200SEG_CONV_HALO3 && path != B200SEG_CONV_HALO_WS) return 0;
  return (yfwd->n == y->n && yfwd->d == y->d && yfwd->h == y->h && yfwd->w == y->w && yfwd->c == y->c &&
          yfwd->dtype == B200SEG_BF16 && (yfwd->ld % 8) == 0 && (reinterpret_cast<uintptr_t>(yfwd->ptr) % 16) == 0)
             ? 1 : 0;
}

int b200seg_conv_bwdstats(int kind, int dims, const b200seg_tensor* x, const void* wpk, int w_dtype,
                          const b200seg_tensor* y, const b200seg_tensor* addend, const b200seg_tensor* yfwd,
                          const b200seg_gn* gn, double* sums, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(y, "y");
  REQ_TENSOR(yfwd, "yfwd");
  OPT_TENSOR(addend, "addend");
  B200_CHECK_ARG(wpk != nullptr && gn != nullptr && sums != nullptr && gn->stats && gn->gamma && gn->beta,
                 "b200seg_conv_bwdstats: null argument");
  B200_CHECK_ARG(b200seg_conv_bwdstats_supported(kind, dims, x, w_dtype, y, addend, yfwd),
                 "b200seg_conv_bwdstats: unsupported shape (query b200seg_conv_bwdstats_supported first)");
  B200_DEVICE(device);
  if (conv_tc_init(device) != B200SEG_OK) return B200SEG_ECUDA;
  if (conv_path(kind, dims, x, w_dtype, y, addend) == B200SEG_CONV_HALO_WS)
    return conv_halows(kind, dims, x, wpk, nullptr, y, nullptr, addend, device, ST(stream), yfwd, gn, sums);
  return conv_halo(kind, dims, x, wpk, nullptr, y, nullptr, addend, device, ST(stream), yfwd, gn, sums);
}

int b200seg_conv_tc_eligible(int kind, int cin, int cout) { return conv_tc_channels_ok(kind, cin, cout); }

int b200seg_conv_halo_eligible(int kind, int cin, int cout) { return conv_halo_channels_ok(kind, cin, cout); }

int b200seg_conv_halo_ws_ntile(int kind, int cin, int cout) { return conv_halows_ntile(kind, cin, cout); }

// the kernel family b200seg_wgrad runs (a, b already validated); b200seg_wgrad switches on it
static int wgrad_path(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b) {
  if (wgrad_halo_mma_supported(kind, dims, a, b)) return B200SEG_WGRAD_HALO_MMA;
  if (wgrad_tc_supported(kind, dims, a, b)) return B200SEG_WGRAD_TC;
  if (stem_mma_wgrad_supported(kind, a, b)) return B200SEG_WGRAD_STEM_MMA;
  if (stem_wgrad_supported(kind, a, b)) return B200SEG_WGRAD_STEM;
  if (smallcin_wgrad_supported(kind, a, b)) return B200SEG_WGRAD_SMALLCIN;
  return B200SEG_WGRAD_GENERIC;
}

int b200seg_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                  b200seg_stream stream) {
  REQ_TENSOR(a, "a");
  REQ_TENSOR(b, "b");
  B200_CHECK_ARG(dwp != nullptr, "b200seg_wgrad: null output");
  B200_CHECK_ARG(dims == 2 || dims == 3, "b200seg_wgrad: dims must be 2 or 3");
  B200_DEVICE(device);
  switch (wgrad_path(kind, dims, a, b)) {
    case B200SEG_WGRAD_HALO_MMA:
      return wgrad_halo_mma(kind, dims, a, b, dwp, device, ST(stream));
    case B200SEG_WGRAD_TC:
      if (conv_tc_init(device) != B200SEG_OK) return B200SEG_ECUDA;
      return wgrad_tc(kind, dims, a, b, dwp, device, ST(stream));
    case B200SEG_WGRAD_STEM_MMA:
      return stem_mma_wgrad(kind, dims, a, b, dwp, device, ST(stream));
    case B200SEG_WGRAD_STEM:
      return stem_wgrad(kind, dims, a, b, dwp, device, ST(stream));
    case B200SEG_WGRAD_SMALLCIN:
      return smallcin_wgrad(kind, dims, a, b, dwp, device, ST(stream));
    default:
      return wgrad_generic(kind, dims, a, b, dwp, device, ST(stream));
  }
}

int b200seg_wgrad_path(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b) {
  REQ_TENSOR(a, "a");
  REQ_TENSOR(b, "b");
  B200_CHECK_ARG(dims == 2 || dims == 3, "b200seg_wgrad_path: dims must be 2 or 3");
  return wgrad_path(kind, dims, a, b);
}

int b200seg_gn_finalize(const double* stats, const float* gamma, const float* beta, const float* scale, int N, int C,
                        int groups, int64_t vox, float eps, float* coef, float* mr, int device,
                        b200seg_stream stream) {
  B200_CHECK_ARG(stats && gamma && beta && coef && mr && N > 0 && C > 0 && groups > 0 && vox > 0,
                 "b200seg_gn_finalize: bad argument");
  B200_DEVICE(device);
  return ew_gn_finalize(stats, gamma, beta, scale, N, C, groups, vox, eps, coef, mr, ST(stream));
}

int b200seg_apply(const b200seg_tensor* y1, const float* coef1, const b200seg_tensor* y2, const float* coef2,
                  const b200seg_tensor* res, const b200seg_tensor* out, int device, b200seg_stream stream) {
  REQ_TENSOR(y1, "y1");
  REQ_TENSOR(out, "out");
  OPT_TENSOR(y2, "y2");
  OPT_TENSOR(res, "res");
  B200_CHECK_ARG(coef1 && (!y2 || coef2), "b200seg_apply: missing coefficients");
  B200_DEVICE(device);
  return ew_apply(y1, coef1, nullptr, y2, coef2, nullptr, res, out, device, ST(stream));
}

static bool valid_gn(const b200seg_gn* g, int C) {
  return g && g->stats && g->gamma && g->beta && g->groups > 0 && (C % g->groups) == 0 && g->vox > 0;
}

int b200seg_apply_gn(const b200seg_tensor* y1, const b200seg_gn* gn1, const b200seg_tensor* y2, const b200seg_gn* gn2,
                     const b200seg_tensor* res, const b200seg_tensor* out, int device, b200seg_stream stream) {
  REQ_TENSOR(y1, "y1");
  REQ_TENSOR(out, "out");
  OPT_TENSOR(y2, "y2");
  OPT_TENSOR(res, "res");
  B200_CHECK_ARG(valid_gn(gn1, y1->c) && (!y2 || valid_gn(gn2, y2->c)), "b200seg_apply_gn: bad GroupNorm reference");
  B200_DEVICE(device);
  return ew_apply(y1, nullptr, gn1, y2, nullptr, gn2, res, out, device, ST(stream));
}

int b200seg_gn_bwd_reduce_gn(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, double* sums,
                             int device, b200seg_stream stream) {
  REQ_TENSOR(g, "g");
  REQ_TENSOR(y, "y");
  B200_CHECK_ARG(valid_gn(gn, y->c) && sums && y->c <= 2048, "b200seg_gn_bwd_reduce_gn: bad argument");
  B200_DEVICE(device);
  return ew_gn_bwd_reduce(g, y, nullptr, gn, sums, device, ST(stream));
}

int b200seg_gn_bwd_apply_gn(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, const double* sums,
                            const b200seg_tensor* dy, float* dgamma, float* dbeta, float* dbias, int sum_y_from_stats,
                            int device, b200seg_stream stream) {
  REQ_TENSOR(g, "g");
  REQ_TENSOR(y, "y");
  REQ_TENSOR(dy, "dy");
  B200_CHECK_ARG(valid_gn(gn, y->c) && sums && dgamma && dbeta, "b200seg_gn_bwd_apply_gn: bad argument");
  B200_DEVICE(device);
  return ew_gn_bwd_apply(g, y, nullptr, nullptr, gn, sums, dgamma, dbeta, dbias, dy, device, ST(stream),
                         sum_y_from_stats);
}

int b200seg_gn_bwd_fused_supported(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_tensor* dy,
                                   int device) {
  if (g == nullptr || y == nullptr || dy == nullptr) return 0;
  if (!ew_gn_bwd_fused_supported(g, y, dy)) return 0;
  return y->n <= num_sms(device) ? 1 : 0;
}

int b200seg_gn_bwd_fused_gn(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, double* sums,
                            unsigned int* counter, const b200seg_tensor* dy, float* dgamma, float* dbeta,
                            float* dbias, int device, b200seg_stream stream) {
  REQ_TENSOR(g, "g");
  REQ_TENSOR(y, "y");
  REQ_TENSOR(dy, "dy");
  B200_CHECK_ARG(valid_gn(gn, y->c) && sums && counter && dgamma && dbeta, "b200seg_gn_bwd_fused_gn: bad argument");
  B200_DEVICE(device);
  return ew_gn_bwd_fused(g, y, gn, sums, counter, dgamma, dbeta, dbias, dy, device, ST(stream));
}

int b200seg_gn_bwd_reduce(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, double* sums, int device,
                          b200seg_stream stream) {
  REQ_TENSOR(g, "g");
  REQ_TENSOR(y, "y");
  B200_CHECK_ARG(coef && sums, "b200seg_gn_bwd_reduce: null argument");
  B200_CHECK_ARG(y->c <= 4096, "b200seg_gn_bwd_reduce: too many channels");
  B200_DEVICE(device);
  return ew_gn_bwd_reduce(g, y, coef, nullptr, sums, device, ST(stream));
}

int b200seg_gn_bwd_finalize(const double* sums, const float* mr, const float* gamma, const float* scale, int N, int C,
                            int groups, int64_t vox, float* coef3, float* dgamma, float* dbeta, float* dbias,
                            int device, b200seg_stream stream) {
  B200_CHECK_ARG(sums && mr && gamma && coef3 && dgamma && dbeta && N > 0 && C > 0 && groups > 0 && vox > 0,
                 "b200seg_gn_bwd_finalize: bad argument");
  B200_DEVICE(device);
  return ew_gn_bwd_finalize(sums, mr, gamma, scale, N, C, groups, vox, coef3, dgamma, dbeta, dbias, ST(stream));
}

int b200seg_gn_bwd_apply(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, const float* coef3,
                         const b200seg_tensor* dy, int device, b200seg_stream stream) {
  REQ_TENSOR(g, "g");
  REQ_TENSOR(y, "y");
  REQ_TENSOR(dy, "dy");
  B200_CHECK_ARG(coef && coef3, "b200seg_gn_bwd_apply: null coefficients");
  B200_DEVICE(device);
  return ew_gn_bwd_apply(g, y, coef, coef3, nullptr, nullptr, nullptr, nullptr, nullptr, dy, device, ST(stream));
}

int b200seg_colsum(const b200seg_tensor* dy, float* out, int device, b200seg_stream stream) {
  REQ_TENSOR(dy, "dy");
  B200_CHECK_ARG(out != nullptr && dy->c <= 4096, "b200seg_colsum: bad argument");
  B200_DEVICE(device);
  return ew_colsum(dy, out, device, ST(stream));
}

int b200seg_stem_gn_supported(const b200seg_tensor* x, int cout, int dims) {
  if (x == nullptr || !valid_tensor(x)) return 0;
  return stem_gn_supported(x, cout, dims);
}

int b200seg_stem_gn_stats(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                          double* stats3, double* stats1, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  B200_DEVICE(device);
  return stem_gn(0, x, w3, b3, w1, b1, nullptr, nullptr, stats3, stats1, nullptr, nullptr, nullptr, nullptr, nullptr,
                 nullptr, nullptr, nullptr, nullptr, nullptr, device, ST(stream));
}

int b200seg_stem_gn_apply(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                          const b200seg_gn* gn3, const b200seg_gn* gn1, const b200seg_tensor* out, int device,
                          b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(out, "out");
  B200_DEVICE(device);
  return stem_gn(1, x, w3, b3, w1, b1, gn3, gn1, nullptr, nullptr, out, nullptr, nullptr, nullptr, nullptr, nullptr,
                 nullptr, nullptr, nullptr, nullptr, device, ST(stream));
}

int b200seg_stem_gn_bwd_sums(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                             const b200seg_gn* gn3, const b200seg_gn* gn1, const b200seg_tensor* g, double* sums3,
                             double* sums1, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(g, "g");
  B200_DEVICE(device);
  return stem_gn(2, x, w3, b3, w1, b1, gn3, gn1, nullptr, nullptr, nullptr, g, sums3, sums1, nullptr, nullptr, nullptr,
                 nullptr, nullptr, nullptr, device, ST(stream));
}

int b200seg_stem_gn_bwd(const b200seg_tensor* x, const void* w3, const float* b3, const void* w1, const float* b1,
                        const b200seg_gn* gn3, const b200seg_gn* gn1, const b200seg_tensor* g, const double* sums3,
                        const double* sums1, float* dw3, float* dw1, float* dgamma, float* dbeta, float* db3,
                        float* db1, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(g, "g");
  B200_DEVICE(device);
  return stem_gn(3, x, w3, b3, w1, b1, gn3, gn1, nullptr, nullptr, nullptr, g, const_cast<double*>(sums3),
                 const_cast<double*>(sums1), dw3, dw1, dgamma, dbeta, db3, db1, device, ST(stream));
}

int b200seg_pool_fwd(const b200seg_tensor* x, const b200seg_tensor* out, int dims, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(out, "out");
  B200_CHECK_ARG(dims == 2 || dims == 3, "b200seg_pool_fwd: dims must be 2 or 3");
  B200_DEVICE(device);
  return ew_pool_fwd(x, out, dims, device, ST(stream));
}

int b200seg_pool_bwd(const b200seg_tensor* x, const b200seg_tensor* g_out, const b200seg_tensor* addend,
                     const b200seg_tensor* g_x, int dims, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(g_out, "g_out");
  REQ_TENSOR(g_x, "g_x");
  OPT_TENSOR(addend, "addend");
  B200_CHECK_ARG(dims == 2 || dims == 3, "b200seg_pool_bwd: dims must be 2 or 3");
  B200_DEVICE(device);
  return ew_pool_bwd(x, g_out, addend, g_x, dims, device, ST(stream));
}

int b200seg_head_fwd(const b200seg_tensor* x, const float* w, const float* bias, float* logits, float* probs, int nc,
                     int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  B200_CHECK_ARG(w && logits, "b200seg_head_fwd: null argument");
  B200_DEVICE(device);
  return head_fwd(x, w, bias, logits, probs, nc, device, ST(stream));
}

int b200seg_head_bwd_supported(int cin, int nc) {
  b200seg_tensor t;
  t.c = cin;
  return head_bwd_supported(&t, nc);
}

int b200seg_head_bwd(const b200seg_tensor* x, const float* dlogits, const float* w, const b200seg_tensor* dx,
                     float* dw, float* db, int nc, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  REQ_TENSOR(dx, "dx");
  B200_CHECK_ARG(dlogits && w && dw && db, "b200seg_head_bwd: null argument");
  B200_DEVICE(device);
  return head_bwd(x, dlogits, w, dx, dw, db, nc, device, ST(stream));
}

int b200seg_head_probs(const float* logits, float* probs, int64_t nvox_, int C, int device, b200seg_stream stream) {
  B200_CHECK_ARG(logits && probs && nvox_ > 0 && C > 0, "b200seg_head_probs: bad argument");
  B200_DEVICE(device);
  return ew_head_probs(logits, probs, nvox_, C, device, ST(stream));
}

int b200seg_loss_partials(const float* logits, const void* labels, int label_dtype, int N, int64_t vox, int C,
                          float gamma, float alpha_f, double* part, double* metric, int device,
                          b200seg_stream stream) {
  B200_CHECK_ARG(logits && labels && part && vox > 0 && N > 0, "b200seg_loss_partials: bad argument");
  B200_DEVICE(device);
  return loss_partials(logits, labels, label_dtype, N, vox, C, gamma, alpha_f, part, metric, device, ST(stream));
}

int b200seg_metric_partials(const float* probs, const void* labels, int label_dtype, int N, int64_t vox, int C,
                            float threshold, double* metric, int device, b200seg_stream stream) {
  B200_CHECK_ARG(probs && labels && metric && vox > 0 && N > 0, "b200seg_metric_partials: bad argument");
  B200_CHECK_ARG(label_dtype == B200SEG_I64 || label_dtype == B200SEG_F32, "b200seg_metric_partials: bad label dtype");
  B200_DEVICE(device);
  return metric_partials(probs, labels, label_dtype, N, vox, C, threshold, metric, device, ST(stream));
}

int b200seg_metric_finalize(const double* metric, int N, int C, float* out, int device, b200seg_stream stream) {
  B200_CHECK_ARG(metric && out && N > 0 && C > 0, "b200seg_metric_finalize: bad argument");
  B200_DEVICE(device);
  return metric_finalize(metric, N, C, out, ST(stream));
}

int b200seg_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float* state,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int decoupled,
                      const float* gscale, int tick, int device, b200seg_stream stream) {
  B200_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && state && n > 0, "b200seg_adam_step: bad argument");
  B200_DEVICE(device);
  return adam_step(param, grad, exp_avg, exp_avg_sq, n, state, lr, beta1, beta2, eps, weight_decay, decoupled, gscale,
                   tick, device, ST(stream));
}

int b200seg_dropout_masks(const int64_t* rng, const int32_t* table, int nmasks, int total, double p_drop, float* out,
                          int device, b200seg_stream stream) {
  B200_CHECK_ARG(rng && table && out, "b200seg_dropout_masks: null argument");
  B200_DEVICE(device);
  return dropout_masks(reinterpret_cast<const long long*>(rng), table, nmasks, total, p_drop, out, ST(stream));
}

int b200seg_head_mask(const b200seg_tensor* x, const float* w, const float* bias, uint8_t* mask, int nc,
                      float threshold, int device, b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  B200_CHECK_ARG(w && mask, "b200seg_head_mask: null argument");
  B200_DEVICE(device);
  return head_mask(x, w, bias, mask, nc, threshold, device, ST(stream));
}

int b200seg_mask_logits(const float* logits, int64_t nvox_, int C, float threshold, uint8_t* mask, int device,
                        b200seg_stream stream) {
  B200_CHECK_ARG(logits && mask && nvox_ > 0 && C > 0, "b200seg_mask_logits: bad argument");
  B200_DEVICE(device);
  return mask_logits(logits, nvox_, C, threshold, mask, device, ST(stream));
}

int b200seg_cls_head_fwd(const b200seg_tensor* x, const float* w1, const float* b1, const float* w2, const float* b2,
                         int hidden_width, int ncls, float* pooled, float* hidden, float* logits, int device,
                         b200seg_stream stream) {
  REQ_TENSOR(x, "x");
  B200_CHECK_ARG(w1 && b1 && w2 && b2 && pooled && hidden && logits, "b200seg_cls_head_fwd: null argument");
  B200_CHECK_ARG(x->n <= 65535, "b200seg_cls_head_fwd: batch must be at most 65535 (got %d)", x->n);
  B200_DEVICE(device);
  return cls_head_fwd(x, w1, b1, w2, b2, hidden_width, ncls, pooled, hidden, logits, ST(stream));
}

int b200seg_cls_head_bwd(const float* dlogits, const float* pooled, const float* hidden, const float* w1,
                         const float* w2, int hidden_width, int ncls, float* work, const b200seg_tensor* dx, float* dw1,
                         float* db1, float* dw2, float* db2, int device, b200seg_stream stream) {
  REQ_TENSOR(dx, "dx");
  B200_CHECK_ARG(dlogits && pooled && hidden && w1 && w2 && work && dw1 && db1 && dw2 && db2,
                 "b200seg_cls_head_bwd: null argument");
  B200_CHECK_ARG(dx->n <= 65535, "b200seg_cls_head_bwd: batch must be at most 65535 (got %d)", dx->n);
  B200_DEVICE(device);
  return cls_head_bwd(dlogits, pooled, hidden, w1, w2, hidden_width, ncls, work, dx, dw1, db1, dw2, db2, device,
                      ST(stream));
}

int b200seg_stage_u8_sums(const uint8_t* img, int n, int64_t per_sample, uint64_t* sums, int device,
                          b200seg_stream stream) {
  B200_CHECK_ARG(img && sums && n > 0 && per_sample > 0, "b200seg_stage_u8_sums: bad argument");
  B200_CHECK_ARG(n <= 65535, "b200seg_stage_u8_sums: at most 65535 samples per call (got %d)", n);
  B200_DEVICE(device);
  return stage_u8_sums(img, n, per_sample, reinterpret_cast<unsigned long long*>(sums), device, ST(stream));
}

int b200seg_stage_u8_normalize(const uint8_t* img, int n, int64_t per_sample, const uint64_t* sums, void* out,
                               int out_dtype, int device, b200seg_stream stream) {
  B200_CHECK_ARG(img && sums && out && n > 0 && per_sample > 0, "b200seg_stage_u8_normalize: bad argument");
  B200_CHECK_ARG(n <= 65535, "b200seg_stage_u8_normalize: at most 65535 samples per call (got %d)", n);
  B200_CHECK_ARG(out_dtype == B200SEG_F32 || out_dtype == B200SEG_BF16, "b200seg_stage_u8_normalize: fp32 or bf16 output");
  B200_DEVICE(device);
  return stage_u8_normalize(img, n, per_sample, reinterpret_cast<const unsigned long long*>(sums), out, out_dtype,
                            device, ST(stream));
}

int b200seg_stage_labels_u8(const uint8_t* lab, int64_t count, int binarize, int64_t* out, int device,
                            b200seg_stream stream) {
  B200_CHECK_ARG(lab && out && count > 0, "b200seg_stage_labels_u8: bad argument");
  B200_DEVICE(device);
  return stage_labels_u8(lab, count, binarize, reinterpret_cast<long long*>(out), device, ST(stream));
}

int b200seg_loss_finalize(const double* part, int C, int terms, const float* alpha, float gamma, float alpha_f,
                          float* loss, float* lcoef, int device, b200seg_stream stream) {
  B200_CHECK_ARG(part && loss && lcoef && C >= 1 && (C == 1 || alpha), "b200seg_loss_finalize: bad argument");
  const int ext = terms & B200SEG_LOSS_EXT_MASK;
  B200_CHECK_ARG((terms > 0 && terms < 8) ||
                     (terms == ext && (ext & (ext - 1)) == 0 && (C == 1 || ext == B200SEG_LOSS_ELDICE)),
                 "b200seg_loss_finalize: bad terms mask %d for %d classes", terms, C);
  B200_DEVICE(device);
  return loss_finalize(part, C, terms, alpha, gamma, alpha_f, loss, lcoef, ST(stream));
}

int b200seg_loss_bwd(const float* logits, const void* labels, int label_dtype, int64_t nvox_, int C,
                     const float* lcoef, const float* gscale, float* dlogits, int device, b200seg_stream stream) {
  B200_CHECK_ARG(logits && labels && lcoef && gscale && dlogits && nvox_ > 0, "b200seg_loss_bwd: bad argument");
  B200_DEVICE(device);
  return loss_bwd(logits, labels, label_dtype, nvox_, C, lcoef, gscale, dlogits, device, ST(stream));
}

int b200seg_loss_partials_ss(const float* logits, const void* labels, int label_dtype, int N, int64_t vox,
                             double* part, double* metric, int device, b200seg_stream stream) {
  B200_CHECK_ARG(logits && labels && part && vox > 0 && N > 0, "b200seg_loss_partials_ss: bad argument");
  B200_CHECK_ARG(label_dtype == B200SEG_I64 || label_dtype == B200SEG_F32, "b200seg_loss_partials_ss: bad label dtype");
  B200_DEVICE(device);
  return loss_partials_ss(logits, labels, label_dtype, N, vox, part, metric, device, ST(stream));
}

int b200seg_loss_bwd_ss(const float* logits, const void* labels, int label_dtype, int64_t nvox_, const float* lcoef,
                        const float* gscale, float* dlogits, int device, b200seg_stream stream) {
  B200_CHECK_ARG(logits && labels && lcoef && gscale && dlogits && nvox_ > 0, "b200seg_loss_bwd_ss: bad argument");
  B200_CHECK_ARG(label_dtype == B200SEG_I64 || label_dtype == B200SEG_F32, "b200seg_loss_bwd_ss: bad label dtype");
  B200_DEVICE(device);
  return loss_bwd_ss(logits, labels, label_dtype, nvox_, lcoef, gscale, dlogits, device, ST(stream));
}

int64_t b200seg_radix_sort_workspace(int nseg, int64_t seg_len) {
  if (nseg < 1 || seg_len < 0) return 0;
  return radix_sort_workspace(nseg, seg_len);
}

int b200seg_radix_sort_pairs(const uint32_t* keys_in, const int32_t* vals_in, uint32_t* keys_out, int32_t* vals_out,
                             int nseg, int64_t seg_len, void* workspace, int64_t workspace_bytes, int device,
                             b200seg_stream stream) {
  B200_CHECK_ARG(seg_len == 0 || (keys_in && vals_in && keys_out && vals_out), "b200seg_radix_sort_pairs: null argument");
  B200_DEVICE(device);
  return radix_sort_pairs(keys_in, vals_in, keys_out, vals_out, nseg, seg_len, workspace, workspace_bytes, ST(stream));
}

int64_t b200seg_lovasz_workspace(int N, int64_t vox, int C, int per_image) {
  if (N < 1 || vox < 1 || C < 1) return 0;
  return lovasz_workspace(N, vox, C, per_image);
}

int b200seg_lovasz_fwd(const float* logits, const int64_t* labels, int N, int64_t vox, int C, int per_image,
                       int has_ignore, int64_t ignore, void* workspace, int64_t workspace_bytes, float* loss,
                       float* coef, float* seg_scale, int device, b200seg_stream stream) {
  B200_CHECK_ARG(logits && labels && loss && coef && seg_scale, "b200seg_lovasz_fwd: null argument");
  B200_DEVICE(device);
  return lovasz_fwd(logits, reinterpret_cast<const long long*>(labels), N, vox, C, per_image, has_ignore, ignore,
                    workspace, workspace_bytes, loss, coef, seg_scale, device, ST(stream));
}

int b200seg_lovasz_bwd(const float* logits, const int64_t* labels, int N, int64_t vox, int C, int per_image,
                       const float* coef, const float* seg_scale, const float* gscale, float* dlogits, int device,
                       b200seg_stream stream) {
  B200_CHECK_ARG(logits && labels && coef && seg_scale && gscale && dlogits, "b200seg_lovasz_bwd: null argument");
  B200_DEVICE(device);
  return lovasz_bwd(logits, reinterpret_cast<const long long*>(labels), N, vox, C, per_image, coef, seg_scale, gscale,
                    dlogits, device, ST(stream));
}

int64_t b200seg_segmetric3d_workspace(int N, int D, int H, int W) {
  if (N < 1 || D < 1 || H < 1 || W < 1) return 0;
  return segmetric3d_workspace(N, D, H, W);
}

int b200seg_segmetric3d(const void* real, int real_dtype, const void* pred, int pred_dtype, int N, int D, int H, int W,
                        const double* spacing_zyx, void* workspace, int64_t workspace_bytes, int64_t* counts,
                        double* metrics, int32_t* flags, int device, b200seg_stream stream) {
  B200_CHECK_ARG(real && pred && spacing_zyx && counts && metrics && flags, "b200seg_segmetric3d: null argument");
  B200_DEVICE(device);
  return segmetric3d(real, real_dtype, pred, pred_dtype, N, D, H, W, spacing_zyx, workspace, workspace_bytes,
                     reinterpret_cast<long long*>(counts), metrics, flags, device, ST(stream));
}

int b200seg_segmetric3d_points(const void* real, int real_dtype, const void* pred, int pred_dtype, int N, int D, int H,
                               int W, const double* spacing_zyx, void* workspace, int64_t workspace_bytes,
                               int64_t cap_r, int64_t cap_p, int64_t* real_idx, int64_t* pred_idx, double* real2pred,
                               double* pred2real, int device, b200seg_stream stream) {
  B200_CHECK_ARG(real && pred && spacing_zyx, "b200seg_segmetric3d_points: null argument");
  B200_CHECK_ARG((cap_r == 0 || (real_idx && real2pred)) && (cap_p == 0 || (pred_idx && pred2real)),
                 "b200seg_segmetric3d_points: null output");
  B200_DEVICE(device);
  return segmetric3d_points(real, real_dtype, pred, pred_dtype, N, D, H, W, spacing_zyx, workspace, workspace_bytes,
                            cap_r, cap_p, reinterpret_cast<long long*>(real_idx),
                            reinterpret_cast<long long*>(pred_idx), real2pred, pred2real, device, ST(stream));
}

int64_t b200seg_ssim_workspace(int dims, int N, int C, int D, int H, int W, int window_size) {
  if ((dims != 2 && dims != 3) || N < 1 || C < 1 || H < 1 || W < 1 || (dims == 3 && D < 1) || window_size < 1 ||
      window_size > 31)
    return 0;
  return ssim_workspace(dims, N, C, D, H, W, window_size);
}

int b200seg_ssim_fwd(int dims, const float* img1, const int64_t* strides1, const float* img2, const int64_t* strides2,
                     int N, int C, int D, int H, int W, int window_size, const float* taps, double* coef,
                     void* workspace, int64_t workspace_bytes, int device, b200seg_stream stream) {
  B200_CHECK_ARG(img1 && img2 && strides1 && strides2, "b200seg_ssim_fwd: null argument");
  B200_DEVICE(device);
  return ssim_fwd(dims, img1, strides1, img2, strides2, N, C, D, H, W, window_size, taps, coef, workspace,
                  workspace_bytes, device, ST(stream));
}

int b200seg_ssim_finalize(int dims, int N, int C, int D, int H, int W, int window_size, int size_average, int reduce,
                          const void* workspace, int64_t workspace_bytes, double* acc, float* value, int device,
                          b200seg_stream stream) {
  B200_CHECK_ARG(acc && value, "b200seg_ssim_finalize: null argument");
  B200_DEVICE(device);
  return ssim_finalize(dims, N, C, D, H, W, window_size, size_average, reduce, workspace, workspace_bytes, acc, value,
                       ST(stream));
}

int b200seg_ssim_bwd(int dims, const float* img1, const int64_t* strides1, const float* img2, const int64_t* strides2,
                     int N, int C, int D, int H, int W, int window_size, const float* taps, const double* coef,
                     int size_average, const float* gout, const double* acc, float* grad1, float* grad2, int device,
                     b200seg_stream stream) {
  B200_CHECK_ARG(img1 && img2 && strides1 && strides2 && coef && gout, "b200seg_ssim_bwd: null argument");
  B200_CHECK_ARG(grad1 || grad2, "b200seg_ssim_bwd: no gradient requested");
  B200_DEVICE(device);
  return ssim_bwd(dims, img1, strides1, img2, strides2, N, C, D, H, W, window_size, taps, coef, size_average, gout,
                  acc, grad1, grad2, device, ST(stream));
}

static bool valid_ratio(const double* r) {
  return r && r[0] > 0.0 && r[1] > 0.0 && r[2] > 0.0 && r[0] < 1e9 && r[1] < 1e9 && r[2] < 1e9;
}

int64_t b200seg_resample_workspace(int norm_mode, int oD, int oH, int oW) {
  if (norm_mode < B200SEG_NORM_NONE || norm_mode > B200SEG_NORM_PCTL || oD < 1 || oH < 1 || oW < 1) return 0;
  return resample_workspace(norm_mode, (long long)oD * oH * oW);
}

int b200seg_resample_linear(const void* src, int src_dtype, int D, int H, int W, const double* ratio_zyx, int oD,
                            int oH, int oW, int norm_mode, float lower, float upper, float* out, void* workspace,
                            int64_t workspace_bytes, int device, b200seg_stream stream) {
  B200_CHECK_ARG(src && out, "b200seg_resample_linear: null argument");
  B200_CHECK_ARG(D >= 1 && H >= 1 && W >= 1 && oD >= 1 && oH >= 1 && oW >= 1,
                 "b200seg_resample_linear: sizes must be >= 1 (%d %d %d -> %d %d %d)", D, H, W, oD, oH, oW);
  B200_CHECK_ARG(src_dtype == B200SEG_U8 || src_dtype == B200SEG_I16 || src_dtype == B200SEG_I32 ||
                     src_dtype == B200SEG_F32,
                 "b200seg_resample_linear: unsupported pixel type %d", src_dtype);
  B200_CHECK_ARG(norm_mode >= B200SEG_NORM_NONE && norm_mode <= B200SEG_NORM_PCTL,
                 "b200seg_resample_linear: bad norm_mode %d", norm_mode);
  B200_CHECK_ARG(valid_ratio(ratio_zyx), "b200seg_resample_linear: ratios must be finite and > 0");
  B200_CHECK_ARG(norm_mode != B200SEG_NORM_PCTL || (long long)oD * oH * oW < (1LL << 31),
                 "b200seg_resample_linear: the percentile sort takes < 2^31 voxels");
  B200_DEVICE(device);
  return resample_linear(src, src_dtype, D, H, W, ratio_zyx, oD, oH, oW, norm_mode, lower, upper, out, workspace,
                         workspace_bytes, ST(stream));
}

int b200seg_normalize(int norm_mode, const float* x, int oD, int oH, int oW, void* workspace, int64_t workspace_bytes,
                      float* out, int device, b200seg_stream stream) {
  B200_CHECK_ARG(x && out && x != out, "b200seg_normalize: null or aliased argument");
  B200_CHECK_ARG(oD >= 1 && oH >= 1 && oW >= 1, "b200seg_normalize: sizes must be >= 1");
  B200_CHECK_ARG(norm_mode == B200SEG_NORM_MEANSTD || norm_mode == B200SEG_NORM_PCTL,
                 "b200seg_normalize: bad norm_mode %d", norm_mode);
  B200_CHECK_ARG(norm_mode != B200SEG_NORM_PCTL || (long long)oD * oH * oW < (1LL << 31),
                 "b200seg_normalize: the percentile sort takes < 2^31 voxels");
  B200_DEVICE(device);
  return normalize_volume(norm_mode, x, (long long)oD * oH * oW, workspace, workspace_bytes, out, device, ST(stream));
}

int b200seg_resample_nearest_u8(const uint8_t* src, int D, int H, int W, const double* ratio_zyx, int vD, int vH,
                                int vW, int oD, int oH, int oW, uint8_t* out, int device, b200seg_stream stream) {
  B200_CHECK_ARG(src && out, "b200seg_resample_nearest_u8: null argument");
  B200_CHECK_ARG(D >= 1 && H >= 1 && W >= 1 && oD >= 1 && oH >= 1 && oW >= 1 && vD >= 0 && vH >= 0 && vW >= 0,
                 "b200seg_resample_nearest_u8: bad sizes");
  B200_CHECK_ARG(valid_ratio(ratio_zyx), "b200seg_resample_nearest_u8: ratios must be finite and > 0");
  B200_DEVICE(device);
  return resample_nearest_u8(src, D, H, W, ratio_zyx, vD, vH, vW, oD, oH, oW, out, device, ST(stream));
}

}  // extern "C"
