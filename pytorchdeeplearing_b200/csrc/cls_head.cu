// Classifier head of ResNet2d / ResNet3d (reference networks/ResNet3d.py:61-118, ResNet2d.py:62-119):
//   GlobalAveragePooling -> Linear(C, Hd) -> ReLU -> Linear(Hd, K)
// on the last encoder activation (N, D, H, W, C) channels-last, bf16 or fp32.  The MLP is a few MFLOP, so it runs on
// CUDA cores.  Every sum (over voxels, inputs and the batch) is taken by one thread or one warp in a fixed order and
// nothing uses atomics, so reruns give identical bits.  No allocation and no host synchronisation: graph-capturable.
//
//   forward  launch 1  cls_pool_kernel      pooled[n][c] = mean over voxels of x[n, :, c]
//            launch 2  cls_mlp_fwd_kernel   hidden = relu(W1 pooled + b1), logits = W2 hidden + b2   (one CTA per sample)
//   backward launch 1  cls_mlp_bwd_kernel   dh = (W2^T dlogits) * [hidden > 0], dp = (W1^T dh) / vox   (one CTA per sample)
//   backward launch 2  cls_grad_kernel      dW1, db1, dW2, db2 (one thread per element, batch summed in order) and the
//                                           broadcast dx[n, v, c] = dp[n][c] (the mean's gradient)
#include "common.cuh"

namespace b200seg {

constexpr int kClsMax = 1024;          // bound on C, Hd and K (shared-memory vectors of one sample)
constexpr int kPoolLanes = 32;         // channels per pooling CTA
constexpr int kPoolRows = 8;           // voxel lanes per pooling CTA

template <typename T>
__global__ void __launch_bounds__(kPoolLanes * kPoolRows) cls_pool_kernel(TV x, float inv_vox,
                                                                           float* __restrict__ pooled) {
  PDL_ENTER();
  __shared__ float part[kPoolRows][kPoolLanes];
  const int n = blockIdx.y;
  const int c = blockIdx.x * kPoolLanes + threadIdx.x;
  const long long vox = (long long)x.d * x.h * x.w;
  const T* base = static_cast<const T*>(x.p) + (long long)n * vox * x.ld;
  float s = 0.f;
  if (c < x.c)
    for (long long v = threadIdx.y; v < vox; v += kPoolRows) s += to_f(base[v * x.ld + c]);
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < x.c) {
    float t = part[0][threadIdx.x];
#pragma unroll
    for (int r = 1; r < kPoolRows; ++r) t += part[r][threadIdx.x];
    pooled[(long long)n * x.c + c] = t * inv_vox;
  }
}

// y[o] = b[o] + sum_i W[o][i] v[i] for o < O: one warp per output row, lanes stride the inputs, fixed-order warp sum
__device__ __forceinline__ void warp_rows(const float* __restrict__ W, const float* __restrict__ b,
                                          const float* __restrict__ v, int I, int O, float* __restrict__ y, bool relu) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int o = warp; o < O; o += nw) {
    const float* row = W + (long long)o * I;
    float s = 0.f;
    for (int i = lane; i < I; i += 32) s = fmaf(row[i], v[i], s);
    s = warp_sum(s);
    if (lane == 0) {
      s += b[o];
      y[o] = relu ? fmaxf(s, 0.f) : s;
    }
  }
}

__global__ void __launch_bounds__(256) cls_mlp_fwd_kernel(const float* __restrict__ pooled, const float* __restrict__ w1,
                                                          const float* __restrict__ b1, const float* __restrict__ w2,
                                                          const float* __restrict__ b2, int C, int Hd, int K,
                                                          float* __restrict__ hidden, float* __restrict__ logits) {
  PDL_ENTER();
  __shared__ float sp[kClsMax];
  __shared__ float sh[kClsMax];
  const int n = blockIdx.x;
  for (int i = threadIdx.x; i < C; i += blockDim.x) sp[i] = pooled[(long long)n * C + i];
  __syncthreads();
  warp_rows(w1, b1, sp, C, Hd, sh, true);
  __syncthreads();
  for (int i = threadIdx.x; i < Hd; i += blockDim.x) hidden[(long long)n * Hd + i] = sh[i];
  warp_rows(w2, b2, sh, Hd, K, logits + (long long)n * K, false);
}

__global__ void __launch_bounds__(256) cls_mlp_bwd_kernel(const float* __restrict__ dlogits,
                                                          const float* __restrict__ hidden, const float* __restrict__ w1,
                                                          const float* __restrict__ w2, int C, int Hd, int K,
                                                          float inv_vox, float* __restrict__ dh,
                                                          float* __restrict__ dp) {
  PDL_ENTER();
  __shared__ float sl[kClsMax];
  __shared__ float sd[kClsMax];
  const int n = blockIdx.x;
  for (int i = threadIdx.x; i < K; i += blockDim.x) sl[i] = dlogits[(long long)n * K + i];
  __syncthreads();
  // column j of W2 (coalesced over j), k summed in order
  for (int j = threadIdx.x; j < Hd; j += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < K; ++k) s = fmaf(w2[(long long)k * Hd + j], sl[k], s);
    s = hidden[(long long)n * Hd + j] > 0.f ? s : 0.f;
    sd[j] = s;
    dh[(long long)n * Hd + j] = s;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < Hd; ++j) s = fmaf(w1[(long long)j * C + c], sd[j], s);
    dp[(long long)n * C + c] = s * inv_vox;
  }
}

// blocks [0, wblocks): one thread per weight / bias element, in state_dict order (fc_layers.0.weight, .0.bias,
// .2.weight, .2.bias), each summing over the batch in order; blocks [wblocks, grid): the broadcast data gradient.
template <typename T>
__global__ void __launch_bounds__(256) cls_grad_kernel(const float* __restrict__ dlogits,
                                                       const float* __restrict__ pooled,
                                                       const float* __restrict__ hidden, const float* __restrict__ dh,
                                                       const float* __restrict__ dp, int N, int C, int Hd, int K,
                                                       int wblocks, float* __restrict__ dw1, float* __restrict__ db1,
                                                       float* __restrict__ dw2, float* __restrict__ db2, TV dx) {
  PDL_ENTER();
  if ((int)blockIdx.x < wblocks) {
    long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n1 = (long long)Hd * C, n2 = n1 + Hd, n3 = n2 + (long long)K * Hd, n4 = n3 + K;
    if (e >= n4) return;
    const float *a, *b;
    int sa, sb;
    float* out;
    if (e < n1) {                       // dW1[j][c] = sum_n dh[n][j] pooled[n][c]
      a = dh + e / C; sa = Hd; b = pooled + e % C; sb = C; out = dw1 + e;
    } else if (e < n2) {                // db1[j] = sum_n dh[n][j]
      e -= n1; a = dh + e; sa = Hd; b = nullptr; sb = 0; out = db1 + e;
    } else if (e < n3) {                // dW2[k][j] = sum_n dlogits[n][k] hidden[n][j]
      e -= n2; a = dlogits + e / Hd; sa = K; b = hidden + e % Hd; sb = Hd; out = dw2 + e;
    } else {                            // db2[k] = sum_n dlogits[n][k]
      e -= n3; a = dlogits + e; sa = K; b = nullptr; sb = 0; out = db2 + e;
    }
    float s = 0.f;
    if (b != nullptr)
      for (int n = 0; n < N; ++n) s = fmaf(a[(long long)n * sa], b[(long long)n * sb], s);
    else
      for (int n = 0; n < N; ++n) s += a[(long long)n * sa];
    *out = s;
    return;
  }
  const long long vox = (long long)dx.d * dx.h * dx.w;
  const long long total = (long long)N * vox * C;
  const long long stride = (long long)(gridDim.x - wblocks) * blockDim.x;
  T* out = static_cast<T*>(dx.p);
  for (long long i = (long long)(blockIdx.x - wblocks) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % C);
    const long long nv = i / C;                        // n * vox + v
    const int n = (int)(nv / vox);
    out[nv * dx.ld + c] = from_f<T>(dp[(long long)n * C + c]);
  }
}

static int cls_check(const char* fn, int C, int Hd, int K) {
  B200_CHECK_ARG(C >= 1 && C <= kClsMax && Hd >= 1 && Hd <= kClsMax && K >= 1 && K <= kClsMax,
                 "%s: channels, hidden width and classes must be in [1, %d] (got C=%d, Hd=%d, K=%d)", fn, kClsMax, C,
                 Hd, K);
  return B200SEG_OK;
}

int cls_head_fwd(const b200seg_tensor* x, const float* w1, const float* b1, const float* w2, const float* b2, int Hd,
                 int K, float* pooled, float* hidden, float* logits, cudaStream_t st) {
  if (int rc = cls_check("b200seg_cls_head_fwd", x->c, Hd, K)) return rc;
  const TV t = tv(x);
  const float inv_vox = (float)(1.0 / (double)nvox(x));
  const dim3 grid((x->c + kPoolLanes - 1) / kPoolLanes, x->n);
  const dim3 block(kPoolLanes, kPoolRows);
  if (x->dtype == B200SEG_BF16)
    launch_k(cls_pool_kernel<bf16>, grid, block, 0, st, t, inv_vox, pooled);
  else
    launch_k(cls_pool_kernel<float>, grid, block, 0, st, t, inv_vox, pooled);
  B200_LAUNCH_CHECK();
  launch_k(cls_mlp_fwd_kernel, x->n, 256, 0, st, (const float*)pooled, w1, b1, w2, b2, x->c, Hd, K, hidden, logits);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int cls_head_bwd(const float* dlogits, const float* pooled, const float* hidden, const float* w1, const float* w2,
                 int Hd, int K, float* work, const b200seg_tensor* dx, float* dw1, float* db1, float* dw2, float* db2,
                 int device, cudaStream_t st) {
  const int N = dx->n, C = dx->c;
  if (int rc = cls_check("b200seg_cls_head_bwd", C, Hd, K)) return rc;
  float* dh = work;                                      // [N][Hd]
  float* dp = work + (long long)N * Hd;                  // [N][C]
  const float inv_vox = (float)(1.0 / (double)nvox(dx));
  launch_k(cls_mlp_bwd_kernel, N, 256, 0, st, dlogits, hidden, w1, w2, C, Hd, K, inv_vox, dh, dp);
  B200_LAUNCH_CHECK();
  const long long nw = (long long)Hd * C + Hd + (long long)K * Hd + K;
  const int wblocks = (int)((nw + 255) / 256);
  long long bb = ((long long)N * nvox(dx) * C + 255) / 256;
  const long long cap = (long long)num_sms(device) * 8;
  if (bb > cap) bb = cap;
  const int grid = wblocks + (int)bb;
  if (dx->dtype == B200SEG_BF16)
    launch_k(cls_grad_kernel<bf16>, grid, 256, 0, st, dlogits, pooled, hidden, (const float*)dh, (const float*)dp, N, C,
             Hd, K, wblocks, dw1, db1, dw2, db2, tv(dx));
  else
    launch_k(cls_grad_kernel<float>, grid, 256, 0, st, dlogits, pooled, hidden, (const float*)dh, (const float*)dp, N,
             C, Hd, K, wblocks, dw1, db1, dw2, db2, tv(dx));
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
