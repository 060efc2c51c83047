// Single-image-channel stem (Cin == 1) on CUDA cores (sm_90a): VNet3d.py:28-29 in_tr.conv1 (3x3x3) /
// in_tr.conv2 (1x1x1), Unet3d.py:67 / Unet2d.py:67 enc1conv1.  These two layers carry 27 (or 1) MACs per output
// element -- no MMA shape fits -- but they touch full-resolution tensors, so they must run at streaming speed:
//
//   conv_stem1_kernel  : a thread owns VPT (1 or 2) voxels adjacent in w.  All KD x 3 x (2+VPT) input values are
//                        fetched first (one batch of independent loads, coalesced along w), then the taps are a
//                        straight-line FMA block against fp32 weights broadcast from shared memory (one LDS.128
//                        per 8 FMAs).  Bias, GroupNorm statistics (fixed summation order) and the 128-bit NDHWC
//                        stores are fused.
//   wgrad_stem1_kernel : dW[tap][co] = sum_v x[v + tap] * dy[v][co].  A thread owns one voxel per trip and the
//                        accumulators of ONE kd-plane of taps (9) x CG output channels (72 registers); the
//                        (kd-plane, channel-group) variants are the fastest grid index so the CTAs that share
//                        dy rows run together and hit L2.  Voxel coordinates advance incrementally (no division
//                        in the loop); the block folds its accumulators once at the end.
//
// smallcin (small_channels.cu) remains the fallback for Cin in 2..4 and odd widths.
#include "common.cuh"

namespace b200seg {

template <typename TX, typename TW, typename TY, int COUT, int KD, int KHW, int VPT>
__global__ void __launch_bounds__(256, 2) conv_stem1_kernel(const TX* __restrict__ x, long long xld,
                                                            const TW* __restrict__ w, const float* __restrict__ bias,
                                                            TY* __restrict__ y, long long yld,
                                                            double* __restrict__ stats, int D, int H, int W) {
  PDL_ENTER();
  constexpr int TAPS = KD * KHW * KHW;
  constexpr int PD = KD / 2, PHW = KHW / 2;
  constexpr int XW = KHW + VPT - 1;                 // input columns covering the thread's VPT voxels along w
  __shared__ __align__(16) float s_w[TAPS * COUT];
  __shared__ float s_b[COUT];
  __shared__ float s_red[8][2 * COUT];
  for (int i = threadIdx.x; i < TAPS * COUT; i += blockDim.x) s_w[i] = to_f(w[i]);
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) s_b[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int n = blockIdx.y;
  const int WG = W / VPT;
  const int items = D * H * WG;
  const long long V = (long long)D * H * W;
  const TX* xb = x + (long long)n * V * xld;
  TY* yb = y + (long long)n * V * yld;
  float ssum[COUT], ssq[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) ssum[c] = ssq[c] = 0.f;
#pragma unroll 1
  for (int pi = blockIdx.x * blockDim.x + threadIdx.x; pi < items; pi += gridDim.x * blockDim.x) {
    const int ow = (pi % WG) * VPT;
    const int t2 = pi / WG;
    const int oh = t2 % H;
    const int od = t2 / H;
    float xv[KD][KHW][XW];
#pragma unroll
    for (int a = 0; a < KD; ++a) {
      const int id = od + a - PD;
#pragma unroll
      for (int b = 0; b < KHW; ++b) {
        const int ih = oh + b - PHW;
        const bool rok = (unsigned)id < (unsigned)D && (unsigned)ih < (unsigned)H;
        const TX* row = xb + ((long long)(rok ? id : 0) * H + (rok ? ih : 0)) * W * xld;
#pragma unroll
        for (int c = 0; c < XW; ++c) {
          const int iw = ow + c - PHW;
          xv[a][b][c] = (rok && (unsigned)iw < (unsigned)W) ? to_f(row[(long long)iw * xld]) : 0.f;
        }
      }
    }
    float acc[VPT][COUT];
#pragma unroll
    for (int v = 0; v < VPT; ++v)
#pragma unroll
      for (int c = 0; c < COUT; ++c) acc[v][c] = s_b[c];
#pragma unroll
    for (int a = 0; a < KD; ++a)
#pragma unroll
      for (int b = 0; b < KHW; ++b)
#pragma unroll
        for (int cc = 0; cc < KHW; ++cc) {
          const float4* wr = reinterpret_cast<const float4*>(s_w + ((a * KHW + b) * KHW + cc) * COUT);
#pragma unroll
          for (int c4 = 0; c4 < COUT / 4; ++c4) {
            const float4 wv = wr[c4];
#pragma unroll
            for (int v = 0; v < VPT; ++v) {
              const float xx = xv[a][b][cc + v];
              acc[v][4 * c4 + 0] = fmaf(xx, wv.x, acc[v][4 * c4 + 0]);
              acc[v][4 * c4 + 1] = fmaf(xx, wv.y, acc[v][4 * c4 + 1]);
              acc[v][4 * c4 + 2] = fmaf(xx, wv.z, acc[v][4 * c4 + 2]);
              acc[v][4 * c4 + 3] = fmaf(xx, wv.w, acc[v][4 * c4 + 3]);
            }
          }
        }
    TY* py = yb + (((long long)od * H + oh) * W + ow) * yld;
#pragma unroll
    for (int v = 0; v < VPT; ++v)
#pragma unroll
      for (int c4 = 0; c4 < COUT / 4; ++c4)
        store4(py + v * yld + 4 * c4,
               make_float4(acc[v][4 * c4], acc[v][4 * c4 + 1], acc[v][4 * c4 + 2], acc[v][4 * c4 + 3]));
    if (stats != nullptr) {
#pragma unroll
      for (int v = 0; v < VPT; ++v)
#pragma unroll
        for (int c = 0; c < COUT; ++c) {
          ssum[c] += acc[v][c];
          ssq[c] = fmaf(acc[v][c], acc[v][c], ssq[c]);
        }
    }
  }
  if (stats != nullptr) {
    // fixed order: lanes (shuffle tree) -> warps (smem rows) -> one fp64 atomic per (channel, moment) per CTA
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < COUT; ++c) {
      const float a = warp_sum(ssum[c]);
      const float b = warp_sum(ssq[c]);
      if (lane == 0) {
        s_red[wid][c] = a;
        s_red[wid][COUT + c] = b;
      }
    }
    __syncthreads();
    if (threadIdx.x < 2 * COUT) {
      double t = 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += (double)s_red[k][threadIdx.x];
      const int which = threadIdx.x / COUT, c = threadIdx.x - which * COUT;
      atomicAdd(stats + ((long long)n * COUT + c) * 2 + which, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------
template <typename TB, int CG> struct DyVec;
template <int CG> struct DyVec<float, CG> {
  static __device__ __forceinline__ void load(const float* p, float* o) {
#pragma unroll
    for (int i = 0; i < CG / 4; ++i) {
      const float4 v = load4(p + 4 * i);
      o[4 * i] = v.x; o[4 * i + 1] = v.y; o[4 * i + 2] = v.z; o[4 * i + 3] = v.w;
    }
  }
};
template <int CG> struct DyVec<bf16, CG> {
  static __device__ __forceinline__ void load(const bf16* p, float* o) {
#pragma unroll
    for (int i = 0; i < CG / 8; ++i) load8(p + 8 * i, o + 8 * i);
  }
};

template <typename TA, typename TB, int COUT, int KD, int KHW, int CG>
__global__ void __launch_bounds__(256) wgrad_stem1_kernel(const TA* __restrict__ a, long long ald,
                                                          const TB* __restrict__ b, long long bld,
                                                          float* __restrict__ dwp, int N, int D, int H, int W) {
  PDL_ENTER();
  constexpr int PD = KD / 2, PHW = KHW / 2;
  constexpr int NCG = COUT / CG;
  constexpr int NVAR = KD * NCG;
  constexpr int NACC = KHW * KHW * CG;
  __shared__ float s_red[8][NACC];
  const int var = blockIdx.x % NVAR;
  const int chunk = blockIdx.x / NVAR;
  const int nchunks = gridDim.x / NVAR;
  const int tg = var / NCG;                      // kd plane of this CTA's taps
  const int cg = var - tg * NCG;                 // output-channel group
  float acc[KHW * KHW][CG];
#pragma unroll
  for (int t = 0; t < KHW * KHW; ++t)
#pragma unroll
    for (int c = 0; c < CG; ++c) acc[t][c] = 0.f;
  const long long V = (long long)D * H * W;
  const long long NV = (long long)N * V;
  const long long step = (long long)nchunks * blockDim.x;
  // decomposition of the stride, so the loop advances (ow, oh, od, n) by add-with-carry
  const int sw = (int)(step % W);
  const int sh = (int)((step / W) % H);
  const int sd = (int)((step / ((long long)W * H)) % D);
  const int sn = (int)(step / V);
  long long gv = (long long)chunk * blockDim.x + threadIdx.x;
  int ow = (int)(gv % W), oh = (int)((gv / W) % H), od = (int)((gv / ((long long)W * H)) % D), n = (int)(gv / V);
#pragma unroll 1
  for (; gv < NV; gv += step) {
    const int id = od + tg - PD;
    if ((unsigned)id < (unsigned)D) {
      float dv[CG];
      DyVec<TB, CG>::load(b + gv * bld + cg * CG, dv);
      float xv[KHW][KHW];
      const TA* plane = a + (((long long)n * D + id) * H) * W * ald;
#pragma unroll
      for (int bb = 0; bb < KHW; ++bb) {
        const int ih = oh + bb - PHW;
        const bool rok = (unsigned)ih < (unsigned)H;
        const TA* row = plane + (long long)(rok ? ih : 0) * W * ald;
#pragma unroll
        for (int cc = 0; cc < KHW; ++cc) {
          const int iw = ow + cc - PHW;
          xv[bb][cc] = (rok && (unsigned)iw < (unsigned)W) ? to_f(row[(long long)iw * ald]) : 0.f;
        }
      }
#pragma unroll
      for (int bb = 0; bb < KHW; ++bb)
#pragma unroll
        for (int cc = 0; cc < KHW; ++cc)
#pragma unroll
          for (int c = 0; c < CG; ++c) acc[bb * KHW + cc][c] = fmaf(xv[bb][cc], dv[c], acc[bb * KHW + cc][c]);
    }
    ow += sw;
    if (ow >= W) { ow -= W; ++oh; }
    oh += sh;
    if (oh >= H) { oh -= H; ++od; }
    od += sd;
    if (od >= D) { od -= D; ++n; }
    n += sn;
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int t = 0; t < KHW * KHW; ++t)
#pragma unroll
    for (int c = 0; c < CG; ++c) {
      const float s = warp_sum(acc[t][c]);
      if (lane == 0) s_red[wid][t * CG + c] = s;
    }
  __syncthreads();
  for (int i = threadIdx.x; i < NACC; i += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += s_red[k][i];
    const int tp = i / CG, c = i - tp * CG;
    const int tap = tg * KHW * KHW + tp;
    atomicAdd(dwp + (long long)tap * COUT + cg * CG + c, t);
  }
}

// ------------------------------------------------------------------------------------------------
// host dispatch
// ------------------------------------------------------------------------------------------------
static bool al16t(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

int stem_conv_supported(int kind, const b200seg_tensor* x, const b200seg_tensor* y, const b200seg_tensor* addend) {
  if (kind != B200SEG_K3 && kind != B200SEG_K1) return 0;
  if (addend != nullptr || x->c != 1) return 0;
  if (y->c != 16 && y->c != 32) return 0;
  if ((y->ld % 8) || !al16t(y->ptr)) return 0;
  if (x->d != y->d || x->h != y->h || x->w != y->w) return 0;
  if ((long long)x->d * x->h * x->w >= (1ll << 31)) return 0;
  return 1;
}

template <typename TX, typename TW, typename TY, int CO>
static int stem_conv_co(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                        const b200seg_tensor* y, double* stats, int device, cudaStream_t st) {
  // voxels per thread along w: 2 shares the input window between neighbours but needs the registers (it spills
  // under the 2-CTA/SM bound for the 27-tap case)
  int vpt = (kind == B200SEG_K1 || dims == 2) ? 2 : 1;
  if (x->w & 1) vpt = 1;
  const long long items = (long long)x->d * x->h * (x->w / vpt);
  long long blocks = (items + 255) / 256;
  const long long cap = ((long long)num_sms(device) * 2 + x->n - 1) / x->n;     // 2 resident CTAs per SM
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks, x->n);
#define STEM_LAUNCH(KD_, KHW_)                                                                                     \
  do {                                                                                                             \
    if (vpt == 2)                                                                                                  \
      launch_k(conv_stem1_kernel<TX, TW, TY, CO, KD_, KHW_, 2>, grid, 256, 0, st, \
          static_cast<const TX*>(x->ptr), x->ld, static_cast<const TW*>(w), bias, static_cast<TY*>(y->ptr), y->ld, \
          stats, x->d, x->h, x->w);                                                                                \
    else                                                                                                           \
      launch_k(conv_stem1_kernel<TX, TW, TY, CO, KD_, KHW_, 1>, grid, 256, 0, st, \
          static_cast<const TX*>(x->ptr), x->ld, static_cast<const TW*>(w), bias, static_cast<TY*>(y->ptr), y->ld, \
          stats, x->d, x->h, x->w);                                                                                \
  } while (0)
  if (kind == B200SEG_K1) STEM_LAUNCH(1, 1);
  else if (dims == 3) STEM_LAUNCH(3, 3);
  else STEM_LAUNCH(1, 3);
#undef STEM_LAUNCH
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

template <typename TX, typename TW, typename TY>
static int stem_conv_typed(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                           const b200seg_tensor* y, double* stats, int device, cudaStream_t st) {
  if (y->c == 16) return stem_conv_co<TX, TW, TY, 16>(kind, dims, x, w, bias, y, stats, device, st);
  return stem_conv_co<TX, TW, TY, 32>(kind, dims, x, w, bias, y, stats, device, st);
}

int stem_conv(int kind, int dims, const b200seg_tensor* x, const void* w, int w_dtype, const float* bias,
              const b200seg_tensor* y, double* stats, int device, cudaStream_t st) {
  const int xd = x->dtype, yd = y->dtype;
  if (w_dtype == B200SEG_F32) {
    B200_CHECK_ARG(xd == B200SEG_F32 && yd == B200SEG_F32, "stem_conv: fp32 weights need fp32 tensors");
    return stem_conv_typed<float, float, float>(kind, dims, x, w, bias, y, stats, device, st);
  }
  B200_CHECK_ARG(yd == B200SEG_BF16, "stem_conv: bf16 weights need a bf16 output");
  if (xd == B200SEG_F32) return stem_conv_typed<float, bf16, bf16>(kind, dims, x, w, bias, y, stats, device, st);
  return stem_conv_typed<bf16, bf16, bf16>(kind, dims, x, w, bias, y, stats, device, st);
}

int stem_wgrad_supported(int kind, const b200seg_tensor* a, const b200seg_tensor* b) {
  if (kind != B200SEG_K3 && kind != B200SEG_K1) return 0;
  if (a->c != 1) return 0;
  if (b->c != 16 && b->c != 32) return 0;
  if ((b->ld % 8) || !al16t(b->ptr)) return 0;
  if (a->d != b->d || a->h != b->h || a->w != b->w) return 0;
  return 1;
}

template <typename TA, typename TB, int CO>
static int stem_wgrad_co(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                         cudaStream_t st) {
  const long long NV = (long long)b->n * b->d * b->h * b->w;
  const int sms = num_sms(device);
#define STEM_WG(KD_, KHW_, CG_)                                                                                    \
  do {                                                                                                             \
    constexpr int nvar = KD_ * (CO / CG_);                                                                         \
    long long nch = ((long long)sms * 2 + nvar - 1) / nvar;                                                        \
    const long long need = (NV + 255) / 256;                                                                       \
    if (nch > need) nch = need;                                                                                    \
    if (nch < 1) nch = 1;                                                                                          \
    launch_k(wgrad_stem1_kernel<TA, TB, CO, KD_, KHW_, CG_>, (unsigned)(nch * nvar), 256, 0, st, \
        static_cast<const TA*>(a->ptr), a->ld, static_cast<const TB*>(b->ptr), b->ld, dwp, b->n, b->d, b->h,       \
        b->w);                                                                                                     \
  } while (0)
  if (kind == B200SEG_K1) STEM_WG(1, 1, 16);
  else if (dims == 3) STEM_WG(3, 3, 8);
  else STEM_WG(1, 3, 8);
#undef STEM_WG
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

template <typename TA, typename TB>
static int stem_wgrad_typed(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp,
                            int device, cudaStream_t st) {
  if (b->c == 16) return stem_wgrad_co<TA, TB, 16>(kind, dims, a, b, dwp, device, st);
  return stem_wgrad_co<TA, TB, 32>(kind, dims, a, b, dwp, device, st);
}

int stem_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
               cudaStream_t st) {
  if (a->dtype == B200SEG_F32 && b->dtype == B200SEG_F32) return stem_wgrad_typed<float, float>(kind, dims, a, b, dwp, device, st);
  if (a->dtype == B200SEG_F32 && b->dtype == B200SEG_BF16) return stem_wgrad_typed<float, bf16>(kind, dims, a, b, dwp, device, st);
  if (a->dtype == B200SEG_BF16 && b->dtype == B200SEG_BF16) return stem_wgrad_typed<bf16, bf16>(kind, dims, a, b, dwp, device, st);
  return stem_wgrad_typed<bf16, float>(kind, dims, a, b, dwp, device, st);
}

}  // namespace b200seg
