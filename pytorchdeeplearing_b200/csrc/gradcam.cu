// Grad-CAM of the 2-D classifier (reference model/visualization.py:112-224, GradCAM): per target stage, the channel
// weights w[n][c] = mean over pixels of d(sum_i logit[i, t_i]) / dA, cam = relu(sum_c w[c] A[:, :, c]), a per-image
// min-max scale and an OpenCV-rule bilinear resize to the input size; then the mean over the stages and a second
// min-max scale.  A and its gradient are channels-last (N, 1, h, w, C), bf16 or fp32; the map is fp32 (N, H, W).
//
//   per stage  launch 1  cam_weights_kernel  fp64 partial sums of g over pixel chunks (fixed order, no atomics)
//              launch 2  cam_map_kernel      w from the partials (fp64), cam per pixel (one warp, fp64 channel sum),
//                                            clamp at 0, per-image min / max by atomics on the fp32 bits
//              launch 3  cam_resize_kernel   scale, resize, accumulate into the output; the last stage divides by the
//                                            number of stages and takes the min / max of the mean
//   finally    launch 4  cam_scale_kernel    the final min-max scale, in place
//   target     cam_target_kernel             the one-hot d loss / d logits (the arg-max of each row, or one class)
//
// Min and max are exact and independent of the order the atomics land in, and every sum has a fixed order, so reruns
// are bit-identical.  The values are >= 0 when the atomics run (clamped cam, scaled maps), so their fp32 bits order
// like the values.  No allocation, no host synchronisation.
#include "common.cuh"

namespace b200seg {

constexpr int kCamLanes = 32;        // channels per weight CTA
constexpr int kCamRows = 8;          // pixel lanes per weight CTA
constexpr int kCamChunk = 512;       // pixels per weight CTA
constexpr int kCamMaxSplit = 64;     // most pixel chunks per image
constexpr int kCamWarps = 8;         // pixels per map CTA (one warp each)
constexpr int kCamThreads = 256;     // resize / scale CTA

// workspace: [final min/max N x 2 u32][stage min/max N x 2 u32] | 256-byte aligned fp64 partials [N][S][C] | fp32 cam
inline int cam_splits(long long hw) {
  long long s = (hw + kCamChunk - 1) / kCamChunk;
  return (int)(s < kCamMaxSplit ? s : kCamMaxSplit);
}
inline long long align256(long long b) { return (b + 255) / 256 * 256; }
inline long long cam_part_offset(int n) { return align256(16LL * n); }
inline long long cam_map_offset(int n, long long hw, int c) {
  return cam_part_offset(n) + align256(8LL * n * cam_splits(hw) * c);
}

long long gradcam_workspace(int n, int h, int w, int c) {
  return cam_map_offset(n, (long long)h * w, c) + align256(4LL * n * h * w);
}

template <typename T>
__global__ void __launch_bounds__(kCamLanes * kCamRows) cam_weights_kernel(TV g, int splits, double* __restrict__ part,
                                                                           unsigned* __restrict__ mm, int reset_final) {
  PDL_ENTER();
  __shared__ double red[kCamRows][kCamLanes];
  const int n = blockIdx.z, s = blockIdx.y;
  const int c = blockIdx.x * kCamLanes + threadIdx.x;
  const long long hw = (long long)g.h * g.w;
  const long long per = (hw + splits - 1) / splits;
  const long long p0 = s * per, p1 = p0 + per < hw ? p0 + per : hw;
  if (blockIdx.x == 0 && s == 0 && threadIdx.y == 0 && threadIdx.x < 2) {
    // this stage's min / max (and, on the first stage, the mean's) start from +inf / 0 (all values are >= 0)
    const unsigned init = threadIdx.x == 0 ? 0x7f800000u : 0u;
    mm[2 * g.n + 2 * n + threadIdx.x] = init;
    if (reset_final) mm[2 * n + threadIdx.x] = init;
  }
  const T* base = static_cast<const T*>(g.p) + (long long)n * hw * g.ld;
  double acc = 0.0;
  if (c < g.c)
    for (long long p = p0 + threadIdx.y; p < p1; p += kCamRows) acc += (double)to_f(base[p * g.ld + c]);
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < g.c) {
    double t = red[0][threadIdx.x];
#pragma unroll
    for (int r = 1; r < kCamRows; ++r) t += red[r][threadIdx.x];
    part[((long long)n * splits + s) * g.c + c] = t;
  }
}

template <typename T>
__global__ void __launch_bounds__(kCamWarps * 32) cam_map_kernel(TV a, int splits, const double* __restrict__ part,
                                                                 float* __restrict__ cam, unsigned* __restrict__ mm) {
  PDL_ENTER();
  extern __shared__ double wsh[];                 // C channel weights
  __shared__ float bmin[kCamWarps], bmax[kCamWarps];
  const int n = blockIdx.y;
  const long long hw = (long long)a.h * a.w;
  const double inv = 1.0 / (double)hw;
  for (int c = threadIdx.x; c < a.c; c += blockDim.x) {
    const double* pp = part + (long long)n * splits * a.c + c;
    double t = 0.0;
    for (int s = 0; s < splits; ++s) t += pp[(long long)s * a.c];
    wsh[c] = t * inv;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long p = (long long)blockIdx.x * kCamWarps + warp;
  float v = 0.f;
  const bool live = p < hw;
  if (live) {
    const T* row = static_cast<const T*>(a.p) + ((long long)n * hw + p) * a.ld;
    double t = 0.0;
    for (int c = lane; c < a.c; c += 32) t = fma(wsh[c], (double)to_f(row[c]), t);
    t = warp_sum(t);
    v = fmaxf((float)t, 0.f);
    if (lane == 0) cam[(long long)n * hw + p] = v;
  }
  if (lane == 0) {
    bmin[warp] = live ? v : __int_as_float(0x7f800000);
    bmax[warp] = live ? v : 0.f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float lo = bmin[0], hi = bmax[0];
    for (int i = 1; i < kCamWarps; ++i) {
      lo = fminf(lo, bmin[i]);
      hi = fmaxf(hi, bmax[i]);
    }
    atomicMin(mm + 2 * a.n + 2 * n, __float_as_uint(lo));
    atomicMax(mm + 2 * a.n + 2 * n + 1, __float_as_uint(hi));
  }
}

// OpenCV's INTER_LINEAR source index and fp32 weight of the far tap for destination index d (resize.cpp, float path):
// fx = (float)((d + 0.5) * (1 / (D / S)) - 0.5), s = floor(fx), fx -= s, both clamped to the source at the borders
__device__ __forceinline__ int cv_coeff(int d, int D, int S, float* frac) {
  const double scale = 1.0 / __ddiv_rn((double)D, (double)S);
  float fx = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
  int s = (int)floorf(fx);
  fx = __fsub_rn(fx, (float)s);
  if (s < 0) {
    fx = 0.f;
    s = 0;
  }
  if (s >= S - 1) {
    fx = 0.f;
    s = S - 1;
  }
  *frac = fx;
  return s;
}

// the reference's scale_cam_image on one value: (v - min) / (1e-7 + (max - min)) in fp32
__device__ __forceinline__ float cam_norm(float v, float lo, float den) { return __fdiv_rn(__fsub_rn(v, lo), den); }

__global__ void __launch_bounds__(kCamThreads) cam_resize_kernel(const float* __restrict__ cam, int n_img, int h, int w,
                                                                 int H, int W, int layer, int nlayers,
                                                                 unsigned* __restrict__ mm, float* __restrict__ out) {
  PDL_ENTER();
  __shared__ float bmin[kCamThreads / 32], bmax[kCamThreads / 32];
  const int n = blockIdx.y;
  const long long HW = (long long)H * W;
  const long long q = (long long)blockIdx.x * kCamThreads + threadIdx.x;
  const bool live = q < HW;
  const float lo = __uint_as_float(mm[2 * n_img + 2 * n]);
  const float den = __fadd_rn(1e-7f, __fsub_rn(__uint_as_float(mm[2 * n_img + 2 * n + 1]), lo));
  const float* src = cam + (long long)n * h * w;
  float m = 0.f;
  if (live) {
    const int oy = (int)(q / W), ox = (int)(q % W);
    float v;
    if (h == H && w == W) {
      v = cam_norm(src[q], lo, den);                      // cv2.resize to the same size is a copy
    } else {
      float fy, fx;
      const int y0 = cv_coeff(oy, H, h, &fy), x0 = cv_coeff(ox, W, w, &fx);
      const int y1 = y0 + 1 < h ? y0 + 1 : h - 1, x1 = x0 + 1 < w ? x0 + 1 : w - 1;
      const float ax = __fsub_rn(1.f, fx), ay = __fsub_rn(1.f, fy);
      // horizontal pass on both source rows, then the vertical pass: each product rounded, then the sum
      const float r0 = __fadd_rn(__fmul_rn(cam_norm(src[y0 * w + x0], lo, den), ax),
                                 __fmul_rn(cam_norm(src[y0 * w + x1], lo, den), fx));
      const float r1 = __fadd_rn(__fmul_rn(cam_norm(src[y1 * w + x0], lo, den), ax),
                                 __fmul_rn(cam_norm(src[y1 * w + x1], lo, den), fx));
      v = __fadd_rn(__fmul_rn(r0, ay), __fmul_rn(r1, fy));
    }
    float* o = out + (long long)n * HW + q;
    m = layer == 0 ? v : __fadd_rn(*o, v);                // np.mean over the stages: sum in stage order, then divide
    if (layer == nlayers - 1) m = __fdiv_rn(m, (float)nlayers);
    *o = m;
  }
  if (layer != nlayers - 1) return;
  float lo2 = live ? m : __int_as_float(0x7f800000), hi2 = live ? m : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo2 = fminf(lo2, __shfl_xor_sync(0xffffffffu, lo2, o));
    hi2 = fmaxf(hi2, __shfl_xor_sync(0xffffffffu, hi2, o));
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    bmin[warp] = lo2;
    bmax[warp] = hi2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < kCamThreads / 32; ++i) {
      lo2 = fminf(lo2, bmin[i]);
      hi2 = fmaxf(hi2, bmax[i]);
    }
    atomicMin(mm + 2 * n, __float_as_uint(lo2));
    atomicMax(mm + 2 * n + 1, __float_as_uint(hi2));
  }
}

__global__ void __launch_bounds__(kCamThreads) cam_scale_kernel(float* __restrict__ out, long long HW,
                                                                const unsigned* __restrict__ mm) {
  PDL_ENTER();
  const int n = blockIdx.y;
  const long long q = (long long)blockIdx.x * kCamThreads + threadIdx.x;
  if (q >= HW) return;
  const float lo = __uint_as_float(mm[2 * n]);
  const float den = __fadd_rn(1e-7f, __fsub_rn(__uint_as_float(mm[2 * n + 1]), lo));
  float* o = out + (long long)n * HW + q;
  *o = cam_norm(*o, lo, den);
}

__global__ void __launch_bounds__(128) cam_target_kernel(const float* __restrict__ logits, int n, int k, int target,
                                                         float* __restrict__ dlogits, long long* __restrict__ category) {
  PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* row = logits + (long long)i * k;
  int t = target;
  if (t < 0) {                                           // arg-max, the first of equal maxima (torch / numpy)
    t = 0;
    for (int j = 1; j < k; ++j)
      if (row[j] > row[t]) t = j;
  }
  for (int j = 0; j < k; ++j) dlogits[(long long)i * k + j] = j == t ? 1.f : 0.f;
  category[i] = t;
}

int gradcam_target(const float* logits, int n, int k, int target, float* dlogits, long long* category,
                   cudaStream_t st) {
  launch_k(cam_target_kernel, dim3((n + 127) / 128), dim3(128), 0, st, logits, n, k, target, dlogits, category);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int gradcam_layer(const b200seg_tensor* act, const b200seg_tensor* grad, int H, int W, int layer, int nlayers,
                  void* ws, float* out, cudaStream_t st) {
  const int n = act->n, c = act->c;
  const long long hw = (long long)act->h * act->w;
  const int splits = cam_splits(hw);
  unsigned char* base = static_cast<unsigned char*>(ws);
  unsigned* mm = reinterpret_cast<unsigned*>(base);
  double* part = reinterpret_cast<double*>(base + cam_part_offset(n));
  float* cam = reinterpret_cast<float*>(base + cam_map_offset(n, hw, c));
  const bool bf = act->dtype == B200SEG_BF16;
  const dim3 gw((c + kCamLanes - 1) / kCamLanes, splits, n);
  if (grad->dtype == B200SEG_BF16)
    launch_k(cam_weights_kernel<bf16>, gw, dim3(kCamLanes, kCamRows), 0, st, tv(grad), splits, part, mm,
             layer == 0 ? 1 : 0);
  else
    launch_k(cam_weights_kernel<float>, gw, dim3(kCamLanes, kCamRows), 0, st, tv(grad), splits, part, mm,
             layer == 0 ? 1 : 0);
  B200_LAUNCH_CHECK();
  const dim3 gm((unsigned)((hw + kCamWarps - 1) / kCamWarps), n);
  const size_t smem = sizeof(double) * c;
  if (bf)
    launch_k(cam_map_kernel<bf16>, gm, dim3(kCamWarps * 32), smem, st, tv(act), splits, (const double*)part, cam, mm);
  else
    launch_k(cam_map_kernel<float>, gm, dim3(kCamWarps * 32), smem, st, tv(act), splits, (const double*)part, cam, mm);
  B200_LAUNCH_CHECK();
  const long long HW = (long long)H * W;
  launch_k(cam_resize_kernel, dim3((unsigned)((HW + kCamThreads - 1) / kCamThreads), n), dim3(kCamThreads), 0, st,
           (const float*)cam, n, act->h, act->w, H, W, layer, nlayers, mm, out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int gradcam_scale(float* out, int n, int H, int W, void* ws, cudaStream_t st) {
  const long long HW = (long long)H * W;
  launch_k(cam_scale_kernel, dim3((unsigned)((HW + kCamThreads - 1) / kCamThreads), n), dim3(kCamThreads), 0, st, out,
           HW, (const unsigned*)ws);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
