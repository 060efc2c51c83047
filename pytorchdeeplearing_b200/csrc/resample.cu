// Whole-volume 3-D inference around the network (sm_90a): what XModel.inference / inference_patch
// (model/modelVNet.py:678-698, model/modelUnet.py:684-763) do on the host with SimpleITK and numpy, done on the device.
//   resample_linear   ResampleImageFilter with an identity transform and a linear interpolator
//                     (dataprocess/utils.py:99-145).  Output index i maps to the continuous input index u = i * r
//                     (r per axis, fp64, from the host).  A sample is taken only where -0.5 <= u < S - 0.5 on every
//                     axis (ITK's inside-buffer rule), else 0.  Trilinear: base = max(floor(u), 0), d = u - base
//                     (no interpolation along an axis where d <= 0), upper neighbour clamped to S - 1, lerps
//                     a + (b - a) * d along W, then H, then D, every operation rounded in fp64.  The result takes
//                     the input's pixel type (integers: clamped to the type's range and truncated toward zero), then
//                     fp32.  Optional fused steps: the truncation of ConvertitkTrunctedValue (utils.py:148-179), the
//                     per-block fp64 sums {sum x, sum x^2} of the meanstd statistics, or the order-preserving fp32
//                     keys of the percentile sort.
//   normalize         MEANSTD: sitk.NormalizeImageFilter: z = (x - mean) / sigma, sigma the N - 1 sample deviation
//                     from (sum x^2 - (sum x)^2 / N) / (N - 1).  PCTL: normalize() (utils.py:182-204): numpy's linear
//                     5th / 95th percentile from a stable radix sort (exact order statistics), the clip, mean and
//                     population std of the nonzero clipped voxels (two passes), and the reference's early return
//                     (either std == 0, tested as "all values equal") as a device-side flag read by the apply pass.
//   resample_nearest  the uint8 mask back to the original grid: index = floor(u + 0.5) (RoundHalfIntegerUp), the same
//                     inside-buffer rule, and the crop / zero pad of inference_patch (modelUnet.py:752-757) fused in.
// Every reduction has a fixed order (reruns are bit-identical); nothing is allocated or synchronised, so the chain can
// be captured in a CUDA graph.
#include <type_traits>

#include "common.cuh"

namespace b200seg {

int radix_sort_pairs(const uint32_t* kin, const int32_t* vin, uint32_t* kout, int32_t* vout, int nseg, long long len,
                     void* ws, long long ws_bytes, cudaStream_t s);
int64_t radix_sort_workspace(int nseg, long long len);

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 1024;
constexpr int kPart = 4;          // fp64 values per block partial
constexpr int kStats = 8;         // fp64 values of the stats block

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
inline int nblocks(long long nvox) {
  const long long b = (nvox + kThreads - 1) / kThreads;
  return (int)(b < 1 ? 1 : (b > kMaxBlocks ? kMaxBlocks : b));
}

struct Layout {
  size_t stats, part, kin, kout, vout, sort, total;
};
Layout layout(int mode, long long nvox) {
  Layout L{};
  size_t o = 0;
  L.stats = o; o += align256(kStats * 8);
  L.part = o; o += align256((size_t)nblocks(nvox) * kPart * 8);
  if (mode == B200SEG_NORM_PCTL) {
    L.kin = o; o += align256((size_t)nvox * 4);
    L.kout = o; o += align256((size_t)nvox * 4);
    L.vout = o; o += align256((size_t)nvox * 4);
    L.sort = o; o += align256((size_t)radix_sort_workspace(1, nvox));
  }
  L.total = o;
  return L;
}

// fixed-order block reduction of one fp64 value (256 threads)
__device__ __forceinline__ double block_sum(double v, double* s_tmp) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_tmp[wid] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) t += s_tmp[w];
  __syncthreads();
  return t;
}
__device__ __forceinline__ double block_min(double v, double* s_tmp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_tmp[wid] = v;
  __syncthreads();
  double t = s_tmp[0];
#pragma unroll
  for (int w = 1; w < kThreads / 32; ++w) t = fmin(t, s_tmp[w]);
  __syncthreads();
  return t;
}

template <typename T> struct PixelRange;
template <> struct PixelRange<uint8_t> { static constexpr double lo = 0.0, hi = 255.0; };
template <> struct PixelRange<int16_t> { static constexpr double lo = -32768.0, hi = 32767.0; };
template <> struct PixelRange<int32_t> { static constexpr double lo = -2147483648.0, hi = 2147483647.0; };

// fp64 interpolated value -> the input's pixel type -> fp32
template <typename T>
__device__ __forceinline__ float cast_pixel(double v) {
  if constexpr (std::is_floating_point<T>::value) {
    return (float)v;
  } else {
    v = fmin(fmax(v, PixelRange<T>::lo), PixelRange<T>::hi);
    return (float)(T)v;                                   // truncation toward zero
  }
}

__device__ __forceinline__ double lerp_rn(double a, double b, double d) {
  return __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), d));
}

__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t b = __float_as_uint(f == 0.0f ? 0.0f : f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// one axis of the linear sample: base index, upper index, distance (0 where ITK does not interpolate); false outside
__device__ __forceinline__ bool axis_linear(long long i, double r, int S, int& i0, int& i1, double& d) {
  const double u = __dmul_rn((double)i, r);
  if (!(u >= -0.5 && u < (double)S - 0.5)) return false;
  const double fl = floor(u);
  i0 = fl < 0.0 ? 0 : (int)fl;
  d = __dsub_rn(u, (double)i0);
  if (d < 0.0) d = 0.0;
  i1 = i0 + 1 < S ? i0 + 1 : S - 1;
  return true;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
resample_linear_kernel(const T* __restrict__ src, int D, int H, int W, double rz, double ry, double rx, int oD, int oH,
                       int oW, int mode, float lower, float upper, float* __restrict__ out,
                       double* __restrict__ part, uint32_t* __restrict__ keys) {
  PDL_ENTER();
  __shared__ double s_tmp[kThreads / 32];
  const long long nvox = (long long)oD * oH * oW;
  const long long plane = (long long)H * W;
  double s1 = 0.0, s2 = 0.0;
  for (long long o = (long long)blockIdx.x * kThreads + threadIdx.x; o < nvox; o += (long long)gridDim.x * kThreads) {
    const long long z = o / ((long long)oH * oW);
    const long long rem = o - z * oH * oW;
    const long long y = rem / oW, x = rem - y * oW;
    int z0, z1, y0, y1, x0, x1;
    double dz, dy, dx;
    double v = 0.0;
    if (axis_linear(z, rz, D, z0, z1, dz) && axis_linear(y, ry, H, y0, y1, dy) && axis_linear(x, rx, W, x0, x1, dx)) {
      const T* p00 = src + z0 * plane + (long long)y0 * W;
      const T* p01 = src + z0 * plane + (long long)y1 * W;
      const T* p10 = src + z1 * plane + (long long)y0 * W;
      const T* p11 = src + z1 * plane + (long long)y1 * W;
      const double c00 = lerp_rn((double)__ldg(p00 + x0), (double)__ldg(p00 + x1), dx);
      const double c01 = lerp_rn((double)__ldg(p01 + x0), (double)__ldg(p01 + x1), dx);
      const double c10 = lerp_rn((double)__ldg(p10 + x0), (double)__ldg(p10 + x1), dx);
      const double c11 = lerp_rn((double)__ldg(p11 + x0), (double)__ldg(p11 + x1), dx);
      v = lerp_rn(lerp_rn(c00, c01, dy), lerp_rn(c10, c11, dy), dz);
    }
    float f = cast_pixel<T>(v);
    if (mode == B200SEG_NORM_MEANSTD) {
      if (f > upper) f = upper;                             // ConvertitkTrunctedValue's order: upper, then lower
      if (f < lower) f = lower;
      const double fd = (double)f;
      s1 = __dadd_rn(s1, fd);
      s2 = __dadd_rn(s2, __dmul_rn(fd, fd));
    } else if (mode == B200SEG_NORM_PCTL) {
      keys[o] = order_key(f);
    }
    out[o] = f;
  }
  if (mode == B200SEG_NORM_MEANSTD) {
    s1 = block_sum(s1, s_tmp);
    s2 = block_sum(s2, s_tmp);
    if (threadIdx.x == 0) {
      part[blockIdx.x * kPart + 0] = s1;
      part[blockIdx.x * kPart + 1] = s2;
    }
  }
}

// stats[0] = mean, stats[1] = sigma (N - 1), stats[5] = N
__global__ void __launch_bounds__(kThreads) meanstd_finalize_kernel(const double* __restrict__ part, int nblk,
                                                                    long long nvox, double* __restrict__ stats) {
  PDL_ENTER();
  __shared__ double s_tmp[kThreads / 32];
  double s1 = 0.0, s2 = 0.0;
  for (int b = threadIdx.x; b < nblk; b += kThreads) {
    s1 += part[b * kPart + 0];
    s2 += part[b * kPart + 1];
  }
  s1 = block_sum(s1, s_tmp);
  s2 = block_sum(s2, s_tmp);
  if (threadIdx.x == 0) {
    const double n = (double)nvox;
    const double mean = s1 / n;
    const double var = (s2 - s1 * s1 / n) / (n - 1.0);
    stats[0] = mean;
    stats[1] = sqrt(var);
    stats[2] = 0.0;
    stats[3] = 0.0;
    stats[4] = 0.0;
    stats[5] = n;
  }
}

__global__ void __launch_bounds__(kThreads) meanstd_apply_kernel(const float* __restrict__ x, long long nvox,
                                                                 const double* __restrict__ stats,
                                                                 float* __restrict__ out) {
  PDL_ENTER();
  const double mean = stats[0], sd = stats[1];
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nvox; i += (long long)gridDim.x * kThreads)
    out[i] = (float)(__dsub_rn((double)x[i], mean) / sd);
}

// numpy.percentile(a, q), method 'linear': vi = (n - 1) * (q / 100), lerp of the two order statistics around vi as
// numpy's _lerp (a + (b - a) * g, or b - (b - a) * (1 - g) for g >= 0.5)
__device__ double percentile_linear(const uint32_t* sorted, long long n, double q) {
  const double vi = __dmul_rn((double)(n - 1), q / 100.0);
  if (vi >= (double)(n - 1)) return (double)key_value(sorted[n - 1]);
  const double prev = floor(vi);
  const long long i = (long long)prev;
  const double g = __dsub_rn(vi, prev);
  const double a = (double)key_value(sorted[i]), b = (double)key_value(sorted[i + 1]);
  const double diff = __dsub_rn(b, a);
  if (g >= 0.5) return __dsub_rn(b, __dmul_rn(diff, __dsub_rn(1.0, g)));
  return __dadd_rn(a, __dmul_rn(diff, g));
}

// stats[2] = 5th percentile t, stats[3] = 95th percentile b (normalize(slice, bottom=95, down=5))
__global__ void pctl_select_kernel(const uint32_t* __restrict__ sorted, long long n, double* __restrict__ stats) {
  PDL_ENTER();
  if (threadIdx.x == 0) {
    stats[2] = percentile_linear(sorted, n, 5.0);
    stats[3] = percentile_linear(sorted, n, 95.0);
  }
}

__device__ __forceinline__ double clip_tb(float x, double t, double b) { return fmin(fmax((double)x, t), b); }

// pass 1 over the clipped volume: per block {sum of nonzero, nonzero count, min nonzero, -max nonzero};
// pass 2 (stats[0] holds the mean): per block {sum (c - mean)^2 over nonzero}
__global__ void __launch_bounds__(kThreads) pctl_sums_kernel(const float* __restrict__ x, long long nvox, int pass,
                                                             const double* __restrict__ stats,
                                                             double* __restrict__ part) {
  PDL_ENTER();
  __shared__ double s_tmp[kThreads / 32];
  const double t = stats[2], b = stats[3], mean = stats[0];
  double s = 0.0, cnt = 0.0, mn = INFINITY, nmx = INFINITY;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nvox; i += (long long)gridDim.x * kThreads) {
    const double c = clip_tb(x[i], t, b);
    if (c != 0.0) {
      if (pass == 0) {
        s = __dadd_rn(s, c);
        cnt += 1.0;
        mn = fmin(mn, c);
        nmx = fmin(nmx, -c);
      } else {
        const double dv = __dsub_rn(c, mean);
        s = __dadd_rn(s, __dmul_rn(dv, dv));
      }
    }
  }
  s = block_sum(s, s_tmp);
  if (pass == 0) {
    cnt = block_sum(cnt, s_tmp);
    mn = block_min(mn, s_tmp);
    nmx = block_min(nmx, s_tmp);
  }
  if (threadIdx.x == 0) {
    part[blockIdx.x * kPart + 0] = s;
    if (pass == 0) {
      part[blockIdx.x * kPart + 1] = cnt;
      part[blockIdx.x * kPart + 2] = mn;
      part[blockIdx.x * kPart + 3] = nmx;
    }
  }
}

// pass 0: stats[0] = mean of the nonzero clipped voxels, stats[4] = 1 where normalize() returns the clipped volume
// unchanged (t == b: the clipped volume is constant; or all nonzero clipped values are equal), stats[5] = count;
// pass 1: stats[1] = population std of the nonzero clipped voxels
__global__ void __launch_bounds__(kThreads) pctl_finalize_kernel(const double* __restrict__ part, int nblk, int pass,
                                                                 double* __restrict__ stats) {
  PDL_ENTER();
  __shared__ double s_tmp[kThreads / 32];
  double s = 0.0, cnt = 0.0, mn = INFINITY, nmx = INFINITY;
  for (int k = threadIdx.x; k < nblk; k += kThreads) {
    s += part[k * kPart + 0];
    if (pass == 0) {
      cnt += part[k * kPart + 1];
      mn = fmin(mn, part[k * kPart + 2]);
      nmx = fmin(nmx, part[k * kPart + 3]);
    }
  }
  s = block_sum(s, s_tmp);
  if (pass == 0) {
    cnt = block_sum(cnt, s_tmp);
    mn = block_min(mn, s_tmp);
    nmx = block_min(nmx, s_tmp);
  }
  if (threadIdx.x == 0) {
    if (pass == 0) {
      stats[0] = s / cnt;
      stats[4] = (stats[2] == stats[3] || mn == -nmx) ? 1.0 : 0.0;
      stats[5] = cnt;
    } else {
      stats[1] = sqrt(s / stats[5]);
    }
  }
}

__global__ void __launch_bounds__(kThreads) pctl_apply_kernel(const float* __restrict__ x, long long nvox,
                                                              const double* __restrict__ stats,
                                                              float* __restrict__ out) {
  PDL_ENTER();
  const double t = stats[2], b = stats[3], mean = stats[0], sd = stats[1];
  const bool keep = stats[4] != 0.0;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < nvox; i += (long long)gridDim.x * kThreads) {
    const double c = clip_tb(x[i], t, b);
    out[i] = keep ? (float)c : (float)(__dsub_rn(c, mean) / sd);
  }
}

// NN sample index along one axis, -1 outside the buffer
__device__ __forceinline__ int axis_nearest(long long i, double r, int S) {
  const double u = __dmul_rn((double)i, r);
  if (!(u >= -0.5 && u < (double)S - 0.5)) return -1;
  const int k = (int)floor(__dadd_rn(u, 0.5));
  return k < S ? k : S - 1;
}

// out [oD][oH][oW]: the first (vD, vH, vW) corner is the NN resample of src, the rest is 0 (inference_patch's pad)
__global__ void __launch_bounds__(kThreads)
resample_nearest_kernel(const uint8_t* __restrict__ src, int D, int H, int W, double rz, double ry, double rx, int vD,
                        int vH, int vW, int oD, int oH, int oW, uint8_t* __restrict__ out) {
  PDL_ENTER();
  const long long nvox = (long long)oD * oH * oW;
  for (long long o = (long long)blockIdx.x * kThreads + threadIdx.x; o < nvox; o += (long long)gridDim.x * kThreads) {
    const long long z = o / ((long long)oH * oW);
    const long long rem = o - z * oH * oW;
    const long long y = rem / oW, x = rem - y * oW;
    uint8_t v = 0;
    if (z < vD && y < vH && x < vW) {
      const int kz = axis_nearest(z, rz, D), ky = axis_nearest(y, ry, H), kx = axis_nearest(x, rx, W);
      if (kz >= 0 && ky >= 0 && kx >= 0) v = __ldg(src + ((long long)kz * H + ky) * W + kx);
    }
    out[o] = v;
  }
}

int grid_for(long long nvox, int device) {
  long long b = (nvox + kThreads - 1) / kThreads;
  const long long cap = (long long)num_sms(device) * 8;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

int64_t resample_workspace(int mode, long long nvox) { return (int64_t)layout(mode, nvox).total; }

int resample_linear(const void* src, int dtype, int D, int H, int W, const double* ratio, int oD, int oH, int oW,
                    int mode, float lower, float upper, float* out, void* ws, long long ws_bytes, cudaStream_t st) {
  const long long nvox = (long long)oD * oH * oW;
  const Layout L = layout(mode, nvox);
  B200_CHECK_ARG(mode == B200SEG_NORM_NONE || (ws && ws_bytes >= (long long)L.total),
                 "b200seg_resample_linear: workspace too small");
  char* w = static_cast<char*>(ws);
  double* part = mode == B200SEG_NORM_MEANSTD ? reinterpret_cast<double*>(w + L.part) : nullptr;
  uint32_t* keys = mode == B200SEG_NORM_PCTL ? reinterpret_cast<uint32_t*>(w + L.kin) : nullptr;
  const int g = nblocks(nvox);      // fixed by the size alone: the partials' order does not depend on the device
  const double rz = ratio[0], ry = ratio[1], rx = ratio[2];
#define B200_RESAMPLE(T)                                                                                         \
  launch_k(resample_linear_kernel<T>, g, kThreads, 0, st, static_cast<const T*>(src), D, H, W, rz, ry, rx, oD, oH, \
           oW, mode, lower, upper, out, part, keys)
  switch (dtype) {
    case B200SEG_U8: B200_RESAMPLE(uint8_t); break;
    case B200SEG_I16: B200_RESAMPLE(int16_t); break;
    case B200SEG_I32: B200_RESAMPLE(int32_t); break;
    default: B200_RESAMPLE(float); break;
  }
#undef B200_RESAMPLE
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int normalize_volume(int mode, const float* x, long long nvox, void* ws, long long ws_bytes, float* out, int device,
                     cudaStream_t st) {
  const Layout L = layout(mode, nvox);
  B200_CHECK_ARG(ws && ws_bytes >= (long long)L.total, "b200seg_normalize: workspace too small");
  char* w = static_cast<char*>(ws);
  double* stats = reinterpret_cast<double*>(w + L.stats);
  double* part = reinterpret_cast<double*>(w + L.part);
  const int nblk = nblocks(nvox);
  const int ga = grid_for(nvox, device);
  if (mode == B200SEG_NORM_MEANSTD) {
    launch_k(meanstd_finalize_kernel, 1, kThreads, 0, st, (const double*)part, nblk, nvox, stats);
    launch_k(meanstd_apply_kernel, ga, kThreads, 0, st, x, nvox, (const double*)stats, out);
    B200_LAUNCH_CHECK();
    return B200SEG_OK;
  }
  const uint32_t* kin = reinterpret_cast<const uint32_t*>(w + L.kin);
  uint32_t* kout = reinterpret_cast<uint32_t*>(w + L.kout);
  int32_t* vout = reinterpret_cast<int32_t*>(w + L.vout);
  // the keys double as the (unused) values of the pair sort
  const int rc = radix_sort_pairs(kin, reinterpret_cast<const int32_t*>(kin), kout, vout, 1, nvox, w + L.sort,
                                  (long long)(L.total - L.sort), st);
  if (rc != B200SEG_OK) return rc;
  launch_k(pctl_select_kernel, 1, 32, 0, st, (const uint32_t*)kout, nvox, stats);
  for (int pass = 0; pass < 2; ++pass) {
    launch_k(pctl_sums_kernel, nblk, kThreads, 0, st, x, nvox, pass, (const double*)stats, part);
    launch_k(pctl_finalize_kernel, 1, kThreads, 0, st, (const double*)part, nblk, pass, stats);
  }
  launch_k(pctl_apply_kernel, ga, kThreads, 0, st, x, nvox, (const double*)stats, out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int resample_nearest_u8(const uint8_t* src, int D, int H, int W, const double* ratio, int vD, int vH, int vW, int oD,
                        int oH, int oW, uint8_t* out, int device, cudaStream_t st) {
  const long long nvox = (long long)oD * oH * oW;
  launch_k(resample_nearest_kernel, grid_for(nvox, device), kThreads, 0, st, src, D, H, W, ratio[0], ratio[1],
           ratio[2], vD, vH, vW, oD, oH, oW, out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
