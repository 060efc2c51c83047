// The reference's 3-D augmentation warp on the device (sm_90a): ImageDataGenerator3D.random_transform followed by
// standardize (dataprocess/Augmentation/images_masks_3dtransform.py), i.e. scipy.ndimage.affine_transform(order=0)
// of every image channel and of the label with one matrix per sample, then the channel shift, the flips and
// "x *= rescale".  Order 0 copies input values, so the result is scipy's bit for bit once the source index is:
//   cc = off[a]; cc += m[a][0] i0; cc += m[a][1] i1; cc += m[a][2] i2  (fp64, every operation rounded on its own:
//   __dmul_rn / __dadd_rn keep nvcc from contracting them into FMAs, which moves the index on ties), then the fill
//   mode's map of cc (scipy's map_coordinate, fp64 as well), k = floor(cc + 0.5) and the fold of an index one past
//   the edge.
// One launch warps a whole batch: grid (blocks per sample, N), each thread walks the sample's output voxels with a
// grid stride, un-flips the output index, computes the three coordinates, gathers the C image values and the label
// and writes both.  The channel shift needs the min and max of the warped sample first: a statistics launch computes
// the same gather and writes per-block min / max partials into the workspace, and each block of the main launch
// folds them.  No allocation, no host synchronisation, no atomics; min and max do not depend on order, so reruns are
// bit-identical.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxStatBlocks = 256;       // partial (min, max) pairs per sample, one per statistics block
constexpr int kMaxMainBlocks = 1024;      // blocks per sample of the warp launch

__host__ __device__ inline int stat_blocks(long long vox) {
  const long long b = (vox + 16LL * kThreads - 1) / (16LL * kThreads);
  return (int)(b < 1 ? 1 : (b > kMaxStatBlocks ? kMaxStatBlocks : b));
}

// scipy's map_coordinate for one input axis of length n, then the index and its fold; false: outside ('constant')
__device__ __forceinline__ bool map_axis(double cc, int n, int mode, int& k) {
  const double len = (double)n;
  const double last = (double)(n - 1);
  if (cc < 0.0 || cc > last) {
    if (mode == B200SEG_AUG_CONSTANT) return false;
    if (mode == B200SEG_AUG_NEAREST) {
      cc = cc < 0.0 ? 0.0 : last;
    } else if (n <= 1) {
      cc = 0.0;
    } else if (mode == B200SEG_AUG_REFLECT) {
      const double s2 = 2.0 * len;
      if (cc < 0.0) {
        if (cc < -s2) cc = __dadd_rn(__dmul_rn(s2, trunc(__ddiv_rn(-cc, s2))), cc);
        cc = cc < -len ? __dadd_rn(cc, s2) : __dsub_rn(cc > -1e-15 ? 1e-15 : -cc, 1.0);
      } else {
        cc = __dsub_rn(cc, __dmul_rn(s2, trunc(__ddiv_rn(cc, s2))));
        if (cc >= len) cc = __dsub_rn(__dsub_rn(s2, cc), 1.0);
      }
    } else if (mode == B200SEG_AUG_MIRROR) {
      const double s2 = 2.0 * len - 2.0;
      if (cc < 0.0) {
        cc = __dadd_rn(__dmul_rn(s2, trunc(__ddiv_rn(-cc, s2))), cc);
        cc = cc <= 1.0 - len ? __dadd_rn(cc, s2) : -cc;
      } else {
        cc = __dsub_rn(cc, __dmul_rn(s2, trunc(__ddiv_rn(cc, s2))));
        if (cc >= len) cc = __dsub_rn(s2, cc);
      }
    } else {  // B200SEG_AUG_WRAP: the old period n - 1
      if (cc < 0.0) cc = __dadd_rn(cc, __dmul_rn(last, __dadd_rn(trunc(__ddiv_rn(-cc, last)), 1.0)));
      else cc = __dsub_rn(cc, __dmul_rn(last, trunc(__ddiv_rn(cc, last))));
    }
  }
  int i = (int)floor(__dadd_rn(cc, 0.5));
  if (i < 0 || i >= n) {      // one past the edge: REFLECT repeats the edge voxel, MIRROR reflects about it
    const int e = mode == B200SEG_AUG_REFLECT ? 1 : 0;
    i = n <= 1 ? 0 : (i < 0 ? -e - i : 2 * n - 2 + e - i);
  }
  k = min(max(i, 0), n - 1);  // never outside the sample, whatever the matrix holds
  return true;
}

struct Geom {
  int D, H, W;
  long long vox;
};

// output voxel v of a sample -> source voxel index, or -1 for the fill value
__device__ __forceinline__ long long source_voxel(const b200seg_aug3d_param& p, const Geom& g, long long v, int mode) {
  int w = (int)(v % g.W);
  const long long t = v / g.W;
  int h = (int)(t % g.H);
  int d = (int)(t / g.H);
  if (p.flip & 1) d = g.D - 1 - d;
  if (p.flip & 2) h = g.H - 1 - h;
  if (p.flip & 4) w = g.W - 1 - w;
  const double i0 = (double)d, i1 = (double)h, i2 = (double)w;
  const int len[3] = {g.D, g.H, g.W};
  int k[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double cc = p.off[a];
    cc = __dadd_rn(cc, __dmul_rn(p.m[3 * a + 0], i0));
    cc = __dadd_rn(cc, __dmul_rn(p.m[3 * a + 1], i1));
    cc = __dadd_rn(cc, __dmul_rn(p.m[3 * a + 2], i2));
    if (!map_axis(cc, len[a], mode, k[a])) return -1;
  }
  return ((long long)k[0] * g.H + k[1]) * g.W + k[2];
}

// numpy's NaN-propagating min / max (np.min, np.max) and clip (max(x, lo) then min(., hi), NaN in x kept)
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a) ? a : ((b != b) ? b : (b < a ? b : a)); }
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a) ? a : ((b != b) ? b : (b > a ? b : a)); }
__device__ __forceinline__ float np_clip(float x, float lo, float hi) {
  const float t = (x != x) ? x : (x > lo ? x : lo);
  return (t != t) ? t : (t < hi ? t : hi);
}

__device__ __forceinline__ void block_minmax(float& lo, float& hi) {
  __shared__ float s_lo[kThreads / 32], s_hi[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    s_lo[wid] = lo;
    s_hi[wid] = hi;
  }
  __syncthreads();
  lo = s_lo[0];
  hi = s_hi[0];
#pragma unroll
  for (int i = 1; i < kThreads / 32; ++i) {
    lo = nan_min(lo, s_lo[i]);
    hi = nan_max(hi, s_hi[i]);
  }
}

// per-block (min, max) of the warped image over every channel: ws[(s * nb + b) * 2 + {0, 1}]
template <int C>
__global__ void __launch_bounds__(kThreads)
augment3d_stats_kernel(const float* __restrict__ x, const b200seg_aug3d_param* __restrict__ params, Geom g, int mode,
                       float fill, float* __restrict__ ws) {
  PDL_ENTER();
  const int s = blockIdx.y;
  const b200seg_aug3d_param p = params[s];
  const float* xs = x + (long long)s * g.vox * C;
  float lo = __int_as_float(0x7f800000), hi = -__int_as_float(0x7f800000);
  for (long long v = (long long)blockIdx.x * kThreads + threadIdx.x; v < g.vox; v += (long long)gridDim.x * kThreads) {
    const long long src = source_voxel(p, g, v, mode);
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float val = src < 0 ? fill : __ldg(xs + src * C + c);
      lo = nan_min(lo, val);
      hi = nan_max(hi, val);
    }
  }
  block_minmax(lo, hi);
  if (threadIdx.x == 0) {
    float* o = ws + ((long long)s * gridDim.x + blockIdx.x) * 2;
    o[0] = lo;
    o[1] = hi;
  }
}

struct LabelArgs {
  const void* y;
  void* y_out;
  int out_kind;       // 0: y's own dtype, 1: int64, 2: int64 (y != 0)
};

template <int C, bool LABEL_U8>
__global__ void __launch_bounds__(kThreads)
augment3d_kernel(const float* __restrict__ x, const b200seg_aug3d_param* __restrict__ params, Geom g, int mode,
                 double cval, int shift, int nstat, double rescale, int rescale_mode, bool vec,
                 float* __restrict__ x_out, LabelArgs lab, const float* __restrict__ ws) {
  PDL_ENTER();
  const int s = blockIdx.y;
  const b200seg_aug3d_param p = params[s];
  float lo = 0.0f, hi = 0.0f;
  if (shift) {
    lo = __int_as_float(0x7f800000);
    hi = -lo;
    for (int i = threadIdx.x; i < nstat; i += kThreads) {
      lo = nan_min(lo, ws[((long long)s * nstat + i) * 2]);
      hi = nan_max(hi, ws[((long long)s * nstat + i) * 2 + 1]);
    }
    block_minmax(lo, hi);
  }
  const float fill = __double2float_rn(cval);
  const float rs32 = __double2float_rn(rescale);
  float lfill;
  if (LABEL_U8) {
    double t = cval > 0.0 ? __dadd_rn(cval, 0.5) : 0.0;
    t = t > 255.0 ? 255.0 : t;
    lfill = (float)(int)t;
  } else {
    lfill = fill;
  }
  const long long base = (long long)s * g.vox;
  const float* xs = x + base * C;
  float* xo = x_out + base * C;
  for (long long v = (long long)blockIdx.x * kThreads + threadIdx.x; v < g.vox; v += (long long)gridDim.x * kThreads) {
    const long long src = source_voxel(p, g, v, mode);
    float val[C];
    if (C == 4 && vec && src >= 0) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(xs) + src);
      val[0] = q.x;
      val[1 % C] = q.y;
      val[2 % C] = q.z;
      val[3 % C] = q.w;
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) val[c] = src < 0 ? fill : __ldg(xs + src * C + c);
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float t = val[c];
      if (shift) t = np_clip(__fadd_rn(t, p.shift[c]), lo, hi);
      if (rescale_mode == B200SEG_RESCALE_F32) t = __fmul_rn(t, rs32);
      else if (rescale_mode == B200SEG_RESCALE_F64) t = __double2float_rn(__dmul_rn((double)t, rescale));
      val[c] = t;
    }
    if (C == 4 && vec) {
      reinterpret_cast<float4*>(xo)[v] = make_float4(val[0], val[1 % C], val[2 % C], val[3 % C]);
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) xo[v * C + c] = val[c];
    }
    // the label: same gather, scipy's cval cast outside
    float lv;
    uint8_t lb = 0;
    if (LABEL_U8) {
      lb = src < 0 ? (uint8_t)lfill : __ldg(static_cast<const uint8_t*>(lab.y) + base + src);
      lv = (float)lb;
    } else {
      lv = src < 0 ? lfill : __ldg(static_cast<const float*>(lab.y) + base + src);
    }
    if (lab.out_kind == 0) {
      if (LABEL_U8) static_cast<uint8_t*>(lab.y_out)[base + v] = lb;
      else static_cast<float*>(lab.y_out)[base + v] = lv;
    } else {
      const long long li = lab.out_kind == 2 ? (long long)(lv != 0.0f) : (LABEL_U8 ? (long long)lb : __float2ll_rz(lv));
      static_cast<long long*>(lab.y_out)[base + v] = li;
    }
  }
}

template <int C>
int launch_augment3d(const float* x, const void* y, bool label_u8, int n, Geom g, const b200seg_aug3d_param* params,
                     int mode, double cval, int shift, double rescale, int rescale_mode, float* x_out, void* y_out,
                     int out_kind, float* ws, cudaStream_t st) {
  const int nstat = stat_blocks(g.vox);
  if (shift) {
    launch_k(augment3d_stats_kernel<C>, dim3(nstat, n), kThreads, 0, st, x, params, g, mode, (float)cval, ws);
    B200_LAUNCH_CHECK();
  }
  const long long want = (g.vox + kThreads - 1) / kThreads;
  const dim3 grid((unsigned)(want < kMaxMainBlocks ? want : kMaxMainBlocks), n);
  const LabelArgs lab{y, y_out, out_kind};
  // 16-byte loads and stores of the four channels when both buffers allow them
  const bool vec = reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(x_out) % 16 == 0;
  if (label_u8)
    launch_k(augment3d_kernel<C, true>, grid, kThreads, 0, st, x, params, g, mode, cval, shift, nstat, rescale,
             rescale_mode, vec, x_out, lab, (const float*)ws);
  else
    launch_k(augment3d_kernel<C, false>, grid, kThreads, 0, st, x, params, g, mode, cval, shift, nstat, rescale,
             rescale_mode, vec, x_out, lab, (const float*)ws);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace

long long augment3d_workspace(int n, long long vox) { return (long long)n * stat_blocks(vox) * 2 * sizeof(float); }

int augment3d(const float* x, const void* y, int y_dtype, int n, int D, int H, int W, int C,
              const b200seg_aug3d_param* params, int mode, double cval, int shift, double rescale, int rescale_mode,
              float* x_out, void* y_out, int label_out, int binarize, void* ws, cudaStream_t st) {
  const Geom g{D, H, W, (long long)D * H * W};
  const bool u8 = y_dtype == B200SEG_U8;
  const int out_kind = binarize ? 2 : (label_out == B200SEG_I64 ? 1 : 0);
  float* w = static_cast<float*>(ws);
  switch (C) {
    case 1: return launch_augment3d<1>(x, y, u8, n, g, params, mode, cval, shift, rescale, rescale_mode, x_out, y_out,
                                       out_kind, w, st);
    case 3: return launch_augment3d<3>(x, y, u8, n, g, params, mode, cval, shift, rescale, rescale_mode, x_out, y_out,
                                       out_kind, w, st);
    default: return launch_augment3d<4>(x, y, u8, n, g, params, mode, cval, shift, rescale, rescale_mode, x_out,
                                        y_out, out_kind, w, st);
  }
}

}  // namespace b200seg
