// The reference's 2-D augmentation (dataprocess/AugData.py, Segmenation_Aug: albumentations' HorizontalFlip,
// VerticalFlip, OneOf(MotionBlur, MedianBlur, Blur), ShiftScaleRotate, RandomBrightnessContrast) on the device, byte
// for byte OpenCV 4.13's uint8 kernels.  Every draw, the motion kernel, the inverse matrix and the 256-byte table are
// made on the host; a b200seg_aug2d_param entry per image carries them.  Two launches per batch:
//   blur_kernel  (only when some entry blurs): flips + blur of those entries into the workspace, at the entry's dst
//                offset.  MotionBlur is filter2D with reflect-101 over the nonzero taps in row-major order, fp32,
//                s = fma(v, w, s) for the row elements i = x * cn + ch < (w * cn) & ~3 (OpenCV's SIMD body and
//                4-unrolled loop) and s = s + v * w rounded separately for the last (w * cn) % 4 elements (its
//                scalar tail); cvRound to uint8.  MedianBlur 3x3 is the exact median with replicated borders, Blur 3x3
//                rint(sum / 9) with reflect-101.
//   warp_kernel  every entry: the flips (when the image was not blurred), warpAffine (when drawn) and the table.
//                warpAffine follows OpenCV's fixed-point remap: with M the inverse matrix (fp64),
//                adelta = rint(M0 x 1024), X0 = rint((M1 y + M2) 1024) + 16 (+ 512 for nearest), each fp64 product
//                and sum rounded on its own; X = (X0 + adelta) >> 5, sx = X >> 5, fx = X & 31 (likewise y); taps
//                reflected (101) one by one; weights (32 - fy)(32 - fx) 32 ... summing to 2^15,
//                v = (sum + 2^14) >> 15.  Nearest: sx = (X0 + adelta) >> 10.  The mask takes the flips and the
//                nearest warp only.
// One thread per pixel (every channel), grid (pixels / 256, n): no reductions, reruns are bit-identical.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ int reflect101(int p, int n) {
  if (n == 1) return 0;
  while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

// flipped-frame (y, x) -> source row-major pixel index
__device__ __forceinline__ long long flip_index(int y, int x, int h, int w, int flags) {
  if (flags & B200SEG_AUG2D_HFLIP) x = w - 1 - x;
  if (flags & B200SEG_AUG2D_VFLIP) y = h - 1 - y;
  return (long long)y * w + x;
}

__device__ __forceinline__ void cswap(int& a, int& b) {
  const int t = min(a, b);
  b = max(a, b);
  a = t;
}

// median of nine (the classic 19-exchange network)
__device__ __forceinline__ int median9(int* p) {
  cswap(p[1], p[2]); cswap(p[4], p[5]); cswap(p[7], p[8]);
  cswap(p[0], p[1]); cswap(p[3], p[4]); cswap(p[6], p[7]);
  cswap(p[1], p[2]); cswap(p[4], p[5]); cswap(p[7], p[8]);
  cswap(p[0], p[3]); cswap(p[5], p[8]); cswap(p[4], p[7]);
  cswap(p[3], p[6]); cswap(p[1], p[4]); cswap(p[2], p[5]);
  cswap(p[4], p[7]); cswap(p[4], p[2]); cswap(p[6], p[4]);
  cswap(p[4], p[2]);
  return p[4];
}

__global__ void __launch_bounds__(kThreads)
blur_kernel(const uint8_t* __restrict__ src, const b200seg_aug2d_param* __restrict__ params, uint8_t* __restrict__ ws) {
  PDL_ENTER();
  const b200seg_aug2d_param& e = params[blockIdx.y];
  const int flags = e.flags;
  if (!(flags & B200SEG_AUG2D_BLUR)) return;
  const int h = e.h, w = e.w, cn = e.c;
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= (long long)h * w) return;
  const int y = (int)(p / w), x = (int)(p % w);
  const uint8_t* img = src + e.src;
  uint8_t* out = ws + e.dst + p * cn;
  const int kind = e.blur;
  if (kind == B200SEG_AUG2D_MOTION) {
    const int fcn = e.filter_cn;
    const int body = (w * fcn) & ~3;                     // row elements of OpenCV's FMA body
    for (int ch = 0; ch < cn; ++ch) {
      const bool fused = x * fcn + ch < body;
      float s = 0.0f;
      for (int t = 0; t < e.ntaps; ++t) {
        const int yy = reflect101(y + e.tap_dy[t], h), xx = reflect101(x + e.tap_dx[t], w);
        const float v = (float)__ldg(img + flip_index(yy, xx, h, w, flags) * cn + ch);
        s = fused ? __fmaf_rn(v, e.tap_w[t], s) : __fadd_rn(s, __fmul_rn(v, e.tap_w[t]));
      }
      out[ch] = (uint8_t)min(max(__float2int_rn(s), 0), 255);
    }
  } else {
    const bool median = kind == B200SEG_AUG2D_MEDIAN;
    long long idx[9];
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int yy = median ? min(max(y + dy, 0), h - 1) : reflect101(y + dy, h);
        const int xx = median ? min(max(x + dx, 0), w - 1) : reflect101(x + dx, w);
        idx[(dy + 1) * 3 + dx + 1] = flip_index(yy, xx, h, w, flags) * cn;
      }
    }
    for (int ch = 0; ch < cn; ++ch) {
      int v[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) v[k] = __ldg(img + idx[k] + ch);
      int r;
      if (median) {
        r = median9(v);
      } else {
        int s = 0;
#pragma unroll
        for (int k = 0; k < 9; ++k) s += v[k];
        r = (2 * s + 9) / 18;                            // rint(s / 9): s / 9 is never a tie
      }
      out[ch] = (uint8_t)r;
    }
  }
}

// OpenCV's per-row and per-column fixed-point terms (imgwarp.cpp, WarpAffineInvoker), fp64 without contraction
__device__ __forceinline__ int fx_row(double m1, double m2, int y) {
  return __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m1, (double)y), m2), 1024.0));
}
__device__ __forceinline__ int fx_col(double m0, int x) { return __double2int_rn(__dmul_rn(__dmul_rn(m0, (double)x), 1024.0)); }

__global__ void __launch_bounds__(kThreads)
warp_kernel(const uint8_t* __restrict__ src, const uint8_t* __restrict__ msrc,
            const b200seg_aug2d_param* __restrict__ params, const uint8_t* __restrict__ ws, uint8_t* __restrict__ out,
            uint8_t* __restrict__ mout) {
  __shared__ uint8_t s_lut[256];
  PDL_ENTER();
  const b200seg_aug2d_param& e = params[blockIdx.y];
  const int flags = e.flags;
  const int h = e.h, w = e.w, cn = e.c;
  const bool lut = flags & B200SEG_AUG2D_LUT;
  if (lut) {
    s_lut[threadIdx.x] = e.lut[threadIdx.x];
    __syncthreads();
  }
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= (long long)h * w) return;
  const int y = (int)(p / w), x = (int)(p % w);
  // the image the warp reads: the blurred one (already flipped) or the source read through the flips
  const bool blurred = flags & B200SEG_AUG2D_BLUR;
  const uint8_t* img = blurred ? ws + e.dst : src + e.src;
  const int iflags = blurred ? 0 : flags;
  uint8_t* o = out + e.dst + p * cn;
  const bool has_mask = e.mask_src >= 0 && msrc != nullptr && mout != nullptr;
  if (flags & B200SEG_AUG2D_WARP) {
    const double m0 = e.minv[0], m1 = e.minv[1], m2 = e.minv[2], m3 = e.minv[3], m4 = e.minv[4], m5 = e.minv[5];
    const int rx = fx_row(m1, m2, y), ry = fx_row(m4, m5, y);
    const int ax = fx_col(m0, x), ay = fx_col(m3, x);
    const int X = (rx + 16 + ax) >> 5, Y = (ry + 16 + ay) >> 5;
    const int sx = X >> 5, sy = Y >> 5, fx = X & 31, fy = Y & 31;
    const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32,
              w11 = fy * fx * 32;
    const int x0 = reflect101(sx, w), x1 = reflect101(sx + 1, w), y0 = reflect101(sy, h), y1 = reflect101(sy + 1, h);
    const long long i00 = flip_index(y0, x0, h, w, iflags) * cn, i01 = flip_index(y0, x1, h, w, iflags) * cn,
                    i10 = flip_index(y1, x0, h, w, iflags) * cn, i11 = flip_index(y1, x1, h, w, iflags) * cn;
    for (int ch = 0; ch < cn; ++ch) {
      const int s = __ldg(img + i00 + ch) * w00 + __ldg(img + i01 + ch) * w01 + __ldg(img + i10 + ch) * w10 +
                    __ldg(img + i11 + ch) * w11;
      const int v = min((s + (1 << 14)) >> 15, 255);
      o[ch] = lut ? s_lut[v] : (uint8_t)v;
    }
    if (has_mask) {
      const int nx = reflect101((rx + 512 + ax) >> 10, w), ny = reflect101((ry + 512 + ay) >> 10, h);
      mout[e.mask_dst + p] = __ldg(msrc + e.mask_src + flip_index(ny, nx, h, w, flags));
    }
  } else {
    const long long i = flip_index(y, x, h, w, iflags) * cn;
    for (int ch = 0; ch < cn; ++ch) {
      const uint8_t v = __ldg(img + i + ch);
      o[ch] = lut ? s_lut[v] : v;
    }
    if (has_mask) mout[e.mask_dst + p] = __ldg(msrc + e.mask_src + flip_index(y, x, h, w, flags));
  }
}

}  // namespace

int augment2d(const uint8_t* src, const uint8_t* msrc, const b200seg_aug2d_param* params, int n, long long max_hw,
              int stages, uint8_t* out, uint8_t* mout, uint8_t* ws, cudaStream_t st) {
  const dim3 grid((unsigned)((max_hw + kThreads - 1) / kThreads), n);
  if (stages & B200SEG_AUG2D_BLUR) {
    launch_k(blur_kernel, grid, kThreads, 0, st, src, params, ws);
    B200_LAUNCH_CHECK();
  }
  launch_k(warp_kernel, grid, kThreads, 0, st, src, msrc, params, (const uint8_t*)ws, out, mout);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
