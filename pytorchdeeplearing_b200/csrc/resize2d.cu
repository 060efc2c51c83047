// OpenCV's uint8 bilinear resize on the device (sm_90a): cv2.resize(img, (W, H)) with the default INTER_LINEAR, as
// the reference's 2-D datasets (model/dataset.py:63,140,154) and 2-D inference methods (model/modelVNet.py:231-242,
// model/modelUnet.py:231-242, model/modelResNet.py:212-221) call it on the host.
//   Per axis (source size s, destination size d, destination index i): scale = 1 / (d / s) in fp64,
//   f = (float)((i + 0.5) * scale - 0.5), k = floor(f), f -= k; along x, k < 0 or k >= s - 1 clamp k and set f = 0,
//   along y only the taps are clamped; c0 = rint((1 - f) * 2048), c1 = rint(f * 2048).  Horizontal pass
//   r = src[k] c0 + src[k + 1] c1 (int32), vertical pass (((b0 (r0 >> 4)) >> 16) + ((b1 (r1 >> 4)) >> 16) + 2) >> 2
//   (OpenCV's fixed-point SIMD form), saturated to [0, 255].  Every coefficient operation is rounded on its own
//   (no FMA contraction), so the bytes equal cv2's.
// One launch resizes a ragged batch: sample n starts at byte desc[n].offset of src and has its own (h, w); the output
// is dense (N, oH, oW), either the uint8 bytes or fp32 (float)((double)v / 255.0) (the reference's "/ 255." then
// .float(), written straight into the network input).  Block = 128 threads x 4 output columns x 8 output rows: the
// column taps live in registers for the block's rows, each output row reads its two source rows, and the four
// columns of a thread are stored with one 4-byte (uint8) or 16-byte (fp32) store when the rows allow it.  No
// allocation, no host synchronisation, no reductions: reruns are bit-identical.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kThreads = 128;
constexpr int kVec = 4;                      // output columns per thread
constexpr int kTileW = kThreads * kVec;      // output columns per block
constexpr int kRows = 8;                     // output rows per block

// one destination index along one axis -> taps k0, k1 and 11-bit coefficients c0, c1
__device__ __forceinline__ void axis_tap(int i, int s, double scale, bool x_axis, int& k0, int& k1, int& c0,
                                         int& c1) {
  float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)i, 0.5), scale), 0.5));
  const float fk = floorf(f);
  int k = (int)fk;
  f = __fsub_rn(f, fk);
  if (x_axis) {
    if (k < 0) {
      k = 0;
      f = 0.0f;
    }
    if (k >= s - 1) {
      k = s - 1;
      f = 0.0f;
    }
    k0 = k;
    k1 = min(k + 1, s - 1);
  } else {
    k0 = min(max(k, 0), s - 1);
    k1 = min(max(k + 1, 0), s - 1);
  }
  c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, f), 2048.0f));
  c1 = __float2int_rn(__fmul_rn(f, 2048.0f));
}

__device__ __forceinline__ double inv_ratio(int d, int s) { return __ddiv_rn(1.0, __ddiv_rn((double)d, (double)s)); }

// F32: write (float)(v / 255.0); VEC: the output rows allow one aligned vector store per thread
template <bool F32, bool VEC>
__global__ void __launch_bounds__(kThreads)
resize_linear_kernel(const uint8_t* __restrict__ src, const b200seg_resize_src* __restrict__ desc, int oH, int oW,
                     void* __restrict__ out) {
  __shared__ float s_unit[F32 ? 256 : 1];
  PDL_ENTER();
  if (F32) {
    for (int v = threadIdx.x; v < 256; v += kThreads) s_unit[v] = __double2float_rn(__ddiv_rn((double)v, 255.0));
    __syncthreads();
  }
  const int n = blockIdx.z;
  const long long offset = desc[n].offset;
  const int h = desc[n].h, w = desc[n].w;
  const int xb = blockIdx.x * kTileW + threadIdx.x * kVec;
  if (h < 1 || w < 1 || xb >= oW) return;
  const uint8_t* img = src + offset;

  const double sx = inv_ratio(oW, w), sy = inv_ratio(oH, h);
  int x0[kVec], x1[kVec], a0[kVec], a1[kVec];
#pragma unroll
  for (int j = 0; j < kVec; ++j) {
    if (xb + j < oW) {
      axis_tap(xb + j, w, sx, true, x0[j], x1[j], a0[j], a1[j]);
    } else {
      x0[j] = x1[j] = 0;
      a0[j] = a1[j] = 0;
    }
  }
  const int y_end = min(oH, (int)blockIdx.y * kRows + kRows);
  for (int y = blockIdx.y * kRows; y < y_end; ++y) {
    int y0, y1, b0, b1;
    axis_tap(y, h, sy, false, y0, y1, b0, b1);
    const uint8_t* r0p = img + (long long)y0 * w;
    const uint8_t* r1p = img + (long long)y1 * w;
    int v[kVec];
#pragma unroll
    for (int j = 0; j < kVec; ++j) {
      const int r0 = (int)__ldg(r0p + x0[j]) * a0[j] + (int)__ldg(r0p + x1[j]) * a1[j];
      const int r1 = (int)__ldg(r1p + x0[j]) * a0[j] + (int)__ldg(r1p + x1[j]) * a1[j];
      const int t = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
      v[j] = min(max(t, 0), 255);
    }
    const long long o = ((long long)n * oH + y) * oW + xb;
    if (F32) {
      float* op = static_cast<float*>(out) + o;
      if (VEC) {
        *reinterpret_cast<float4*>(op) = make_float4(s_unit[v[0]], s_unit[v[1]], s_unit[v[2]], s_unit[v[3]]);
      } else {
#pragma unroll
        for (int j = 0; j < kVec; ++j)
          if (xb + j < oW) op[j] = s_unit[v[j]];
      }
    } else {
      uint8_t* op = static_cast<uint8_t*>(out) + o;
      if (VEC) {
        *reinterpret_cast<uint32_t*>(op) =
            (uint32_t)v[0] | ((uint32_t)v[1] << 8) | ((uint32_t)v[2] << 16) | ((uint32_t)v[3] << 24);
      } else {
#pragma unroll
        for (int j = 0; j < kVec; ++j)
          if (xb + j < oW) op[j] = (uint8_t)v[j];
      }
    }
  }
}

}  // namespace

int resize_linear_u8(const uint8_t* src, const b200seg_resize_src* desc, int n, int oH, int oW, void* out,
                     int out_mode, cudaStream_t st) {
  const dim3 grid((oW + kTileW - 1) / kTileW, (oH + kRows - 1) / kRows, n);
  const bool f32 = out_mode == B200SEG_F32;
  const bool vec = oW % kVec == 0 && reinterpret_cast<uintptr_t>(out) % (f32 ? 16 : 4) == 0;
  if (f32) {
    if (vec) launch_k(resize_linear_kernel<true, true>, grid, kThreads, 0, st, src, desc, oH, oW, out);
    else launch_k(resize_linear_kernel<true, false>, grid, kThreads, 0, st, src, desc, oH, oW, out);
  } else {
    if (vec) launch_k(resize_linear_kernel<false, true>, grid, kThreads, 0, st, src, desc, oH, oW, out);
    else launch_k(resize_linear_kernel<false, false>, grid, kThreads, 0, st, src, desc, oH, oW, out);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
