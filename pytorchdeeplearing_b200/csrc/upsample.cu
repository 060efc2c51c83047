// 2x trilinear upsample fused with the skip add, and its adjoint (UNet3dthin's decoder: networks/Unet3dthin.py:40-54,
// nn.Upsample(scale_factor=2, mode='trilinear') then torch.add with the encoder output).
//
//   forward   S[fine] = sum over 2 x 2 x 2 coarse taps of wz*wy*wx * a[coarse] + e[fine]
//   backward  ga[coarse] = sum over <= 4 x 4 x 4 fine taps of wz*wy*wx * gS[fine]
//
// The tap weights are those of torch's upsample_trilinear3d with align_corners=False and scale 2 (source coordinate
// dst/2 - 0.25, clamped below at 0; at the top edge both taps land on the last index).  Per axis, with n coarse cells:
//   fine 2k   reads coarse (k-1, k) with (0.25, 0.75); fine 0 reads coarse 0 with 1
//   fine 2k+1 reads coarse (k, k+1) with (0.75, 0.25); fine 2n-1 reads coarse n-1 with 1
// and the adjoint gathers, for coarse k, fine (2k-1, 2k, 2k+1, 2k+2) with (0.25, 0.75, 0.75, 0.25): coarse 0 drops
// fine -1 and takes fine 0 with 1, coarse n-1 drops fine 2n and takes fine 2n-1 with 1.  Every weight product is a
// dyadic number, so it is exact in fp32; sums are accumulated in fp32 in a fixed order and rounded once to the storage
// type.  The backward is a gather (no atomics): reruns are bit-identical.
//
// One thread per (voxel, 8-channel chunk): 16-byte bf16 accesses, two 16-byte fp32 accesses.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kUpThreads = 256;

template <typename T>
struct Chunk8;
template <>
struct Chunk8<bf16> {
  static __device__ __forceinline__ void load(const bf16* p, float* v) { load8(p, v); }
  static __device__ __forceinline__ void store(bf16* p, const float* v) { store8(p, v); }
};
template <>
struct Chunk8<float> {
  static __device__ __forceinline__ void load(const float* p, float* v) {
    const float4 a = load4(p), b = load4(p + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* v) {
    store4(p, make_float4(v[0], v[1], v[2], v[3]));
    store4(p + 4, make_float4(v[4], v[5], v[6], v[7]));
  }
};

// the two coarse taps of fine index j on an axis of n coarse cells
__device__ __forceinline__ void fwd_taps(int j, int n, int* i0, int* i1, float* w0, float* w1) {
  const int k = j >> 1;
  if (j & 1) {
    if (k == n - 1) { *i0 = k; *i1 = k; *w0 = 1.f; *w1 = 0.f; }
    else { *i0 = k; *i1 = k + 1; *w0 = 0.75f; *w1 = 0.25f; }
  } else {
    if (k == 0) { *i0 = 0; *i1 = 0; *w0 = 1.f; *w1 = 0.f; }
    else { *i0 = k - 1; *i1 = k; *w0 = 0.25f; *w1 = 0.75f; }
  }
}

// weight of fine index 2k - 1 + t (t = 0..3) in the adjoint at coarse k; 0 where the tap does not exist
__device__ __forceinline__ float bwd_weight(int k, int n, int t) {
  if (t == 0) return k == 0 ? 0.f : 0.25f;
  if (t == 3) return k == n - 1 ? 0.f : 0.25f;
  if (t == 1) return k == 0 ? 1.f : 0.75f;
  return k == n - 1 ? 1.f : 0.75f;
}

template <typename T>
__global__ void __launch_bounds__(kUpThreads) upsample2_add_kernel(TV a, TV e, TV s) {
  PDL_ENTER();
  const int G = s.c >> 3;
  const int FD = s.d, FH = s.h, FW = s.w;
  const long long total = (long long)s.n * FD * FH * FW * G;
  const T* __restrict__ ap = static_cast<const T*>(a.p);
  const T* __restrict__ ep = static_cast<const T*>(e.p);
  T* __restrict__ sp = static_cast<T*>(s.p);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % G) << 3;
    long long v = i / G;
    const int x = (int)(v % FW);
    v /= FW;
    const int y = (int)(v % FH);
    v /= FH;
    const int z = (int)(v % FD);
    const int n = (int)(v / FD);
    int zi[2], yi[2], xi[2];
    float zw[2], yw[2], xw[2];
    fwd_taps(z, a.d, &zi[0], &zi[1], &zw[0], &zw[1]);
    fwd_taps(y, a.h, &yi[0], &yi[1], &yw[0], &yw[1]);
    fwd_taps(x, a.w, &xi[0], &xi[1], &xw[0], &xw[1]);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
          const float w = zw[dz] * yw[dy] * xw[dx];
          const long long cv = (((long long)n * a.d + zi[dz]) * a.h + yi[dy]) * a.w + xi[dx];
          float t[8];
          Chunk8<T>::load(ap + cv * a.ld + c0, t);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = fmaf(w, t[j], acc[j]);
        }
    const long long fv = (((long long)n * FD + z) * FH + y) * FW + x;
    float t[8];
    Chunk8<T>::load(ep + fv * e.ld + c0, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += t[j];
    Chunk8<T>::store(sp + fv * s.ld + c0, acc);
  }
}

template <typename T>
__global__ void __launch_bounds__(kUpThreads) upsample2_bwd_kernel(TV gs, TV ga) {
  PDL_ENTER();
  const int G = ga.c >> 3;
  const int CD = ga.d, CH = ga.h, CW = ga.w;
  const long long total = (long long)ga.n * CD * CH * CW * G;
  const T* __restrict__ gp = static_cast<const T*>(gs.p);
  T* __restrict__ op = static_cast<T*>(ga.p);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % G) << 3;
    long long v = i / G;
    const int x = (int)(v % CW);
    v /= CW;
    const int y = (int)(v % CH);
    v /= CH;
    const int z = (int)(v % CD);
    const int n = (int)(v / CD);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int tz = 0; tz < 4; ++tz) {
      const float wz = bwd_weight(z, CD, tz);
      if (wz == 0.f) continue;
      const int fz = 2 * z - 1 + tz;
      for (int ty = 0; ty < 4; ++ty) {
        const float wy = bwd_weight(y, CH, ty);
        if (wy == 0.f) continue;
        const int fy = 2 * y - 1 + ty;
        const float wzy = wz * wy;
#pragma unroll
        for (int tx = 0; tx < 4; ++tx) {
          const float wx = bwd_weight(x, CW, tx);
          if (wx == 0.f) continue;
          const float w = wzy * wx;
          const long long fv = (((long long)n * gs.d + fz) * gs.h + fy) * gs.w + (2 * x - 1 + tx);
          float t[8];
          Chunk8<T>::load(gp + fv * gs.ld + c0, t);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = fmaf(w, t[j], acc[j]);
        }
      }
    }
    Chunk8<T>::store(op + ((((long long)n * CD + z) * CH + y) * CW + x) * ga.ld + c0, acc);
  }
}

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

inline bool chunk_ok(const b200seg_tensor* t) { return t->c % 8 == 0 && t->ld % 8 == 0 && al16(t->ptr); }

inline bool twice(const b200seg_tensor* coarse, const b200seg_tensor* fine) {
  return coarse->n == fine->n && coarse->c == fine->c && fine->d == 2 * coarse->d && fine->h == 2 * coarse->h &&
         fine->w == 2 * coarse->w;
}

inline int grid_for(long long total, int device) {
  long long blocks = (total + kUpThreads - 1) / kUpThreads;
  const long long cap = (long long)num_sms(device) * 16;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace

int upsample2_add(const b200seg_tensor* a, const b200seg_tensor* e, const b200seg_tensor* s, int device,
                  cudaStream_t st) {
  B200_CHECK_ARG(twice(a, s) && same_geom(e, s), "upsample2_add: S and e must be (N, 2d, 2h, 2w, C) for a (N, d, h, w, C)");
  B200_CHECK_ARG(a->dtype == s->dtype && e->dtype == s->dtype, "upsample2_add: a, e and S must share one dtype");
  B200_CHECK_ARG(chunk_ok(a) && chunk_ok(e) && chunk_ok(s),
                 "upsample2_add: C and every pitch must be multiples of 8, every pointer 16-byte aligned");
  const long long total = (long long)s->n * nvox(s) * (s->c / 8);
  if (s->dtype == B200SEG_BF16)
    launch_k(upsample2_add_kernel<bf16>, grid_for(total, device), kUpThreads, 0, st, tv(a), tv(e), tv(s));
  else
    launch_k(upsample2_add_kernel<float>, grid_for(total, device), kUpThreads, 0, st, tv(a), tv(e), tv(s));
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int upsample2_bwd(const b200seg_tensor* gs, const b200seg_tensor* ga, int device, cudaStream_t st) {
  B200_CHECK_ARG(twice(ga, gs), "upsample2_bwd: gS must be (N, 2d, 2h, 2w, C) for a (N, d, h, w, C) ga");
  B200_CHECK_ARG(gs->dtype == ga->dtype, "upsample2_bwd: gS and ga must share one dtype");
  B200_CHECK_ARG(chunk_ok(gs) && chunk_ok(ga),
                 "upsample2_bwd: C and every pitch must be multiples of 8, every pointer 16-byte aligned");
  const long long total = (long long)ga->n * nvox(ga) * (ga->c / 8);
  if (ga->dtype == B200SEG_BF16)
    launch_k(upsample2_bwd_kernel<bf16>, grid_for(total, device), kUpThreads, 0, st, tv(gs), tv(ga));
  else
    launch_k(upsample2_bwd_kernel<float>, grid_for(total, device), kUpThreads, 0, st, tv(gs), tv(ga));
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
