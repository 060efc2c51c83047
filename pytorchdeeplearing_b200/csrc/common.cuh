// Shared device/host helpers of the b200seg kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <utility>

#include "../../include/b200seg.h"

namespace b200seg {

void set_error(const char* fmt, ...);

#define B200_CHECK_ARG(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      b200seg::set_error(__VA_ARGS__);            \
      return B200SEG_EINVAL;                      \
    }                                             \
  } while (0)

#define B200_CUDA(call)                                                                     \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) {                                                                \
      b200seg::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return B200SEG_ECUDA;                                                                 \
    }                                                                                       \
  } while (0)

#define B200_LAUNCH_CHECK()                                                                 \
  do {                                                                                      \
    cudaError_t _e = cudaPeekAtLastError();                                                 \
    if (_e != cudaSuccess) {                                                                \
      b200seg::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      (void)cudaGetLastError();                                                             \
      return B200SEG_ECUDA;                                                                 \
    }                                                                                       \
  } while (0)

// RAII device selection without touching the caller's current device permanently.
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    want = dev;
  }
  ~DeviceGuard() {
    if (prev >= 0 && prev != want) cudaSetDevice(prev);
  }
  int want = -1;
};

#define B200_DEVICE(dev)                                   \
  b200seg::DeviceGuard _guard(dev);                        \
  if (!_guard.ok) {                                        \
    b200seg::set_error("cannot select CUDA device %d", dev); \
    (void)cudaGetLastError();                              \
    return B200SEG_ECUDA;                                  \
  }

// Tensor view passed by value to kernels.
struct TV {
  void* p;
  int n, d, h, w, c;
  long long ld;
};
inline TV tv(const b200seg_tensor* t) { return TV{t->ptr, t->n, t->d, t->h, t->w, t->c, (long long)t->ld}; }
inline long long nvox(const b200seg_tensor* t) { return (long long)t->d * t->h * t->w; }
inline bool same_geom(const b200seg_tensor* a, const b200seg_tensor* b) {
  return a->n == b->n && a->d == b->d && a->h == b->h && a->w == b->w && a->c == b->c;
}

typedef __nv_bfloat16 bf16;

// geometry of one conv kind (gather taps / strides / pads, or the depth-to-space factors of UP)
struct ConvGeom {
  int kd, kh, kw;   // taps of the gather (1,1,1 for UP)
  int sd, sh, sw;   // strides
  int pd, ph, pw;   // zero padding
  int up;           // 1 -> depth-to-space store, cols = (tap, cout)
  int ud, uh, uw;   // UP: upsampling factors
};
int conv_geometry(int kind, int dims, ConvGeom* g);

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }

// 4 consecutive elements <-> float4 (16-byte aligned for float, 8-byte for bf16)
__device__ __forceinline__ float4 load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 load4(const bf16* p) {
  uint2 u = *reinterpret_cast<const uint2*>(p);
  __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&u.x);
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&u.y);
  float2 fa = __bfloat1622float2(a), fb = __bfloat1622float2(b);
  return make_float4(fa.x, fa.y, fb.x, fb.y);
}
__device__ __forceinline__ void store4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void store4(bf16* p, float4 v) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y);
  __nv_bfloat162 b = __floats2bfloat162_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<unsigned*>(&a);
  u.y = *reinterpret_cast<unsigned*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
// 8 consecutive bf16 <-> 8 floats (16-byte access)
__device__ __forceinline__ void load8(const bf16* p, float* o) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __bfloat1622float2(h[i]);
    o[2 * i] = f.x;
    o[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void store8(bf16* p, const float* v) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------------------
// Programmatic dependent launch.  A step is a chain of ~150 short kernels; every kernel starts with
// ``griddepcontrol.wait`` (all memory of the kernels before it in the stream is visible after it) followed by
// ``griddepcontrol.launch_dependents``, and every launch carries the programmatic-stream-serialization attribute:
// the next kernel of the chain is launched and its CTAs are scheduled while the last wave of this one is still
// running, so the launch latency (~2-3 us per boundary inside a CUDA graph) leaves the critical path.  Because the
// wait is the first instruction, every kernel still sees the complete output of ALL its predecessors (the chain is
// transitive).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
#define PDL_ENTER() b200seg::pdl_enter()
// Split form for kernels with an on-chip prologue (mbarrier init, shared-memory clears): trigger
// first, run the prologue, THEN wait -- the prologue overlaps the tail of the kernel before.  Nothing before
// PDL_WAIT() may touch global memory: a chain of triggered kernels can be resident before ANY of them has completed,
// so not even data written many launches ago (packed weights) is safe to read early.  Every thread executes the wait.
#define PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")

template <typename... KArgs, typename... Args>
inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);     // errors surface in B200_LAUNCH_CHECK
}

inline int num_sms(int dev) {
  static int cached[64] = {0};
  if (dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    cached[dev] = v;
  }
  return cached[dev];
}

}  // namespace b200seg
