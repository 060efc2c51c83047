// wgmma / TMA / mbarrier PTX wrappers and the lazily-resolved cuTensorMapEncodeTiled entry point,
// shared by the tensor-core kernels (conv_tc.cu, wgrad_tc.cu, conv_halo.cu, conv_halo_ws.cu).  sm_90a.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace b200seg {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// driver entry point (no -lcuda: resolved lazily so the library loads on machines without a driver);
// returns nullptr (and sets the error text) on failure.  Defined in conv_tc.cu.
EncodeTiledFn tc_encode_fn();
// 128-voxel box (bw x bh x bd, powers of two) with the least padding for a W x H x D volume
void tc_pick_box(int W, int H, int D, int* bw, int* bh, int* bd);
int tc_max_smem(int device);

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// per-thread register count of the executing warpgroup (all four warps execute it); the kernel's counts of all its
// warpgroups together must stay within what it was launched with
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void tma_load_5d(const CUtensorMap* tm, void* dst, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, void* dst, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// wgmma: a warpgroup (four warps, the first a multiple of four) computes 64 rows into fp32 registers; thread t (warp
// w = t/32, lane l) holds in d[i] row 16w + l/4 + 8((i/2)&1), column 8(i/4) + 2(l&3) + (i&1).  wgmma_fence reconverges
// the warp first (the instructions are .aligned; barrier waits can leave it diverged).
__device__ __forceinline__ void wgmma_fence() {
  __syncwarp();
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// waits until at most N committed groups of this warpgroup are still in flight (N = 1: the previous chain is complete
// while the one just committed keeps the tensor core busy)
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void frag_zero(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}
// accumulator fragment (64 rows starting at row0) <-> a row-major fp32 tile in shared memory, `pitch` floats per row
template <int R>
__device__ __forceinline__ void frag_store(float* s, int pitch, int row0, const float (&d)[R], int wt) {
  const int r = row0 + 16 * (wt >> 5) + ((wt & 31) >> 2), c = 2 * (wt & 3);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    *reinterpret_cast<float2*>(s + r * pitch + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(s + (r + 8) * pitch + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
template <int R>
__device__ __forceinline__ void frag_load(const float* s, int pitch, int row0, float (&d)[R], int wt) {
  const int r = row0 + 16 * (wt >> 5) + ((wt & 31) >> 2), c = 2 * (wt & 3);
#pragma unroll
  for (int j = 0; j < R / 4; ++j) {
    const float2 a = *reinterpret_cast<const float2*>(s + r * pitch + 8 * j + c);
    const float2 b = *reinterpret_cast<const float2*>(s + (r + 8) * pitch + 8 * j + c);
    d[4 * j] = a.x; d[4 * j + 1] = a.y; d[4 * j + 2] = b.x; d[4 * j + 3] = b.y;
  }
}
// 16 consecutive fp32 of one accumulator row in shared memory (16-byte aligned)
__device__ __forceinline__ void acc_ld16(const float* s, float* v) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 f = reinterpret_cast<const float4*>(s)[j];
    v[4 * j] = f.x; v[4 * j + 1] = f.y; v[4 * j + 2] = f.z; v[4 * j + 3] = f.w;
  }
}

// Shared-memory matrix descriptors (layout type in bits 62-63: 1 = 128-byte, 2 = 64-byte, 3 = 32-byte swizzle).
// K-major, swizzled operand tile (rows of `swizzle_bytes`, 8-row atoms): SBO = 8 * swizzle_bytes
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr, uint32_t swizzle_bytes) {
  const uint64_t layout = swizzle_bytes == 128 ? 1ull : (swizzle_bytes == 64 ? 2ull : 3ull);
  const uint64_t sbo = (uint64_t)(8u * swizzle_bytes) >> 4;
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (sbo << 32) | (layout << 62);
}


// MN-major, swizzled operand tile: rows (K index) of `swizzle_bytes` holding swizzle_bytes/2 bf16 MN-elements,
// 8-row atoms (SBO = 8 * swizzle_bytes); the next group of MN-elements starts `lbo_bytes` further on.
__device__ __forceinline__ uint64_t make_mnmajor_desc(uint32_t smem_addr, uint32_t swizzle_bytes, uint32_t lbo_bytes) {
  const uint64_t layout = swizzle_bytes == 128 ? 1ull : (swizzle_bytes == 64 ? 2ull : 3ull);
  const uint64_t sbo = (uint64_t)(8u * swizzle_bytes) >> 4;
  const uint64_t lbo = (uint64_t)lbo_bytes >> 4;
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (lbo << 16) | (sbo << 32) | (layout << 62);
}

}  // namespace b200seg
