// wgmma + TMA weight-gradient kernel for sm_90a (bf16 operands, fp32 accumulation in registers).
//
//   dwp[t][ka][kb] += sum_{n,o} a[n, o + t - p, ka] * b[n, o, kb]        (stride-1 kinds: 3x3x3 / 3x3 / 1x1)
//
// GEMM view: M = flattened (tap, ka) rows, N = kb, K = output voxels.  Both operands sit in shared
// memory exactly as TMA delivers NDHWC boxes -- [voxel rows][channels] -- which is the MN-major
// canonical wgmma layout (rows = K index, 32/64/128-byte swizzled rows of MN elements), so no
// transposition is ever materialised:
//   A stage : 128/CA sub-tiles, each the activation box of one (tap, 16/32/64-channel block) shifted
//             by the tap offset (TMA zero fill = conv padding); consecutive sub-tiles are consecutive
//             MN atoms (descriptor LBO = sub-tile bytes), i.e. several taps are STACKED along M so
//             that 16- and 32-channel layers still fill the 128-row accumulator block.
//   B stage : the dy box of the same 128 voxels, the CTA's NC kb channels in 64-channel sub-tiles.
//   MMA     : 2 x 8 wgmma (two M64 halves x N=NC x K16 voxels) per stage, both operands MN-major.
// A CTA owns one accumulator block (128 rows x NC columns, in the registers of its MMA warpgroup) and a contiguous
// chunk of voxel tiles; at the end the warpgroup adds the block into dwp with fp32 atomics (split-K over the grid).
// Warp roles (256 threads): warp 0 TMA producer, warps 1-3 idle, warps 4-7 MMA warpgroup + epilogue.
#include <stdlib.h>

#include "tc_common.cuh"

namespace b200seg {

struct WgArgs {
  float* dwp;
  int N, D, H, W;
  int Ka, Kb, Rtot;          // rows per tap, columns, taps*Ka
  int kd, kh, kw, pd, ph, pw, sd, sh, sw;
  int bw, bh, bd, tw, th, td, ntiles;
  int CA, CB;                // channels per A / B sub-tile (<= 64)
  int mblocks_total;
  int nstages;
};

constexpr int kWgMaxStages = 6;
constexpr int kWgThreads = 256;

// grid: x = split-K over the voxel tiles, y = accumulator block (128 rows of (tap, ka)), z = group of NC columns
template <int NC>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                 const __grid_constant__ CUtensorMap tmB, const WgArgs p) {
  PDL_TRIGGER();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t A_SUB = 128u * (uint32_t)p.CA * 2u;          // bytes of one A sub-tile
  const uint32_t A_BYTES = 128u * 128u * 2u;                  // 128/CA sub-tiles
  const uint32_t B_SUB = 128u * (uint32_t)p.CB * 2u;
  const uint32_t nbsub = (uint32_t)(NC / p.CB);
  const uint32_t B_BYTES = B_SUB * nbsub;
  const uint32_t STAGE = A_BYTES + B_BYTES;
  uint8_t* tail = smem + (size_t)p.nstages * STAGE;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* empty = full + kWgMaxStages;
  int4* s_sub = reinterpret_cast<int4*>(empty + kWgMaxStages);   // [128/CA] : channel, dw, dh, dd of a sub-tile

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int tiles_per_cta = (p.ntiles + gridDim.x - 1) / gridDim.x;
  const int tile_begin = blockIdx.x * tiles_per_cta;
  const int tile_end = min(p.ntiles, tile_begin + tiles_per_cta);
  const int mb = blockIdx.y;
  const int col0 = blockIdx.z * NC;
  const int nasub = 128 / p.CA;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nstages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);      // one arrive per MMA warp
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  // tap decode of every A sub-tile of this CTA's block (keeps integer division out of the producer loop)
  for (int j = threadIdx.x; j < nasub; j += blockDim.x) {
    const int R = mb * 128 + j * p.CA;
    int4 e = make_int4(-1, 0, 0, 0);
    if (R < p.Rtot) {
      const int tap = R / p.Ka;
      e.x = R - tap * p.Ka;
      e.y = tap % p.kw - p.pw;
      e.z = (tap / p.kw) % p.kh - p.ph;
      e.w = tap / (p.kw * p.kh) - p.pd;
    }
    s_sub[j] = e;
  }
  __syncthreads();
  PDL_WAIT();               // everything above is on-chip set-up: it runs under the tail of the previous kernel
  if (tile_begin >= tile_end) return;

  if (warp == 0) {
    // ===================================================== TMA producer
    if (elect_one()) {
      // the last M block may be partial: skip (and do not expect) the sub-tiles that do not exist
      int valid = 0;
      for (int j = 0; j < nasub; ++j) valid += s_sub[j].x >= 0 ? 1 : 0;
      uint32_t it = 0;
      for (int tile = tile_begin; tile < tile_end; ++tile, ++it) {
        int t = tile;
        const int iw = t % p.tw; t /= p.tw;
        const int ih = t % p.th; t /= p.th;
        const int id = t % p.td;
        const int n = t / p.td;
        const int w0 = iw * p.bw, h0 = ih * p.bh, d0 = id * p.bd;
        const uint32_t s = it % p.nstages;
        const uint32_t ph = (it / p.nstages) & 1u;
        mbar_wait(&empty[s], ph ^ 1u);
        uint8_t* sa = smem + (size_t)s * STAGE;
        mbar_expect_tx(&full[s], (uint32_t)valid * A_SUB + B_BYTES);
        for (int j = 0; j < valid; ++j) {
          const int4 e = s_sub[j];
          tma_load_5d(&tmA, sa + (size_t)j * A_SUB, &full[s], e.x, w0 * p.sw + e.y, h0 * p.sh + e.z, d0 * p.sd + e.w, n);
        }
        for (uint32_t j = 0; j < nbsub; ++j)
          tma_load_5d(&tmB, sa + A_BYTES + (size_t)j * B_SUB, &full[s], col0 + (int)j * p.CB, w0, h0, d0, n);
      }
    }
  } else if (warp >= 4) {
    // ===================================================== MMA warpgroup, then the dW epilogue
    const int wt = threadIdx.x - 128;
    const uint32_t swa = (uint32_t)p.CA * 2u, swb = (uint32_t)p.CB * 2u;
    float d0[NC / 2], d1[NC / 2];
    frag_zero(d0);
    frag_zero(d1);
    uint32_t it = 0;
    for (int tile = tile_begin; tile < tile_end; ++tile, ++it) {
      const uint32_t s = it % p.nstages;
      const uint32_t ph = (it / p.nstages) & 1u;
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * STAGE);
      const uint64_t adesc = make_mnmajor_desc(sa, swa, A_SUB);
      const uint64_t bdesc = make_mnmajor_desc(sa + A_BYTES, swb, B_SUB);
      wgmma_fence_regs(d0);
      wgmma_fence_regs(d1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        // 16 voxel rows per K step: advance the start address by 16 rows of the operand's row pitch; rows 64..127 of
        // the block are the A sub-tiles 64 MN elements (16 KB) further on
        const uint64_t ka = (uint64_t)((16u * swa * (uint32_t)k) >> 4);
        const uint64_t kb = (uint64_t)((16u * swb * (uint32_t)k) >> 4);
        Wgmma<NC, 1, 1>::mma(d0, adesc + ka, bdesc + kb);
        Wgmma<NC, 1, 1>::mma(d1, adesc + (uint64_t)(16384u >> 4) + ka, bdesc + kb);
      }
      wgmma_commit();
      wgmma_wait0();
      wgmma_fence_regs(d0);
      wgmma_fence_regs(d1);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // fragment element i of half h: row 64h + 16w + l/4 + 8*((i/2)&1), column 8*(i/4) + 2*(l&3) + (i&1)
    const int r0 = mb * 128 + 16 * (wt >> 5) + ((wt & 31) >> 2);
    const int c = col0 + 2 * (wt & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < NC / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int R = r0 + 64 * h + 8 * e;
          const float x0 = h ? d1[4 * j + 2 * e] : d0[4 * j + 2 * e];
          const float x1 = h ? d1[4 * j + 2 * e + 1] : d0[4 * j + 2 * e + 1];
          if (R < p.Rtot) atomicAdd(reinterpret_cast<float2*>(p.dwp + (size_t)R * p.Kb + c + 8 * j), make_float2(x0, x1));
        }
  }
}

// ------------------------------------------------------------------------------------------------
static bool al16w(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

static int sub_channels(int c) {
  if (c % 64 == 0) return 64;
  if (c == 32) return 32;
  if (c == 16) return 16;
  return 0;
}

int wgrad_tc_init(int device, int maxsm) {
  (void)device;
  B200_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
  B200_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
  B200_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
  B200_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
  return B200SEG_OK;
}

int wgrad_tc_supported(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b) {
  ConvGeom g;
  if (conv_geometry(kind, dims, &g) != 0 || g.up) return 0;
  if (a->dtype != B200SEG_BF16 || b->dtype != B200SEG_BF16) return 0;
  if (sub_channels(a->c) == 0 || sub_channels(b->c) == 0) return 0;
  if (a->c > 256 || b->c > 256) return 0;
  if ((a->ld % 8) || (b->ld % 8) || !al16w(a->ptr) || !al16w(b->ptr)) return 0;
  if (a->n != b->n || a->d != b->d * g.sd || a->h != b->h * g.sh || a->w != b->w * g.sw) return 0;
  return 1;
}

static int encode_box_map(CUtensorMap* tm, const b200seg_tensor* t, int cbox, int bw, int bh, int bd, int sw_ = 1,
                          int sh_ = 1, int sd_ = 1) {
  EncodeTiledFn enc = tc_encode_fn();
  if (!enc) return B200SEG_ECUDA;
  const CUtensorMapSwizzle sw = cbox == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                           : (cbox == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  cuuint64_t dims5[5] = {(cuuint64_t)t->c, (cuuint64_t)t->w, (cuuint64_t)t->h, (cuuint64_t)t->d, (cuuint64_t)t->n};
  cuuint64_t strides[4] = {(cuuint64_t)t->ld * 2, (cuuint64_t)t->ld * 2 * t->w, (cuuint64_t)t->ld * 2 * t->w * t->h,
                           (cuuint64_t)t->ld * 2 * t->w * t->h * t->d};
  cuuint32_t box[5] = {(cuuint32_t)cbox, (cuuint32_t)(bw * sw_), (cuuint32_t)(bh * sh_), (cuuint32_t)(bd * sd_), 1};
  cuuint32_t estr[5] = {1, (cuuint32_t)sw_, (cuuint32_t)sh_, (cuuint32_t)sd_, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, t->ptr, dims5, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_CHECK_ARG(r == CUDA_SUCCESS, "wgrad_tc: cuTensorMapEncodeTiled failed with %d", (int)r);
  return B200SEG_OK;
}

int wgrad_tc(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
             cudaStream_t st) {
  ConvGeom g;
  conv_geometry(kind, dims, &g);
  WgArgs p;
  p.dwp = dwp;
  p.N = b->n; p.D = b->d; p.H = b->h; p.W = b->w;
  p.Ka = a->c; p.Kb = b->c;
  p.kd = g.kd; p.kh = g.kh; p.kw = g.kw; p.pd = g.pd; p.ph = g.ph; p.pw = g.pw;
  p.sd = g.sd; p.sh = g.sh; p.sw = g.sw;
  p.Rtot = g.kd * g.kh * g.kw * p.Ka;
  tc_pick_box(p.W, p.H, p.D, &p.bw, &p.bh, &p.bd);
  p.tw = (p.W + p.bw - 1) / p.bw;
  p.th = (p.H + p.bh - 1) / p.bh;
  p.td = (p.D + p.bd - 1) / p.bd;
  p.ntiles = p.N * p.td * p.th * p.tw;
  p.CA = sub_channels(p.Ka);
  p.CB = sub_channels(p.Kb);
  p.mblocks_total = (p.Rtot + 127) / 128;
  // Decomposition: grid.y = accumulator blocks (128 rows of (tap, ka) each), grid.z = column groups of NC <= 128 kb
  // channels (the block lives in 128 registers per thread of one warpgroup), grid.x = split-K over the voxel tiles
  // for the rest of the chip.  Every K split adds its partial dW with fp32 atomics.
  const int nc = p.Kb % 128 == 0 ? 128 : (p.Kb % 64 == 0 ? 64 : p.Kb);
  const int gy = p.mblocks_total, gz = p.Kb / nc;
  const uint32_t stage = 128u * 128u * 2u + 128u * (uint32_t)nc * 2u;
  const uint32_t tail = 2 * kWgMaxStages * 8 + (uint32_t)(128 / p.CA) * 16;
  const int maxsm = tc_max_smem(device);
  int nst = (int)((maxsm - 1024 - (int)tail - 256) / (int)stage);
  if (nst > kWgMaxStages) nst = kWgMaxStages;
  B200_CHECK_ARG(nst >= 2, "wgrad_tc: stage does not fit in shared memory (Kb=%d)", p.Kb);
  p.nstages = nst;
  const size_t smem_bytes = 1024 + (size_t)nst * stage + tail + 128;
  CUtensorMap tmA, tmB;
  int rc = encode_box_map(&tmA, a, p.CA, p.bw, p.bh, p.bd, g.sw, g.sh, g.sd);
  if (rc != B200SEG_OK) return rc;
  rc = encode_box_map(&tmB, b, p.CB, p.bw, p.bh, p.bd);
  if (rc != B200SEG_OK) return rc;
  int gx = num_sms(device) / (gy * gz);
  if (gx < 1) gx = 1;
  if (gx > p.ntiles) gx = p.ntiles;
  dim3 grid(gx, gy, gz);
  if (nc == 128) launch_k(wgrad_tc_kernel<128>, grid, kWgThreads, smem_bytes, st, tmA, tmB, p);
  else if (nc == 64) launch_k(wgrad_tc_kernel<64>, grid, kWgThreads, smem_bytes, st, tmA, tmB, p);
  else if (nc == 32) launch_k(wgrad_tc_kernel<32>, grid, kWgThreads, smem_bytes, st, tmA, tmB, p);
  else launch_k(wgrad_tc_kernel<16>, grid, kWgThreads, smem_bytes, st, tmA, tmB, p);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
