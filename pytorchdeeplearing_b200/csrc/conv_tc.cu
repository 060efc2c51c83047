// wgmma + TMA implicit-GEMM convolution for sm_90a (bf16 operands, fp32 accumulation in registers).
//
// Covers the dense-MMA-shaped members of the conv family in PERF mode: 3x3x3 / 3x3 (pad 1) and
// 1x1x1 convolutions, forward and data-gradient form, Cin in {16, 32, 64k}, Cout = 16..256 (x16).
//
// GEMM view per CTA tile: M = 128 output voxels (a bw x bh x bd box of one sample), N = Cout,
// K = taps x Cin.  One pipeline stage = one tap x one 16/32/64-channel block:
//   A tile  : TMA 5-D tiled load of the NDHWC activation box shifted by the tap offset; the
//             hardware zero-fills out-of-bounds voxels = the conv's zero padding; 128 rows of
//             BKC*2 bytes land K-major with the 32/64/128-byte swizzle the wgmma descriptor names.
//   B tile  : TMA 2-D load of the [tap*Cout + co][ci] packed weights (K-major, same swizzle).
//   MMA     : the MMA warpgroup issues 2 x BKC/16 wgmma (two M64 halves x N x K16) per stage into register
//             accumulators (N <= 64), then releases the smem stage; at the end of the K loop it writes the
//             accumulator tile to one of two fp32 staging slots in shared memory and publishes it.
// Warp roles (512 threads): warp 0 TMA producer, warps 1-3 idle, warps 4-7 MMA warpgroup, warps 8-15 epilogue in two
// groups of four (group e drains the tiles with local index = e mod 2, one thread per tile row):
// staged accumulator row -> +bias -> GroupNorm sum/sumsq partials -> +addend -> bf16 NDHWC stores.
// The two staging slots let the MMA warpgroup run one tile ahead of each epilogue group; CTAs are persistent over
// contiguous tile ranges (grid = min(tiles, #SM)).
#include <stdlib.h>

#include <mutex>

#include "tc_common.cuh"

namespace b200seg {

// ------------------------------------------------------------------------------------------------
// driver entry point
// ------------------------------------------------------------------------------------------------
static EncodeTiledFn g_encode = nullptr;

EncodeTiledFn tc_encode_fn() {
  if (g_encode) return g_encode;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
    (void)cudaGetLastError();
    set_error("cannot resolve cuTensorMapEncodeTiled from the CUDA driver");
    return nullptr;
  }
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return g_encode;
}

// ------------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------------
struct TcArgs {
  bf16* y;
  const bf16* addend;
  const float* bias;
  double* stats;          // [N][Cout][2] or null
  long long yld, ald;
  int N, D, H, W;         // tile-space dims: output dims (gather kinds) or input dims (UP)
  int Cin, Cout;
  int kd, kh, kw, pd, ph, pw;
  int sd, sh, sw;         // gather strides (2 for the k2s2 down conv)
  int up, ud, uh, uw;     // UP: columns are (tap, cout), depth-to-space store with these factors
  int Ntile, ngroups;     // MMA N (columns per accumulator) and number of column groups per voxel tile
  int bw, bh, bd;         // M-tile box, bw*bh*bd == 128
  int tw, th, td;         // tiles per dim
  int ntiles;             // N * td * th * tw
  int nstages;
  int nacc;               // accumulator staging slots in shared memory (== kMaxAcc)
  int acc_pitch;          // floats per row of the staging tile: nacc*Ntile + 4
  // split-K (deep, small levels): the (tap, channel-block) loop of one (voxel tile, column group) is cut into
  // `ksplit` ranges, one work item each; every item leaves its fp32 partial in its own slab of `ws`, and the item
  // that arrives last (counted in cnt[tile, group]) adds the slabs in split order and runs the usual epilogue
  int ksplit;
  float4* ws;             // [tile*group][ksplit][Ntile/4][128 rows] float4
  unsigned int* cnt;      // [tile*group], zero between launches (the last arriver resets its word)
};

constexpr int kMaxStages = 8;
constexpr int kEpiWarps = 4;          // warps per epilogue group (32 tile rows each)
constexpr int kEpiGroups = 2;         // group e drains accumulator slot e: two tiles are in the epilogue at a time
constexpr int kTcThreads = 256 + 32 * kEpiWarps * kEpiGroups;
constexpr int kMaxAcc = 2;            // accumulator staging slots (one per epilogue group)
constexpr int kTcMaxN = 64;           // MMA N per tile: both M64 halves of the accumulator stay in registers

// butterfly transpose-reduce of 16 per-lane column values (and their squares) over the 32 lanes of a warp:
// afterwards every EVEN lane L holds in s[0] / q[0] the warp totals of column stat_col(L)
__device__ __forceinline__ void stat_butterfly(float* s, float* qq, int lane) {
#pragma unroll
  for (int half = 8, off = 16; half >= 1; half >>= 1, off >>= 1) {
    const bool up = (lane & off) != 0;
#pragma unroll
    for (int j = 0; j < half; ++j) {
      const float keep_s = up ? s[j + half] : s[j];
      const float send_s = up ? s[j] : s[j + half];
      const float keep_q = up ? qq[j + half] : qq[j];
      const float send_q = up ? qq[j] : qq[j + half];
      s[j] = keep_s + __shfl_xor_sync(0xffffffffu, send_s, off);
      qq[j] = keep_q + __shfl_xor_sync(0xffffffffu, send_q, off);
    }
  }
  s[0] += __shfl_xor_sync(0xffffffffu, s[0], 1);
  qq[0] += __shfl_xor_sync(0xffffffffu, qq[0], 1);
}
// column owned by an even lane after stat_butterfly: bit k of the index is bit (4-k) of the lane for k = 0..3
__device__ __forceinline__ int stat_col(int lane) {
  return ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
}

template <int BKC, int N>
__device__ __forceinline__ void tc_mma_role(const TcArgs& p, const uint8_t* smem, uint32_t STAGE, uint64_t* full,
                                            uint64_t* empty, uint64_t* tfull, uint64_t* tempty, float* s_acc,
                                            int tile_begin, int tile_end, int kblocks, int wt) {
  constexpr uint32_t SWZ = BKC * 2;
  constexpr uint32_t A_BYTES = 128u * SWZ;
  constexpr int R = N / 2;
  const int S = p.ksplit;
  const int lane = wt & 31;
  uint32_t it = 0;
  int local = 0;
  for (int item = tile_begin; item < tile_end; ++item, ++local) {
    const uint32_t as = (uint32_t)local % (uint32_t)p.nacc;
    const uint32_t aph = ((uint32_t)local / (uint32_t)p.nacc) & 1u;
    float d0[R], d1[R];
    frag_zero(d0);
    frag_zero(d1);
    const int sp = item % S;
    const int kb0 = sp * kblocks / S, kb1 = (sp + 1) * kblocks / S;
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const uint32_t s = it % p.nstages;
      const uint32_t ph = (it / p.nstages) & 1u;
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * STAGE);
      const uint64_t adesc = make_kmajor_desc(sa, SWZ);
      const uint64_t bdesc = make_kmajor_desc(sa + A_BYTES, SWZ);
      wgmma_fence_regs(d0);
      wgmma_fence_regs(d1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BKC / 16; ++k) {
        // +32 bytes (2 x 16-byte units) per K=16 step inside the swizzle atom; rows 64..127 start 64 rows further on
        Wgmma<N, 0, 0>::mma(d0, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k));
        Wgmma<N, 0, 0>::mma(d1, adesc + (uint64_t)((64u * SWZ) >> 4) + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k));
      }
      wgmma_commit();
      wgmma_wait0();
      wgmma_fence_regs(d0);
      wgmma_fence_regs(d1);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // the epilogue group of this slot has drained the previous tile
    mbar_wait(&tempty[as], aph ^ 1u);
    float* acc = s_acc + as * N;
    frag_store(acc, p.acc_pitch, 0, d0, wt);
    frag_store(acc, p.acc_pitch, 64, d1, wt);
    __syncwarp();
    if (lane == 0) mbar_arrive(&tfull[as]);
  }
}

// NCH > 0 (Cout == 16 * NCH <= 32): the layers with few MACs per output element (1x1x1, 2x2x2 stride 2 and its
// transpose at 16/32 channels) are bound by the epilogue, so their GroupNorm statistics are accumulated per
// thread in registers across all of the CTA's tiles and folded over the warp once per sample, and the bias lives
// in registers.  NCH == 0: generic Cout, per-chunk butterfly.
template <int BKC, int NCH>
__global__ void __launch_bounds__(kTcThreads, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                         const __grid_constant__ CUtensorMap tmB, const TcArgs p) {
  PDL_TRIGGER();
  constexpr uint32_t SWZ = BKC * 2;                 // bytes per smem row = swizzle span
  constexpr uint32_t A_BYTES = 128u * SWZ;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t b_bytes_real = (uint32_t)p.Ntile * SWZ;
  const uint32_t B_BYTES = (b_bytes_real + 1023u) & ~1023u;
  const uint32_t STAGE = A_BYTES + B_BYTES;
  uint8_t* tail = smem + (size_t)p.nstages * STAGE;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* empty = full + kMaxStages;
  uint64_t* tfull = empty + kMaxStages;
  uint64_t* tempty = tfull + kMaxAcc;
  float* s_stat = reinterpret_cast<float*>(tempty + kMaxAcc);  // [2 groups][4 epilogue warps][2][Cout]
  unsigned int* s_flag = reinterpret_cast<unsigned int*>(s_stat + 8 * kEpiGroups * p.Cout);   // [2 groups]
  float* s_acc = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(s_flag + kEpiGroups) + 15) & ~(uintptr_t)15);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // work item = (voxel tile, column group, K range); consecutive items of a CTA share the voxel tile
  const int S = p.ksplit;
  const int nitems = p.ntiles * p.ngroups * S;
  const int items_per_cta = (nitems + gridDim.x - 1) / gridDim.x;
  const int tile_begin = blockIdx.x * items_per_cta;
  const int tile_end = min(nitems, tile_begin + items_per_cta);
  const int taps = p.kd * p.kh * p.kw;
  const int cblocks = p.Cin / BKC;
  const int kblocks = taps * cblocks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nstages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);      // one arrive per MMA warp
    }
    for (int a = 0; a < kMaxAcc; ++a) {
      mbar_init(&tfull[a], 4);
      mbar_init(&tempty[a], kEpiWarps);
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  for (int i = threadIdx.x; i < 8 * kEpiGroups * p.Cout; i += blockDim.x) s_stat[i] = 0.f;
  __syncthreads();
  PDL_WAIT();               // everything above is on-chip set-up: it runs under the tail of the previous kernel

  if (warp == 0) {
    // ===================================================== TMA producer
    if (elect_one()) {
      uint32_t it = 0;
      for (int item = tile_begin; item < tile_end; ++item) {
        const int sp = item % S;
        const int tg = item / S;
        int t = tg / p.ngroups;
        const int ng = tg - t * p.ngroups;
        const int iw = t % p.tw; t /= p.tw;
        const int ih = t % p.th; t /= p.th;
        const int id = t % p.td;
        const int n = t / p.td;
        const int w0 = iw * p.bw * p.sw, h0 = ih * p.bh * p.sh, d0 = id * p.bd * p.sd;
        const int kb0 = sp * kblocks / S, kb1 = (sp + 1) * kblocks / S;
        int tap = kb0 / cblocks, cb = kb0 - tap * cblocks;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int kw_ = tap % p.kw, kh_ = (tap / p.kw) % p.kh, kd_ = tap / (p.kw * p.kh);
          const uint32_t s = it % p.nstages;
          const uint32_t ph = (it / p.nstages) & 1u;
          mbar_wait(&empty[s], ph ^ 1u);
          uint8_t* sa = smem + (size_t)s * STAGE;
          mbar_expect_tx(&full[s], A_BYTES + b_bytes_real);
          tma_load_5d(&tmA, sa, &full[s], cb * BKC, w0 + kw_ - p.pw, h0 + kh_ - p.ph, d0 + kd_ - p.pd, n);
          tma_load_2d(&tmB, sa + A_BYTES, &full[s], cb * BKC, p.up ? ng * p.Ntile : tap * p.Cout + ng * p.Ntile);
          if (++cb == cblocks) {
            cb = 0;
            ++tap;
          }
        }
      }
    }
  } else if (warp >= 4 && warp < 8) {
    // ===================================================== MMA warpgroup
    const int wt = threadIdx.x - 128;
    switch (p.Ntile) {
      case 16: tc_mma_role<BKC, 16>(p, smem, STAGE, full, empty, tfull, tempty, s_acc, tile_begin, tile_end, kblocks, wt); break;
      case 32: tc_mma_role<BKC, 32>(p, smem, STAGE, full, empty, tfull, tempty, s_acc, tile_begin, tile_end, kblocks, wt); break;
      case 48: tc_mma_role<BKC, 48>(p, smem, STAGE, full, empty, tfull, tempty, s_acc, tile_begin, tile_end, kblocks, wt); break;
      default: tc_mma_role<BKC, 64>(p, smem, STAGE, full, empty, tfull, tempty, s_acc, tile_begin, tile_end, kblocks, wt); break;
    }
  } else if (warp >= 8) {
    // ===================================================== epilogue warps (8..15), two groups of four
    const int eg = (warp - 8) >> 2;               // group = accumulator slot it drains
    const int q = warp & 3;                       // quarter of the tile rows this warp handles
    const int row = q * 32 + lane;                // row of the M tile = voxel of the box
    const int rw = row % p.bw;
    const int rh = (row / p.bw) % p.bh;
    const int rd = row / (p.bw * p.bh);
    const int etid = (threadIdx.x - 256) & 127;   // 0..127 inside the group
    float* s_stat_g = s_stat + eg * 8 * p.Cout;   // [4 warps][2][Cout] of this group
    int cur_n = -1;
    constexpr int NR = NCH > 0 ? NCH : 1;
    float rs[NR][16], rq[NR][16], rb[NR][16];
#pragma unroll
    for (int ci = 0; ci < NR; ++ci)
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        rs[ci][j] = 0.f;
        rq[ci][j] = 0.f;
        rb[ci][j] = (NCH > 0 && p.bias != nullptr) ? __ldg(p.bias + ci * 16 + j) : 0.f;
      }
    auto flush_stats = [&](int n) {
      if (NCH > 0 && p.stats != nullptr) {
#pragma unroll
        for (int ci = 0; ci < NR; ++ci) {
          stat_butterfly(rs[ci], rq[ci], lane);
          if ((lane & 1) == 0) {
            float* sw_ = s_stat_g + q * 2 * p.Cout;
            sw_[ci * 16 + stat_col(lane)] += rs[ci][0];
            sw_[p.Cout + ci * 16 + stat_col(lane)] += rq[ci][0];
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            rs[ci][j] = 0.f;
            rq[ci][j] = 0.f;
          }
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + eg) : "memory");
      if (p.stats != nullptr && n >= 0) {
        for (int i = etid; i < 2 * p.Cout; i += 128) {
          const int which = i / p.Cout, c = i - which * p.Cout;
          double t = 0.0;
#pragma unroll
          for (int wq = 0; wq < 4; ++wq) {
            t += (double)s_stat_g[wq * 2 * p.Cout + i];
            s_stat_g[wq * 2 * p.Cout + i] = 0.f;
          }
          atomicAdd(p.stats + ((long long)n * p.Cout + c) * 2 + which, t);
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + eg) : "memory");
    };
    for (int item = tile_begin + eg, local = eg; item < tile_end; item += kEpiGroups, local += kEpiGroups) {
      const int sp = item % S;
      const int tg = item / S;
      int t = tg / p.ngroups;
      const int ng = tg - t * p.ngroups;
      const int iw = t % p.tw; t /= p.tw;
      const int ih = t % p.th; t /= p.th;
      const int id = t % p.td;
      const int n = t / p.td;
      const int ow = iw * p.bw + rw, oh = ih * p.bh + rh, od = id * p.bd + rd;
      const bool valid = ow < p.W && oh < p.H && od < p.D;
      const long long vox = (((long long)n * p.D + od) * p.H + oh) * p.W + ow;
      const uint32_t as = (uint32_t)local % (uint32_t)p.nacc;
      const uint32_t aph = ((uint32_t)local / (uint32_t)p.nacc) & 1u;
      mbar_wait(&tfull[as], aph);
      const float* tacc = s_acc + row * p.acc_pitch + as * p.Ntile;
      const float4* slabs = nullptr;
      if (S > 1) {
        // partial sums of this K range -> own slab; the accumulator is free as soon as it has been read
        float4* mine = p.ws + ((size_t)tg * S + sp) * (size_t)(p.Ntile / 4) * 128 + row;
        for (int cc = 0; cc < p.Ntile; cc += 16) {
          float v[16];
          acc_ld16(tacc + cc, v);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            __stcg(mine + (size_t)(cc / 4 + j) * 128, make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&tempty[as]);
        __threadfence();
        asm volatile("bar.sync %0, 128;" ::"r"(1 + eg) : "memory");
        if (etid == 0) s_flag[eg] = atomicAdd(p.cnt + tg, 1u);
        asm volatile("bar.sync %0, 128;" ::"r"(1 + eg) : "memory");
        if (s_flag[eg] != (unsigned int)(S - 1)) continue;      // not the last K range of this (tile, group) to finish
        __threadfence();
        if (etid == 0) p.cnt[tg] = 0u;                           // ready for the next launch
        slabs = p.ws + (size_t)tg * S * (size_t)(p.Ntile / 4) * 128 + row;
      }
      if (n != cur_n) {
        if (cur_n >= 0 && p.stats != nullptr) flush_stats(cur_n);
        cur_n = n;
      }
      for (int cc = 0; cc < p.Ntile; cc += 16) {
        float v[16];
        if (S == 1) {
          acc_ld16(tacc + cc, v);
        } else {
          // fixed order over the K ranges: the result does not depend on which range finished last
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = 0.f;
#pragma unroll 2
          for (int s_ = 0; s_ < S; ++s_) {
            const float4* sl = slabs + (size_t)s_ * (size_t)(p.Ntile / 4) * 128 + (size_t)(cc / 4) * 128;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 f = __ldcg(sl + (size_t)j * 128);
              v[4 * j] += f.x; v[4 * j + 1] += f.y; v[4 * j + 2] += f.z; v[4 * j + 3] += f.w;
            }
          }
        }
        // channel block of this 16-column chunk (UP: columns are (tap, cout); otherwise column group ng of Cout)
        int c0 = ng * p.Ntile + cc;
        long long ovox = vox;
        if (p.up) {
          const int col = ng * p.Ntile + cc;
          const int tp = col / p.Cout;
          c0 = col - tp * p.Cout;
          const int fc = tp % p.uw, fb = (tp / p.uw) % p.uh, fa = tp / (p.uw * p.uh);
          ovox = (((long long)n * (p.D * p.ud) + (od * p.ud + fa)) * (p.H * p.uh) + (oh * p.uh + fb)) * (p.W * p.uw) +
                 (ow * p.uw + fc);
        }
        if (NCH > 0) {
          const int ci = c0 >> 4;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            v[j] += (NCH == 1 || ci == 0) ? rb[0][j] : rb[NR - 1][j];
            const float sv = valid ? v[j] : 0.f;
            if (NCH == 1 || ci == 0) {
              rs[0][j] += sv;
              rq[0][j] = fmaf(sv, sv, rq[0][j]);
            } else {
              rs[NR - 1][j] += sv;
              rq[NR - 1][j] = fmaf(sv, sv, rq[NR - 1][j]);
            }
          }
        } else {
          if (p.bias != nullptr) {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] += __ldg(p.bias + c0 + j);
          }
          if (p.stats != nullptr) {
            float s[16], qq[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              s[j] = valid ? v[j] : 0.f;
              qq[j] = s[j] * s[j];
            }
            stat_butterfly(s, qq, lane);
            if ((lane & 1) == 0) {
              // this lane is the only writer of its column in this warp's private row: no atomics, fixed order
              float* sw_ = s_stat_g + q * 2 * p.Cout;
              sw_[c0 + stat_col(lane)] += s[0];
              sw_[p.Cout + c0 + stat_col(lane)] += qq[0];
            }
          }
        }
        if (valid) {
          if (p.addend != nullptr) {
            float r[16];
            load8(p.addend + ovox * p.ald + c0, r);
            load8(p.addend + ovox * p.ald + c0 + 8, r + 8);
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] += r[j];
          }
          store8(p.y + ovox * p.yld + c0, v);
          store8(p.y + ovox * p.yld + c0 + 8, v + 8);
        }
      }
      if (S == 1) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&tempty[as]);
      }
    }
    if (p.stats != nullptr && cur_n >= 0) flush_stats(cur_n);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static bool al16p(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

static int pick_bkc(int cin) {
  if (cin % 64 == 0) return 64;
  if (cin == 32) return 32;
  if (cin == 16) return 16;
  return 0;
}

int conv_tc_channels_ok(int kind, int cin, int cout) {
  if (kind < B200SEG_K3 || kind > B200SEG_UP) return 0;
  if (pick_bkc(cin) == 0) return 0;
  if (cout < 16 || cout > 256 || (cout % 16) != 0) return 0;
  // transposed conv: the (tap, cout) columns are split into groups of <= 256 whole taps
  if (kind == B200SEG_UP && (cout & (cout - 1)) != 0) return 0;
  return 1;
}

int conv_tc_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                      const b200seg_tensor* addend) {
  if (w_dtype != B200SEG_BF16_TC) return 0;
  if (!conv_tc_channels_ok(kind, x->c, y->c)) return 0;
  if (x->dtype != B200SEG_BF16 || y->dtype != B200SEG_BF16) return 0;
  if (addend && addend->dtype != B200SEG_BF16) return 0;
  if ((x->ld % 8) || (y->ld % 8) || !al16p(x->ptr) || !al16p(y->ptr)) return 0;
  if (addend && ((addend->ld % 8) || !al16p(addend->ptr))) return 0;
  ConvGeom g;
  if (conv_geometry(kind, dims, &g) != 0) return 0;
  if (g.up) {
    if (y->d != x->d * g.ud || y->h != x->h * g.uh || y->w != x->w * g.uw) return 0;
  } else {
    if (x->d != y->d * g.sd || x->h != y->h * g.sh || x->w != y->w * g.sw) return 0;
  }
  return 1;
}

void tc_pick_box(int W, int H, int D, int* bw, int* bh, int* bd) {
  long long best = -1;
  int bb[3] = {16, 8, 1};
  for (int w = 1; w <= 128; w *= 2)
    for (int h = 1; w * h <= 128; h *= 2) {
      int d = 128 / (w * h);
      if (d > 128) continue;
      long long padded = (long long)((W + w - 1) / w * w) * ((H + h - 1) / h * h) * ((D + d - 1) / d * d);
      // prefer less padding, then wider rows (longer contiguous runs in memory)
      long long score = padded * 1024 - w * 4 - h;
      if (best < 0 || score < best) {
        best = score;
        bb[0] = w; bb[1] = h; bb[2] = d;
      }
    }
  *bw = bb[0]; *bh = bb[1]; *bd = bb[2];
}

static int g_smem_optin[64] = {0};

// split-K scratch: kKsPool slabs per device, handed to streams in order of first use (no CUDA call at hand-out time, so
// a stream first seen during graph capture still gets one); launches on one stream are ordered, so they share a slab
constexpr int kKsPool = 4;
constexpr size_t kKsBytes = 12u << 20;
constexpr int kKsCntWords = 1024;
struct KsSlab {
  void* base = nullptr;
  cudaStream_t owner = nullptr;
  bool taken = false;
};
static KsSlab g_ks[64][kKsPool];
static std::mutex g_ks_mutex;

static bool ks_workspace(int device, cudaStream_t st, float4** ws, unsigned int** cnt) {
  if (device < 0 || device >= 64) return false;
  std::lock_guard<std::mutex> lock(g_ks_mutex);
  for (int i = 0; i < kKsPool; ++i) {
    KsSlab& k = g_ks[device][i];
    if (k.base == nullptr) return false;
    if (!k.taken) {
      k.taken = true;
      k.owner = st;
    }
    if (k.owner == st) {
      *cnt = static_cast<unsigned int*>(k.base);
      *ws = reinterpret_cast<float4*>(static_cast<char*>(k.base) + kKsCntWords * sizeof(unsigned int));
      return true;
    }
  }
  return false;
}

int wgrad_tc_init(int device, int maxsm);
int tc_max_smem(int device) { return (device >= 0 && device < 64 && g_smem_optin[device] > 0) ? g_smem_optin[device] : 227 * 1024; }

int conv_tc_init(int device) {
  if (device < 0 || device >= 64) return B200SEG_OK;
  if (g_smem_optin[device]) return B200SEG_OK;
  int maxsm = 0;
  B200_CUDA(cudaDeviceGetAttribute(&maxsm, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
#define TC_ATTR(B, C) \
  B200_CUDA(cudaFuncSetAttribute(conv_tc_kernel<B, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm))
  TC_ATTR(16, 0); TC_ATTR(16, 1); TC_ATTR(16, 2);
  TC_ATTR(32, 0); TC_ATTR(32, 1); TC_ATTR(32, 2);
  TC_ATTR(64, 0); TC_ATTR(64, 1); TC_ATTR(64, 2);
#undef TC_ATTR
  if (wgrad_tc_init(device, maxsm) != B200SEG_OK) return B200SEG_ECUDA;
  for (int i = 0; i < kKsPool; ++i) {
    void* base = nullptr;
    const size_t bytes = kKsCntWords * sizeof(unsigned int) + kKsBytes;
    if (cudaMalloc(&base, bytes) != cudaSuccess || cudaMemset(base, 0, kKsCntWords * sizeof(unsigned int)) != cudaSuccess) {
      cudaGetLastError();     // no scratch: the split-K form is simply not used
      break;
    }
    std::lock_guard<std::mutex> lock(g_ks_mutex);
    g_ks[device][i].base = base;
  }
  g_smem_optin[device] = maxsm;
  return B200SEG_OK;
}

int conv_tc(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias, const b200seg_tensor* y,
            double* stats, const b200seg_tensor* addend, int device, cudaStream_t st) {
  if (tc_encode_fn() == nullptr) return B200SEG_ECUDA;
  if (conv_tc_init(device) != B200SEG_OK) return B200SEG_ECUDA;
  ConvGeom g;
  conv_geometry(kind, dims, &g);
  TcArgs p;
  p.y = static_cast<bf16*>(y->ptr);
  p.addend = addend ? static_cast<const bf16*>(addend->ptr) : nullptr;
  p.bias = bias;
  p.stats = stats;
  p.yld = y->ld;
  p.ald = addend ? addend->ld : 0;
  p.N = x->n;
  if (g.up) { p.D = x->d; p.H = x->h; p.W = x->w; } else { p.D = y->d; p.H = y->h; p.W = y->w; }
  p.Cin = x->c; p.Cout = y->c;
  p.kd = g.kd; p.kh = g.kh; p.kw = g.kw; p.pd = g.pd; p.ph = g.ph; p.pw = g.pw;
  p.sd = g.sd; p.sh = g.sh; p.sw = g.sw;
  p.up = g.up; p.ud = g.ud; p.uh = g.uh; p.uw = g.uw;
  const int ncols = g.up ? g.ud * g.uh * g.uw * p.Cout : p.Cout;
  p.Ntile = kTcMaxN;
  while (ncols % p.Ntile) p.Ntile -= 16;       // widest column group (multiple of 16, <= 64) that divides the columns
  p.ngroups = ncols / p.Ntile;
  p.ksplit = 1;
  p.ws = nullptr;
  p.cnt = nullptr;
  {
    // few voxel tiles (deep, small levels): spread the layer over the chip.  With a long (tap, channel-block) loop,
    // cut the loop (split-K, column groups of >= 64 so the activation tile is not re-read more than needed); else
    // split the output channels only: every group re-reads the activation tile (cheap, it is L2 resident) but only
    // its own weights
    int bw_, bh_, bd_;
    tc_pick_box(p.W, p.H, p.D, &bw_, &bh_, &bd_);
    const int tiles = p.N * ((p.W + bw_ - 1) / bw_) * ((p.H + bh_ - 1) / bh_) * ((p.D + bd_ - 1) / bd_);
    const int sms = num_sms(device);
    const int kblocks = g.kd * g.kh * g.kw * (p.Cin / pick_bkc(p.Cin));
    // B200SEG_TC_KSPLIT (0: off, n >= 2: at most n ranges, unset: automatic) is read on every call: it is how the
    // split-K test reaches the unsplit kernel on the same shape as its reference, and how it caps the ranges
    const char* e = getenv("B200SEG_TC_KSPLIT");
    const int ks_max = e ? atoi(e) : 16;
    if (!g.up && kblocks >= 16 && ks_max >= 2) {
      int nt = p.Ntile, ngp = p.ngroups;
      while (tiles * ngp * 2 <= sms && nt >= 128 && (nt / 2) % 16 == 0) {
        nt /= 2;
        ngp *= 2;
      }
      int S = sms / (tiles * ngp);
      if (S > kblocks / 4) S = kblocks / 4;
      if (S > ks_max) S = ks_max;
      if (S >= 2 && tiles * ngp <= kKsCntWords && (size_t)tiles * ngp * S * 128 * nt * sizeof(float) <= kKsBytes &&
          ks_workspace(device, st, &p.ws, &p.cnt)) {
        p.Ntile = nt;
        p.ngroups = ngp;
        p.ksplit = S;
      }
    }
    while (p.ksplit == 1 && !g.up && tiles * p.ngroups * 2 <= sms && p.Ntile >= 64 && (p.Ntile / 2) % 16 == 0) {
      p.Ntile /= 2;
      p.ngroups *= 2;
    }
  }
  tc_pick_box(p.W, p.H, p.D, &p.bw, &p.bh, &p.bd);
  p.tw = (p.W + p.bw - 1) / p.bw;
  p.th = (p.H + p.bh - 1) / p.bh;
  p.td = (p.D + p.bd - 1) / p.bd;
  p.ntiles = p.N * p.td * p.th * p.tw;
  const int bkc = pick_bkc(p.Cin);
  const uint32_t swz = bkc * 2;
  const uint32_t a_bytes = 128u * swz;
  const uint32_t b_bytes = (((uint32_t)p.Ntile * swz) + 1023u) & ~1023u;
  const uint32_t stage = a_bytes + b_bytes;
  // barriers, statistics rows, flags and the accumulator staging tile (128 rows of nacc*Ntile + 4 floats)
  const uint32_t tail = (2 * kMaxStages + 2 * kMaxAcc) * 8 + 8 * kEpiGroups * p.Cout * 4 + 16 + 16 +
                        128u * (uint32_t)(kMaxAcc * p.Ntile + 4) * 4u;
  const int maxsm = g_smem_optin[device] > 0 ? g_smem_optin[device] : 227 * 1024;
  int nst = (int)((maxsm - 1024 - (int)tail - 256) / (int)stage);
  if (nst > kMaxStages) nst = kMaxStages;
  B200_CHECK_ARG(nst >= 2, "conv_tc: tile does not fit in shared memory (Cin=%d Cout=%d)", p.Cin, p.Cout);
  p.nstages = nst;
  p.nacc = kMaxAcc;
  p.acc_pitch = p.nacc * p.Ntile + 4;
  const size_t smem_bytes = 1024 + (size_t)nst * stage + tail + 128;

  // ---- tensor maps
  CUtensorMap tmA, tmB;
  const CUtensorMapSwizzle sw = bkc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                          : (bkc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  {
    cuuint64_t dims5[5] = {(cuuint64_t)p.Cin, (cuuint64_t)x->w, (cuuint64_t)x->h, (cuuint64_t)x->d, (cuuint64_t)p.N};
    cuuint64_t strides[4] = {(cuuint64_t)x->ld * 2, (cuuint64_t)x->ld * 2 * x->w, (cuuint64_t)x->ld * 2 * x->w * x->h,
                             (cuuint64_t)x->ld * 2 * x->w * x->h * x->d};
    // strided gather (k2s2 down conv): the box spans s*b positions traversed with element stride s
    cuuint32_t box[5] = {(cuuint32_t)bkc, (cuuint32_t)(p.bw * p.sw), (cuuint32_t)(p.bh * p.sh),
                         (cuuint32_t)(p.bd * p.sd), 1};
    cuuint32_t estr[5] = {1, (cuuint32_t)p.sw, (cuuint32_t)p.sh, (cuuint32_t)p.sd, 1};
    CUresult r = g_encode(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, x->ptr, dims5, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_CHECK_ARG(r == CUDA_SUCCESS, "conv_tc: cuTensorMapEncodeTiled(A) failed with %d", (int)r);
  }
  {
    const int rows = g.up ? ncols : g.kd * g.kh * g.kw * p.Cout;
    cuuint64_t dims2[2] = {(cuuint64_t)p.Cin, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)p.Cin * 2};
    cuuint32_t box[2] = {(cuuint32_t)bkc, (cuuint32_t)p.Ntile};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(&tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(wpk), dims2, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_CHECK_ARG(r == CUDA_SUCCESS, "conv_tc: cuTensorMapEncodeTiled(B) failed with %d", (int)r);
  }
  int grid = num_sms(device);
  if (grid > p.ntiles * p.ngroups * p.ksplit) grid = p.ntiles * p.ngroups * p.ksplit;
  const int nch = p.Cout == 16 ? 1 : (p.Cout == 32 ? 2 : 0);
#define TC_LAUNCH(B)                                                                         \
  do {                                                                                       \
    if (nch == 1) launch_k(conv_tc_kernel<B, 1>, grid, kTcThreads, smem_bytes, st, tmA, tmB, p);          \
    else if (nch == 2) launch_k(conv_tc_kernel<B, 2>, grid, kTcThreads, smem_bytes, st, tmA, tmB, p);     \
    else launch_k(conv_tc_kernel<B, 0>, grid, kTcThreads, smem_bytes, st, tmA, tmB, p);                   \
  } while (0)
  if (bkc == 64) TC_LAUNCH(64);
  else if (bkc == 32) TC_LAUNCH(32);
  else TC_LAUNCH(16);
#undef TC_LAUNCH
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
