// Halo-staged wgmma 3x3x3 convolution with STREAMED weights for the 64/128-channel pyramid levels (sm_90a, bf16).
//
// At 24^3 / 12^3 voxels the TMA im2col path (conv_tc.cu) is bound by what one SM can ingest: every 128-voxel tile
// pulls 27 shifted copies of its activation box plus all 27 tap blocks of the weights through L2->smem
// (0.66 MB per tile at 64 channels) while the tensor core waits.  This kernel removes both multipliers:
//   * activations: as in conv_halo.cu, an (8 wide x 16 high) output column keeps its input d-slices (one-voxel
//     halo, zero filled = conv padding) channel-planar in shared memory and all 27 taps are descriptor VIEWS of
//     them (no-swizzle K-major canonical layout: SBO = one halo row, LBO = one 8-channel plane);
//   * weights: a work item covers NACC consecutive output slices of the column and NT output channels.  Each of the
//     27 tap blocks ([Cin/8][NT][8] bf16, 4-8 KB) is streamed ONCE per item through a cp.async.bulk ring (as deep as
//     the shared memory left over allows: the blocks in flight hide the L2 latency of the stream) and
//     multiplied into all NACC accumulators (registers of the MMA warpgroup, NACC x NT columns) before the next
//     block is needed: weight traffic per tile drops by NACC, activation traffic by ~27 / (1 + 2/NACC).  At the end
//     of an item the accumulators go to a staging tile in shared memory (double buffered where it fits).
// Items = samples x columns x ceil(D / NACC) x (Cout / NT), so even the 12^3 level spreads over ~100 CTAs.
// Warp roles (544 threads): warps 0-3 MMA warpgroup, warps 4-7 epilogue (bias, GroupNorm statistics, residual
// addend, bf16 NDHWC stores), warps 8-15 slice loaders (cp.async, zero fill), warp 16 weight streamer.
#include "tc_common.cuh"

namespace b200seg {

constexpr int WS_TW = 8, WS_TH = 16;                 // output tile (w, h); M = 128 rows = (hh, ww)
constexpr int WS_PW = WS_TW + 2, WS_PH = WS_TH + 2;
constexpr int kWsMaxSlices = 8;
constexpr int kWsLoaderWarps = 8;
constexpr int kWsThreads = 32 * (4 + 4 + kWsLoaderWarps + 1);
constexpr int kWsMaxWStages = 16;     // weight ring depth is chosen at launch from the shared memory left over

struct HaloWsArgs {
  const bf16* x;
  const bf16* w;          // packed [group][tap][Cin/8][NT][8]
  bf16* y;
  const bf16* addend;
  const float* bias;
  double* stats;
  long long xld, yld, ald;
  int N, D, H, W;
  int Cin, Cout;
  int tw, th;             // tiles along w, h
  int ndchunks;           // items along d (NACC output slices each)
  int ngroups;            // output-channel groups of NT columns
  int nitems;             // N * th * tw * ndchunks * ngroups
  int nslices;            // ring size (>= NACC + 2)
  int wstages;            // weight ring depth (tap blocks in flight)
  int accslots;           // accumulator staging slots in shared memory (1 or 2)
  int acc_pitch;          // floats per staging row: accslots * NACC * NT + 4
  // GroupNorm-backward sums fused into the data-gradient epilogue (b200seg_conv_bwdstats; see conv_halo.cu)
  const bf16* yfwd;
  long long yfld;
  const double* gstats;
  const float* ggamma;
  const float* gbeta;
  const float* gscale;
  int ggroups;
  double gm;
  float geps;
};

__device__ __forceinline__ uint64_t ws_nosw_desc(uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}

template <int CIN, int NT, int NACC, bool BWD>
__global__ void __launch_bounds__(kWsThreads, 1) conv_halows_kernel(const HaloWsArgs p) {
  PDL_TRIGGER();
  constexpr int CP = CIN / 8;                                // 8-channel planes
  constexpr uint32_t PLANE = WS_PH * WS_PW * 16u;            // bytes of one plane of one slice
  constexpr uint32_t SLICE = (uint32_t)CP * PLANE;
  constexpr int TAPS = 27;
  constexpr uint32_t TAP_BYTES = (uint32_t)CIN * NT * 2u;
  constexpr int NSL = NACC + 2;                              // input slices of a full item
  constexpr int kMaxPieces = (WS_PH * WS_PW * CP + 32 * kWsLoaderWarps - 1) / (32 * kWsLoaderWarps);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  uint8_t* s_w = smem;
  uint8_t* s_ring = smem + (size_t)p.wstages * TAP_BYTES;
  uint8_t* tail = s_ring + (size_t)p.nslices * SLICE;
  uint64_t* sfull = reinterpret_cast<uint64_t*>(tail);
  uint64_t* sempty = sfull + kWsMaxSlices;
  uint64_t* tfull = sempty + kWsMaxSlices;
  uint64_t* tempty = tfull + 2;
  uint64_t* wfull = tempty + 2;
  uint64_t* wempty = wfull + kWsMaxWStages;
  float* s_stat = reinterpret_cast<float*>(wempty + kWsMaxWStages);   // [4 epilogue warps][2][Cout]
  float* s_ab = s_stat + 8 * p.Cout;                         // [2][Cout]: A, B of the sample being processed (BWD)
  double* s_gd = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(s_ab + 2 * p.Cout) + 7) & ~(uintptr_t)7);
  float* s_acc = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(s_gd + 2 * p.Cout + 16) + 15) & ~(uintptr_t)15);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int items_per_cta = (p.nitems + gridDim.x - 1) / gridDim.x;
  const int item_begin = blockIdx.x * items_per_cta;
  const int item_end = min(p.nitems, item_begin + items_per_cta);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nslices; ++s) {
      mbar_init(&sfull[s], 32 * kWsLoaderWarps);     // one deferred cp.async arrive per loader thread
      mbar_init(&sempty[s], 4);                      // one arrive per MMA warp
    }
    for (int a = 0; a < 2; ++a) {
      mbar_init(&tfull[a], 4);
      mbar_init(&tempty[a], 4);
    }
    for (int a = 0; a < p.wstages; ++a) {
      mbar_init(&wfull[a], 1);
      mbar_init(&wempty[a], 4);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 8 * p.Cout; i += blockDim.x) s_stat[i] = 0.f;
  fence_proxy_async();
  __syncthreads();
  PDL_WAIT();               // barriers and the statistics rows are set up under the tail of the previous kernel

  // item -> (sample, column, first output slice, slices, channel group); the channel group is the fastest index
  auto decode = [&](int item, int& n, int& h0, int& w0, int& d0, int& nd, int& ng) {
    int t = item / p.ngroups;
    ng = item - t * p.ngroups;
    const int dc = t % p.ndchunks; t /= p.ndchunks;
    const int iw = t % p.tw; t /= p.tw;
    const int ih = t % p.th;
    n = t / p.th;
    w0 = iw * WS_TW;
    h0 = ih * WS_TH;
    d0 = dc * NACC;
    nd = min(NACC, p.D - d0);
  };

  if (warp < 4) {
    // ===================================================== MMA warpgroup
    const int wt = threadIdx.x;
    const uint64_t a_hi = ws_nosw_desc(PLANE, WS_PW * 16u);
    const uint64_t b_hi = ws_nosw_desc((uint32_t)NT * 16u, 128u);
    const uint32_t ring_u32 = smem_u32(s_ring);
    const uint32_t w_u32 = smem_u32(s_w);
    constexpr int kchunks = CIN / 16;
    uint32_t gs = 0;    // slices consumed so far
    uint32_t gi = 0;    // items done (accumulator slot = gi % accslots)
    uint32_t wst = 0;   // weight blocks consumed so far
    for (int item = item_begin; item < item_end; ++item, ++gi) {
      int n, h0, w0, d0, nd, ng;
      decode(item, n, h0, w0, d0, nd, ng);
      const int nsl = nd + 2;
      const uint32_t as = gi % (uint32_t)p.accslots;
      float acc0[NACC][NT / 2], acc1[NACC][NT / 2];
#pragma unroll
      for (int j = 0; j < NACC; ++j) {
        frag_zero(acc0[j]);
        frag_zero(acc1[j]);
      }
      // slices are waited for when first needed: kd = 0 touches slices 0..nd-1, every further kd one more,
      // so the multiplications start while the tail of the item's slices is still in flight
      auto wait_slice = [&](int k) {
        const uint32_t sl = gs + (uint32_t)k;
        mbar_wait(&sfull[sl % (uint32_t)p.nslices], (sl / (uint32_t)p.nslices) & 1u);
      };
#pragma unroll
      for (int kd_ = 0; kd_ < 3; ++kd_) {
        if (kd_ == 0) {
          for (int k = 0; k < nd; ++k) wait_slice(k);
        } else {
          wait_slice(nd - 1 + kd_);
        }
        fence_proxy_async();      // cp.async (generic proxy) writes -> tensor core (async proxy) reads
#pragma unroll
        for (int kh_ = 0; kh_ < 3; ++kh_)
#pragma unroll
          for (int kw_ = 0; kw_ < 3; ++kw_) {
            const uint32_t wq = wst + (uint32_t)((kd_ * 3 + kh_) * 3 + kw_);
            const uint32_t stg = wq % (uint32_t)p.wstages;
            mbar_wait(&wfull[stg], (wq / (uint32_t)p.wstages) & 1u);
            const uint64_t b_tap = b_hi | (uint64_t)((w_u32 + stg * TAP_BYTES) >> 4);
#pragma unroll
            for (int j = 0; j < NACC; ++j) {
              wgmma_fence_regs(acc0[j]);
              wgmma_fence_regs(acc1[j]);
            }
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < NACC; ++j) {
              if (NACC == 1 || j < nd) {
                const uint32_t sl = gs + (uint32_t)(j + kd_);
                const uint64_t a_base = a_hi | (uint64_t)((ring_u32 + (sl % (uint32_t)p.nslices) * SLICE) >> 4);
#pragma unroll
                for (int kc = 0; kc < kchunks; ++kc) {
                  const uint32_t a_off = ((uint32_t)(2 * kc) * PLANE + (uint32_t)(kh_ * WS_PW + kw_) * 16u) >> 4;
                  const uint32_t b_off = ((uint32_t)(kc * 2 * NT) * 16u) >> 4;
                  Wgmma<NT, 0, 0>::mma(acc0[j], a_base + a_off, b_tap + b_off);
                  // rows 64..127 of the tile (hh = 8..15) start 8 halo rows further on
                  Wgmma<NT, 0, 0>::mma(acc1[j], a_base + a_off + (8u * WS_PW * 16u >> 4), b_tap + b_off);
                }
              }
            }
            wgmma_commit();
            wgmma_wait0();
#pragma unroll
            for (int j = 0; j < NACC; ++j) {
              wgmma_fence_regs(acc0[j]);
              wgmma_fence_regs(acc1[j]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&wempty[stg]);
          }
      }
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int k = 0; k < NSL; ++k)
          if (k < nsl) mbar_arrive(&sempty[(gs + (uint32_t)k) % (uint32_t)p.nslices]);
      }
      mbar_wait(&tempty[as], ((gi / (uint32_t)p.accslots) & 1u) ^ 1u);
#pragma unroll
      for (int j = 0; j < NACC; ++j) {
        float* acc = s_acc + as * (uint32_t)(NACC * NT) + j * NT;
        frag_store(acc, p.acc_pitch, 0, acc0[j], wt);
        frag_store(acc, p.acc_pitch, 64, acc1[j], wt);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&tfull[as]);
      gs += (uint32_t)nsl;
      wst += TAPS;
    }
  } else if (warp == 8 + kWsLoaderWarps) {
    // ===================================================== weight streamer: tap blocks -> ring (one lane)
    if (lane == 0) {
      uint32_t wst = 0;
      for (int item = item_begin; item < item_end; ++item) {
        int n, h0, w0, d0, nd, ng;
        decode(item, n, h0, w0, d0, nd, ng);
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + (size_t)ng * TAPS * TAP_BYTES;
        for (int tap = 0; tap < TAPS; ++tap, ++wst) {
          const uint32_t stg = wst % (uint32_t)p.wstages;
          mbar_wait(&wempty[stg], ((wst / (uint32_t)p.wstages) & 1u) ^ 1u);
          mbar_expect_tx(&wfull[stg], TAP_BYTES);
          asm volatile(
              "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                  smem_u32(s_w + (size_t)stg * TAP_BYTES)),
              "l"(wsrc + (size_t)tap * TAP_BYTES), "r"(TAP_BYTES), "r"(smem_u32(&wfull[stg]))
              : "memory");
        }
      }
    }
  } else if (warp >= 8) {
    // ===================================================== slice loaders (8 warps, cp.async with zero fill)
    constexpr int LT = 32 * kWsLoaderWarps;
    const int lt = threadIdx.x - 256;
    const int pieces = WS_PH * WS_PW * CP;
    int poff[kMaxPieces], phh[kMaxPieces], pww[kMaxPieces];
    bool pval[kMaxPieces];
#pragma unroll
    for (int j = 0; j < kMaxPieces; ++j) {
      const int q = lt + j * LT;
      pval[j] = q < pieces;
      const int qq = pval[j] ? q : 0;
      const int v = qq / CP, plane = qq - v * CP;
      phh[j] = v / WS_PW;
      pww[j] = (v - phh[j] * WS_PW) | (plane << 16);
      poff[j] = plane * (int)PLANE + v * 16;
    }
    uint32_t sl = 0;
    for (int item = item_begin; item < item_end; ++item) {
      int n, h0, w0, d0, nd, ng;
      decode(item, n, h0, w0, d0, nd, ng);
      const int nsl = nd + 2;
      for (int i = 0; i < nsl; ++i, ++sl) {
        const uint32_t slot = sl % (uint32_t)p.nslices;
        mbar_wait(&sempty[slot], ((sl / (uint32_t)p.nslices) & 1u) ^ 1u);
        const uint32_t dst = smem_u32(s_ring + (size_t)slot * SLICE);
        const int d = d0 - 1 + i;
        const bool dok = (unsigned)d < (unsigned)p.D;
        const bf16* src = p.x + (((long long)n * p.D + (dok ? d : 0)) * p.H) * p.W * p.xld;
#pragma unroll
        for (int j = 0; j < kMaxPieces; ++j) {
          if (!pval[j]) continue;
          const int plane = pww[j] >> 16, ww = pww[j] & 0xffff;
          const int h = h0 - 1 + phh[j], w = w0 - 1 + ww;
          const bool ok = dok && (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
          const bf16* g = ok ? src + ((long long)h * p.W + w) * p.xld + plane * 8 : p.x;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + (uint32_t)poff[j]), "l"(g),
                       "r"(ok ? 16 : 0)
                       : "memory");
        }
        asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&sfull[slot])) : "memory");
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // ===================================================== epilogue warps 4..7
    const int q = warp & 3;
    const int row = q * 32 + lane;
    const int rw = row % WS_TW, rh = row / WS_TW;
    const int etid = (warp - 4) * 32 + lane;
    uint32_t gi = 0;
    int cur_n = -1;
    auto flush_stats = [&](int n) {
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (p.stats != nullptr && n >= 0) {
        for (int i = etid; i < 2 * p.Cout; i += 128) {
          const int which = i / p.Cout, c = i - which * p.Cout;
          double t = 0.0;
#pragma unroll
          for (int wq = 0; wq < 4; ++wq) {
            t += (double)s_stat[wq * 2 * p.Cout + i];
            s_stat[wq * 2 * p.Cout + i] = 0.f;
          }
          atomicAdd(p.stats + ((long long)n * p.Cout + c) * (BWD ? 3 : 2) + which, t);
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    };
    // A, B of sample n for the ReLU mask of the backward sums: same expressions and precision as gn_cta_coefs
    auto load_coefs = [&](int n) {
      const int C = p.Cout, cpg = C / p.ggroups;
      for (int c = etid; c < C; c += 128) {
        const double* q_ = p.gstats + ((long long)n * C + c) * 2;
        s_gd[c] = q_[0];
        s_gd[C + c] = q_[1];
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (etid < p.ggroups) {
        double sm = 0.0, sq = 0.0;
        for (int k_ = 0; k_ < cpg; ++k_) {
          sm += s_gd[etid * cpg + k_];
          sq += s_gd[C + etid * cpg + k_];
        }
        const double mean = sm / p.gm;
        double var = sq / p.gm - mean * mean;
        if (var < 0.0) var = 0.0;
        s_gd[2 * C + etid * 2 + 0] = mean;
        s_gd[2 * C + etid * 2 + 1] = rsqrt(var + (double)p.geps);
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      for (int c = etid; c < C; c += 128) {
        const int g_ = c / cpg;
        const double mean = s_gd[2 * C + g_ * 2 + 0], rstd = s_gd[2 * C + g_ * 2 + 1];
        const double sc = p.gscale ? (double)p.gscale[(long long)n * C + c] : 1.0;
        const double ga = (double)p.ggamma[c], be = (double)p.gbeta[c];
        s_ab[c] = (float)(rstd * ga * sc);
        s_ab[C + c] = (float)((be - mean * rstd * ga) * sc);
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    };
    for (int item = item_begin; item < item_end; ++item, ++gi) {
      int n, h0, w0, d0, nd, ng;
      decode(item, n, h0, w0, d0, nd, ng);
      if (n != cur_n) {
        if (cur_n >= 0 && p.stats != nullptr) flush_stats(cur_n);
        cur_n = n;
        if constexpr (BWD) load_coefs(n);
      }
      const int oh = h0 + rh, ow = w0 + rw;
      const bool valid = oh < p.H && ow < p.W;
      const int cbase = ng * NT;
      const uint32_t as = gi % (uint32_t)p.accslots;
      mbar_wait(&tfull[as], (gi / (uint32_t)p.accslots) & 1u);
      const float* tacc = s_acc + row * p.acc_pitch + as * (NACC * NT);
      // GroupNorm statistics: per-thread (row) partials over the item's tiles, ONE warp fold per 16-column chunk
      // and item (chunk-outer order keeps only one chunk's partials in registers)
#pragma unroll 1
      for (int c = 0; c < NT / 16; ++c) {
        const int c0 = cbase + c * 16;
        float rs[16], rq[16], bv[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          rs[j] = rq[j] = 0.f;
          bv[j] = p.bias != nullptr ? __ldg(p.bias + c0 + j) : 0.f;
        }
        for (int o = 0; o < nd; ++o) {
          const long long vox = (((long long)n * p.D + (d0 + o)) * p.H + oh) * p.W + ow;
          uint4 yfv[2];
          if constexpr (BWD) {
            yfv[0] = yfv[1] = make_uint4(0u, 0u, 0u, 0u);
            if (valid) {
              yfv[0] = *reinterpret_cast<const uint4*>(p.yfwd + vox * p.yfld + c0);
              yfv[1] = *reinterpret_cast<const uint4*>(p.yfwd + vox * p.yfld + c0 + 8);
            }
          }
          float v[16];
          acc_ld16(tacc + o * NT + c * 16, v);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            v[j] += bv[j];
            if constexpr (!BWD) {
              const float sv = valid ? v[j] : 0.f;
              rs[j] += sv;
              rq[j] = fmaf(sv, sv, rq[j]);
            }
          }
          if (valid) {
            if (p.addend != nullptr) {
              float r[16];
              load8(p.addend + vox * p.ald + c0, r);
              load8(p.addend + vox * p.ald + c0 + 8, r + 8);
#pragma unroll
              for (int j = 0; j < 16; ++j) v[j] += r[j];
            }
            if constexpr (!BWD) {
              store8(p.y + vox * p.yld + c0, v);
              store8(p.y + vox * p.yld + c0 + 8, v + 8);
            } else {
              // g is rounded to bf16 once: what is stored is what the sums see (as a separate reduce pass would)
#pragma unroll
              for (int h_ = 0; h_ < 2; ++h_) {
                uint4 pk;
                __nv_bfloat162* g2 = reinterpret_cast<__nv_bfloat162*>(&pk);
#pragma unroll
                for (int j = 0; j < 4; ++j) g2[j] = __floats2bfloat162_rn(v[8 * h_ + 2 * j], v[8 * h_ + 2 * j + 1]);
                *reinterpret_cast<uint4*>(p.y + vox * p.yld + c0 + 8 * h_) = pk;
                const __nv_bfloat162* y2 = reinterpret_cast<const __nv_bfloat162*>(&yfv[h_]);
                const int cb = c0 + 8 * h_;
                const float4 a0 = *reinterpret_cast<const float4*>(s_ab + cb), a1 = *reinterpret_cast<const float4*>(s_ab + cb + 4);
                const float4 b0 = *reinterpret_cast<const float4*>(s_ab + p.Cout + cb);
                const float4 b1 = *reinterpret_cast<const float4*>(s_ab + p.Cout + cb + 4);
                const float aa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float2 yy = __bfloat1622float2(y2[j]);
                  const float2 gg = __bfloat1622float2(g2[j]);
                  const float d0_ = fmaf(yy.x, aa[2 * j], bb[2 * j]) > 0.f ? gg.x : 0.f;
                  const float d1_ = fmaf(yy.y, aa[2 * j + 1], bb[2 * j + 1]) > 0.f ? gg.y : 0.f;
                  rs[8 * h_ + 2 * j] += d0_;
                  rs[8 * h_ + 2 * j + 1] += d1_;
                  rq[8 * h_ + 2 * j] = fmaf(d0_, yy.x, rq[8 * h_ + 2 * j]);
                  rq[8 * h_ + 2 * j + 1] = fmaf(d1_, yy.y, rq[8 * h_ + 2 * j + 1]);
                }
              }
            }
          }
        }
        if (c == NT / 16 - 1) {
          // the accumulators are drained: hand them back before the last (register-only) statistics fold
          __syncwarp();
          if (lane == 0) mbar_arrive(&tempty[as]);
        }
        if (p.stats != nullptr) {
#pragma unroll
          for (int half = 8, off = 16; half >= 1; half >>= 1, off >>= 1) {
            const bool up = (lane & off) != 0;
#pragma unroll
            for (int j = 0; j < half; ++j) {
              const float keep_s = up ? rs[j + half] : rs[j];
              const float send_s = up ? rs[j] : rs[j + half];
              const float keep_q = up ? rq[j + half] : rq[j];
              const float send_q = up ? rq[j] : rq[j + half];
              rs[j] = keep_s + __shfl_xor_sync(0xffffffffu, send_s, off);
              rq[j] = keep_q + __shfl_xor_sync(0xffffffffu, send_q, off);
            }
          }
          rs[0] += __shfl_xor_sync(0xffffffffu, rs[0], 1);
          rq[0] += __shfl_xor_sync(0xffffffffu, rq[0], 1);
          if ((lane & 1) == 0) {
            const int col = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
            float* sw_ = s_stat + q * 2 * p.Cout;     // this warp's private row: no atomics, fixed order
            sw_[c0 + col] += rs[0];
            sw_[p.Cout + c0 + col] += rq[0];
          }
        }
      }
    }
    if (p.stats != nullptr && cur_n >= 0) flush_stats(cur_n);
  }
}

// ------------------------------------------------------------------------------------------------
static bool al16w(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

// columns per work item for a given input channel count (0: not handled by this kernel)
int conv_halows_ntile(int kind, int cin, int cout) {
  if (kind != B200SEG_K3) return 0;
  if (cin != 64 && cin != 128) return 0;
  if (cout % 64 != 0 || cout > 256) return 0;
  return 64;
}

int conv_halows_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                          const b200seg_tensor* addend) {
  if (w_dtype != B200SEG_BF16_HALO_WS || dims != 3) return 0;
  if (conv_halows_ntile(kind, x->c, y->c) == 0) return 0;
  if (x->dtype != B200SEG_BF16 || y->dtype != B200SEG_BF16) return 0;
  if (addend && addend->dtype != B200SEG_BF16) return 0;
  if ((x->ld % 8) || (y->ld % 8) || !al16w(x->ptr) || !al16w(y->ptr)) return 0;
  if (addend && ((addend->ld % 8) || !al16w(addend->ptr))) return 0;
  if (x->d != y->d || x->h != y->h || x->w != y->w) return 0;
  return 1;
}

static int g_ws_init[64] = {0};

template <int CIN, int NT, int NACC>
static int conv_halows_launch(HaloWsArgs& p, int device, int maxsm, cudaStream_t st) {
  // (tail: + A/B table and its fp64 scratch for the backward-sums epilogue)
  const uint32_t slice = (uint32_t)(CIN / 8) * WS_PH * WS_PW * 16u;
  const uint32_t tap_bytes = (uint32_t)CIN * NT * 2u;
  const uint32_t tail0 = (2 * kWsMaxSlices + 4 + 2 * kWsMaxWStages) * 8 + 16 + 10 * p.Cout * 4 + 64 +
                         (2 * p.Cout + 16) * 8 + 8 + 16;
  // one item's slices stay resident; the staging tile is double buffered if four weight blocks still fit beside it;
  // the rest is the weight ring (tap blocks in flight hide the L2 latency of the stream)
  const int ns = NACC + 2;
  int wst = 0;
  uint32_t tail = 0;
  for (p.accslots = 2; p.accslots >= 1; --p.accslots) {
    p.acc_pitch = p.accslots * NACC * NT + 4;
    tail = tail0 + 128u * (uint32_t)p.acc_pitch * 4u;
    wst = (maxsm - 256 - (int)tail - ns * (int)slice) / (int)tap_bytes;
    if (wst >= 4 || p.accslots == 1) break;
  }
  if (wst > kWsMaxWStages) wst = kWsMaxWStages;
  B200_CHECK_ARG(wst >= 2, "conv_halows: slices do not fit in shared memory");
  p.nslices = ns;
  p.wstages = wst;
  const uint32_t wbytes = (uint32_t)wst * tap_bytes;
  p.ndchunks = (p.D + NACC - 1) / NACC;
  p.ngroups = p.Cout / NT;
  p.nitems = p.N * p.th * p.tw * p.ndchunks * p.ngroups;
  const size_t smem_bytes = 128 + wbytes + (size_t)ns * slice + tail;
  const int sms = num_sms(device);
  const int grid = sms < p.nitems ? sms : p.nitems;
  if (p.yfwd != nullptr) launch_k(conv_halows_kernel<CIN, NT, NACC, true>, grid, kWsThreads, smem_bytes, st, p);
  else launch_k(conv_halows_kernel<CIN, NT, NACC, false>, grid, kWsThreads, smem_bytes, st, p);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int conv_halows(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias,
                const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device, cudaStream_t st,
                const b200seg_tensor* yfwd, const b200seg_gn* gn, double* sums) {
  (void)kind; (void)dims;
  const int maxsm = tc_max_smem(device);
  if (device >= 0 && device < 64 && !g_ws_init[device]) {
    B200_CUDA(cudaFuncSetAttribute(conv_halows_kernel<64, 64, 1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
    B200_CUDA(cudaFuncSetAttribute(conv_halows_kernel<128, 64, 1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
    B200_CUDA(cudaFuncSetAttribute(conv_halows_kernel<64, 64, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
    B200_CUDA(cudaFuncSetAttribute(conv_halows_kernel<128, 64, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
    g_ws_init[device] = 1;
  }
  HaloWsArgs p;
  p.x = static_cast<const bf16*>(x->ptr);
  p.w = static_cast<const bf16*>(wpk);
  p.y = static_cast<bf16*>(y->ptr);
  p.addend = addend ? static_cast<const bf16*>(addend->ptr) : nullptr;
  p.bias = bias;
  p.stats = stats;
  p.xld = x->ld; p.yld = y->ld; p.ald = addend ? addend->ld : 0;
  p.N = x->n; p.D = x->d; p.H = x->h; p.W = x->w;
  p.Cin = x->c; p.Cout = y->c;
  p.tw = (p.W + WS_TW - 1) / WS_TW;
  p.th = (p.H + WS_TH - 1) / WS_TH;
  p.yfwd = nullptr; p.yfld = 0; p.gstats = nullptr; p.ggamma = nullptr; p.gbeta = nullptr; p.gscale = nullptr;
  p.ggroups = 1; p.gm = 1.0; p.geps = 0.f;
  if (yfwd != nullptr) {
    B200_CHECK_ARG(gn != nullptr && sums != nullptr && stats == nullptr && same_geom(yfwd, y) &&
                       yfwd->dtype == B200SEG_BF16 && (yfwd->ld % 8) == 0 && al16w(yfwd->ptr) && gn->groups > 0 &&
                       gn->groups <= 8 && (y->c % gn->groups) == 0,
                   "conv_halows: bad forward tensor / GroupNorm reference for the backward statistics");
    p.yfwd = static_cast<const bf16*>(yfwd->ptr);
    p.yfld = yfwd->ld;
    p.gstats = gn->stats; p.ggamma = gn->gamma; p.gbeta = gn->beta; p.gscale = gn->scale;
    p.ggroups = gn->groups;
    p.gm = (double)(y->c / gn->groups) * (double)gn->vox;
    p.geps = gn->eps;
    p.stats = sums;
  }
  // NT = 64 columns per MMA (narrower groups re-read A for less work); NACC = 1 keeps the warpgroup at 64
  // accumulator registers per thread, within the budget of a 544-thread CTA
  if (p.Cin == 64) return conv_halows_launch<64, 64, 1>(p, device, maxsm, st);
  return conv_halows_launch<128, 64, 1>(p, device, maxsm, st);
}

}  // namespace b200seg
