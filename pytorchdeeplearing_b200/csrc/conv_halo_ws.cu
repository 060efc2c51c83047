// Halo-staged wgmma 3x3x3 convolution with STREAMED weights for the 64/128-channel pyramid levels (sm_90a, bf16).
//
// At 24^3 / 12^3 voxels the TMA im2col path (conv_tc.cu) is bound by what one SM can ingest: every 128-voxel tile
// pulls 27 shifted copies of its activation box plus all 27 tap blocks of the weights through L2->smem
// (0.66 MB per tile at 64 channels) while the tensor core waits.  This kernel removes both multipliers:
//   * activations: as in conv_halo.cu, an (8 wide x 16 high) output column keeps its input d-slices (one-voxel
//     halo, zero filled = conv padding) channel-planar in shared memory and all 27 taps are descriptor VIEWS of
//     them (no-swizzle K-major canonical layout: SBO = one halo row, LBO = one 8-channel plane);
//   * weights: the 27 tap blocks ([Cin/8][NT][8] bf16, 8-16 KB) of an output-channel group are too large to stay
//     resident beside the slices, so they are streamed through a cp.async.bulk ring (as deep as the shared memory
//     left over allows: the blocks in flight hide the L2 latency of the stream).
// Output tile geometry (M = 128 rows), chosen per launch by shape (conv_halows_geometry):
//   * column: 8 wide x 16 high.  One core matrix is one 8-voxel output row, so the tile covers a plane exactly only
//     where 8 | W and 16 | H (UNet3d's 32^2 / 16^2 planes); 128 input channels always use it;
//   * flattened padded rows: with P = W + 2 the padded row pitch, output (h, w) is anchor position q = h*P + w and
//     tap (kh, kw) reads padded position q + kh*P + kw, one constant offset over a run of consecutive positions.  A
//     tile is 128 consecutive anchors [q0, q0 + 128); its slice window is padded positions [q0, q0 + 128 + 2P + 2)
//     (SBO = 16 B x 8 positions).  The two wrap-around anchors per padded row (w = W, W + 1) are computed and
//     dropped by the epilogue.  A 24 x 24 plane takes 5 such tiles (640 rows) instead of 2 x 3 column tiles (768),
//     and a tile whose upper M64 half lies wholly past the last anchor issues only its lower half's MMAs.
//   Both read the same packed weights in the same (kd, kh, kw, kc) order: every output value is the same in either.
// Work split: the output space is T = N * th * tw * (Cout / NT) * D units, one (slice tile, NT-channel group)
// each, ordered (n, h tile, w tile, group, d) (flat: th = tiles, tw = 1).  CTA b of G owns [b*T/G, (b+1)*T/G) and
// walks it as column segments (n, tile, group, d_a, nd); every role takes its segments from ws_segment, so their
// slice, tap-block and output sequences, and with them the mbarrier parities, agree.  A segment stages its input
// slices d_a-1 .. d_a+nd once.
//   * items: a segment is cut into items of NACC consecutive output slices (the last one may be shorter).  Each
//     streamed tap block is multiplied into all of the item's accumulators (registers of the MMA warpgroup), so the
//     weight traffic per output tile drops by NACC.  Every output sums its 27 taps x Cin/16 K chunks in the order
//     (kd, kh, kw, kc), from zero, in one accumulator;
//   * pipelined chains: the chain of tap t+1 is issued before the one of tap t is waited for (wgmma wait_group 1),
//     and tap t's weight stage is released as soon as that wait returns.  An input slice goes back to the loaders
//     as soon as the item's last chain reading it has completed and the next item of the segment does not need it,
//     so the loaders stage the next item's slices while this one still computes;
//   * finished outputs pass one at a time through an fp32 staging tile in shared memory (double buffered where the
//     shared memory allows) to the epilogue: bias, GroupNorm statistics (per-row sums over a segment, one warp fold
//     per segment, flushed when a range crosses into the next sample), residual addend, bf16 NDHWC stores, or the
//     fused GroupNorm-backward sums of b200seg_conv_bwdstats;
//   * registers per role (setmaxnreg): the loader warpgroup gives most of its share to the MMA warpgroup
//     (NACC outputs' accumulators) and to the epilogue (per-row sums of every channel of the group).
// NACC = 2 at 64 input channels.  At 128 the four input slices of a 2-slice item (4 x 45 KB) leave no room for the
// staging tile and the weight ring, so NACC = 1 there.
// Warp roles (384 threads): warps 0-3 MMA warpgroup, warps 4-7 epilogue, warps 8-10 slice loaders (cp.async, zero
// fill), warp 11 weight streamer.
#include <type_traits>

#include "gn_coef.cuh"
#include "tc_common.cuh"

namespace b200seg {

constexpr int WS_TW = 8, WS_TH = 16;                 // column output tile (w, h); M = 128 rows = (hh, ww)
constexpr int WS_PW = WS_TW + 2, WS_PH = WS_TH + 2;
constexpr int WS_M = WS_TW * WS_TH;                  // output rows per tile (both geometries)
// flat tiles are used only while their slice window (128 + 2P + 2 positions) is no longer than 184 positions (W <= 25),
// about the column window's 18 x 10 = 180: the shared-memory split of conv_halows_launch stays what it was
constexpr int kWsFlatMaxPos = 184;
constexpr int kWsMaxSlices = 8;
constexpr int kWsSliceLoaders = 3;                   // warps 8..10; warp 11 streams the weights
constexpr int kWsThreads = 32 * (4 + 4 + 4);         // 384 threads
constexpr int kWsMaxWStages = 16;     // weight ring depth is chosen at launch from the shared memory left over
// Registers per thread after setmaxnreg.  One CTA of 384 threads starts every thread at 168 (65536 / 384, rounded
// down to a multiple of 8), and the three warpgroups may hold at most 3 * 168 between them.  The MMA warpgroup holds
// NACC x 2 M64 halves x NT/2 = 128 fp32 accumulators at NACC = 2, NT = 64, plus descriptors and ring counters; the
// epilogue holds the per-row GroupNorm sums of the group's NT channels (2 x NT = 128) plus one 16-column chunk; the
// loaders and the weight streamer hold addresses only (64: at 56 the 128-channel loader spills).
constexpr uint32_t kWsRegsMma = 224, kWsRegsEpi = 216, kWsRegsLoad = 64;
static_assert(kWsRegsMma + kWsRegsEpi + kWsRegsLoad <= 3 * 168, "register budget of conv_halows_kernel");
static_assert(2 * 2 * (64 / 2) + 64 <= kWsRegsMma, "NACC = 2 accumulators at NT = 64 plus addressing");

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
  int tw, th;             // tiles along w, h (flat: tw = 1, th = tiles of 128 anchors)
  int P;                  // flat: padded row pitch W + 2
  int span;               // flat: anchors of a plane, (H - 1) * P + W
  int npos;               // positions of one staged slice plane (flat: 128 + 2P + 2, column: 18 x 10)
  int ngroups;            // output-channel groups of NT columns
  int nslices;            // input slice ring size (>= NACC + 2)
  int wstages;            // weight ring depth (tap blocks in flight)
  int accslots;           // output staging slots in shared memory (1 or 2)
  int acc_pitch;          // floats per staging row: accslots * NT + 4
  // GroupNorm-backward sums fused into the data-gradient epilogue (b200seg_conv_bwdstats; see conv_halo.cu)
  const bf16* yfwd;
  long long yfld;
  GnRef gn;
};

__device__ __forceinline__ uint64_t ws_nosw_desc(uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}

// this CTA's share [begin, end) of the N * th * tw * ngroups * D (slice tile, channel group) units
__device__ __forceinline__ void ws_range(const HaloWsArgs& p, int& begin, int& end) {
  const long long nunits = (long long)p.N * p.th * p.tw * p.ngroups * p.D;
  begin = (int)(nunits * blockIdx.x / gridDim.x);
  end = (int)(nunits * (blockIdx.x + 1) / gridDim.x);
}

// one column segment of a CTA's range: nd output slices from (n, d0) of the (h0, w0) column (flat: of the tile whose
// first anchor is q0), channel group g
struct WsSeg {
  int n, h0, w0, q0, g, d0, nd;
};
// the segment starting at unit u of a CTA range that ends at `end` (units ordered (n, h tile, w tile, group, d))
__device__ __forceinline__ WsSeg ws_segment(const HaloWsArgs& p, int u, int end) {
  WsSeg s;
  s.d0 = u % p.D;
  int c = u / p.D;
  s.g = c % p.ngroups;
  c /= p.ngroups;
  const int iw = c % p.tw;
  c /= p.tw;
  const int ih = c % p.th;
  s.n = c / p.th;
  s.w0 = iw * WS_TW;
  s.h0 = ih * WS_TH;
  s.q0 = ih * WS_M;
  s.nd = min(p.D - s.d0, end - u);
  return s;
}

template <int CIN, int NT, int NACC, bool BWD, bool FLAT>
__global__ void __launch_bounds__(kWsThreads, 1) conv_halows_kernel(const HaloWsArgs p) {
  PDL_TRIGGER();
  constexpr int CP = CIN / 8;                                // 8-channel planes
  const int npos = FLAT ? p.npos : WS_PH * WS_PW;            // positions of one plane of one slice
  const uint32_t PLANE = (uint32_t)npos * 16u;               // bytes of one plane of one slice
  const uint32_t SLICE = (uint32_t)CP * PLANE;
  constexpr int TAPS = 27;
  constexpr uint32_t TAP_BYTES = (uint32_t)CIN * NT * 2u;
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
  float* s_bias = s_stat + 8 * p.Cout;                       // [Cout]
  float* s_ab = s_bias + p.Cout;                             // [2][Cout]: A, B of the sample being processed (BWD)
  double* s_gd = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(s_ab + 2 * p.Cout) + 7) & ~(uintptr_t)7);
  // staging tile [128 rows][accslots x NT] fp32: finished outputs on their way from the MMA warpgroup to the epilogue
  float* s_acc = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(s_gd + 2 * p.Cout + 16) + 15) & ~(uintptr_t)15);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t ns = (uint32_t)p.nslices, nw = (uint32_t)p.wstages, na = (uint32_t)p.accslots;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nslices; ++s) {
      mbar_init(&sfull[s], 1);                       // ONE arrive: by the loader warp that staged the slice
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
  __syncthreads();
  PDL_WAIT();               // barriers and the statistics rows are set up under the tail of the previous kernel
  for (int i = threadIdx.x; i < p.Cout; i += blockDim.x) s_bias[i] = p.bias != nullptr ? p.bias[i] : 0.f;
  fence_proxy_async();
  __syncthreads();

  int u_begin, u_end;
  ws_range(p, u_begin, u_end);

  if (warp < 4) {
    // ===================================================== MMA warpgroup
    setmaxnreg_inc<kWsRegsMma>();
    const int wt = threadIdx.x;
    // column: one core matrix = one 8-voxel halo row (SBO = one halo row); flat: 8 consecutive positions (SBO = 128 B)
    const uint64_t a_hi = ws_nosw_desc(PLANE, FLAT ? 128u : WS_PW * 16u);
    const uint32_t pitch = FLAT ? (uint32_t)p.P : (uint32_t)WS_PW;   // positions from one kh to the next
    // rows 64..127 of the tile: 8 halo rows further on (column), 64 positions further on (flat)
    constexpr uint32_t hi_off = (FLAT ? 64u * 16u : 8u * WS_PW * 16u) >> 4;
    const uint64_t b_hi = ws_nosw_desc((uint32_t)NT * 16u, 128u);
    const uint32_t ring_u32 = smem_u32(s_ring);
    const uint32_t w_u32 = smem_u32(s_w);
    constexpr int kchunks = CIN / 16;
    uint32_t gs = 0;    // input slices of earlier segments (ring position of the segment's first slice)
    uint32_t go = 0;    // outputs handed to the epilogue so far
    uint32_t wq = 0;    // weight blocks consumed so far
    auto release_slice = [&](uint32_t sl) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&sempty[sl % ns]);
    };
    auto release_wstage = [&](uint32_t q) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&wempty[q % nw]);
    };
    for (int u = u_begin; u < u_end;) {
      const WsSeg s = ws_segment(p, u, u_end);
      // a flat tile whose upper M64 half lies wholly past the plane's last anchor computes its lower half only (its
      // upper accumulators stay zero and the epilogue drops those rows)
      const bool upper = !FLAT || s.q0 + 64 < p.span;
      for (int o0 = 0; o0 < s.nd; o0 += NACC) {
        const bool last = o0 + NACC >= s.nd;       // last item of the segment
        const uint32_t f = gs + (uint32_t)o0;      // ring position of the item's first input slice
        // one item of NA output slices: reads input slices f .. f + NA + 1, output j and tap kd read slice f + j + kd
        auto item = [&](auto na_, auto up_) {
          constexpr int NA = decltype(na_)::value;
          constexpr bool UP = decltype(up_)::value;   // the upper M64 half is computed (a compile-time choice: a
                                                      // branch inside the chain would make ptxas serialise the wgmmas)
          float acc[NA][2][NT / 2];
#pragma unroll
          for (int j = 0; j < NA; ++j) {
            frag_zero(acc[j][0]);
            frag_zero(acc[j][1]);
          }
          auto wait_slice = [&](uint32_t sl) { mbar_wait(&sfull[sl % ns], (sl / ns) & 1u); };
#pragma unroll 1
          for (int kd = 0; kd < 3; ++kd) {
            // slices are waited for when first needed: kd = 0 reads slices 0 .. NA-1 of the item, every further kd
            // one more (the loader warp that staged a slice fenced it for the async proxy before its arrive)
            if (kd == 0) {
#pragma unroll
              for (int j = 0; j < NA; ++j) wait_slice(f + (uint32_t)j);
            } else {
              wait_slice(f + (uint32_t)(kd + NA - 1));
            }
#pragma unroll
            for (int t9 = 0; t9 < 9; ++t9) {
              const uint32_t stg = wq % nw;
              mbar_wait(&wfull[stg], (wq / nw) & 1u);
              const uint64_t b_tap = b_hi | (uint64_t)((w_u32 + stg * TAP_BYTES) >> 4);
#pragma unroll
              for (int j = 0; j < NA; ++j) {
                wgmma_fence_regs(acc[j][0]);
                wgmma_fence_regs(acc[j][1]);
              }
              wgmma_fence();
#pragma unroll
              for (int j = 0; j < NA; ++j) {
                const uint32_t sl = f + (uint32_t)(j + kd);
                const uint64_t a_base = a_hi | (uint64_t)((ring_u32 + (sl % ns) * SLICE) >> 4);
#pragma unroll
                for (int kc = 0; kc < kchunks; ++kc) {
                  const uint32_t a_off = ((uint32_t)(2 * kc) * PLANE + ((uint32_t)(t9 / 3) * pitch + t9 % 3) * 16u) >> 4;
                  const uint32_t b_off = ((uint32_t)(kc * 2 * NT) * 16u) >> 4;
                  Wgmma<NT, 0, 0>::mma(acc[j][0], a_base + a_off, b_tap + b_off);
                  if constexpr (UP) Wgmma<NT, 0, 0>::mma(acc[j][1], a_base + a_off + hi_off, b_tap + b_off);
                }
              }
              wgmma_commit();
              // the chain of the previous tap is complete once at most this one is in flight
              wgmma_wait<1>();
#pragma unroll
              for (int j = 0; j < NA; ++j) {
                wgmma_fence_regs(acc[j][0]);
                wgmma_fence_regs(acc[j][1]);
              }
              if (t9 > 0 || kd > 0) release_wstage(wq - 1u);
              // every chain of tap block kd-1 has completed: the item's input slice kd-1 had its last use there; it
              // goes back to the loaders unless the next item of the segment starts on it
              if (t9 == 0 && kd > 0 && (kd - 1 < NA || last)) release_slice(f + (uint32_t)(kd - 1));
              ++wq;
            }
          }
          wgmma_wait0();
#pragma unroll
          for (int j = 0; j < NA; ++j) {
            wgmma_fence_regs(acc[j][0]);
            wgmma_fence_regs(acc[j][1]);
          }
          release_wstage(wq - 1u);
          if (last) {
#pragma unroll
            for (int i = 2; i < NA + 2; ++i) release_slice(f + (uint32_t)i);
          }
#pragma unroll
          for (int j = 0; j < NA; ++j) {
            const uint32_t o = go + (uint32_t)j;
            const uint32_t as = o % na;
            mbar_wait(&tempty[as], ((o / na) & 1u) ^ 1u);
            frag_store(s_acc + as * NT, p.acc_pitch, 0, acc[j][0], wt);
            frag_store(s_acc + as * NT, p.acc_pitch, 64, acc[j][1], wt);
            __syncwarp();
            if (lane == 0) mbar_arrive(&tfull[as]);
          }
          go += (uint32_t)NA;
        };
        auto halves = [&](auto up_) {
          if (o0 + NACC <= s.nd) item(std::integral_constant<int, NACC>{}, up_);
          else item(std::integral_constant<int, 1>{}, up_);   // NACC = 2: the odd last slice of a segment
        };
        if (upper) halves(std::true_type{});
        else if constexpr (FLAT) halves(std::false_type{});
      }
      gs += (uint32_t)(s.nd + 2);
      u += s.nd;
    }
  } else if (warp >= 8) {
    setmaxnreg_dec<kWsRegsLoad>();
    if (warp == 8 + kWsSliceLoaders) {
      // ===================================================== weight streamer: the 27 tap blocks of the segment's channel
      // group, once per item, into the ring (one lane)
      if (lane == 0) {
        uint32_t q = 0;
        for (int u = u_begin; u < u_end;) {
          const WsSeg s = ws_segment(p, u, u_end);
          const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w) + (size_t)s.g * TAPS * TAP_BYTES;
          for (int o0 = 0; o0 < s.nd; o0 += NACC) {
            for (int tap = 0; tap < TAPS; ++tap, ++q) {
              const uint32_t stg = q % nw;
              mbar_wait(&wempty[stg], ((q / nw) & 1u) ^ 1u);
              mbar_expect_tx(&wfull[stg], TAP_BYTES);
              asm volatile(
                  "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                      smem_u32(s_w + (size_t)stg * TAP_BYTES)),
                  "l"(wsrc + (size_t)tap * TAP_BYTES), "r"(TAP_BYTES), "r"(smem_u32(&wfull[stg]))
                  : "memory");
            }
          }
          u += s.nd;
        }
      }
    } else {
      // ===================================================== slice loaders: warp w stages the input slices sl = w (mod 3)
      // of the CTA's sequence on its own (all pieces of the slice, 16-byte cp.async with zero fill = conv padding),
      // waits for them to land and signals the slice with ONE mbarrier arrive.  A slice is signalled before the warp
      // takes its next one: the ring may hold just one item's NACC + 2 slices, and the slot of a later slice is only
      // freed once the MMA warpgroup has read this one.
      const int lw = warp - 8;
      const int pieces = npos * CP;
      int u = u_begin, it_i = 0, it_nsl = 0;
      WsSeg s{0, 0, 0, 0, 0, 0, 0};
      auto load_seg = [&]() {
        if (u < u_end) {
          s = ws_segment(p, u, u_end);
          it_nsl = s.nd + 2;
        }
      };
      auto advance = [&](int steps) {
        it_i += steps;
        while (u < u_end && it_i >= it_nsl) {
          it_i -= it_nsl;
          u += s.nd;
          load_seg();
        }
      };
      load_seg();
      advance(lw);
      uint32_t sl = (uint32_t)lw;
      while (u < u_end) {
        const uint32_t slot = sl % ns;
        mbar_wait(&sempty[slot], ((sl / ns) & 1u) ^ 1u);
        const uint32_t dst = smem_u32(s_ring + (size_t)slot * SLICE);
        const int d = s.d0 - 1 + it_i;
        const bool dok = (unsigned)d < (unsigned)p.D;
        const bf16* src = p.x + (((long long)s.n * p.D + (dok ? d : 0)) * p.H) * p.W * p.xld;
        if constexpr (FLAT) {
          // a lane keeps one 8-channel plane (32 % CP == 0) and walks positions v = lane / CP + k * 32 / CP; padded
          // position q0 + v = (hp, wp) holds source voxel (hp - 1, wp - 1), stepped without a division per piece
          constexpr int VSTEP = 32 / CP;
          const int plane = lane % CP;
          int v = lane / CP;
          int hp = (int)((unsigned)(s.q0 + v) / (unsigned)p.P);
          int wp = s.q0 + v - hp * p.P;
#pragma unroll 4
          for (; v < npos; v += VSTEP) {
            const int h = hp - 1, w = wp - 1;
            const bool ok = dok && (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
            const bf16* g = ok ? src + ((long long)h * p.W + w) * p.xld + plane * 8 : p.x;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + (uint32_t)(plane * (int)PLANE + v * 16)),
                         "l"(g), "r"(ok ? 16 : 0)
                         : "memory");
            wp += VSTEP;
            while (wp >= p.P) {
              wp -= p.P;
              ++hp;
            }
          }
        } else {
#pragma unroll 4
          for (int q = lane; q < pieces; q += 32) {
            const int v = q / CP, plane = q - v * CP;
            const int hh = v / WS_PW, ww = v - hh * WS_PW;
            const int h = s.h0 - 1 + hh, w = s.w0 - 1 + ww;
            const bool ok = dok && (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
            const bf16* g = ok ? src + ((long long)h * p.W + w) * p.xld + plane * 8 : p.x;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + (uint32_t)(plane * (int)PLANE + v * 16)),
                         "l"(g), "r"(ok ? 16 : 0)
                         : "memory");
          }
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        fence_proxy_async();            // landed cp.async data -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&sfull[slot]);
        advance(kWsSliceLoaders);
        sl += kWsSliceLoaders;
      }
    }
  } else {
    // ===================================================== epilogue warps 4..7
    // GroupNorm statistics: per-thread (= per output row) partial sums in registers over ALL outputs of a segment, one
    // butterfly fold over the warp per segment; the staging buffer is released right after its last chunk is read.
    setmaxnreg_inc<kWsRegsEpi>();
    const int q = warp & 3;
    const int row = q * 32 + lane;
    const int rw = row % WS_TW, rh = row / WS_TW;
    const int etid = (warp - 4) * 32 + lane;
    constexpr int sstride = BWD ? 3 : 2;
    const bool want_stats = p.stats != nullptr;
    uint32_t go = 0;
    int cur_n = -1;
    auto flush_stats = [&](int n) {
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (want_stats && n >= 0) {
        for (int i = etid; i < 2 * p.Cout; i += 128) {
          const int which = i / p.Cout, c = i - which * p.Cout;
          double t = 0.0;
#pragma unroll
          for (int wq = 0; wq < 4; ++wq) {
            t += (double)s_stat[wq * 2 * p.Cout + i];
            s_stat[wq * 2 * p.Cout + i] = 0.f;
          }
          atomicAdd(p.stats + ((long long)n * p.Cout + c) * sstride + which, t);
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    };
    for (int u = u_begin; u < u_end;) {
      const WsSeg sg = ws_segment(p, u, u_end);
      const int n = sg.n, d0 = sg.d0, nd = sg.nd;
      u += nd;
      // a CTA's range can cross into the next sample: its statistics go to that sample's rows from here on
      if (n != cur_n) {
        if (cur_n >= 0 && want_stats) flush_stats(cur_n);
        cur_n = n;
        // A, B of sample n for the ReLU mask of the backward sums (gn_coefs, as gn_bwd_apply derives them)
        if constexpr (BWD)
          gn_coefs<false, false>(GnNamedBarrier<1, 128>{etid}, p.gn, nullptr, n, p.Cout, s_gd, nullptr, s_ab,
                                 s_ab + p.Cout, nullptr, nullptr, nullptr);
      }
      int oh = sg.h0 + rh, ow = sg.w0 + rw;
      if constexpr (FLAT) {
        // anchor q = oh * P + ow; the wrap-around anchors (ow = W, W + 1) and those past the plane are not outputs
        const int qa = sg.q0 + row;
        oh = (int)((unsigned)qa / (unsigned)p.P);
        ow = qa - oh * p.P;
      }
      const bool valid = oh < p.H && ow < p.W;
      const int cbase = sg.g * NT;
      float rs[NT], rq[NT];
#pragma unroll
      for (int j = 0; j < NT; ++j) rs[j] = rq[j] = 0.f;
      for (int o = 0; o < nd; ++o, ++go) {
        const long long vox = (((long long)n * p.D + (d0 + o)) * p.H + oh) * p.W + ow;
        const uint32_t as = go % na;
        mbar_wait(&tfull[as], (go / na) & 1u);
        const float* tacc = s_acc + row * p.acc_pitch + as * NT;
#pragma unroll
        for (int c = 0; c < NT / 16; ++c) {
          const int c0 = cbase + c * 16;
          uint4 yfv[2];
          if constexpr (BWD) {
            yfv[0] = yfv[1] = make_uint4(0u, 0u, 0u, 0u);
            if (valid) {
              yfv[0] = *reinterpret_cast<const uint4*>(p.yfwd + vox * p.yfld + c0);
              yfv[1] = *reinterpret_cast<const uint4*>(p.yfwd + vox * p.yfld + c0 + 8);
            }
          }
          float v[16];
          acc_ld16(tacc + c * 16, v);
          if (c == NT / 16 - 1) {
            // every column of the buffer is read: release it before the arithmetic
            __syncwarp();
            if (lane == 0) mbar_arrive(&tempty[as]);
          }
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            const float4 b4 = *reinterpret_cast<const float4*>(s_bias + c0 + j);
            v[j] += b4.x; v[j + 1] += b4.y; v[j + 2] += b4.z; v[j + 3] += b4.w;
          }
          if constexpr (!BWD) {
            if (want_stats && valid) {
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                rs[c * 16 + j] += v[j];
                rq[c * 16 + j] = fmaf(v[j], v[j], rq[c * 16 + j]);
              }
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
                  const int k_ = c * 16 + 8 * h_ + 2 * j;
                  rs[k_] += d0_;
                  rs[k_ + 1] += d1_;
                  rq[k_] = fmaf(d0_, yy.x, rq[k_]);
                  rq[k_ + 1] = fmaf(d1_, yy.y, rq[k_ + 1]);
                }
              }
            }
          }
        }
      }
      if (want_stats) {
        // fold the 32 rows of this warp: after the butterfly lane pair (2k, 2k+1) holds column col(k) of the chunk
#pragma unroll
        for (int c = 0; c < NT / 16; ++c) {
          float s[16], qq[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            s[j] = rs[c * 16 + j];
            qq[j] = rq[c * 16 + j];
          }
          stat_butterfly(s, qq, lane);
          if ((lane & 1) == 0) {
            const int col = stat_col(lane);
            float* sw_ = s_stat + q * 2 * p.Cout;     // this warp's private row: no atomics, fixed order
            sw_[cbase + c * 16 + col] += s[0];
            sw_[p.Cout + cbase + c * 16 + col] += qq[0];
          }
        }
      }
    }
    if (want_stats && cur_n >= 0) flush_stats(cur_n);
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

// The output tile geometry of a layer with Cin input channels and an H x W plane: flattened padded rows at 64 input
// channels where they need fewer tiles per plane than the 8 x 16 column tile and their slice window fits the
// column's shared-memory budget; a tie keeps the column tile.  Fewer tiles means fewer units, and so fewer per CTA:
// 24 x 24 takes 5 flat tiles instead of 6 (64 -> 64 at 2 x 24^3 on an H100: 31.5 -> 29.5 us forward, 39.6 -> 35.6 us
// for the data gradient with GroupNorm-backward sums).  Fewer MMA rows alone do not pay: at 12 x 12 the flat split is
// one full tile and one lower-half tile, two units per (n, d, group) as with two column tiles, and a trial of it at
// 128 channels measured no faster, so 128 input channels and the planes the column tile covers exactly (8 | W,
// 16 | H) stay on the column tile.
// Where flat is chosen no CTA gets more units than under the column split.  b200seg_conv_halo_ws_geometry reports
// this same value.
int conv_halows_geometry(int cin, int h, int w) {
  if (cin != 64) return B200SEG_WS_GEOM_COLUMN;
  const long long col_tiles = (long long)((h + WS_TH - 1) / WS_TH) * ((w + WS_TW - 1) / WS_TW);
  const int P = w + 2;
  if (WS_M + 2 * P + 2 > kWsFlatMaxPos) return B200SEG_WS_GEOM_COLUMN;
  const long long flat_tiles = ((long long)(h - 1) * P + w + WS_M - 1) / WS_M;
  return flat_tiles < col_tiles ? B200SEG_WS_GEOM_FLAT : B200SEG_WS_GEOM_COLUMN;
}

static int g_ws_init[64] = {0};

template <int CIN, int NT, int NACC, bool FLAT>
static int conv_halows_set_smem(int maxsm) {
  B200_CUDA(cudaFuncSetAttribute(conv_halows_kernel<CIN, NT, NACC, false, FLAT>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
  B200_CUDA(cudaFuncSetAttribute(conv_halows_kernel<CIN, NT, NACC, true, FLAT>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm));
  return B200SEG_OK;
}

template <int CIN, int NT, int NACC>
static int conv_halows_launch(HaloWsArgs& p, int flat, int device, int maxsm, cudaStream_t st) {
  // (tail: barriers, statistics rows, bias, the A/B table and its fp64 scratch for the backward-sums epilogue)
  const int slice = (CIN / 8) * p.npos * 16;
  const int tap_bytes = CIN * NT * 2;
  const int tail0 = (2 * kWsMaxSlices + 4 + 2 * kWsMaxWStages) * 8 + 16 + 11 * p.Cout * 4 + 64 +
                    (2 * p.Cout + 16) * 8 + 8 + 16;
  // the slices of one item (NACC + 2) at least; the staging tile is double buffered if four weight blocks still fit
  // beside it; one more slice where the weight ring keeps six blocks in flight; the rest is the weight ring
  int ns = NACC + 2;
  int avail = 0, wst = 0;
  for (p.accslots = 2; p.accslots >= 1; --p.accslots) {
    p.acc_pitch = p.accslots * NT + 4;
    avail = maxsm - 256 - tail0 - 128 * p.acc_pitch * 4;
    wst = (avail - ns * slice) / tap_bytes;
    if (wst >= 4 || p.accslots == 1) break;
  }
  while (ns < kWsMaxSlices && (avail - (ns + 1) * slice) / tap_bytes >= 6) {
    ++ns;
    wst = (avail - ns * slice) / tap_bytes;
  }
  if (wst > kWsMaxWStages) wst = kWsMaxWStages;
  B200_CHECK_ARG(wst >= 2, "conv_halows: slices do not fit in shared memory");
  p.nslices = ns;
  p.wstages = wst;
  p.ngroups = p.Cout / NT;
  const size_t smem_bytes = 128 + (size_t)wst * tap_bytes + (size_t)ns * slice + (size_t)tail0 +
                            128u * (size_t)p.acc_pitch * 4u;
  // the N * th * tw * ngroups * D units are split evenly over at most one CTA per SM.  Flat tiles take just enough
  // CTAs for the largest share, ceil(units / SMs): 240 units at 2 x 24^3 go two to each of 120 CTAs, so with an even
  // D every CTA's pair is one NACC = 2 item of one column (one weight stream), where 132 CTAs would leave some pairs
  // split across two columns.  The largest share, and so the statistics fold count per CTA, is the same either way.
  const long long nunits = (long long)p.N * p.th * p.tw * p.ngroups * p.D;
  const int sms = num_sms(device);
  int grid = nunits < sms ? (int)nunits : sms;
  if (flat) {
    const long long share = (nunits + grid - 1) / grid;
    grid = (int)((nunits + share - 1) / share);
  }
  if (flat) {
    if (p.yfwd != nullptr) launch_k(conv_halows_kernel<CIN, NT, NACC, true, true>, grid, kWsThreads, smem_bytes, st, p);
    else launch_k(conv_halows_kernel<CIN, NT, NACC, false, true>, grid, kWsThreads, smem_bytes, st, p);
  } else {
    if (p.yfwd != nullptr) launch_k(conv_halows_kernel<CIN, NT, NACC, true, false>, grid, kWsThreads, smem_bytes, st, p);
    else launch_k(conv_halows_kernel<CIN, NT, NACC, false, false>, grid, kWsThreads, smem_bytes, st, p);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int conv_halows(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias,
                const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device, cudaStream_t st,
                const b200seg_tensor* yfwd, const b200seg_gn* gn, double* sums) {
  (void)kind; (void)dims;
  const int maxsm = tc_max_smem(device);
  if (device >= 0 && device < 64 && !g_ws_init[device]) {
    if (conv_halows_set_smem<64, 64, 2, false>(maxsm) != B200SEG_OK ||
        conv_halows_set_smem<128, 64, 1, false>(maxsm) != B200SEG_OK ||
        conv_halows_set_smem<64, 64, 2, true>(maxsm) != B200SEG_OK ||
        conv_halows_set_smem<128, 64, 1, true>(maxsm) != B200SEG_OK)
      return B200SEG_ECUDA;
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
  const int flat = conv_halows_geometry(p.Cin, p.H, p.W) == B200SEG_WS_GEOM_FLAT;
  if (flat) {
    p.P = p.W + 2;
    p.span = (p.H - 1) * p.P + p.W;
    p.npos = WS_M + 2 * p.P + 2;
    p.tw = 1;
    p.th = (p.span + WS_M - 1) / WS_M;
  } else {
    p.P = 0;
    p.span = 0;
    p.npos = WS_PH * WS_PW;
    p.tw = (p.W + WS_TW - 1) / WS_TW;
    p.th = (p.H + WS_TH - 1) / WS_TH;
  }
  p.yfwd = nullptr; p.yfld = 0; p.gn = gn_ref(nullptr, 0);
  if (yfwd != nullptr) {
    B200_CHECK_ARG(gn != nullptr && sums != nullptr && stats == nullptr && same_geom(yfwd, y) &&
                       yfwd->dtype == B200SEG_BF16 && (yfwd->ld % 8) == 0 && al16w(yfwd->ptr) && gn->groups > 0 &&
                       gn->groups <= 8 && (y->c % gn->groups) == 0,
                   "conv_halows: bad forward tensor / GroupNorm reference for the backward statistics");
    p.yfwd = static_cast<const bf16*>(yfwd->ptr);
    p.yfld = yfwd->ld;
    p.gn = gn_ref(gn, y->c);
    p.stats = sums;
  }
  // NT = 64 columns per MMA (narrower groups re-read A for less work).  Two output slices share each streamed tap
  // block at 64 input channels; at 128 the four input slices that takes do not fit beside the staging tile.
  if (p.Cin == 64) return conv_halows_launch<64, 64, 2>(p, flat, device, maxsm, st);
  return conv_halows_launch<128, 64, 1>(p, flat, device, maxsm, st);
}

}  // namespace b200seg
