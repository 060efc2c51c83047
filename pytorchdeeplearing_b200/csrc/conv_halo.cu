// Halo-staged wgmma convolution for the full-resolution 16/32-channel 3x3(x3) layers (sm_90a, bf16).
//
// conv_tc.cu loads one shifted activation box per tap through TMA: 27 L2->smem transfers of the same
// voxels per output tile, which makes the 16/32-channel layers (80 % of the network's bytes) L2-bound.
// This kernel stages each input d-slice ONCE in shared memory and lets the 27 taps read shifted VIEWS of it:
//   * a CTA owns an (8 wide x 16 high) output column and marches along d; a ring of input slices
//     (18 x 10 voxels each, one-voxel halo, zero filled = conv padding) lives in smem, so each input voxel
//     is fetched ~1.4x instead of 27x;
//   * slices are stored channel-planar, [C/8 planes][18][10][8 ch], i.e. every voxel contributes one 16-byte
//     K-chunk per plane and 8 consecutive voxels along w form one wgmma core matrix (8 rows x 16 B).  In the
//     no-swizzle K-major canonical layout the 16 core-matrix rows of the M = 128 tile are then a constant
//     SBO = 160 B (one halo row) apart and the two K-chunks LBO = one plane apart, for EVERY tap: the tap only
//     moves the descriptor start address by (kh*10 + kw)*16 B inside the slice selected by kd;
//   * the packed weights of all taps stay resident in smem for the CTA's lifetime;
//   * loader warps move global -> smem with 16-byte cp.async (zero fill = conv padding); the MMA warpgroup (two
//     M64 halves, register accumulators), the double-buffered accumulator staging tile in shared memory and the
//     epilogue (bias, GroupNorm statistics, residual addend, bf16 NDHWC stores) follow conv_tc.cu.
// conv_halo_kernel below is the 2-D (1x3x3) form; the 3-D layers take the input-slice-major conv_halo3_kernel.
// Warp roles (512 threads): warps 0-3 MMA warpgroup, warps 4-7 epilogue, warps 8-15 loaders.
#include "gn_coef.cuh"
#include "tc_common.cuh"

namespace b200seg {

constexpr int HT_W = 8, HT_H = 16;            // output tile (w, h); M = 128 rows = (hh, ww)
constexpr int HP_W = HT_W + 2, HP_H = HT_H + 2;
constexpr int kHaloMaxSlices = 16;
constexpr int kLoaderWarps = 8;
constexpr int kHaloThreads = 32 * (4 + 4 + kLoaderWarps);
constexpr int kMaxPieces = (HP_H * HP_W * 4 + 32 * kLoaderWarps - 1) / (32 * kLoaderWarps);   // Cin <= 32

struct HaloArgs {
  const bf16* x;
  const bf16* w;          // packed [tap][Cin/8][Cout][8]
  bf16* y;
  const bf16* addend;
  const float* bias;
  double* stats;
  long long xld, yld, ald;
  int N, D, H, W;
  int Cin, Cout;
  int kd;                 // 3 (3-D) or 1 (2-D)
  int tw, th;             // tiles along w, h
  int dchunk, ndchunks;   // 2-D kernel: output slices per work item, items along d
  int nitems;             // 2-D kernel: N * th * tw * ndchunks
  int nslices;            // ring size
  int acc_pitch;          // floats per row of the accumulator staging tile in shared memory
  // GroupNorm-backward sums fused into the data-gradient epilogue (b200seg_conv_bwdstats): the output of this conv is
  // g = dL/d(act) of the layer whose raw output is yfwd; with m = [yfwd*A + B > 0] (A, B = that layer's GroupNorm /
  // dropout coefficients, derived here from its statistics with gn_coefs) the epilogue accumulates
  // sums[n][c][0] += g*m, sums[n][c][1] += g*m*yfwd  (stride 3: [2] = sum yfwd is taken from the forward statistics).
  const bf16* yfwd;       // nullptr: forward statistics mode (stats = [N][Cout][2])
  long long yfld;
  GnRef gn;               // the GroupNorm of the layer being differentiated
};

__device__ __forceinline__ uint64_t make_nosw_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) |
         ((uint64_t)(sbo_bytes >> 4) << 32);
}

template <int CIN, int COUT>
__global__ void __launch_bounds__(kHaloThreads, 1) conv_halo_kernel(const HaloArgs p) {
  PDL_ENTER();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  constexpr int CP = CIN / 8;                                // 8-channel planes
  constexpr uint32_t PLANE = HP_H * HP_W * 16u;              // bytes of one plane of one slice
  constexpr uint32_t SLICE = (uint32_t)CP * PLANE;
  constexpr int taps = 9;
  constexpr uint32_t W_BYTES = (uint32_t)taps * CIN * COUT * 2u;
  uint8_t* s_w = smem;
  uint8_t* s_ring = smem + ((W_BYTES + 127u) & ~127u);
  uint8_t* tail = s_ring + (size_t)p.nslices * SLICE;
  tail = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tail) + 15) & ~(uintptr_t)15);
  uint64_t* sfull = reinterpret_cast<uint64_t*>(tail);
  uint64_t* sempty = sfull + kHaloMaxSlices;
  uint64_t* tfull = sempty + kHaloMaxSlices;
  uint64_t* tempty = tfull + 2;
  float* s_stat = reinterpret_cast<float*>(tempty + 2);      // [4 epilogue warps][2][Cout]
  float* s_acc = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(s_stat + 8 * COUT) + 15) & ~(uintptr_t)15);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int items_per_cta = (p.nitems + gridDim.x - 1) / gridDim.x;
  const int item_begin = blockIdx.x * items_per_cta;
  const int item_end = min(p.nitems, item_begin + items_per_cta);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nslices; ++s) {
      mbar_init(&sfull[s], 32 * kLoaderWarps);   // one (deferred, cp.async) arrive per loader thread
      mbar_init(&sempty[s], 4);     // one arrive per MMA warp
    }
    for (int a = 0; a < 2; ++a) {
      mbar_init(&tfull[a], 4);
      mbar_init(&tempty[a], 4);
    }
    fence_barrier_init();
  }
  // resident weights: straight 16-byte copy of the pre-packed smem image
  for (uint32_t i = threadIdx.x * 16u; i < W_BYTES; i += blockDim.x * 16u)
    *reinterpret_cast<uint4*>(s_w + i) = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.w) + i);
  for (int i = threadIdx.x; i < 8 * p.Cout; i += blockDim.x) s_stat[i] = 0.f;
  fence_proxy_async();
  __syncthreads();

  auto decode = [&](int item, int& n, int& h0, int& w0, int& d0, int& nd) {
    int t = item;
    const int dc = t % p.ndchunks; t /= p.ndchunks;
    const int iw = t % p.tw; t /= p.tw;
    const int ih = t % p.th;
    n = t / p.th;
    w0 = iw * HT_W;
    h0 = ih * HT_H;
    d0 = dc * p.dchunk;
    nd = min(p.dchunk, p.D - d0);
  };

  if (warp < 4) {
    // ===================================================== MMA warpgroup
    const int wt = threadIdx.x;
    const uint64_t a_hi = make_nosw_desc(0, PLANE, HP_W * 16u);
    const uint64_t b_hi = make_nosw_desc(0, (uint32_t)COUT * 16u, 128u);
    const uint32_t ring_u32 = smem_u32(s_ring);
    const uint64_t b_base = b_hi | (uint64_t)(smem_u32(s_w) >> 4);
    constexpr int kchunks = CIN / 16;
    uint32_t go = 0;   // output slice-tiles produced so far = input slices consumed (output o reads input slice o)
    for (int item = item_begin; item < item_end; ++item) {
      int n, h0, w0, d0, nd;
      decode(item, n, h0, w0, d0, nd);
      for (int o = 0; o < nd; ++o, ++go) {
        const uint32_t slot = go % p.nslices;
        mbar_wait(&sfull[slot], (go / p.nslices) & 1u);
        const uint32_t as = go & 1u;
        // slices written by cp.async (generic proxy) must be ordered before the tensor core's async-proxy reads
        fence_proxy_async();
        float acc0[COUT / 2], acc1[COUT / 2];
        frag_zero(acc0);
        frag_zero(acc1);
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        wgmma_fence();
        {
          // straight-line issue: every descriptor is (slice base) + compile-time offset, in 16-byte units;
          // rows 64..127 of the tile (hh = 8..15) start 8 halo rows further on
          const uint64_t a_base = a_hi | (uint64_t)((ring_u32 + slot * SLICE) >> 4);
#pragma unroll
          for (int kh_ = 0; kh_ < 3; ++kh_)
#pragma unroll
            for (int kw_ = 0; kw_ < 3; ++kw_)
#pragma unroll
              for (int kc = 0; kc < kchunks; ++kc) {
                const uint32_t a_off = ((uint32_t)(2 * kc) * PLANE + (uint32_t)(kh_ * HP_W + kw_) * 16u) >> 4;
                const uint32_t b_off = ((uint32_t)(((kh_ * 3 + kw_) * kchunks + kc) * 2 * COUT) * 16u) >> 4;
                Wgmma<COUT, 0, 0>::mma(acc0, a_base + a_off, b_base + b_off);
                Wgmma<COUT, 0, 0>::mma(acc1, a_base + a_off + (8u * HP_W * 16u >> 4), b_base + b_off);
              }
        }
        wgmma_commit();
        wgmma_wait0();
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sempty[slot]);   // input slice o is no longer needed
        mbar_wait(&tempty[as], ((go >> 1) & 1u) ^ 1u);
        frag_store(s_acc + as * COUT, p.acc_pitch, 0, acc0, wt);
        frag_store(s_acc + as * COUT, p.acc_pitch, 64, acc1, wt);
        __syncwarp();
        if (lane == 0) mbar_arrive(&tfull[as]);
      }
    }
  } else if (warp >= 8) {
    // ===================================================== loaders (8 warps)
    constexpr int LT = 32 * kLoaderWarps;
    const int lt = threadIdx.x - 256;
    const int pieces = HP_H * HP_W * CP;
    // this thread's pieces: q = lt + j*LT  ->  (voxel v, plane) -> smem offset and (hh, ww)
    int poff[kMaxPieces], phh[kMaxPieces], pww[kMaxPieces];
    bool pval[kMaxPieces];
#pragma unroll
    for (int j = 0; j < kMaxPieces; ++j) {
      const int q = lt + j * LT;
      pval[j] = q < pieces;
      const int qq = pval[j] ? q : 0;
      const int v = qq / CP, plane = qq - v * CP;
      phh[j] = v / HP_W;
      pww[j] = v - phh[j] * HP_W;
      poff[j] = plane * (int)PLANE + v * 16;
      // global element offset of the plane is added per slice below
      pww[j] |= plane << 16;
    }
    // iterator over (item, slice)
    int it_item = item_begin, it_i = 0, n = 0, h0 = 0, w0 = 0, d0 = 0, nd = 0;
    if (it_item < item_end) decode(it_item, n, h0, w0, d0, nd);
    // fully asynchronous: as many slices in flight as the ring has free slots
    uint32_t sl = 0;
    while (it_item < item_end) {
      const uint32_t slot = sl % p.nslices;
      mbar_wait(&sempty[slot], ((sl / p.nslices) & 1u) ^ 1u);
      const uint32_t dst = smem_u32(s_ring + (size_t)slot * SLICE);
      const bf16* src = p.x + (((long long)n * p.D + d0 + it_i) * p.H) * p.W * p.xld;
#pragma unroll
      for (int j = 0; j < kMaxPieces; ++j) {
        if (!pval[j]) continue;
        const int plane = pww[j] >> 16, ww = pww[j] & 0xffff;
        const int h = h0 - 1 + phh[j], w = w0 - 1 + ww;
        const bool ok = (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
        const bf16* g = ok ? src + ((long long)h * p.W + w) * p.xld + plane * 8 : p.x;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + (uint32_t)poff[j]), "l"(g),
                     "r"(ok ? 16 : 0)
                     : "memory");
      }
      asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&sfull[slot])) : "memory");
      ++it_i;
      if (it_i == nd) {
        ++it_item;
        it_i = 0;
        if (it_item < item_end) decode(it_item, n, h0, w0, d0, nd);
      }
      ++sl;
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else {
    // ===================================================== epilogue warps 4..7
    const int q = warp & 3;
    const int row = q * 32 + lane;
    const int rw = row % HT_W, rh = row / HT_W;
    const int etid = (warp - 4) * 32 + lane;
    uint32_t go = 0;
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
          atomicAdd(p.stats + ((long long)n * p.Cout + c) * 2 + which, t);
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    };
    for (int item = item_begin; item < item_end; ++item) {
      int n, h0, w0, d0, nd;
      decode(item, n, h0, w0, d0, nd);
      if (n != cur_n) {
        if (cur_n >= 0 && p.stats != nullptr) flush_stats(cur_n);
        cur_n = n;
      }
      const int oh = h0 + rh, ow = w0 + rw;
      const bool valid = oh < p.H && ow < p.W;
      for (int o = 0; o < nd; ++o, ++go) {
        const long long vox = (((long long)n * p.D + (d0 + o)) * p.H + oh) * p.W + ow;
        const uint32_t as = go & 1u;
        mbar_wait(&tfull[as], (go >> 1) & 1u);
        const float* tacc = s_acc + row * p.acc_pitch + as * COUT;
        for (int c0 = 0; c0 < p.Cout; c0 += 16) {
          float v[16];
          acc_ld16(tacc + c0, v);
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
              const int col = stat_col(lane);
              // this lane is the only writer of its column in this warp's private row: no atomics, fixed order
              float* sw_ = s_stat + q * 2 * p.Cout;
              sw_[c0 + col] += s[0];
              sw_[p.Cout + c0 + col] += qq[0];
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
            store8(p.y + vox * p.yld + c0, v);
            store8(p.y + vox * p.yld + c0 + 8, v + 8);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&tempty[as]);
      }
    }
    if (p.stats != nullptr && cur_n >= 0) flush_stats(cur_n);
  }
}


// ------------------------------------------------------------------------------------------------
// Input-slice-major form of the 3-D kernel (KD = 3): every staged input slice is multiplied ONCE per (kh, kw, K chunk)
// against the weights of all three kd taps side by side, B = [W(kd=2) | W(kd=1) | W(kd=0)] (N = 3*Cout columns), and
// accumulates into the three output slices (i-2, i-1, i) it contributes to.  An MMA instruction re-reads its A operand
// (the voxel rows) from shared memory whatever N is, so 9 instructions of N = 3*Cout per input slice instead of 27 of
// N = Cout per output slice do the same MACs with a third of the A reads.
//   * work split: the output space is T = N * th * tw * D slice tiles ordered (n, h tile, w tile, d); CTA b of G owns
//     [b*T/G, (b+1)*T/G) and walks it as column segments (n, h0, w0, d_a, nd).  A segment stages input slices
//     d_a-1 .. d_a+nd (zero filled outside the volume).  All three roles take their segments from halo3_segment, so
//     their slice and output sequences, and with them the mbarrier parities, agree;
//   * accumulators: the MMA warpgroup holds the three outputs of the slice being multiplied in registers, 3*Cout/2
//     fp32 per M64 half, in one fixed order: columns [0, Cout) output i-2, then i-1, then i.  A wgmma instruction
//     takes its accumulator as one contiguous register range, so the three outputs cannot rotate in place from slice
//     to slice (ptxas would copy them between the instructions and wait for each one); they shift down by one output
//     per slice instead, 2*Cout register moves per thread;
//   * every slice runs the full N = 3*Cout: at the ends of a segment the outputs before d_a and from d_a+nd on
//     accumulate into columns that are zeroed before their first real use.  That keeps one instruction shape for
//     2/(nd+2) extra tensor work, and every real output still sums exactly its three slices, in the same order, from
//     zero;
//   * the chain of slice i is waited for right after its issue (a wait further on, behind the mbarrier traffic, makes
//     ptxas serialise every instruction of the chain); output i-2 is then complete and is written once to a
//     double-buffered fp32 staging tile in shared memory (tfull / tempty, as in the 2-D kernel) for the epilogue;
//   * registers per role (setmaxnreg): the loader warpgroup gives most of its share to the MMA warpgroup (three outputs'
//     accumulators plus descriptors) and the epilogue (per-row GroupNorm sums of every channel);
//   * the weight image in smem is the packed image permuted at load time to [(kh,kw)][Cin/8][kd reversed][Cout][8].
// 384 threads (4 MMA, 4 epilogue, 4 loader warps), one CTA per SM.
// ------------------------------------------------------------------------------------------------
constexpr int kH3Loaders = 4;          // loader warps of the input-slice-major kernel (warps 8..11)
constexpr int kH3Threads = 32 * (4 + 4 + kH3Loaders);   // 384 threads
// registers per thread after setmaxnreg; at 1 CTA of 384 threads each thread starts with 168 and the three roles
// (one warpgroup each) may hold at most 3 * 168 between them
constexpr uint32_t kH3RegsMma = 224, kH3RegsEpi = 224, kH3RegsLoad = 56;
static_assert(kH3RegsMma + kH3RegsEpi + kH3RegsLoad <= 3 * 168, "register budget of conv_halo3_kernel");

// this CTA's share [begin, end) of the N * th * tw * D output slice tiles
__device__ __forceinline__ void halo3_range(const HaloArgs& p, int& begin, int& end) {
  const long long ntiles = (long long)p.N * p.th * p.tw * p.D;
  begin = (int)(ntiles * blockIdx.x / gridDim.x);
  end = (int)(ntiles * (blockIdx.x + 1) / gridDim.x);
}

// one column segment of a CTA's output range: nd output slices from (n, d0) of the (h0, w0) column
struct Halo3Seg {
  int n, h0, w0, d0, nd;
};
// the segment starting at output slice tile t of a CTA range that ends at `end` (tiles ordered (n, h tile, w tile, d))
__device__ __forceinline__ Halo3Seg halo3_segment(const HaloArgs& p, int t, int end) {
  Halo3Seg s;
  s.d0 = t % p.D;
  int c = t / p.D;
  const int iw = c % p.tw;
  c /= p.tw;
  const int ih = c % p.th;
  s.n = c / p.th;
  s.w0 = iw * HT_W;
  s.h0 = ih * HT_H;
  s.nd = min(p.D - s.d0, end - t);
  return s;
}

template <int CIN, int COUT, bool BWD>
__global__ void __launch_bounds__(kH3Threads, 1) conv_halo3_kernel(const HaloArgs p) {
  PDL_TRIGGER();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
  constexpr int KD = 3;
  constexpr int CP = CIN / 8;                                // 8-channel planes
  constexpr uint32_t PLANE = HP_H * HP_W * 16u;              // bytes of one plane of one slice
  constexpr uint32_t SLICE = (uint32_t)CP * PLANE;
  constexpr int taps = 27;
  constexpr uint32_t W_BYTES = (uint32_t)taps * CIN * COUT * 2u;
  uint8_t* s_w = smem;
  uint8_t* s_ring = smem + ((W_BYTES + 127u) & ~127u);
  uint8_t* tail = s_ring + (size_t)p.nslices * SLICE;
  tail = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tail) + 15) & ~(uintptr_t)15);
  uint64_t* sfull = reinterpret_cast<uint64_t*>(tail);
  uint64_t* sempty = sfull + kHaloMaxSlices;
  uint64_t* tfull = sempty + kHaloMaxSlices;
  uint64_t* tempty = tfull + 2;
  float* s_stat = reinterpret_cast<float*>(tempty + 2);      // [4 epilogue warps][2][Cout]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nslices; ++s) {
      mbar_init(&sfull[s], 1);                   // ONE arrive: by the loader warp that staged the slice
      mbar_init(&sempty[s], 4);                  // one arrive per MMA warp
    }
    for (int a = 0; a < 2; ++a) {
      mbar_init(&tfull[a], 4);
      mbar_init(&tempty[a], 4);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 8 * p.Cout; i += blockDim.x) s_stat[i] = 0.f;
  float* s_bias = s_stat + 8 * COUT;
  float* s_ab = s_bias + COUT;                                       // [2][Cout]: A, B of the sample being processed
  double* s_gd = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(s_ab + 2 * COUT) + 7) & ~(uintptr_t)7);   // [2][Cout] + [8][2]
  // staging tile [128 rows][2 buffers x Cout] fp32: completed outputs on their way from the MMA warpgroup to the epilogue
  float* s_acc = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(s_gd + 2 * COUT + 16) + 15) & ~(uintptr_t)15);
  __syncthreads();
  // everything above is on-chip set-up and runs under the tail of the previous kernel; global memory from here on
  PDL_WAIT();
  // resident weights: 16-byte granules of the packed image [tap = (kd,kh,kw)][plane][co] -> [(kh,kw)][plane][2-kd][co]
  for (uint32_t g = threadIdx.x; g < W_BYTES / 16u; g += blockDim.x) {
    const uint32_t co = g % COUT;
    const uint32_t t1 = g / COUT;
    const uint32_t plane = t1 % CP;
    const uint32_t tap = t1 / CP;
    const uint32_t kd = tap / 9u, t9 = tap - kd * 9u;
    const uint32_t dst = ((t9 * CP + plane) * 3u + (2u - kd)) * COUT + co;
    *reinterpret_cast<uint4*>(s_w + dst * 16u) = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.w) + g * 16u);
  }
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) s_bias[i] = p.bias != nullptr ? p.bias[i] : 0.f;
  fence_proxy_async();
  __syncthreads();
  constexpr int pd = 1;

  if (warp < 4) {
    // ===================================================== MMA warpgroup
    setmaxnreg_inc<kH3RegsMma>();
    const int wt = threadIdx.x;
    const uint64_t a_hi = make_nosw_desc(0, PLANE, HP_W * 16u);
    const uint64_t b_base = make_nosw_desc(smem_u32(s_w), 3u * COUT * 16u, 128u);
    const uint32_t ring_u32 = smem_u32(s_ring);
    constexpr int kchunks = CIN / 16;
    constexpr int F = COUT / 2;   // fragment registers of one output (Cout columns) per M64 half
    // [M64 half][3 outputs x F]: while slice i is multiplied in, columns [0, F) hold output i-2, [F, 2F) output i-1
    // and [2F, 3F) output i
    float acc0[3 * F], acc1[3 * F];
    frag_zero(acc0);
    frag_zero(acc1);
    int t_begin, t_end;
    halo3_range(p, t_begin, t_end);
    uint32_t gs = 0;   // input slices of earlier segments (ring position of the segment's first slice)
    uint32_t go = 0;   // outputs of earlier segments (staging position of the segment's first output)
    for (int t = t_begin; t < t_end;) {
      const Halo3Seg s = halo3_segment(p, t, t_end);
      const int nsl = s.nd + KD - 1;
      for (int i = 0; i < nsl; ++i) {
        // [i-3, i-2, i-1] -> [i-2, i-1, i (zero)]
#pragma unroll
        for (int j = 0; j < 2 * F; ++j) {
          acc0[j] = acc0[j + F];
          acc1[j] = acc1[j + F];
        }
#pragma unroll
        for (int j = 2 * F; j < 3 * F; ++j) acc0[j] = acc1[j] = 0.f;
        const uint32_t sl = gs + (uint32_t)i;
        mbar_wait(&sfull[sl % p.nslices], (sl / p.nslices) & 1u);
        // (the loader warp that staged the slice has waited for its cp.async group and executed
        //  fence.proxy.async BEFORE the arrive: the data is already ordered for the tensor core's async-proxy reads)
        const uint64_t a_base = a_hi | (uint64_t)((ring_u32 + (sl % p.nslices) * SLICE) >> 4);
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        wgmma_fence();
        // straight-line issue: every descriptor is (slice / weight base) + compile-time offset, in 16-byte units
#pragma unroll
        for (int t9 = 0; t9 < 9; ++t9)
#pragma unroll
          for (int kc = 0; kc < kchunks; ++kc) {
            const uint32_t a_off = ((uint32_t)(2 * kc) * PLANE + (uint32_t)((t9 / 3) * HP_W + (t9 % 3)) * 16u) >> 4;
            const uint32_t b_off = ((uint32_t)(t9 * CP + 2 * kc) * 3u * COUT * 16u) >> 4;
            Wgmma<3 * COUT, 0, 0>::mma(acc0, a_base + a_off, b_base + b_off);
            Wgmma<3 * COUT, 0, 0>::mma(acc1, a_base + a_off + (8u * HP_W * 16u >> 4), b_base + b_off);   // hh 8..15
          }
        wgmma_commit();
        wgmma_wait0();
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&sempty[sl % p.nslices]);   // this input slice is consumed
        if (i >= 2) {
          // output i-2 has all three contributions
          const uint32_t o = go + (uint32_t)(i - 2);
          const uint32_t as = o & 1u;
          mbar_wait(&tempty[as], ((o >> 1) & 1u) ^ 1u);
          frag_store(s_acc + as * COUT, p.acc_pitch, 0, reinterpret_cast<const float(&)[F]>(acc0[0]), wt);
          frag_store(s_acc + as * COUT, p.acc_pitch, 64, reinterpret_cast<const float(&)[F]>(acc1[0]), wt);
          __syncwarp();
          if (lane == 0) mbar_arrive(&tfull[as]);
        }
      }
      gs += (uint32_t)nsl;
      go += (uint32_t)s.nd;
      t += s.nd;
    }
  } else if (warp >= 8) {
    // ===================================================== loaders: 4 warps, warp w stages the input slices
    // sl = w (mod 4) on its own (all pieces of the slice, 16-byte cp.async with zero fill = conv padding), waits
    // for them to land and signals the slice with ONE mbarrier arrive.  The warps run independently: four slices
    // are in flight per CTA.
    setmaxnreg_dec<kH3RegsLoad>();
    const int lw = warp - 8;
    constexpr int pieces = HP_H * HP_W * CP;
    int t_begin, t_end;
    halo3_range(p, t_begin, t_end);
    int t = t_begin, it_i = 0, it_nsl = 0;
    Halo3Seg s{0, 0, 0, 0, 0};
    auto load_seg = [&]() {
      if (t < t_end) {
        s = halo3_segment(p, t, t_end);
        it_nsl = s.nd + KD - 1;
      }
    };
    auto advance = [&](int steps) {
      it_i += steps;
      while (t < t_end && it_i >= it_nsl) {
        it_i -= it_nsl;
        t += s.nd;
        load_seg();
      }
    };
    load_seg();
    advance(lw);
    uint32_t sl = (uint32_t)lw, prev_sl = 0u;
    bool have_prev = false;
    auto signal = [&](uint32_t which) {
      fence_proxy_async();            // landed cp.async data -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(&sfull[which % p.nslices]);
    };
    while (t < t_end) {
      const uint32_t slot = sl % p.nslices;
      mbar_wait(&sempty[slot], ((sl / p.nslices) & 1u) ^ 1u);
      const uint32_t dst = smem_u32(s_ring + (size_t)slot * SLICE);
      const int d = s.d0 - pd + it_i;
      const bool dok = (unsigned)d < (unsigned)p.D;
      const bf16* src = p.x + (((long long)s.n * p.D + (dok ? d : 0)) * p.H) * p.W * p.xld;
#pragma unroll 4
      for (int q = lane; q < pieces; q += 32) {
        const int v = q / CP, plane = q - v * CP;
        const int hh = v / HP_W, ww = v - hh * HP_W;
        const int h = s.h0 - 1 + hh, w = s.w0 - 1 + ww;
        const bool ok = dok && (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
        const bf16* g = ok ? src + ((long long)h * p.W + w) * p.xld + plane * 8 : p.x;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + (uint32_t)(plane * (int)PLANE + v * 16)),
                     "l"(g), "r"(ok ? 16 : 0)
                     : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      // two cp.async groups in flight per warp; signal the older one
      if (have_prev) {
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        signal(prev_sl);
      }
      prev_sl = sl;
      have_prev = true;
      advance(kH3Loaders);
      sl += kH3Loaders;
    }
    if (have_prev) {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      signal(prev_sl);
    }
  } else {
    // ===================================================== epilogue warps 4..7
    // GroupNorm statistics: per-thread (= per output row) partial sums in registers over ALL slices of a segment, one
    // butterfly fold over the warp per segment (not per slice); bias from shared memory; the staging buffer is
    // released right after the read, before the arithmetic.
    setmaxnreg_inc<kH3RegsEpi>();
    const int q = warp & 3;
    const int row = q * 32 + lane;
    const int rw = row % HT_W, rh = row / HT_W;
    const int etid = (warp - 4) * 32 + lane;
    uint32_t go = 0;
    int cur_n = -1;
    constexpr bool bwd = BWD;                 // backward-sums epilogue (b200seg_conv_bwdstats): its own instantiation,
    constexpr int sstride = BWD ? 3 : 2;      // so the plain kernel does not carry its registers
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
          atomicAdd(p.stats + ((long long)n * p.Cout + c) * sstride + which, t);
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    };
    const bool want_stats = p.stats != nullptr;
    int t_begin, t_end;
    halo3_range(p, t_begin, t_end);
    for (int t = t_begin; t < t_end;) {
      const Halo3Seg sg = halo3_segment(p, t, t_end);
      const int n = sg.n, h0 = sg.h0, w0 = sg.w0, d0 = sg.d0, nd = sg.nd;
      t += nd;
      // a CTA's range can cross into the next sample: its statistics go to that sample's rows from here on
      if (n != cur_n) {
        if (cur_n >= 0 && want_stats) flush_stats(cur_n);
        cur_n = n;
        // A, B of sample n for the ReLU mask of the backward sums: gn_coefs, so the mask here equals the one
        // gn_bwd_apply derives later
        if (bwd)
          gn_coefs<false, false>(GnNamedBarrier<1, 128>{etid}, p.gn, nullptr, n, COUT, s_gd, nullptr, s_ab,
                                 s_ab + COUT, nullptr, nullptr, nullptr);
      }
      const int oh = h0 + rh, ow = w0 + rw;
      const bool valid = oh < p.H && ow < p.W;
      float rs[COUT], rq[COUT];
#pragma unroll
      for (int j = 0; j < COUT; ++j) rs[j] = rq[j] = 0.f;
      for (int o = 0; o < nd; ++o, ++go) {
        const long long vox = (((long long)n * p.D + (d0 + o)) * p.H + oh) * p.W + ow;
        // backward-sums form: the epilogue's global operands (residual addend, the producer's raw output) are requested
        // BEFORE waiting for the accumulator
        uint4 adv[BWD ? COUT / 8 : 1], yfv[BWD ? COUT / 8 : 1];
        if constexpr (BWD) {
#pragma unroll
          for (int k_ = 0; k_ < COUT / 8; ++k_) {
            adv[k_] = make_uint4(0u, 0u, 0u, 0u);
            yfv[k_] = make_uint4(0u, 0u, 0u, 0u);
          }
          if (valid) {
            if (p.addend != nullptr) {
#pragma unroll
              for (int k_ = 0; k_ < COUT / 8; ++k_)
                adv[k_] = *reinterpret_cast<const uint4*>(p.addend + vox * p.ald + 8 * k_);
            }
#pragma unroll
            for (int k_ = 0; k_ < COUT / 8; ++k_)
              yfv[k_] = *reinterpret_cast<const uint4*>(p.yfwd + vox * p.yfld + 8 * k_);
          }
        }
        const uint32_t as = go & 1u;
        mbar_wait(&tfull[as], (go >> 1) & 1u);
        const float* tacc = s_acc + row * p.acc_pitch + as * COUT;
#pragma unroll
        for (int c0 = 0; c0 < COUT; c0 += 16) {
          float v[16];
          acc_ld16(tacc + c0, v);
          if (c0 + 16 >= COUT) {
            // every column of the buffer is read: release it before the arithmetic
            __syncwarp();
            if (lane == 0) mbar_arrive(&tempty[as]);
          }
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            const float4 b4 = *reinterpret_cast<const float4*>(s_bias + c0 + j);
            v[j] += b4.x; v[j + 1] += b4.y; v[j + 2] += b4.z; v[j + 3] += b4.w;
          }
          if (want_stats && valid && !bwd) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              rs[c0 + j] += v[j];
              rq[c0 + j] = fmaf(v[j], v[j], rq[c0 + j]);
            }
          }
          if (valid) {
            if (p.addend != nullptr) {
              if constexpr (BWD) {
#pragma unroll
                for (int h_ = 0; h_ < 2; ++h_) {
                  const __nv_bfloat162* a2 = reinterpret_cast<const __nv_bfloat162*>(&adv[c0 / 8 + h_]);
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
                    const float2 f = __bfloat1622float2(a2[j]);
                    v[8 * h_ + 2 * j] += f.x;
                    v[8 * h_ + 2 * j + 1] += f.y;
                  }
                }
              } else {
                float r[16];
                load8(p.addend + vox * p.ald + c0, r);
                load8(p.addend + vox * p.ald + c0 + 8, r + 8);
#pragma unroll
                for (int j = 0; j < 16; ++j) v[j] += r[j];
              }
            }
            if constexpr (!BWD) {
              store8(p.y + vox * p.yld + c0, v);
              store8(p.y + vox * p.yld + c0 + 8, v + 8);
            } else {
              // round g to bf16 once: the packed values are what is stored AND what the sums see (a separate reduce
              // pass would read the stored tensor); coefficients come as 128-bit shared-memory loads
#pragma unroll
              for (int h_ = 0; h_ < 2; ++h_) {
                uint4 pk;
                __nv_bfloat162* g2 = reinterpret_cast<__nv_bfloat162*>(&pk);
#pragma unroll
                for (int j = 0; j < 4; ++j) g2[j] = __floats2bfloat162_rn(v[8 * h_ + 2 * j], v[8 * h_ + 2 * j + 1]);
                *reinterpret_cast<uint4*>(p.y + vox * p.yld + c0 + 8 * h_) = pk;
                const __nv_bfloat162* y2 = reinterpret_cast<const __nv_bfloat162*>(&yfv[c0 / 8 + h_]);
                const int cb = c0 + 8 * h_;
                const float4 a0 = *reinterpret_cast<const float4*>(s_ab + cb), a1 = *reinterpret_cast<const float4*>(s_ab + cb + 4);
                const float4 b0 = *reinterpret_cast<const float4*>(s_ab + COUT + cb);
                const float4 b1 = *reinterpret_cast<const float4*>(s_ab + COUT + cb + 4);
                const float aa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float2 yy = __bfloat1622float2(y2[j]);
                  const float2 gg = __bfloat1622float2(g2[j]);
                  const float d0_ = fmaf(yy.x, aa[2 * j], bb[2 * j]) > 0.f ? gg.x : 0.f;
                  const float d1_ = fmaf(yy.y, aa[2 * j + 1], bb[2 * j + 1]) > 0.f ? gg.y : 0.f;
                  rs[cb + 2 * j] += d0_;
                  rs[cb + 2 * j + 1] += d1_;
                  rq[cb + 2 * j] = fmaf(d0_, yy.x, rq[cb + 2 * j]);
                  rq[cb + 2 * j + 1] = fmaf(d1_, yy.y, rq[cb + 2 * j + 1]);
                }
              }
            }
          }
        }
      }
      if (want_stats) {
        // fold the 32 rows of this warp: after the butterfly lane pair (2k, 2k+1) holds column col(k) of the chunk
#pragma unroll
        for (int c0 = 0; c0 < COUT; c0 += 16) {
          float s[16], qq[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            s[j] = rs[c0 + j];
            qq[j] = rq[c0 + j];
          }
          stat_butterfly(s, qq, lane);
          if ((lane & 1) == 0) {
            const int col = stat_col(lane);
            float* sw_ = s_stat + (warp - 4) * 2 * p.Cout;   // this warp's private row: no atomics, fixed order
            sw_[c0 + col] += s[0];
            sw_[p.Cout + c0 + col] += qq[0];
          }
        }
      }
    }
    if (want_stats && cur_n >= 0) flush_stats(cur_n);
  }
}

// ------------------------------------------------------------------------------------------------
static bool al16h(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

int conv_halo_channels_ok(int kind, int cin, int cout) {
  if (kind != B200SEG_K3) return 0;
  if (cin != 16 && cin != 32) return 0;
  if (cout != 16 && cout != 32) return 0;
  return 1;
}

// the packed-weight image: [tap][Cin/8][Cout][8]  (== T taps, K = Cin/8 chunks, N2 = Cout, N1 = 8)
int conv_halo_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                        const b200seg_tensor* addend) {
  (void)dims;
  if (w_dtype != B200SEG_BF16_HALO) return 0;
  if (!conv_halo_channels_ok(kind, x->c, y->c)) return 0;
  if (x->dtype != B200SEG_BF16 || y->dtype != B200SEG_BF16) return 0;
  if (addend && addend->dtype != B200SEG_BF16) return 0;
  if ((x->ld % 8) || (y->ld % 8) || !al16h(x->ptr) || !al16h(y->ptr)) return 0;
  if (addend && ((addend->ld % 8) || !al16h(addend->ptr))) return 0;
  if (x->d != y->d || x->h != y->h || x->w != y->w) return 0;
  return 1;
}

static int g_halo_init[64] = {0};

int conv_halo(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias, const b200seg_tensor* y,
              double* stats, const b200seg_tensor* addend, int device, cudaStream_t st, const b200seg_tensor* yfwd,
              const b200seg_gn* gn, double* sums) {
  (void)kind;
  const int maxsm = tc_max_smem(device);
  if (device >= 0 && device < 64 && !g_halo_init[device]) {
#define HALO_ATTR(CI, CO) \
  B200_CUDA(cudaFuncSetAttribute(conv_halo_kernel<CI, CO>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm))
    HALO_ATTR(16, 16); HALO_ATTR(16, 32); HALO_ATTR(32, 16); HALO_ATTR(32, 32);
#undef HALO_ATTR
#define HALO3_ATTR(CI, CO) \
  B200_CUDA(cudaFuncSetAttribute(conv_halo3_kernel<CI, CO, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm)); \
  B200_CUDA(cudaFuncSetAttribute(conv_halo3_kernel<CI, CO, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)); \
  B200_CUDA(cudaFuncSetAttribute(conv_halo3_kernel<CI, CO, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsm)); \
  B200_CUDA(cudaFuncSetAttribute(conv_halo3_kernel<CI, CO, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100))
    HALO3_ATTR(16, 16); HALO3_ATTR(16, 32); HALO3_ATTR(32, 16); HALO3_ATTR(32, 32);
#undef HALO3_ATTR
    g_halo_init[device] = 1;
  }
  HaloArgs p;
  p.x = static_cast<const bf16*>(x->ptr);
  p.w = static_cast<const bf16*>(wpk);
  p.y = static_cast<bf16*>(y->ptr);
  p.addend = addend ? static_cast<const bf16*>(addend->ptr) : nullptr;
  p.bias = bias;
  p.stats = stats;
  p.xld = x->ld; p.yld = y->ld; p.ald = addend ? addend->ld : 0;
  p.N = x->n; p.D = x->d; p.H = x->h; p.W = x->w;
  p.Cin = x->c; p.Cout = y->c;
  p.kd = dims == 3 ? 3 : 1;
  p.yfwd = nullptr; p.yfld = 0; p.gn = gn_ref(nullptr, 0);
  if (yfwd != nullptr) {
    B200_CHECK_ARG(dims == 3 && gn != nullptr && sums != nullptr && stats == nullptr,
                   "conv_halo: backward statistics need the 3-D input-slice-major kernel");
    B200_CHECK_ARG(same_geom(yfwd, y) && yfwd->dtype == B200SEG_BF16 && (yfwd->ld % 8) == 0 && al16h(yfwd->ptr) &&
                       gn->groups > 0 && (y->c % gn->groups) == 0 && gn->groups <= 8,
                   "conv_halo: bad forward tensor / GroupNorm reference for the backward statistics");
    p.yfwd = static_cast<const bf16*>(yfwd->ptr);
    p.yfld = yfwd->ld;
    p.gn = gn_ref(gn, y->c);
    p.stats = sums;
  }
  p.tw = (p.W + HT_W - 1) / HT_W;
  p.th = (p.H + HT_H - 1) / HT_H;
  const int cols = p.N * p.th * p.tw;
  const int sms = num_sms(device);
  // one CTA per SM with a deep slice ring; the 2-D kernel splits d so that the grid covers the chip
  const uint32_t slice = (uint32_t)(p.Cin / 8) * HP_H * HP_W * 16u;
  const uint32_t wbytes = ((uint32_t)(p.kd * 9) * p.Cin * p.Cout * 2u + 127u) & ~127u;
  uint32_t tail;
  p.acc_pitch = 2 * p.Cout + 4;
  if (p.kd == 3) {
    tail = (2 * kHaloMaxSlices + 4) * 8 + 16 + 11 * p.Cout * 4 + 64 + (2 * p.Cout + 16) * 8 + 8 + 16 +
           128u * (uint32_t)p.acc_pitch * 4u;
  } else {
    tail = (2 * kHaloMaxSlices + 4) * 8 + 16 + 8 * p.Cout * 4 + 64 + 16 + 128u * (uint32_t)p.acc_pitch * 4u;
  }
  const int slots = sms;
  int grid;
  if (p.kd == 3) {
    // the 3-D kernel splits the N * th * tw * D output slice tiles evenly over the CTAs
    const long long ntiles = (long long)cols * p.D;
    grid = ntiles < slots ? (int)ntiles : slots;
  } else {
    int ndch = 1;
    if (cols < slots) {
      ndch = slots / cols;               // items <= slots: one item per CTA, no second wave
      if (ndch > p.D) ndch = p.D;
      if (ndch < 1) ndch = 1;
    }
    p.dchunk = (p.D + ndch - 1) / ndch;
    p.ndchunks = (p.D + p.dchunk - 1) / p.dchunk;
    p.nitems = cols * p.ndchunks;
    grid = slots < p.nitems ? slots : p.nitems;
  }
  const int budget = maxsm;
  int ns = (int)((budget - 256 - (int)wbytes - (int)tail) / (int)slice);
  if (ns > kHaloMaxSlices) ns = kHaloMaxSlices;
  B200_CHECK_ARG(ns >= p.kd + 1, "conv_halo: slices do not fit in shared memory");
  p.nslices = ns;
  const size_t smem_bytes = 128 + wbytes + (size_t)ns * slice + tail;
#define HALO_LAUNCH(CI, CO) launch_k(conv_halo_kernel<CI, CO>, grid, kHaloThreads, smem_bytes, st, p)
#define HALO3_LAUNCH(CI, CO)                                                                             \
  do {                                                                                                   \
    if (p.yfwd != nullptr) launch_k(conv_halo3_kernel<CI, CO, true>, grid, kH3Threads, smem_bytes, st, p);  \
    else launch_k(conv_halo3_kernel<CI, CO, false>, grid, kH3Threads, smem_bytes, st, p);                \
  } while (0)
  if (p.kd == 3) {
    if (p.Cin == 16 && p.Cout == 16) HALO3_LAUNCH(16, 16);
    else if (p.Cin == 16) HALO3_LAUNCH(16, 32);
    else if (p.Cout == 16) HALO3_LAUNCH(32, 16);
    else HALO3_LAUNCH(32, 32);
  } else {
    if (p.Cin == 16 && p.Cout == 16) HALO_LAUNCH(16, 16);
    else if (p.Cin == 16) HALO_LAUNCH(16, 32);
    else if (p.Cout == 16) HALO_LAUNCH(32, 16);
    else HALO_LAUNCH(32, 32);
  }
#undef HALO_LAUNCH
#undef HALO3_LAUNCH
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
