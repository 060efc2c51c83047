// Fused input block of VNet3d / ResNet3d (VNet3d.py:25-43): two single-image-channel stems -- conv1 3x3x3 and
// conv2 1x1x1, 16 channels each -- normalised by ONE GroupNorm(8, 16) with their own statistics, dropped, ReLU'd
// and summed.  With one fp32 image channel in (4 B per voxel) and 2 x 16 bf16 channels out (64 B per voxel), the
// stored stem outputs y_a, y_b are 16x the bytes of what they are computed from.  These kernels never store them:
// every pass recomputes both from the image, with the instruction sequence of stem_mma.cu on the same operands
// (same bf16 rounding of the image, same bias add, same mma.sync fragments, same bf16 rounding of y), so the
// recomputed values are bit-identical to what the stem convolution would have written.
//
//   STATS   per-(n, c) sum y, sum y^2 of both branches (fp64; the stem epilogue's order and convention: sums of the
//           fp32 accumulators, lanes -> warps -> one fp64 atomic per CTA and sample)
//   APPLY   out = relu(y_a*A_a + B_a) + relu(y_b*A_b + B_b), A/B derived per CTA from the statistics, gamma, beta
//           and the dropout scale exactly as apply_kernel does (gn_cta_coefs), written into a pitched buffer
//   BSUMS   per-(n, c) sum g*m, sum g*m*y, sum y of both branches (m = ReLU mask), the layout gn_bwd_apply_gn reads
//   BWD     dy = g*m*P + y*Q + R per branch (rounded to bf16 as the stored dy is), kept on chip and fed straight into
//           both stem weight gradients (the fragment path of wgrad_stem_mma_kernel); d gamma, d beta and both bias
//           gradients from the sums (param_grads_of_sample).  The input block has no data gradient.
//
// A CTA walks the stem's tile sequence (8 rows x TW columns of one (n, d) slice); the image window of tile i+1 (and
// the g tile, cp.async) is loaded while tile i is computed.  Each warp takes 16-voxel groups; per group it recomputes
// both branches with 6 mma.sync (2 k-steps x 2 n-tiles for the 27 taps, 1 x 2 for the single tap: the 1x1x1 branch
// reads the centre of the same halo tile).
#include "stem_mma.cuh"
#include "gn_coef.cuh"

namespace b200seg {

enum { SG_STATS = 0, SG_APPLY = 1, SG_BSUMS = 2, SG_BWD = 3 };

constexpr int SG_C = 16;                       // output channels of each branch
constexpr int SG_GROUPS = 8;                   // GroupNorm(8, 16)

struct StemGnParams {
  const bf16* wa;                              // [27][16] packed forward operand of the 3x3x3 branch
  const float* ba;
  const bf16* wb;                              // [1][16] of the 1x1x1 branch
  const float* bb;
  GnRef gna, gnb;                              // APPLY / BSUMS / BWD (stats in)
  double* stats_a;                             // STATS out, [N][16][2] (zero on entry)
  double* stats_b;
  bf16* out;                                   // APPLY out
  long long ldo;
  const bf16* g;                               // BSUMS / BWD: activation gradient of the block output
  long long ldg;
  double* sums_a;                              // BSUMS out (zero on entry) / BWD in, [N][16][3]
  double* sums_b;
  float* dwa;                                  // BWD: += [27][16]
  float* dwb;                                  // BWD: += [1][16]
  float* dgamma;                               // BWD: += [16]
  float* dbeta;
  float* dba;                                  // BWD: += [16] (may be null)
  float* dbb;
};

// shared-memory carve-up (bytes); identical on host and device
struct SgSmem {
  size_t x, coef, red, gt, dys, total;
};
__host__ __device__ inline SgSmem sg_smem(int mode, int TW) {
  SgSmem s;
  s.x = 0;
  const size_t xb = (((size_t)2 * 3 * (SM_TH + 2) * (TW + 2) * 2) + 15) & ~(size_t)15;
  s.coef = xb;                                                                   // doubles first (8-byte aligned)
  const size_t coefb = gn_cta_doubles(SG_C, SG_GROUPS, true) * sizeof(double) + (size_t)(3 + 2 * 5 + 2) * SG_C * sizeof(float);
  s.red = s.coef + ((coefb + 15) & ~(size_t)15);
  const size_t redb = (size_t)8 * 2 * 3 * SG_C * sizeof(float);
  s.gt = s.red + redb;
  size_t gtb = 0;
  if (mode >= SG_BSUMS) {
    gtb = (size_t)2 * SM_TH * TW * SG_C * 2;
    const size_t fold = (size_t)8 * SG_C * 32 * sizeof(float);                  // BWD: the cross-warp dW fold
    if (mode == SG_BWD && gtb < fold) gtb = fold;
  }
  s.dys = s.gt + gtb;
  const size_t dysb = mode == SG_BWD ? (size_t)8 * 2 * 16 * SG_C * 2 : 0;
  s.total = s.dys + dysb;
  return s;
}

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// BWD keeps 20 weight-gradient accumulators on top of the recompute: one CTA per SM (144 registers, no spills); the
// other passes run two
template <int MODE>
__global__ void __launch_bounds__(SM_THREADS, MODE == SG_BWD ? 1 : 2)
    stem_gn_kernel(const float* __restrict__ x, const __grid_constant__ StemGnParams p, const StemGeom g) {
  PDL_ENTER();
  constexpr int KD = 3, KHW = 3, PAD = 1;
  constexpr int TAPS = 27, KS = 2, NT = 2;     // 3x3x3 branch: 32 padded taps = 2 k-steps; 16 channels = 2 n-tiles
  constexpr int C = SG_C;
  constexpr bool BWD = MODE == SG_BWD;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SgSmem L = sg_smem(MODE, g.TW);
  const int XP = g.TW + 2 * PAD;
  const int xtile = XStage<float, KD, PAD>::ROWS * XP;
  unsigned short* xs0 = reinterpret_cast<unsigned short*>(smem_raw);
  double* s_d = reinterpret_cast<double*>(smem_raw + L.coef);
  float* s_f = reinterpret_cast<float*>(s_d + gn_cta_doubles(C, SG_GROUPS, true));
  float* s_cf = s_f + 3 * C;                   // [2 branches][A, B, P, Q, R][C]
  float* s_bias = s_cf + 10 * C;               // [2 branches][C]
  float* s_red = reinterpret_cast<float*>(smem_raw + L.red);
  unsigned char* gt0 = smem_raw + L.gt;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, tq = lane & 3;
  const int gtile = SM_TH * g.TW * C;          // bf16 elements per g buffer

  // weight fragments and tap offsets of the 3x3x3 branch (as conv_stem_mma_kernel<float, 16, 3, 3>)
  uint32_t wa[KS][NT][2];
  int off[KS][4];
#pragma unroll
  for (int s = 0; s < KS; ++s) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int tap = s * 16 + 2 * tq + (j & 1) + (j >> 1) * 8;
      const int o = tap_offset<KD, KHW>(tap, XP);
      off[s][j] = o < 0 ? 0 : o;
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t0 = s * 16 + 2 * tq + 8 * h;
        const int co = nt * 8 + gq;
        const unsigned short lo = t0 < TAPS ? bf16_bits(p.wa[t0 * C + co]) : (unsigned short)0;
        const unsigned short hi = t0 + 1 < TAPS ? bf16_bits(p.wa[(t0 + 1) * C + co]) : (unsigned short)0;
        wa[s][nt][h] = pack16(lo, hi);
      }
  }
  // 1x1x1 branch: one tap (the centre of the halo tile); the padding taps of its k-step have zero weights
  const int cen = ((KD / 2) * (SM_TH + 2 * PAD) + PAD) * XP + PAD;
  uint32_t wb[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int co = nt * 8 + gq;
    wb[nt][0] = pack16(tq == 0 ? bf16_bits(p.wb[co]) : (unsigned short)0, 0);
    wb[nt][1] = 0u;
  }
  // conv biases (read per 16-voxel group from shared memory: registers are the scarce resource here)
  if ((int)threadIdx.x < 2 * C) {
    const float* bsrc = threadIdx.x < C ? p.ba : p.bb;
    s_bias[threadIdx.x] = bsrc ? bsrc[threadIdx.x & (C - 1)] : 0.f;
  }

  // per-lane partial sums: STATS {sum, sumsq}, BSUMS {g*m, g*m*y, y}, per branch, per (n-tile, channel of the pair)
  float f1[2][NT][2], f2[2][NT][2], f3[2][NT][2];
#pragma unroll
  for (int b = 0; b < 2; ++b)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) f1[b][nt][j] = f2[b][nt][j] = f3[b][nt][j] = 0.f;

  // BWD: weight-gradient accumulators and the B-operand tap offsets (as wgrad_stem_mma_kernel)
  constexpr int WNT = 4;                       // n-tiles of 8 taps covering 27
  float acc_wa[WNT][4], acc_wb[4];
  int woff[WNT];
#pragma unroll
  for (int nt = 0; nt < WNT; ++nt) {
    const int o = tap_offset<KD, KHW>(nt * 8 + gq, XP);        // < 0 (padding tap) only for nt = 3, gq >= 3
    woff[nt] = (o < 0 ? 0 : o) + 2 * tq;
#pragma unroll
    for (int k = 0; k < 4; ++k) acc_wa[nt][k] = 0.f;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) acc_wb[k] = 0.f;

  // coefficients of sample n, both branches, into s_cf (every thread calls: block barriers).  The lanes read them
  // from shared memory where they are used: the registers go to the prefetched image window and the accumulators.
  auto load_coefs = [&](int n) {
    gn_cta_coefs<BWD>(p.gna, p.sums_a, n, C, s_d, s_f, s_cf, s_cf + C, s_cf + 2 * C, s_cf + 3 * C, s_cf + 4 * C);
    float* cb = s_cf + 5 * C;
    gn_cta_coefs<BWD>(p.gnb, p.sums_b, n, C, s_d, s_f, cb, cb + C, cb + 2 * C, cb + 3 * C, cb + 4 * C);
  };
  // coefficient k (0..4 = A, B, P, Q, R) of branch b for the lane's channel pair of n-tile nt
  auto cf = [&](int b, int k, int nt) {
    return *reinterpret_cast<const float2*>(s_cf + (b * 5 + k) * C + nt * 8 + 2 * tq);
  };

  // fold the lane partials of sample n: lanes of a channel pair -> per-warp rows -> fp64 over warps -> one atomic
  auto flush_sums = [&](int n) {
    constexpr int K = MODE == SG_STATS ? 2 : 3;
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          float v[3] = {f1[b][nt][j], f2[b][nt][j], f3[b][nt][j]};
#pragma unroll
          for (int k = 0; k < K; ++k) {
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
            if (gq == 0) s_red[((warp * 2 + b) * K + k) * C + nt * 8 + 2 * tq + j] = v[k];
          }
          f1[b][nt][j] = f2[b][nt][j] = f3[b][nt][j] = 0.f;
        }
    __syncthreads();
    if ((int)threadIdx.x < 2 * K * C) {
      const int b = threadIdx.x / (K * C), r = threadIdx.x - b * K * C, k = r / C, c = r - k * C;
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += (double)s_red[((w * 2 + b) * K + k) * C + c];
      double* dst = MODE == SG_STATS ? (b ? p.stats_b : p.stats_a) : (b ? p.sums_b : p.sums_a);
      atomicAdd(dst + ((long long)n * C + c) * K + k, t);
    }
    __syncthreads();
  };

  auto load_g = [&](int buf, int n, int d, int h0, int w0) {
    // one tile row per warp; 16-byte chunks straight into [vox][16] rows
    const bf16* src = p.g + ((((long long)n * g.D + d) * g.H + h0 + warp) * g.W + w0) * p.ldg;
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(gt0 + ((size_t)buf * gtile + (size_t)warp * g.TW * C) * 2);
    const int chunks = g.TW * (C / 8);
    for (int q = lane; q < chunks; q += 32) {
      const int vox = q >> 1, part = q & 1;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)(vox * C + part * 8) * 2),
                   "l"(src + (long long)vox * p.ldg + part * 8)
                   : "memory");
    }
  };

  const int tpc = (g.tiles + gridDim.x - 1) / gridDim.x;
  const int first = blockIdx.x * tpc;
  const int last = min(g.tiles, first + tpc);
  XStage<float, KD, PAD> st;
  int n = 0, d = 0, h0 = 0, w0 = 0;
  if (first < last) {
    stem_decode(g, first, n, d, h0, w0);
    st.load(x, g, n, d, h0, w0, warp, lane);
    if (MODE >= SG_BSUMS) load_g(0, n, d, h0, w0);
    st.store(xs0, XP, g.TW, warp, lane);
    if (MODE >= SG_BSUMS) asm volatile("cp.async.wait_all;" ::: "memory");
  }
  __syncthreads();
  if (MODE != SG_STATS && first < last) load_coefs(n);
  const int segs = g.TW / 16;
  int cur_n = n;
  for (int tile = first; tile < last; ++tile) {
    const int buf = (tile - first) & 1;
    const unsigned short* xs = xs0 + buf * xtile;
    int nn = 0, nd = 0, nh0 = 0, nw0 = 0;
    const bool more = tile + 1 < last;
    if (more) {
      stem_decode(g, tile + 1, nn, nd, nh0, nw0);
      st.load(x, g, nn, nd, nh0, nw0, warp, lane);
      if (MODE >= SG_BSUMS) load_g(buf ^ 1, nn, nd, nh0, nw0);
    }
    const bf16* gtb = reinterpret_cast<const bf16*>(gt0) + (size_t)buf * gtile;
    for (int ks = warp; ks < SM_TH * segs; ks += 8) {
      const int row = ks / segs, seg = ks - row * segs;
      const int pp = row * XP + seg * 16 + gq;
      // ---- recompute both branches: ya / yb[nt][0..3] = (voxel gq, ch 2tq, 2tq+1), (voxel gq+8, same channels)
      float ya[NT][4], yb[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const float2 ba = *reinterpret_cast<const float2*>(s_bias + nt * 8 + 2 * tq);
        const float2 bb = *reinterpret_cast<const float2*>(s_bias + C + nt * 8 + 2 * tq);
        ya[nt][0] = ya[nt][2] = ba.x;
        ya[nt][1] = ya[nt][3] = ba.y;
        yb[nt][0] = yb[nt][2] = bb.x;
        yb[nt][1] = yb[nt][3] = bb.y;
      }
#pragma unroll
      for (int s = 0; s < KS; ++s) {
        uint32_t a[4];
        a[0] = pack16(xs[off[s][0] + pp], xs[off[s][1] + pp]);
        a[1] = pack16(xs[off[s][0] + pp + 8], xs[off[s][1] + pp + 8]);
        a[2] = pack16(xs[off[s][2] + pp], xs[off[s][3] + pp]);
        a[3] = pack16(xs[off[s][2] + pp + 8], xs[off[s][3] + pp + 8]);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_bf16_16816(ya[nt], a, wa[s][nt][0], wa[s][nt][1]);
      }
      {
        const unsigned short c0 = xs[cen + pp], c8 = xs[cen + pp + 8];
        uint32_t a[4] = {pack16(c0, c0), pack16(c8, c8), pack16(c0, c0), pack16(c8, c8)};
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_bf16_16816(yb[nt], a, wb[nt][0], wb[nt][1]);
      }
      const long long v0 = (((long long)n * g.D + d) * g.H + h0 + row) * g.W + w0 + seg * 16 + gq;
      if constexpr (MODE == SG_STATS) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          f1[0][nt][0] += ya[nt][0] + ya[nt][2];
          f1[0][nt][1] += ya[nt][1] + ya[nt][3];
          f2[0][nt][0] = fmaf(ya[nt][0], ya[nt][0], fmaf(ya[nt][2], ya[nt][2], f2[0][nt][0]));
          f2[0][nt][1] = fmaf(ya[nt][1], ya[nt][1], fmaf(ya[nt][3], ya[nt][3], f2[0][nt][1]));
          f1[1][nt][0] += yb[nt][0] + yb[nt][2];
          f1[1][nt][1] += yb[nt][1] + yb[nt][3];
          f2[1][nt][0] = fmaf(yb[nt][0], yb[nt][0], fmaf(yb[nt][2], yb[nt][2], f2[1][nt][0]));
          f2[1][nt][1] = fmaf(yb[nt][1], yb[nt][1], fmaf(yb[nt][3], yb[nt][3], f2[1][nt][1]));
        }
      } else {
        // the values a stored stem output would hold
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            ya[nt][k] = bf16_round(ya[nt][k]);
            yb[nt][k] = bf16_round(yb[nt][k]);
          }
        if constexpr (MODE == SG_APPLY) {
          bf16* po = p.out + v0 * p.ldo + 2 * tq;
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const float2 A0 = cf(0, 0, nt), B0 = cf(0, 1, nt), A1 = cf(1, 0, nt), B1 = cf(1, 1, nt);
            float o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const bool j = k & 1;
              o[k] = fmaxf(fmaf(ya[nt][k], j ? A0.y : A0.x, j ? B0.y : B0.x), 0.f);
              o[k] += fmaxf(fmaf(yb[nt][k], j ? A1.y : A1.x, j ? B1.y : B1.x), 0.f);
            }
            *reinterpret_cast<__nv_bfloat162*>(po + nt * 8) = __floats2bfloat162_rn(o[0], o[1]);
            *reinterpret_cast<__nv_bfloat162*>(po + 8 * p.ldo + nt * 8) = __floats2bfloat162_rn(o[2], o[3]);
          }
        } else {
          // g of the lane's two voxels and four channels from the staged tile
          const bf16* gp = gtb + (size_t)(row * g.TW + seg * 16 + gq) * C + 2 * tq;
          float gv[NT][4];
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(gp + nt * 8));
            const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(gp + 8 * C + nt * 8));
            gv[nt][0] = lo.x;
            gv[nt][1] = lo.y;
            gv[nt][2] = hi.x;
            gv[nt][3] = hi.y;
          }
          if constexpr (MODE == SG_BSUMS) {
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
              const float2 A0 = cf(0, 0, nt), B0 = cf(0, 1, nt), A1 = cf(1, 0, nt), B1 = cf(1, 1, nt);
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const int j = k & 1;
                const float da = fmaf(ya[nt][k], j ? A0.y : A0.x, j ? B0.y : B0.x) > 0.f ? gv[nt][k] : 0.f;
                const float db = fmaf(yb[nt][k], j ? A1.y : A1.x, j ? B1.y : B1.x) > 0.f ? gv[nt][k] : 0.f;
                f1[0][nt][j] += da;
                f2[0][nt][j] = fmaf(da, ya[nt][k], f2[0][nt][j]);
                f3[0][nt][j] += ya[nt][k];
                f1[1][nt][j] += db;
                f2[1][nt][j] = fmaf(db, yb[nt][k], f2[1][nt][j]);
                f3[1][nt][j] += yb[nt][k];
              }
            }
          } else {
            // dy of both branches -> this warp's [2][16 vox][16 ch] bf16 scratch -> dY^T fragments (ldmatrix.trans)
            bf16* dys = reinterpret_cast<bf16*>(smem_raw + L.dys) + (size_t)warp * 2 * 16 * C;
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
              for (int nt = 0; nt < NT; ++nt) {
                const float2 A = cf(b, 0, nt), B = cf(b, 1, nt), P = cf(b, 2, nt), Q = cf(b, 3, nt), R = cf(b, 4, nt);
                float o[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  const bool j = k & 1;
                  const float yv = b ? yb[nt][k] : ya[nt][k];
                  const float dm = fmaf(yv, j ? A.y : A.x, j ? B.y : B.x) > 0.f ? gv[nt][k] * (j ? P.y : P.x) : 0.f;
                  o[k] = dm + fmaf(yv, j ? Q.y : Q.x, j ? R.y : R.x);
                }
                bf16* q = dys + (size_t)b * 16 * C + gq * C + nt * 8 + 2 * tq;
                *reinterpret_cast<__nv_bfloat162*>(q) = __floats2bfloat162_rn(o[0], o[1]);
                *reinterpret_cast<__nv_bfloat162*>(q + 8 * C) = __floats2bfloat162_rn(o[2], o[3]);
              }
            __syncwarp();
            const uint32_t dyb = (uint32_t)__cvta_generic_to_shared(dys);
            const int vrow = (lane >> 4) * 8 + (lane & 7);
            const int pw = row * XP + seg * 16;
            uint32_t af[4];
            auto ldm = [&](int b) {
              const uint32_t addr = dyb + (uint32_t)(b * 16 * C + vrow * C + ((lane >> 3) & 1) * 8) * 2;
              asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                           : "=r"(af[0]), "=r"(af[1]), "=r"(af[2]), "=r"(af[3])
                           : "r"(addr));
            };
            ldm(0);
#pragma unroll
            for (int nt = 0; nt < WNT; ++nt) {
              uint32_t b0 = 0u, b1 = 0u;
              if (nt < 3 || 24 + gq < TAPS) {
                const unsigned short* q = xs + woff[nt] + pw;
                b0 = pack16(q[0], q[1]);
                b1 = pack16(q[8], q[9]);
              }
              mma_bf16_16816(acc_wa[nt], af, b0, b1);
            }
            ldm(1);
            __syncwarp();                      // the scratch is rewritten by the next group
            {
              uint32_t b0 = 0u, b1 = 0u;
              if (gq == 0) {
                const unsigned short* q = xs + cen + 2 * tq + pw;
                b0 = pack16(q[0], q[1]);
                b1 = pack16(q[8], q[9]);
              }
              mma_bf16_16816(acc_wb, af, b0, b1);
            }
          }
        }
      }
    }
    if (more) {
      st.store(xs0 + (buf ^ 1) * xtile, XP, g.TW, warp, lane);
      if (MODE >= SG_BSUMS) asm volatile("cp.async.wait_all;" ::: "memory");
    }
    __syncthreads();
    if (more) {
      if (nn != cur_n) {
        if (MODE == SG_STATS || MODE == SG_BSUMS) flush_sums(cur_n);
        if (MODE != SG_STATS) load_coefs(nn);
        cur_n = nn;
      }
      n = nn; d = nd; h0 = nh0; w0 = nw0;
    }
  }
  if constexpr (MODE == SG_STATS || MODE == SG_BSUMS) {
    if (first < last) flush_sums(cur_n);
  }
  if constexpr (MODE == SG_BWD) {
    // fold the 8 warps: red[warp][co][32 taps] over the g buffers, then one atomic per (tap, co) per CTA
    float* red = reinterpret_cast<float*>(gt0);
    __syncthreads();
#pragma unroll
    for (int nt = 0; nt < WNT; ++nt) {
      float* r0 = red + ((size_t)warp * C + gq) * 32 + nt * 8 + 2 * tq;
      r0[0] = acc_wa[nt][0];
      r0[1] = acc_wa[nt][1];
      r0[8 * 32] = acc_wa[nt][2];
      r0[8 * 32 + 1] = acc_wa[nt][3];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C * 32; i += blockDim.x) {
      const int co = i >> 5, tap = i & 31;
      if (tap < TAPS) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += red[((size_t)k * C + co) * 32 + tap];
        atomicAdd(p.dwa + (long long)tap * C + co, t);
      }
    }
    __syncthreads();
    {
      float* r0 = red + ((size_t)warp * C + gq) * 32 + 2 * tq;
      r0[0] = acc_wb[0];
      r0[1] = acc_wb[1];
      r0[8 * 32] = acc_wb[2];
      r0[8 * 32 + 1] = acc_wb[3];
    }
    __syncthreads();
    if ((int)threadIdx.x < C) {
      const int co = threadIdx.x;
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += red[((size_t)k * C + co) * 32];
      atomicAdd(p.dwb + co, t);
    }
    // d gamma, d beta, d bias of both branches: one CTA per sample, from the sums (as gn_bwd_apply_kernel)
    for (int s = blockIdx.x; s < g.N; s += gridDim.x) {
      __syncthreads();
      const double* grp = gn_cta_coefs<true>(p.gna, p.sums_a, s, C, s_d, s_f, s_cf, s_cf + C, s_cf + 2 * C,
                                             s_cf + 3 * C, s_cf + 4 * C);
      param_grads_of_sample(p.gna, p.sums_a, grp, s_f, s, C, p.dgamma, p.dbeta, p.dba);
      __syncthreads();
      grp = gn_cta_coefs<true>(p.gnb, p.sums_b, s, C, s_d, s_f, s_cf, s_cf + C, s_cf + 2 * C, s_cf + 3 * C,
                               s_cf + 4 * C);
      param_grads_of_sample(p.gnb, p.sums_b, grp, s_f, s, C, p.dgamma, p.dbeta, p.dbb);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int stem_gn_supported(const b200seg_tensor* x, int cout, int dims) {
  if (x == nullptr || dims != 3 || cout != SG_C || x->dtype != B200SEG_F32) return 0;
  b200seg_tensor y = *x;
  y.c = SG_C;
  y.ld = SG_C;
  y.dtype = B200SEG_BF16;
  StemGeom g;
  return stem_mma_geom(x, &y, &g) ? 1 : 0;
}

static GnRef sg_gnref(const b200seg_gn* gn) {
  GnRef r;
  r.stats = gn->stats; r.gamma = gn->gamma; r.beta = gn->beta; r.scale = gn->scale; r.groups = gn->groups;
  r.m = (double)(SG_C / gn->groups) * (double)gn->vox;
  r.eps = gn->eps;
  r.sum_y_from_stats = 0;
  return r;
}

template <int MODE>
static int stem_gn_launch(const b200seg_tensor* x, const StemGnParams& p, int device, cudaStream_t st) {
  StemGeom g;
  b200seg_tensor y = *x;
  y.c = SG_C;
  y.ld = SG_C;
  y.dtype = B200SEG_BF16;
  B200_CHECK_ARG(stem_mma_geom(x, &y, &g), "b200seg_stem_gn: unsupported geometry");
  const size_t smem = sg_smem(MODE, g.TW).total;
  static int attr_done[64] = {0};
  if (smem > 48 * 1024 && device >= 0 && device < 64 && !attr_done[device]) {
    B200_CUDA(cudaFuncSetAttribute(stem_gn_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr_done[device] = 1;
  }
  const int grid = MODE == SG_BWD ? (g.tiles < num_sms(device) ? g.tiles : num_sms(device)) : stem_grid(g, device);
  launch_k(stem_gn_kernel<MODE>, grid, SM_THREADS, smem, st, static_cast<const float*>(x->ptr), p, g);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

static bool sg_gn_ok(const b200seg_gn* gn, const b200seg_tensor* x) {
  return gn && gn->stats && gn->gamma && gn->beta && gn->groups == SG_GROUPS &&
         gn->vox == (long long)x->d * x->h * x->w;
}

static bool sg_act_ok(const b200seg_tensor* t, const b200seg_tensor* x) {
  return t && t->ptr && t->dtype == B200SEG_BF16 && t->c == SG_C && t->n == x->n && t->d == x->d && t->h == x->h &&
         t->w == x->w && (t->ld % 8) == 0 && al16m(t->ptr);
}

int stem_gn(int mode, const b200seg_tensor* x, const void* wa, const float* ba, const void* wb, const float* bb,
            const b200seg_gn* gna, const b200seg_gn* gnb, double* stats_a, double* stats_b,
            const b200seg_tensor* out, const b200seg_tensor* gr, double* sums_a, double* sums_b, float* dwa,
            float* dwb, float* dgamma, float* dbeta, float* dba, float* dbb, int device, cudaStream_t st) {
  B200_CHECK_ARG(stem_gn_supported(x, SG_C, 3), "b200seg_stem_gn: unsupported image (fp32, one channel, 3-D, H %% 8 == 0, "
                 "W a multiple of 16)");
  B200_CHECK_ARG(wa && wb, "b200seg_stem_gn: null weights");
  StemGnParams p;
  memset(&p, 0, sizeof(p));
  p.wa = static_cast<const bf16*>(wa);
  p.ba = ba;
  p.wb = static_cast<const bf16*>(wb);
  p.bb = bb;
  if (mode == SG_STATS) {
    B200_CHECK_ARG(stats_a && stats_b, "b200seg_stem_gn_stats: null statistics");
    p.stats_a = stats_a;
    p.stats_b = stats_b;
    return stem_gn_launch<SG_STATS>(x, p, device, st);
  }
  B200_CHECK_ARG(sg_gn_ok(gna, x) && sg_gn_ok(gnb, x), "b200seg_stem_gn: bad GroupNorm reference (8 groups, vox = D*H*W)");
  p.gna = sg_gnref(gna);
  p.gnb = sg_gnref(gnb);
  if (mode == SG_APPLY) {
    B200_CHECK_ARG(sg_act_ok(out, x) && (out->ld % 2) == 0, "b200seg_stem_gn_apply: bad output tensor");
    p.out = static_cast<bf16*>(out->ptr);
    p.ldo = out->ld;
    return stem_gn_launch<SG_APPLY>(x, p, device, st);
  }
  B200_CHECK_ARG(sg_act_ok(gr, x), "b200seg_stem_gn: bad gradient tensor (bf16, 16 channels, 16-byte aligned rows)");
  B200_CHECK_ARG(sums_a && sums_b, "b200seg_stem_gn: null backward sums");
  p.g = static_cast<const bf16*>(gr->ptr);
  p.ldg = gr->ld;
  p.sums_a = sums_a;
  p.sums_b = sums_b;
  if (mode == SG_BSUMS) return stem_gn_launch<SG_BSUMS>(x, p, device, st);
  B200_CHECK_ARG(mode == SG_BWD && dwa && dwb && dgamma && dbeta, "b200seg_stem_gn_bwd: null gradient");
  p.dwa = dwa;
  p.dwb = dwb;
  p.dgamma = dgamma;
  p.dbeta = dbeta;
  p.dba = dba;
  p.dbb = dbb;
  return stem_gn_launch<SG_BWD>(x, p, device, st);
}

}  // namespace b200seg
