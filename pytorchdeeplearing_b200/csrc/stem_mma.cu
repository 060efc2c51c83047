// bf16 stem (Cin == 1) on the warp-level tensor-core path (mma.sync m16n8k16, sm_90a).
//
// The stem has one input channel: as a GEMM its K dimension is just the taps (27 -> padded to 32), far too thin
// for a wgmma tile, and on CUDA cores the 27-tap stencil is bound by shared-memory weight broadcasts (forward)
// or by load latency with 72 live accumulators (weight gradient).  Both directions are re-stated here as tiny
// im2col GEMMs whose operand fragments are gathered straight from a halo tile of the image in shared memory:
//
//   forward   Y[16 vox][COUT] += X[16 vox][32 taps] * W[32 taps][COUT]     (VNet3d.py:28-29, Unet3d.py:67)
//   wgrad     dW[COUT][32 taps] += dY^T[COUT][16 vox] * X[16 vox][32 taps]
//
// A CTA (8 warps) walks a contiguous range of tiles of 8 rows x TW columns of one (n, d) slice.  Per tile the
// image window (KD x 10 x (TW+2) values, zero halo = conv padding) is converted to bf16 in shared memory; the
// loads of tile i+1 are in flight (registers / cp.async) while tile i is multiplied.  A 16-voxel group costs
// ~16 LDS.U16 + 4 MMAs, so the kernels run at the speed of their HBM streams (image in, activations out / dY in).
// Bias, GroupNorm statistics (fixed order: lanes -> warps -> one fp64 atomic per CTA and sample) and the bf16
// NDHWC stores are fused into the forward epilogue.
#include "stem_mma.cuh"

namespace b200seg {

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
template <typename TA, int COUT, int KD, int KHW>
__global__ void __launch_bounds__(SM_THREADS, 2)
    conv_stem_mma_kernel(const TA* __restrict__ x, const bf16* __restrict__ w /*[taps][COUT]*/,
                         const float* __restrict__ bias, bf16* __restrict__ y, long long yld,
                         double* __restrict__ stats, const StemGeom g) {
  PDL_ENTER();
  constexpr int TAPS = KD * KHW * KHW;
  constexpr int PAD = KHW / 2;
  constexpr int KS = (TAPS + 15) / 16;
  constexpr int NT = COUT / 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int XP = g.TW + 2 * PAD;
  const int xtile = XStage<TA, KD, PAD>::ROWS * XP;                 // elements per buffer
  unsigned short* xs0 = reinterpret_cast<unsigned short*>(smem_raw);
  float* s_red = reinterpret_cast<float*>(smem_raw + (((size_t)2 * xtile * 2 + 15) & ~(size_t)15));   // [8][2*COUT]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, tq = lane & 3;

  // weight fragments (constant over the kernel) and this lane's tap offsets
  uint32_t wb[KS][NT][2];
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
        const unsigned short lo = t0 < TAPS ? bf16_bits(w[t0 * COUT + co]) : (unsigned short)0;
        const unsigned short hi = t0 + 1 < TAPS ? bf16_bits(w[(t0 + 1) * COUT + co]) : (unsigned short)0;
        wb[s][nt][h] = pack16(lo, hi);
      }
  }
  float bv[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bv[nt][0] = bias ? bias[nt * 8 + 2 * tq] : 0.f;
    bv[nt][1] = bias ? bias[nt * 8 + 2 * tq + 1] : 0.f;
  }
  float ssum[NT][2], ssq[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) ssum[nt][0] = ssum[nt][1] = ssq[nt][0] = ssq[nt][1] = 0.f;

  auto flush_stats = [&](int n) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float a = ssum[nt][j], b = ssq[nt][j];
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if (gq == 0) {
          s_red[warp * 2 * COUT + nt * 8 + 2 * tq + j] = a;
          s_red[warp * 2 * COUT + COUT + nt * 8 + 2 * tq + j] = b;
        }
        ssum[nt][j] = 0.f;
        ssq[nt][j] = 0.f;
      }
    __syncthreads();
    if (threadIdx.x < 2 * COUT) {
      double t = 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += (double)s_red[k * 2 * COUT + threadIdx.x];
      const int which = threadIdx.x / COUT, c = threadIdx.x - which * COUT;
      atomicAdd(stats + ((long long)n * COUT + c) * 2 + which, t);
    }
    __syncthreads();
  };

  const int tpc = (g.tiles + gridDim.x - 1) / gridDim.x;
  const int first = blockIdx.x * tpc;
  const int last = min(g.tiles, first + tpc);
  if (first >= last) return;
  XStage<TA, KD, PAD> st;
  int n, d, h0, w0;
  stem_decode(g, first, n, d, h0, w0);
  st.load(x, g, n, d, h0, w0, warp, lane);
  st.store(xs0, XP, g.TW, warp, lane);
  __syncthreads();
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
    }
    for (int ks = warp; ks < SM_TH * segs; ks += 8) {
      const int row = ks / segs, seg = ks - row * segs;
      const int p = row * XP + seg * 16 + gq;
      float acc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        acc[nt][0] = acc[nt][2] = bv[nt][0];
        acc[nt][1] = acc[nt][3] = bv[nt][1];
      }
#pragma unroll
      for (int s = 0; s < KS; ++s) {
        uint32_t a[4];
        a[0] = pack16(xs[off[s][0] + p], xs[off[s][1] + p]);
        a[1] = pack16(xs[off[s][0] + p + 8], xs[off[s][1] + p + 8]);
        a[2] = pack16(xs[off[s][2] + p], xs[off[s][3] + p]);
        a[3] = pack16(xs[off[s][2] + p + 8], xs[off[s][3] + p + 8]);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_bf16_16816(acc[nt], a, wb[s][nt][0], wb[s][nt][1]);
      }
      const long long v0 = (((long long)n * g.D + d) * g.H + h0 + row) * g.W + w0 + seg * 16 + gq;
      bf16* py = y + v0 * yld + 2 * tq;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        *reinterpret_cast<__nv_bfloat162*>(py + nt * 8) = __floats2bfloat162_rn(acc[nt][0], acc[nt][1]);
        *reinterpret_cast<__nv_bfloat162*>(py + 8 * yld + nt * 8) = __floats2bfloat162_rn(acc[nt][2], acc[nt][3]);
        ssum[nt][0] += acc[nt][0] + acc[nt][2];
        ssum[nt][1] += acc[nt][1] + acc[nt][3];
        ssq[nt][0] = fmaf(acc[nt][0], acc[nt][0], fmaf(acc[nt][2], acc[nt][2], ssq[nt][0]));
        ssq[nt][1] = fmaf(acc[nt][1], acc[nt][1], fmaf(acc[nt][3], acc[nt][3], ssq[nt][1]));
      }
    }
    if (more) st.store(xs0 + (buf ^ 1) * xtile, XP, g.TW, warp, lane);
    __syncthreads();
    if (more) {
      if (nn != cur_n) {
        if (stats != nullptr) flush_stats(cur_n);
        cur_n = nn;
      }
      n = nn; d = nd; h0 = nh0; w0 = nw0;
    }
  }
  if (stats != nullptr) flush_stats(cur_n);
}

// ------------------------------------------------------------------------------------------------
// weight gradient
// ------------------------------------------------------------------------------------------------
template <typename TA, int COUT, int KD, int KHW>
__global__ void __launch_bounds__(SM_THREADS, 2)
    wgrad_stem_mma_kernel(const TA* __restrict__ x, const bf16* __restrict__ dy, long long bld,
                          float* __restrict__ dwp /*[taps][COUT]*/, const StemGeom g) {
  PDL_ENTER();
  constexpr int TAPS = KD * KHW * KHW;
  constexpr int PAD = KHW / 2;
  constexpr int NT = (TAPS + 7) / 8;         // n-tiles of 8 taps
  constexpr int MT = COUT / 16;              // m-tiles of 16 output channels
  constexpr int CPV = COUT / 8;              // 16-byte chunks per voxel of dY
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int XP = g.TW + 2 * PAD;
  const int xtile = XStage<TA, KD, PAD>::ROWS * XP;
  const int dtile = SM_TH * g.TW * COUT;                                    // bf16 elements per dY buffer
  unsigned short* xs0 = reinterpret_cast<unsigned short*>(smem_raw);
  unsigned char* dy0 = smem_raw + (((size_t)2 * xtile * 2 + 15) & ~(size_t)15);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, tq = lane & 3;

  int off[NT];
  bool tapok[NT];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int o = tap_offset<KD, KHW>(nt * 8 + gq, XP);
    tapok[nt] = o >= 0;
    off[nt] = (o < 0 ? 0 : o) + 2 * tq;
  }
  float acc[MT][NT][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[mt][nt][k] = 0.f;

  auto load_dy = [&](int buf, int n, int d, int h0, int w0) {
    // one tile row per warp; 16-byte chunks straight into [vox][COUT] rows
    const bf16* src = dy + ((((long long)n * g.D + d) * g.H + h0 + warp) * g.W + w0) * bld;
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(dy0 + ((size_t)buf * dtile + (size_t)warp * g.TW * COUT) * 2);
    const int chunks = g.TW * CPV;
    for (int q = lane; q < chunks; q += 32) {
      const int vox = q / CPV, part = q - vox * CPV;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)(vox * COUT + part * 8) * 2),
                   "l"(src + (long long)vox * bld + part * 8)
                   : "memory");
    }
  };

  const int tpc = (g.tiles + gridDim.x - 1) / gridDim.x;
  const int first = blockIdx.x * tpc;
  const int last = min(g.tiles, first + tpc);
  XStage<TA, KD, PAD> st;
  int n = 0, d = 0, h0 = 0, w0 = 0;
  if (first < last) {
    stem_decode(g, first, n, d, h0, w0);
    st.load(x, g, n, d, h0, w0, warp, lane);
    load_dy(0, n, d, h0, w0);
    st.store(xs0, XP, g.TW, warp, lane);
    asm volatile("cp.async.wait_all;" ::: "memory");
  }
  __syncthreads();
  const int segs = g.TW / 16;
  for (int tile = first; tile < last; ++tile) {
    const int buf = (tile - first) & 1;
    const unsigned short* xs = xs0 + buf * xtile;
    const bool more = tile + 1 < last;
    if (more) {
      int nn, nd, nh0, nw0;
      stem_decode(g, tile + 1, nn, nd, nh0, nw0);
      st.load(x, g, nn, nd, nh0, nw0, warp, lane);
      load_dy(buf ^ 1, nn, nd, nh0, nw0);
    }
    const uint32_t dyb = (uint32_t)__cvta_generic_to_shared(dy0 + (size_t)buf * dtile * 2);
    for (int ks = warp; ks < SM_TH * segs; ks += 8) {
      const int row = ks / segs, seg = ks - row * segs;
      // A = dY^T: ldmatrix.trans of the [vox][co] rows; matrix m of the x4 = (vox half m>>1, co half m&1)
      uint32_t a[MT][4];
      const int vrow = row * g.TW + seg * 16 + (lane >> 4) * 8 + (lane & 7);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const uint32_t addr = dyb + (uint32_t)(vrow * COUT + mt * 16 + ((lane >> 3) & 1) * 8) * 2;
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                     : "=r"(a[mt][0]), "=r"(a[mt][1]), "=r"(a[mt][2]), "=r"(a[mt][3])
                     : "r"(addr));
      }
      const int p = row * XP + seg * 16;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        uint32_t b0 = 0u, b1 = 0u;
        if (tapok[nt]) {
          const unsigned short* q = xs + off[nt] + p;
          b0 = pack16(q[0], q[1]);
          b1 = pack16(q[8], q[9]);
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) mma_bf16_16816(acc[mt][nt], a[mt], b0, b1);
      }
    }
    if (more) {
      st.store(xs0 + (buf ^ 1) * xtile, XP, g.TW, warp, lane);
      asm volatile("cp.async.wait_all;" ::: "memory");
    }
    __syncthreads();
  }
  // fold the 8 warps: red[warp][co][32 taps] over the dY buffers, then one atomic per (tap, co) per CTA
  float* red = reinterpret_cast<float*>(dy0);
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      float* r0 = red + ((size_t)warp * COUT + mt * 16 + gq) * 32 + nt * 8 + 2 * tq;
      r0[0] = acc[mt][nt][0];
      r0[1] = acc[mt][nt][1];
      r0[8 * 32] = acc[mt][nt][2];
      r0[8 * 32 + 1] = acc[mt][nt][3];
    }
  __syncthreads();
  for (int i = threadIdx.x; i < COUT * 32; i += blockDim.x) {
    const int co = i >> 5, tap = i & 31;
    if (tap < TAPS) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += red[((size_t)k * COUT + co) * 32 + tap];
      atomicAdd(dwp + (long long)tap * COUT + co, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------

int stem_mma_conv_supported(int kind, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                            const b200seg_tensor* addend) {
  if (kind != B200SEG_K3 && kind != B200SEG_K1) return 0;
  if (addend != nullptr || w_dtype != B200SEG_BF16 || y->dtype != B200SEG_BF16) return 0;
  if (x->dtype != B200SEG_F32 && x->dtype != B200SEG_BF16) return 0;
  if ((y->ld % 8) || !al16m(y->ptr)) return 0;
  StemGeom g;
  return stem_mma_geom(x, y, &g) ? 1 : 0;
}


template <typename TA, int CO>
static int stem_mma_conv_co(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                            const b200seg_tensor* y, double* stats, const StemGeom& g, int device, cudaStream_t st) {
  const int grid = stem_grid(g, device);
#define SMC_LAUNCH(KD_, KHW_)                                                                                     \
  do {                                                                                                            \
    const size_t smem = stem_x_bytes<KD_, KHW_ / 2>(g.TW) + (size_t)8 * 2 * CO * sizeof(float);                   \
    launch_k(conv_stem_mma_kernel<TA, CO, KD_, KHW_>, grid, SM_THREADS, smem, st, \
        static_cast<const TA*>(x->ptr), static_cast<const bf16*>(w), bias, static_cast<bf16*>(y->ptr), y->ld,     \
        stats, g);                                                                                                \
  } while (0)
  if (kind == B200SEG_K1) SMC_LAUNCH(1, 1);
  else if (dims == 3) SMC_LAUNCH(3, 3);
  else SMC_LAUNCH(1, 3);
#undef SMC_LAUNCH
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int stem_mma_conv(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                  const b200seg_tensor* y, double* stats, int device, cudaStream_t st) {
  StemGeom g;
  B200_CHECK_ARG(stem_mma_geom(x, y, &g), "stem_mma_conv: unsupported geometry");
  if (x->dtype == B200SEG_F32) {
    if (y->c == 16) return stem_mma_conv_co<float, 16>(kind, dims, x, w, bias, y, stats, g, device, st);
    return stem_mma_conv_co<float, 32>(kind, dims, x, w, bias, y, stats, g, device, st);
  }
  if (y->c == 16) return stem_mma_conv_co<bf16, 16>(kind, dims, x, w, bias, y, stats, g, device, st);
  return stem_mma_conv_co<bf16, 32>(kind, dims, x, w, bias, y, stats, g, device, st);
}

int stem_mma_wgrad_supported(int kind, const b200seg_tensor* a, const b200seg_tensor* b) {
  if (kind != B200SEG_K3 && kind != B200SEG_K1) return 0;
  if (b->dtype != B200SEG_BF16) return 0;
  if (a->dtype != B200SEG_F32 && a->dtype != B200SEG_BF16) return 0;
  if ((b->ld % 8) || !al16m(b->ptr)) return 0;
  StemGeom g;
  return stem_mma_geom(a, b, &g) ? 1 : 0;
}

template <typename TA, int CO>
static int stem_mma_wgrad_co(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp,
                             const StemGeom& g, int device, cudaStream_t st) {
  const int grid = stem_grid(g, device);
#define SMW_LAUNCH(KD_, KHW_)                                                                                     \
  do {                                                                                                            \
    size_t dyb = (size_t)2 * SM_TH * g.TW * CO * 2;              /* two dY buffers ... */                         \
    const size_t redb = (size_t)8 * CO * 32 * sizeof(float);     /* ... reused for the cross-warp fold */         \
    if (dyb < redb) dyb = redb;                                                                                   \
    const size_t smem = stem_x_bytes<KD_, KHW_ / 2>(g.TW) + dyb;                                                  \
    static int attr_done[64] = {0};                                                                               \
    if (smem > 48 * 1024 && device >= 0 && device < 64 && !attr_done[device]) {                                   \
      B200_CUDA(cudaFuncSetAttribute(wgrad_stem_mma_kernel<TA, CO, KD_, KHW_>,                                    \
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));                   \
      attr_done[device] = 1;                                                                                      \
    }                                                                                                             \
    launch_k(wgrad_stem_mma_kernel<TA, CO, KD_, KHW_>, grid, SM_THREADS, smem, st, \
        static_cast<const TA*>(a->ptr), static_cast<const bf16*>(b->ptr), b->ld, dwp, g);                         \
  } while (0)
  if (kind == B200SEG_K1) SMW_LAUNCH(1, 1);
  else if (dims == 3) SMW_LAUNCH(3, 3);
  else SMW_LAUNCH(1, 3);
#undef SMW_LAUNCH
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int stem_mma_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st) {
  StemGeom g;
  B200_CHECK_ARG(stem_mma_geom(a, b, &g), "stem_mma_wgrad: unsupported geometry");
  if (a->dtype == B200SEG_F32) {
    if (b->c == 16) return stem_mma_wgrad_co<float, 16>(kind, dims, a, b, dwp, g, device, st);
    return stem_mma_wgrad_co<float, 32>(kind, dims, a, b, dwp, g, device, st);
  }
  if (b->c == 16) return stem_mma_wgrad_co<bf16, 16>(kind, dims, a, b, dwp, g, device, st);
  return stem_mma_wgrad_co<bf16, 32>(kind, dims, a, b, dwp, g, device, st);
}

}  // namespace b200seg
