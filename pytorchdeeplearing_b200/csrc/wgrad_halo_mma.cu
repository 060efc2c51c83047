// Weight gradient of the full-resolution 3x3x3 layers (16/32 channels) from halo slices, on mma.sync (sm_90a, bf16).
//
//   dW[tap][ci][co] += sum_v x[v + tap][ci] * dy[v][co]
//
// wgrad_tc.cu feeds the tensor core with one TMA box per tap: for 16/32-channel tensors those are 32/64-byte rows
// and the kernel runs at the TMA row rate.  Here every tap is a shifted ldmatrix view of halo slices in shared memory:
//   * the N * th * tw * D output slice tiles (8 x TW voxels of one d-slice) are split evenly over the grid, and a CTA
//     walks its range as column segments (n, h0, w0, d0 .. d0 + nd), as conv_halo3_kernel does.  A segment stages
//     input slices d0 - 1 .. d0 + nd ONCE, each (10 x (TW + 2) voxels, zero fill = conv padding) into a ring of
//     WH_RING slots, and dy[d] into a double buffer; output slice d reads input slices d - 1, d, d + 1 (kd = 0, 1, 2).
//     While slice d computes, the loads of the next step are in flight: one input slice and dy[d + 1], or at a
//     segment boundary the three first slices of the next segment (hence 6 slots);
//   * GEMM per tap: D[ci][co] += X^T[ci][16 vox] * dY[16 vox][co]  (m16n8k16, fp32 accumulators in registers);
//     both operands are stored [voxel][channel] and fetched with ldmatrix.trans (the K index -- voxels -- runs
//     across smem rows); rows are padded by 16 B so the 8 rows of an 8x8 block hit distinct banks;
//   * warp role = (kd, 16 input channels, 16 output channels) with all nine (kh, kw) taps: 72 accumulators; warp
//     strip = (16-voxel column segment, 8 / RS dy rows), as many strips as give 12 warps.  The x fragment of padded
//     row j at shift kw is the operand of taps (kd, kh, kw) for dy rows j - kh, so it is loaded ONCE and multiplied
//     into the three kh accumulators, against dy rows j, j - 1, j - 2 that stay in registers as a sliding window of B
//     fragments: per pair of m16n8k16 (16 x 16 x 16) 0.42 ldmatrix.x4 of x and 0.11 of dy at 8 rows per strip;
//   * a CTA folds its accumulators once at the end: strips through shared memory, then one fp32 atomic per weight.
#include "common.cuh"

namespace b200seg {

constexpr int WH_TH = 8;                 // tile rows
constexpr int WH_RING = 6;               // input slices in the shared-memory ring

struct WhGeom {
  int N, D, H, W;
  int tiles_w, tiles_h;
  long long units;                       // N * tiles_h * tiles_w * D output slice tiles
};

template <int CIN, int COUT, int TW>
struct WhCfg {
  static constexpr int MB = CIN / 16, NB = COUT / 16;
  static constexpr int R = 3 * MB * NB;                  // roles
  static constexpr int S = 4 / (MB * NB);                // strips
  static constexpr int SEGS = TW / 16;
  static constexpr int RS = S / SEGS;                    // dy row parts
  static constexpr int THREADS = 32 * R * S;
  static constexpr int XP = CIN * 2 + 16;                // bytes per voxel row of an x slice (16 B pad: bank spread)
  static constexpr int YP = COUT * 2 + 16;
  static constexpr int PW = TW + 2, PH = WH_TH + 2;
  static constexpr int XSLICE = PH * PW * XP, YSLICE = WH_TH * TW * YP;
  static constexpr int PIPE = WH_RING * XSLICE + 2 * YSLICE;
  static constexpr int RED = 27 * CIN * COUT * 4;
  static constexpr int SMEM = PIPE > RED ? PIPE : RED;
};

__device__ __forceinline__ void wh_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void wh_ldsm4t(uint32_t* r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// one column segment of a CTA's range: nd output slices from (n, d0) of the (h0, w0) column
struct WhSeg {
  int n, h0, w0, d0, nd;
};
// the segment starting at output slice tile t of a range that ends at `end` (tiles ordered (n, h tile, w tile, d))
template <int TW>
__device__ __forceinline__ WhSeg wh_segment(const WhGeom& g, long long t, long long end) {
  WhSeg s;
  s.d0 = (int)(t % g.D);
  long long c = t / g.D;
  s.w0 = (int)(c % g.tiles_w) * TW;
  c /= g.tiles_w;
  s.h0 = (int)(c % g.tiles_h) * WH_TH;
  s.n = (int)(c / g.tiles_h);
  s.nd = (int)min((long long)(g.D - s.d0), end - t);
  return s;
}

template <int CIN, int COUT, int TW>
__global__ void __launch_bounds__(WhCfg<CIN, COUT, TW>::THREADS, 1)
    wgrad_halo_mma_kernel(const bf16* __restrict__ x, long long xld, const bf16* __restrict__ dy, long long bld,
                          float* __restrict__ dwp, const WhGeom g) {
  PDL_ENTER();
  using C = WhCfg<CIN, COUT, TW>;
  constexpr int XP = C::XP, YP = C::YP, PW = C::PW, PH = C::PH;
  constexpr int RPS = WH_TH / C::RS;                // dy rows per strip
  static_assert(C::S * C::MB * C::NB == 4 && C::S % C::SEGS == 0 && WH_TH % C::RS == 0, "12 warps");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(smem_raw);
  const uint32_t ybase = ring + WH_RING * C::XSLICE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = warp % C::R, strip = warp / C::R;
  const int kd = role % 3, mb = (role / 3) % C::MB, nb = role / (3 * C::MB);
  const int seg = strip % C::SEGS, rp = strip / C::SEGS;
  const int gq = lane >> 2, tq = lane & 3;

  float acc[3][3][2][4];                             // [kw][kh][8 output channels][m16n8 fragment]
#pragma unroll
  for (int kw = 0; kw < 3; ++kw)
#pragma unroll
    for (int kh = 0; kh < 3; ++kh)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[kw][kh][nt][k] = 0.f;

  // the loaders' loops stay rolled: unrolled, their addresses take registers the accumulators need (and spill)
  // input slice id (zero outside the volume) of column (n, h0, w0) -> ring slot
  auto load_x = [&](int slot, int n, int id, int h0, int w0) {
    constexpr int XCH = CIN / 8;
    const uint32_t xs = ring + (uint32_t)(slot * C::XSLICE);
    const bool dok = (unsigned)id < (unsigned)g.D;
#pragma unroll 1
    for (int q = threadIdx.x; q < PH * PW * XCH; q += C::THREADS) {
      const int v = q / XCH, part = q - v * XCH;
      const int c = v % PW, rr = v / PW;
      const int ih = h0 + rr - 1, iw = w0 + c - 1;
      const bool ok = dok && (unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W;
      const bf16* src = ok ? x + ((((long long)n * g.D + id) * g.H + ih) * g.W + iw) * xld + part * 8 : x;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(xs + (uint32_t)(v * XP + part * 16)), "l"(src),
                   "r"(ok ? 16 : 0)
                   : "memory");
    }
  };
  auto load_dy = [&](int buf, int n, int d, int h0, int w0) {
    constexpr int YCH = COUT / 8;
    const uint32_t ys = ybase + (uint32_t)(buf * C::YSLICE);
#pragma unroll 1
    for (int q = threadIdx.x; q < WH_TH * TW * YCH; q += C::THREADS) {
      const int v = q / YCH, part = q - v * YCH;
      const int c = v % TW, rr = v / TW;
      const bf16* src = dy + ((((long long)n * g.D + d) * g.H + h0 + rr) * g.W + w0 + c) * bld + part * 8;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ys + (uint32_t)(v * YP + part * 16)), "l"(src)
                   : "memory");
    }
  };

  // this CTA's share [t, end) of the output slice tiles
  long long t = g.units * blockIdx.x / gridDim.x;
  const long long end = g.units * (blockIdx.x + 1) / gridDim.x;
  // input slices are numbered along the walk: a segment stages nd + 2 of them from number gs on, number q sits in
  // ring slot q % WH_RING, and output i of the segment reads numbers gs + i + kd
  WhSeg s{};
  int gs = 0, i = 0;
  if (t < end) {
    s = wh_segment<TW>(g, t, end);
    for (int k = 0; k < 3; ++k) load_x(k, s.n, s.d0 - 1 + k, s.h0, s.w0);
    load_dy(0, s.n, s.d0, s.h0, s.w0);
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  // lane constants of the ldmatrix addresses: matrix m = lane >> 3, row = lane & 7
  const int lm = lane >> 3, lr = lane & 7;
  // A (x^T): m -> (voxel half m >> 1, channel half m & 1);  B (dy): m -> (voxel half m & 1, channel half m >> 1)
  const int a_lane = ((lm >> 1) * 8 + lr) * XP + (lm & 1) * 16;
  const int b_lane = ((lm & 1) * 8 + lr) * YP + (lm >> 1) * 16;
  const int r0 = rp * RPS;
  // x padded row r0 at column seg * 16, channels mb * 16; dy row r0 at column seg * 16, channels nb * 16
  const int a_off = (r0 * PW + seg * 16) * XP + a_lane + mb * 32;
  const int b_off = (r0 * TW + seg * 16) * YP + b_lane + nb * 32;

  for (int step = 0; t < end; ++step) {
    // the next step's input slices beyond this step's three, and its dy
    WhSeg ns = s;
    int ngs = gs, ni = i + 1;
    if (t + 1 < end) {
      if (ni < s.nd) {
        load_x((gs + ni + 2) % WH_RING, s.n, s.d0 + ni + 1, s.h0, s.w0);
      } else {
        ns = wh_segment<TW>(g, t + 1, end);
        ngs = gs + s.nd + 2;
        ni = 0;
        for (int k = 0; k < 3; ++k) load_x((ngs + k) % WH_RING, ns.n, ns.d0 - 1 + k, ns.h0, ns.w0);
      }
      load_dy((step + 1) & 1, ns.n, ns.d0 + ni, ns.h0, ns.w0);
    }
    const uint32_t xa = ring + (uint32_t)(((gs + i + kd) % WH_RING) * C::XSLICE + a_off);
    const uint32_t yb = ybase + (uint32_t)((step & 1) * C::YSLICE + b_off);
    uint32_t bfr[3][4];                             // dy rows jj, jj - 1, jj - 2 in slots jj % 3
#pragma unroll
    for (int jj = 0; jj < RPS + 2; ++jj) {
      if (jj < RPS) wh_ldsm4t(bfr[jj % 3], yb + (uint32_t)(jj * TW * YP));
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        uint32_t afr[4];
        wh_ldsm4t(afr, xa + (uint32_t)((jj * PW + kw) * XP));
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          const int r = jj - kh;
          if (r < 0 || r >= RPS) continue;
          wh_mma(acc[kw][kh][0], afr, bfr[r % 3][0], bfr[r % 3][1]);
          wh_mma(acc[kw][kh][1], afr, bfr[r % 3][2], bfr[r % 3][3]);
        }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    s = ns;
    gs = ngs;
    i = ni;
    ++t;
  }

  // fold the strips through shared memory (red[tap][ci][co]), then one atomic per weight and CTA
  float* red = reinterpret_cast<float*>(smem_raw);
  for (int st = 0; st < C::S; ++st) {
    if (strip == st) {
#pragma unroll
      for (int kw = 0; kw < 3; ++kw)
#pragma unroll
        for (int kh = 0; kh < 3; ++kh)
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) {
            const int tap = (kd * 3 + kh) * 3 + kw;
            float* r0p = red + ((size_t)tap * CIN + mb * 16 + gq) * COUT + (nb * 2 + nt) * 8 + 2 * tq;
            const float* a4 = acc[kw][kh][nt];
            if (st == 0) {
              r0p[0] = a4[0];
              r0p[1] = a4[1];
              r0p[8 * COUT] = a4[2];
              r0p[8 * COUT + 1] = a4[3];
            } else {
              r0p[0] += a4[0];
              r0p[1] += a4[1];
              r0p[8 * COUT] += a4[2];
              r0p[8 * COUT + 1] += a4[3];
            }
          }
    }
    __syncthreads();
  }
  for (int q = threadIdx.x; q < 27 * CIN * COUT; q += C::THREADS) atomicAdd(dwp + q, red[q]);
}

// ------------------------------------------------------------------------------------------------
static bool al16h2(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

static int wh_tile_w(int cin, int W) {
  const int want = cin == 16 ? 32 : 16;
  if (W % want == 0) return want;
  if (W % 16 == 0) return 16;
  return 0;
}

int wgrad_halo_mma_supported(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b) {
  if (kind != B200SEG_K3 || dims != 3) return 0;
  if (a->dtype != B200SEG_BF16 || b->dtype != B200SEG_BF16) return 0;
  if ((a->c != 16 && a->c != 32) || (b->c != 16 && b->c != 32)) return 0;
  if ((a->ld % 8) || (b->ld % 8) || !al16h2(a->ptr) || !al16h2(b->ptr)) return 0;
  if (a->n != b->n || a->d != b->d || a->h != b->h || a->w != b->w) return 0;
  if ((a->h % WH_TH) != 0 || wh_tile_w(a->c, a->w) == 0) return 0;
  // only where the TMA kernel is row-rate bound: large volumes
  if ((long long)a->d * a->h * a->w < 32768) return 0;
  return 1;
}

template <int CIN, int COUT, int TW>
static int wh_launch(const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device, cudaStream_t st) {
  using C = WhCfg<CIN, COUT, TW>;
  WhGeom g;
  g.N = a->n; g.D = a->d; g.H = a->h; g.W = a->w;
  g.tiles_w = a->w / TW;
  g.tiles_h = a->h / WH_TH;
  g.units = (long long)a->n * g.tiles_h * g.tiles_w * a->d;
  static int attr_done[64] = {0};
  if (device >= 0 && device < 64 && !attr_done[device]) {
    B200_CUDA(cudaFuncSetAttribute(wgrad_halo_mma_kernel<CIN, COUT, TW>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    attr_done[device] = 1;
  }
  const int sms = num_sms(device);
  const int grid = g.units < sms ? (int)g.units : sms;
  launch_k(wgrad_halo_mma_kernel<CIN, COUT, TW>, grid, C::THREADS, C::SMEM, st,
           static_cast<const bf16*>(a->ptr), a->ld, static_cast<const bf16*>(b->ptr), b->ld, dwp, g);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int wgrad_halo_mma(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st) {
  (void)kind; (void)dims;
  const int tw = wh_tile_w(a->c, a->w);
  if (a->c == 16 && b->c == 16) {
    if (tw == 32) return wh_launch<16, 16, 32>(a, b, dwp, device, st);
    return wh_launch<16, 16, 16>(a, b, dwp, device, st);
  }
  if (a->c == 16 && b->c == 32) {
    if (tw == 32) return wh_launch<16, 32, 32>(a, b, dwp, device, st);
    return wh_launch<16, 32, 16>(a, b, dwp, device, st);
  }
  if (a->c == 32 && b->c == 16) return wh_launch<32, 16, 16>(a, b, dwp, device, st);
  return wh_launch<32, 32, 16>(a, b, dwp, device, st);
}

}  // namespace b200seg
