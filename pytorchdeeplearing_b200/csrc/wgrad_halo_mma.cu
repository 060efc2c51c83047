// Weight gradient of the full-resolution 3x3x3 layers (16/32 channels) from halo tiles, on mma.sync (sm_90a, bf16).
//
//   dW[tap][ci][co] += sum_v x[v + tap][ci] * dy[v][co]
//
// wgrad_tc.cu feeds the tensor core with one TMA box per tap: for 16/32-channel tensors those are 32/64-byte rows
// and the kernel runs at the TMA row rate (0.28 ms for the 16-channel 96^3 layer).  Here a CTA stages ONE halo tile
// of x (3 x 10 x (TW+2) voxels) and the matching dy tile (8 x TW voxels) in shared memory per step and every tap is a
// shifted ldmatrix view of it:
//   * GEMM per tap: D[ci][co] += X^T[ci][16 vox] * dY[16 vox][co]  (m16n8k16, fp32 accumulators in registers);
//     both operands are stored [voxel][channel] and fetched with ldmatrix.trans (the K index -- voxels -- runs
//     across smem rows); rows are padded by 16 B so the 8 rows of an 8x8 block hit distinct banks;
//   * warp roles: role r owns TPW taps (9 = one kd plane, or 3 = one (kd, kh) row when the accumulators would not
//     fit), stream s owns every S-th 16-voxel group of the tile: warps = (27 / TPW) x S, all reading the same tile;
//   * tiles are double buffered with cp.async (zero fill = conv padding); a CTA walks a contiguous tile range and
//     folds its accumulators once at the end: streams through shared memory, then one fp32 atomic per weight.
#include "common.cuh"

namespace b200seg {

constexpr int WH_TH = 8;                 // tile rows

struct WhGeom {
  int N, D, H, W;
  int tiles_w, tiles_h, tiles;           // tiles = N * D * tiles_h * tiles_w
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

template <int CIN, int COUT, int TW, int TPW, int S>
__global__ void __launch_bounds__(32 * (27 / TPW) * S, 1)
    wgrad_halo_mma_kernel(const bf16* __restrict__ x, long long xld, const bf16* __restrict__ dy, long long bld,
                          float* __restrict__ dwp, const WhGeom g) {
  PDL_ENTER();
  constexpr int R = 27 / TPW;                       // tap groups (warp roles)
  constexpr int NTHREADS = 32 * R * S;
  constexpr int XP = CIN * 2 + 16;                  // bytes per voxel row of the x tile (16 B pad: bank spread)
  constexpr int YP = COUT * 2 + 16;
  constexpr int PW = TW + 2, PH = WH_TH + 2;
  constexpr int XVOX = 3 * PH * PW;
  constexpr int YVOX = WH_TH * TW;
  constexpr int XBYTES = XVOX * XP, YBYTES = YVOX * YP;
  constexpr int MT = CIN / 16, NT = COUT / 8, NB = COUT / 16;
  constexpr int SEGS = TW / 16;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = warp % R, stream = warp / R;
  const int gq = lane >> 2, tq = lane & 3;

  float acc[TPW][MT][NT][4];
#pragma unroll
  for (int t = 0; t < TPW; ++t)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[t][mt][nt][k] = 0.f;

  auto decode = [&](int tile, int& n, int& d, int& h0, int& w0) {
    int t = tile;
    const int wb = t % g.tiles_w; t /= g.tiles_w;
    const int hb = t % g.tiles_h; t /= g.tiles_h;
    d = t % g.D;
    n = t / g.D;
    h0 = hb * WH_TH;
    w0 = wb * TW;
  };
  auto load_tile = [&](int buf, int tile) {
    int n, d, h0, w0;
    decode(tile, n, d, h0, w0);
    unsigned char* xb = smem_raw + (size_t)buf * (XBYTES + YBYTES);
    const uint32_t xs = (uint32_t)__cvta_generic_to_shared(xb);
    const uint32_t ys = xs + XBYTES;
    constexpr int XCH = CIN / 8, YCH = COUT / 8;
    for (int q = threadIdx.x; q < XVOX * XCH; q += NTHREADS) {
      const int v = q / XCH, part = q - v * XCH;
      const int c = v % PW, rr = (v / PW) % PH, pl = v / (PW * PH);
      const int id = d + pl - 1, ih = h0 + rr - 1, iw = w0 + c - 1;
      const bool ok = (unsigned)id < (unsigned)g.D && (unsigned)ih < (unsigned)g.H && (unsigned)iw < (unsigned)g.W;
      const bf16* src = ok ? x + ((((long long)n * g.D + id) * g.H + ih) * g.W + iw) * xld + part * 8 : x;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(xs + (uint32_t)(v * XP + part * 16)), "l"(src),
                   "r"(ok ? 16 : 0)
                   : "memory");
    }
    for (int q = threadIdx.x; q < YVOX * YCH; q += NTHREADS) {
      const int v = q / YCH, part = q - v * YCH;
      const int c = v % TW, rr = v / TW;
      const bf16* src = dy + ((((long long)n * g.D + d) * g.H + h0 + rr) * g.W + w0 + c) * bld + part * 8;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ys + (uint32_t)(v * YP + part * 16)), "l"(src)
                   : "memory");
    }
  };

  const int tpc = (g.tiles + gridDim.x - 1) / gridDim.x;
  const int first = blockIdx.x * tpc;
  const int last = min(g.tiles, first + tpc);
  if (first < last) {
    load_tile(0, first);
    asm volatile("cp.async.wait_all;" ::: "memory");
  }
  __syncthreads();

  // lane constants of the ldmatrix addresses: matrix m = lane >> 3, row = lane & 7
  const int lm = lane >> 3, lr = lane & 7;
  // A (x^T): m -> (voxel half m >> 1, channel half m & 1);  B (dy): m -> (voxel half m & 1, channel half m >> 1)
  const int a_lane = ((lm >> 1) * 8 + lr) * XP + (lm & 1) * 16;
  const int b_lane = ((lm & 1) * 8 + lr) * YP + (lm >> 1) * 16;
  // taps of this role
  int tap_off[TPW];
#pragma unroll
  for (int t = 0; t < TPW; ++t) {
    const int tap = role * TPW + t;
    const int kw = tap % 3, kh = (tap / 3) % 3, kd = tap / 9;
    tap_off[t] = ((kd * PH + kh) * PW + kw) * XP;
  }

  for (int tile = first; tile < last; ++tile) {
    const int buf = (tile - first) & 1;
    if (tile + 1 < last) load_tile(buf ^ 1, tile + 1);
    const uint32_t xs = (uint32_t)__cvta_generic_to_shared(smem_raw + (size_t)buf * (XBYTES + YBYTES));
    const uint32_t ys = xs + XBYTES;
    for (int ks = stream; ks < WH_TH * SEGS; ks += S) {
      const int row = ks / SEGS, seg = ks - row * SEGS;
      uint32_t bfr[NB][4];
#pragma unroll
      for (int nb = 0; nb < NB; ++nb)
        wh_ldsm4t(bfr[nb], ys + (uint32_t)((row * TW + seg * 16) * YP + b_lane + nb * 32));
      const uint32_t xrow = xs + (uint32_t)((row * PW + seg * 16) * XP + a_lane);
#pragma unroll
      for (int t = 0; t < TPW; ++t) {
        uint32_t afr[MT][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) wh_ldsm4t(afr[mt], xrow + (uint32_t)(tap_off[t] + mt * 32));
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int nb = 0; nb < NB; ++nb) {
            wh_mma(acc[t][mt][2 * nb], afr[mt], bfr[nb][0], bfr[nb][1]);
            wh_mma(acc[t][mt][2 * nb + 1], afr[mt], bfr[nb][2], bfr[nb][3]);
          }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
  }

  // fold the streams through shared memory (red[tap][ci][co]), then one atomic per weight and CTA
  float* red = reinterpret_cast<float*>(smem_raw);
  for (int s = 0; s < S; ++s) {
    if (stream == s) {
#pragma unroll
      for (int t = 0; t < TPW; ++t)
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            float* r0 = red + ((size_t)(role * TPW + t) * CIN + mt * 16 + gq) * COUT + nt * 8 + 2 * tq;
            if (s == 0) {
              r0[0] = acc[t][mt][nt][0];
              r0[1] = acc[t][mt][nt][1];
              r0[8 * COUT] = acc[t][mt][nt][2];
              r0[8 * COUT + 1] = acc[t][mt][nt][3];
            } else {
              r0[0] += acc[t][mt][nt][0];
              r0[1] += acc[t][mt][nt][1];
              r0[8 * COUT] += acc[t][mt][nt][2];
              r0[8 * COUT + 1] += acc[t][mt][nt][3];
            }
          }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 27 * CIN * COUT; i += NTHREADS) atomicAdd(dwp + i, red[i]);
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

template <int CIN, int COUT, int TW, int TPW, int S>
static int wh_launch(const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device, cudaStream_t st) {
  WhGeom g;
  g.N = a->n; g.D = a->d; g.H = a->h; g.W = a->w;
  g.tiles_w = a->w / TW;
  g.tiles_h = a->h / WH_TH;
  g.tiles = a->n * a->d * g.tiles_h * g.tiles_w;
  constexpr int XBYTES = 3 * (WH_TH + 2) * (TW + 2) * (CIN * 2 + 16);
  constexpr int YBYTES = WH_TH * TW * (COUT * 2 + 16);
  size_t smem = (size_t)2 * (XBYTES + YBYTES);
  const size_t redb = (size_t)27 * CIN * COUT * sizeof(float);
  if (smem < redb) smem = redb;
  static int attr_done[64] = {0};
  if (device >= 0 && device < 64 && !attr_done[device]) {
    B200_CUDA(cudaFuncSetAttribute(wgrad_halo_mma_kernel<CIN, COUT, TW, TPW, S>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_done[device] = 1;
  }
  const int sms = num_sms(device);
  const int grid = g.tiles < sms ? g.tiles : sms;
  launch_k(wgrad_halo_mma_kernel<CIN, COUT, TW, TPW, S>, grid, 32 * (27 / TPW) * S, smem, st, static_cast<const bf16*>(a->ptr), a->ld, static_cast<const bf16*>(b->ptr), b->ld, dwp, g);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int wgrad_halo_mma(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st) {
  (void)kind; (void)dims;
  const int tw = wh_tile_w(a->c, a->w);
  if (a->c == 16 && b->c == 16) {
    if (tw == 32) return wh_launch<16, 16, 32, 9, 4>(a, b, dwp, device, st);
    return wh_launch<16, 16, 16, 9, 4>(a, b, dwp, device, st);
  }
  if (a->c == 16 && b->c == 32) {
    if (tw == 32) return wh_launch<16, 32, 32, 9, 3>(a, b, dwp, device, st);
    return wh_launch<16, 32, 16, 9, 3>(a, b, dwp, device, st);
  }
  if (a->c == 32 && b->c == 16) return wh_launch<32, 16, 16, 9, 3>(a, b, dwp, device, st);
  return wh_launch<32, 32, 16, 3, 1>(a, b, dwp, device, st);
}

}  // namespace b200seg
