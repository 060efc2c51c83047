// Shared pieces of the single-image-channel stem on mma.sync (stem_mma.cu) and of the fused input block
// (stem_gn.cu): tile geometry and walk, halo staging of the image, fragment helpers.  Every kernel that
// computes a stem output runs this code on the same operands, so recomputed outputs are bit-identical.
#pragma once

#include "common.cuh"

namespace b200seg {

constexpr int SM_TH = 8;               // tile rows (one per warp for the dY loader)
constexpr int SM_THREADS = 256;
constexpr int SM_XC = 5;               // column chunks of 32 covering TW + 2 <= 130

struct StemGeom {
  int N, D, H, W;
  int TW;                              // tile width: multiple of 16 that divides W, <= 128
  int tiles_w, tiles_h, tiles;         // tiles = N * D * tiles_h * tiles_w
};

__device__ __forceinline__ void stem_decode(const StemGeom& g, int tile, int& n, int& d, int& h0, int& w0) {
  int t = tile;
  const int wb = t % g.tiles_w;
  t /= g.tiles_w;
  const int hb = t % g.tiles_h;
  t /= g.tiles_h;
  d = t % g.D;
  n = t / g.D;
  h0 = hb * SM_TH;
  w0 = wb * g.TW;
}

__device__ __forceinline__ uint32_t pack16(unsigned short lo, unsigned short hi) {
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

__device__ __forceinline__ unsigned short bf16_bits(float v) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
__device__ __forceinline__ unsigned short bf16_bits(bf16 v) { return __bfloat16_as_ushort(v); }

__device__ __forceinline__ void mma_bf16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// image window of one tile -> registers (bf16 bits); rows r = warp + 8 i over KD*(TH+2P) rows, columns lane + 32 j
template <typename TA, int KD, int PAD>
struct XStage {
  static constexpr int ROWS = KD * (SM_TH + 2 * PAD);
  static constexpr int XR = (ROWS + 7) / 8;
  unsigned short v[XR][SM_XC];

  __device__ __forceinline__ void load(const TA* __restrict__ x, const StemGeom& g, int n, int d, int h0, int w0,
                                       int warp, int lane) {
    constexpr int PD = KD / 2;
    const int cols = g.TW + 2 * PAD;
#pragma unroll
    for (int i = 0; i < XR; ++i) {
      const int r = warp + 8 * i;
      const int plane = r / (SM_TH + 2 * PAD), rr = r - plane * (SM_TH + 2 * PAD);
      const int id = d + plane - PD, ih = h0 + rr - PAD;
      const bool rok = r < ROWS && (unsigned)id < (unsigned)g.D && (unsigned)ih < (unsigned)g.H;
      const TA* row = x + (((long long)n * g.D + (rok ? id : 0)) * g.H + (rok ? ih : 0)) * g.W;
#pragma unroll
      for (int j = 0; j < SM_XC; ++j) {
        const int c = lane + 32 * j;
        const int iw = w0 + c - PAD;
        const bool ok = rok && c < cols && (unsigned)iw < (unsigned)g.W;
        v[i][j] = ok ? bf16_bits(row[iw]) : (unsigned short)0;
      }
    }
  }
  __device__ __forceinline__ void store(unsigned short* xs, int XP, int TW, int warp, int lane) const {
    const int cols = TW + 2 * PAD;
#pragma unroll
    for (int i = 0; i < XR; ++i) {
      const int r = warp + 8 * i;
      if (r < ROWS) {
#pragma unroll
        for (int j = 0; j < SM_XC; ++j) {
          const int c = lane + 32 * j;
          if (c < cols) xs[r * XP + c] = v[i][j];
        }
      }
    }
  }
};

// smem offset of tap (kd, kh, kw) relative to the voxel position inside the halo tile; -1 for a padding tap
template <int KD, int KHW>
__device__ __forceinline__ int tap_offset(int tap, int XP) {
  constexpr int PAD = KHW / 2;
  if (tap >= KD * KHW * KHW) return -1;
  const int kw = tap % KHW, kh = (tap / KHW) % KHW, kd = tap / (KHW * KHW);
  return (kd * (SM_TH + 2 * PAD) + kh) * XP + kw;
}

// host side
inline bool al16m(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

inline int stem_tile_width(int W) {
  static const int cand[] = {128, 112, 96, 80, 64, 48, 32, 16};
  for (int c : cand)
    if (W % c == 0) return c;
  return 0;
}

inline bool stem_mma_geom(const b200seg_tensor* x, const b200seg_tensor* y, StemGeom* g) {
  if (x->c != 1 || x->ld != 1) return false;
  if (y->c != 16 && y->c != 32) return false;
  if (x->d != y->d || x->h != y->h || x->w != y->w || x->n != y->n) return false;
  if ((x->h % SM_TH) != 0) return false;
  const int tw = stem_tile_width(x->w);
  if (tw == 0) return false;
  if ((long long)x->n * x->d * x->h * x->w >= (1ll << 31)) return false;
  g->N = x->n; g->D = x->d; g->H = x->h; g->W = x->w;
  g->TW = tw;
  g->tiles_w = x->w / tw;
  g->tiles_h = x->h / SM_TH;
  g->tiles = x->n * x->d * g->tiles_h * g->tiles_w;
  return true;
}

template <int KD, int PAD>
inline size_t stem_x_bytes(int TW) {
  return (((size_t)2 * KD * (SM_TH + 2 * PAD) * (TW + 2 * PAD) * 2) + 15) & ~(size_t)15;
}

inline int stem_grid(const StemGeom& g, int device) {
  const int cap = num_sms(device) * 2;
  return g.tiles < cap ? g.tiles : cap;
}

}  // namespace b200seg
