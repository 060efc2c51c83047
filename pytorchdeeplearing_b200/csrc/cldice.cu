// Soft-clDice of model/lossescldice.py (soft skeletonisation by 3x3(x3) min / max pooling), forward and backward
// (sm_90a).
//
// One round of the repaired soft_skeletonize is, in fp32:  m = minpool(x), M = maxpool(m), c = relu(M - m),
// x' = relu(x - c), every pool 3x3x3 (3x3 for 2-D, run as D = 1), stride 1, padding 1, padded positions never taken.
// torch runs it as five full-tensor operators; here one launch per round does all of it over a shared-memory tile.
//
//   cldice_round_kernel<SUMS>  forward round.  One CTA per (n*c, tile of TD x TH x TW voxels) stages x with a 2-voxel
//                              halo, forms m over the tile plus 1, then M, c and x' over the tile.  Only max, min,
//                              subtraction and comparisons: nothing contracts into an FMA, so x' is bit-identical to
//                              torch's fp32 sequence (the min / max pick the FIRST extremum in (kd, kh, kw) order, as
//                              torch's pooling does, so even the sign of a zero agrees).  With SUMS (the last round of
//                              a loss pass) the epilogue writes the CTA's fp64 sums {sum x' * other, sum x'}; the first
//                              round of a one-hot pass also counts labels outside [0, C).
//   cldice_finalize_kernel     one CTA: fixed-order sums of the partials per (n, c), iflat / tflat, the per-group sums
//                              {sum iflat*tflat, sum iflat, sum tflat} (one group, or one per class), the loss and the
//                              derivatives d loss / d iflat, d loss / d tflat per (n, c).  reduce = 0 starts from the
//                              group sums (after a data-parallel all-reduce of them).
//   cldice_round_bwd_kernel    adjoint of one round, as a gather: with a = [x - c > 0], b = [M - m > 0],
//                                g_m(u) = (a b g')(u) - sum_{w: argmax(w) = u} (a b g')(w)
//                                g_x(v) = (a g')(v)   + sum_{u: argmin(u) = v} g_m(u)
//                              over each voxel's <= 27 neighbours in a fixed order (no atomics: reruns are
//                              bit-identical).  The CTA recomputes m, M and both routings from x_r with a 4-voxel
//                              halo; the forward stored x_1 .. x_T.  The last adjoint round (r = T-1) seeds g' from
//                              the loss, the first one (r = 0) adds the tflat term directly.
//   cldice_norm_kernel /       norm_intersection on its own: per-(n, c) fp64 sums, one CTA each, and its elementwise
//   cldice_norm_bwd_kernel     gradient.
// Sums run in fp64 with fixed orders; nothing is allocated or synchronised.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxRounds = 64;
constexpr int kPart = 3;                    // per CTA: {sum x' * other, sum x', labels outside [0, C)}
constexpr int kStats = 8;                   // per (n, c): {A_p, S_p, A_t, S_t, iflat, tflat, dL/diflat, dL/dtflat}

struct ClGeom {
  int N, C, D, H, W;
  int TD, TH, TW;                           // tile
  int hd;                                   // 1 when the window reaches along D (D > 1)
  int nDT, nHT, nWT;
};

struct Field {                              // a (N, C, D, H, W) fp32 field, or the one-hot of int64 labels
  const float* p;
  const long long* lab;                     // [N][D][H][W]; value (lab == c)
  long long sn, sc, sd, sh, sw;
};

ClGeom make_geom(int N, int C, int D, int H, int W) {
  ClGeom G;
  G.N = N; G.C = C; G.D = D; G.H = H; G.W = W;
  G.hd = D > 1 ? 1 : 0;
  G.TW = 32;
  G.TH = G.hd ? 8 : 32;
  G.TD = G.hd ? 4 : 1;
  G.nDT = (D + G.TD - 1) / G.TD;
  G.nHT = (H + G.TH - 1) / G.TH;
  G.nWT = (W + G.TW - 1) / G.TW;
  return G;
}

__host__ __device__ inline long long ntiles(const ClGeom& G) { return (long long)G.nDT * G.nHT * G.nWT; }

__host__ __device__ inline int reg_size(const ClGeom& G, int k) {
  return (G.TD + 2 * k * G.hd) * (G.TH + 2 * k) * (G.TW + 2 * k);
}

Field dense_field(const float* p, const ClGeom& G) {
  const long long hw = (long long)G.H * G.W, dhw = hw * G.D;
  return Field{p, nullptr, G.C * dhw, dhw, hw, (long long)G.W, 1};
}

struct Tile {
  int n, c, nc, z0, y0, x0;
  long long t;
};

__device__ __forceinline__ Tile tile_of(const ClGeom& G) {
  Tile T;
  long long t = blockIdx.x;
  T.t = t;
  const int wt = (int)(t % G.nWT);
  t /= G.nWT;
  const int ht = (int)(t % G.nHT);
  const int dt = (int)(t / G.nHT);
  T.nc = blockIdx.y;
  T.n = T.nc / G.C;
  T.c = T.nc % G.C;
  T.z0 = dt * G.TD;
  T.y0 = ht * G.TH;
  T.x0 = wt * G.TW;
  return T;
}

// local index i of the region with halo k -> global coordinates
__device__ __forceinline__ void coords(const ClGeom& G, const Tile& T, int k, int i, int& z, int& y, int& x) {
  const int ew = G.TW + 2 * k, eh = G.TH + 2 * k;
  x = i % ew;
  i /= ew;
  y = i % eh;
  z = i / eh;
  z += T.z0 - k * G.hd;
  y += T.y0 - k;
  x += T.x0 - k;
}

// global coordinates -> local index in the region with halo k
__device__ __forceinline__ int lidx(const ClGeom& G, const Tile& T, int k, int z, int y, int x) {
  const int ew = G.TW + 2 * k, eh = G.TH + 2 * k;
  return ((z - T.z0 + k * G.hd) * eh + (y - T.y0 + k)) * ew + (x - T.x0 + k);
}

__device__ __forceinline__ bool inb(const ClGeom& G, int z, int y, int x) {
  return z >= 0 && z < G.D && y >= 0 && y < G.H && x >= 0 && x < G.W;
}

__device__ __forceinline__ float fetch(const Field& f, const ClGeom& G, int n, int c, int z, int y, int x) {
  if (f.lab) return f.lab[(((long long)n * G.D + z) * G.H + y) * G.W + x] == c ? 1.f : 0.f;
  return f.p[n * f.sn + c * f.sc + z * f.sd + y * f.sh + x * f.sw];
}

// torch.relu keeps -0.0 and maps negatives to +0.0
__device__ __forceinline__ float relu(float v) { return v < 0.f ? 0.f : v; }

// window offsets in (kd, kh, kw) scan order; code (dz+1)*9 + (dy+1)*3 + (dx+1); the reverse offset has code 26 - code
#define CL_FOR_WINDOW(z, y, x)                                       \
  for (int dz = -1; dz <= 1; ++dz)                                   \
    for (int dy = -1; dy <= 1; ++dy)                                 \
      for (int dx = -1; dx <= 1; ++dx)                               \
        if (inb(G, (z) + dz, (y) + dy, (x) + dx))

// first minimum (MIN) or maximum of the region-k array s over the in-bounds window of (z, y, x)
template <bool MIN>
__device__ __forceinline__ float window_pick(const float* s, const ClGeom& G, const Tile& T, int k, int z, int y, int x,
                                             int& code) {
  float best = 0.f;
  code = -1;
  CL_FOR_WINDOW(z, y, x) {
    const float v = s[lidx(G, T, k, z + dz, y + dy, x + dx)];
    if (code < 0 || (MIN ? v < best : v > best)) {
      best = v;
      code = (dz + 1) * 9 + (dy + 1) * 3 + (dx + 1);
    }
  }
  return best;
}

// fixed-order CTA sum of kPart doubles; thread 0 gets the result
__device__ void block_sum3(double* red, double v[kPart]) {
  __syncthreads();
  for (int j = 0; j < kPart; ++j) red[j * kThreads + threadIdx.x] = v[j];
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o)
      for (int j = 0; j < kPart; ++j) red[j * kThreads + threadIdx.x] += red[j * kThreads + threadIdx.x + o];
    __syncthreads();
  }
  for (int j = 0; j < kPart; ++j) v[j] = red[j * kThreads];
}

template <bool SUMS>
__global__ void __launch_bounds__(kThreads) cldice_round_kernel(const ClGeom G, const Field in, float* __restrict__ out,
                                                                const Field other, double* __restrict__ part,
                                                                int count_bad) {
  PDL_ENTER();
  extern __shared__ __align__(16) unsigned char smem[];
  const Tile T = tile_of(G);
  float* xs = reinterpret_cast<float*>(smem);             // x, halo 2
  float* ms = xs + reg_size(G, 2);                         // m, halo 1
  for (int i = threadIdx.x; i < reg_size(G, 2); i += kThreads) {
    int z, y, x;
    coords(G, T, 2, i, z, y, x);
    xs[i] = inb(G, z, y, x) ? fetch(in, G, T.n, T.c, z, y, x) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < reg_size(G, 1); i += kThreads) {
    int z, y, x, code;
    coords(G, T, 1, i, z, y, x);
    ms[i] = inb(G, z, y, x) ? window_pick<true>(xs, G, T, 2, z, y, x, code) : 0.f;
  }
  __syncthreads();
  double acc[kPart] = {0.0, 0.0, 0.0};
  const long long vox = (long long)G.D * G.H * G.W;
  for (int i = threadIdx.x; i < reg_size(G, 0); i += kThreads) {
    int z, y, x, code;
    coords(G, T, 0, i, z, y, x);
    if (!inb(G, z, y, x)) continue;
    const float m = ms[lidx(G, T, 1, z, y, x)];
    const float M = window_pick<false>(ms, G, T, 1, z, y, x, code);
    const float c = relu(__fsub_rn(M, m));
    const float xo = relu(__fsub_rn(xs[lidx(G, T, 2, z, y, x)], c));
    const long long e = (long long)T.nc * vox + ((long long)z * G.H + y) * G.W + x;
    out[e] = xo;
    if (SUMS) {
      acc[0] += (double)xo * (double)fetch(other, G, T.n, T.c, z, y, x);
      acc[1] += (double)xo;
    }
    if (count_bad && T.c == 0) {
      const long long l = in.lab[(((long long)T.n * G.D + z) * G.H + y) * G.W + x];
      acc[2] += (l < 0 || l >= G.C) ? 1.0 : 0.0;
    }
  }
  if (SUMS || count_bad) {
    double* red = reinterpret_cast<double*>(smem);
    block_sum3(red, acc);
    if (threadIdx.x == 0) {
      double* p = part + ((long long)T.nc * ntiles(G) + T.t) * kPart;
      if (SUMS) { p[0] = acc[0]; p[1] = acc[1]; }
      if (count_bad) p[2] = acc[2];
    }
  }
}


// shared-memory bytes of the backward round: g_m (fp64, halo 1) | x (halo 4) | m (halo 3) | a b g', a g' (halo 2) |
// argmin codes (halo 3) | argmax codes (halo 2)
size_t bwd_smem(const ClGeom& G) {
  return (size_t)reg_size(G, 1) * 8 + ((size_t)reg_size(G, 4) + reg_size(G, 3) + 2 * (size_t)reg_size(G, 2)) * 4 +
         reg_size(G, 3) + reg_size(G, 2);
}

size_t fwd_smem(const ClGeom& G) {
  const size_t s = ((size_t)reg_size(G, 2) + reg_size(G, 1)) * 4;
  return s > (size_t)kPart * kThreads * 8 ? s : (size_t)kPart * kThreads * 8;
}

// gin: d loss / d x_{r+1} (dense), or NULL for the loss seed (t - iflat) dL/diflat / (S_p + 1) of the last round;
// skt: the target's skeleton for the direct tflat term of round 0, or NULL
__global__ void __launch_bounds__(kThreads) cldice_round_bwd_kernel(const ClGeom G, const Field in,
                                                                    const float* __restrict__ gin, const Field tgt,
                                                                    const double* __restrict__ stats,
                                                                    const float* __restrict__ gout,
                                                                    const float* __restrict__ skt,
                                                                    float* __restrict__ gx) {
  PDL_ENTER();
  extern __shared__ __align__(16) unsigned char smem[];
  const Tile T = tile_of(G);
  double* gms = reinterpret_cast<double*>(smem);
  float* xs = reinterpret_cast<float*>(gms + reg_size(G, 1));
  float* ms = xs + reg_size(G, 4);
  float* hs = ms + reg_size(G, 3);
  float* ags = hs + reg_size(G, 2);
  unsigned char* amin = reinterpret_cast<unsigned char*>(ags + reg_size(G, 2));
  unsigned char* amax = amin + reg_size(G, 3);
  const long long vox = (long long)G.D * G.H * G.W;
  const double* st = stats + (long long)T.nc * kStats;
  double ki = 0.0, kb = 0.0, kt = 0.0;
  if (!gin) {                               // d iflat / d sk_v = (t_v - iflat) / (S_p + 1)
    ki = (double)gout[0] * st[6] / (st[1] + 1.0);
    kb = -ki * st[4];
  }
  if (skt) kt = (double)gout[0] * st[7] / (st[3] + 1.0);   // d tflat / d p_v = st_v / (S_t + 1)

  for (int i = threadIdx.x; i < reg_size(G, 4); i += kThreads) {
    int z, y, x;
    coords(G, T, 4, i, z, y, x);
    xs[i] = inb(G, z, y, x) ? fetch(in, G, T.n, T.c, z, y, x) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < reg_size(G, 3); i += kThreads) {
    int z, y, x, code = 0;
    coords(G, T, 3, i, z, y, x);
    ms[i] = inb(G, z, y, x) ? window_pick<true>(xs, G, T, 4, z, y, x, code) : 0.f;
    amin[i] = (unsigned char)code;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < reg_size(G, 2); i += kThreads) {
    int z, y, x, code = 0;
    coords(G, T, 2, i, z, y, x);
    float h = 0.f, ag = 0.f;
    if (inb(G, z, y, x)) {
      const float m = ms[lidx(G, T, 3, z, y, x)];
      const float M = window_pick<false>(ms, G, T, 3, z, y, x, code);
      const float d = __fsub_rn(M, m);
      const float e = __fsub_rn(xs[lidx(G, T, 4, z, y, x)], relu(d));
      const long long o = (long long)T.nc * vox + ((long long)z * G.H + y) * G.W + x;
      const float g = gin ? gin[o] : (float)(ki * (double)fetch(tgt, G, T.n, T.c, z, y, x) + kb);
      ag = e > 0.f ? g : 0.f;
      h = d > 0.f ? ag : 0.f;
    }
    hs[i] = h;
    ags[i] = ag;
    amax[i] = (unsigned char)code;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < reg_size(G, 1); i += kThreads) {
    int z, y, x;
    coords(G, T, 1, i, z, y, x);
    double g = 0.0;
    if (inb(G, z, y, x)) {
      g = (double)hs[lidx(G, T, 2, z, y, x)];
      CL_FOR_WINDOW(z, y, x) {              // w = u + delta routes to u when its argmax code is that of -delta
        const int j = lidx(G, T, 2, z + dz, y + dy, x + dx);
        if (amax[j] == 26 - ((dz + 1) * 9 + (dy + 1) * 3 + (dx + 1))) g -= (double)hs[j];
      }
    }
    gms[i] = g;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < reg_size(G, 0); i += kThreads) {
    int z, y, x;
    coords(G, T, 0, i, z, y, x);
    if (!inb(G, z, y, x)) continue;
    double g = (double)ags[lidx(G, T, 2, z, y, x)];
    CL_FOR_WINDOW(z, y, x) {
      if (amin[lidx(G, T, 3, z + dz, y + dy, x + dx)] == 26 - ((dz + 1) * 9 + (dy + 1) * 3 + (dx + 1)))
        g += gms[lidx(G, T, 1, z + dz, y + dy, x + dx)];
    }
    const long long o = (long long)T.nc * vox + ((long long)z * G.H + y) * G.W + x;
    if (skt) g += kt * (double)skt[o];
    gx[o] = (float)g;
  }
}

// fixed-order CTA sum of one double; every thread gets the result
__device__ double block_sum(double* red, double v) {
  __syncthreads();
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  return red[0];
}

// stats: [N*C][kStats] then the group sums [G][3] = {sum iflat*tflat, sum iflat, sum tflat}, then the count of labels
// outside [0, C); group g is class g (per_class) or everything (binary)
__global__ void __launch_bounds__(kThreads) cldice_finalize_kernel(const ClGeom G, const double* __restrict__ part,
                                                                   int per_class, int labels,
                                                                   const float* __restrict__ alpha, double smooth,
                                                                   double eps, int reduce, double* stats,
                                                                   float* loss) {
  PDL_ENTER();
  __shared__ double red[kThreads];
  const int NC = G.N * G.C, ng = per_class ? G.C : 1;
  const long long nt = ntiles(G);
  double* gs = stats + (long long)NC * kStats;
  if (reduce) {
    double bad = 0.0;
    for (int nc = 0; nc < NC; ++nc) {
      for (int q = 0; q < 4; ++q) {         // {A_p, S_p} from pass 0, {A_t, S_t} from pass 1
        const double* p = part + ((long long)(q / 2) * NC + nc) * nt * kPart + (q % 2);
        double s = 0.0;
        for (long long t = threadIdx.x; t < nt; t += kThreads) s += p[t * kPart];
        s = block_sum(red, s);
        if (threadIdx.x == 0) stats[(long long)nc * kStats + q] = s;
      }
      if (labels && nc % G.C == 0) {
        const double* p = part + ((long long)NC + nc) * nt * kPart + 2;
        double s = 0.0;
        for (long long t = threadIdx.x; t < nt; t += kThreads) s += p[t * kPart];
        bad += block_sum(red, s);
      }
    }
    if (threadIdx.x == 0) {
      for (int g = 0; g < 3 * ng; ++g) gs[g] = 0.0;
      for (int nc = 0; nc < NC; ++nc) {
        double* s = stats + (long long)nc * kStats;
        s[4] = (s[0] + 1.0) / (s[1] + 1.0);            // norm_intersection's smooth = 1
        s[5] = (s[2] + 1.0) / (s[3] + 1.0);
        double* g = gs + 3 * (per_class ? nc % G.C : 0);
        g[0] += s[4] * s[5];
        g[1] += s[4];
        g[2] += s[5];
      }
      gs[3 * ng] = bad;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double total = 0.0;
    for (int g = 0; g < ng; ++g) {
      const double num = 2.0 * gs[3 * g] + smooth, raw = gs[3 * g + 1] + gs[3 * g + 2] + smooth;
      const double den = raw < eps ? eps : raw;
      const double w = per_class ? (double)alpha[g] / G.C : 1.0;
      total += w * (1.0 - num / den);
    }
    loss[0] = (float)total;
    for (int nc = 0; nc < NC; ++nc) {
      double* s = stats + (long long)nc * kStats;
      const int g = per_class ? nc % G.C : 0;
      const double num = 2.0 * gs[3 * g] + smooth, raw = gs[3 * g + 1] + gs[3 * g + 2] + smooth;
      const double den = raw < eps ? eps : raw;
      const double w = per_class ? (double)alpha[g] / G.C : 1.0;
      const double dden = raw >= eps ? num / (den * den) : 0.0;   // clamp_min passes the gradient where raw >= eps
      s[6] = -w * (2.0 * s[5] / den - dden);
      s[7] = -w * (2.0 * s[4] / den - dden);
    }
  }
}

// norm_intersection(cl, v) per (n, c): r = (sum cl*v + 1) / (sum cl + 1); sums[nc] = {sum cl*v, sum cl}
__global__ void __launch_bounds__(1024) cldice_norm_kernel(const ClGeom G, const Field cl, const Field ves,
                                                           double* __restrict__ sums, float* __restrict__ r) {
  PDL_ENTER();
  __shared__ double red[1024];
  const int nc = blockIdx.x, n = nc / G.C, c = nc % G.C;
  const long long vox = (long long)G.D * G.H * G.W;
  double a = 0.0, s = 0.0;
  for (long long i = threadIdx.x; i < vox; i += blockDim.x) {
    const int x = (int)(i % G.W), y = (int)((i / G.W) % G.H), z = (int)(i / ((long long)G.W * G.H));
    const double u = fetch(cl, G, n, c, z, y, x);
    a += u * (double)fetch(ves, G, n, c, z, y, x);
    s += u;
  }
  a = block_sum(red, a);
  s = block_sum(red, s);
  if (threadIdx.x == 0) {
    sums[2 * nc] = a;
    sums[2 * nc + 1] = s;
    r[nc] = (float)((a + 1.0) / (s + 1.0));
  }
}

// g_cl = g (v - r) / (S + 1), g_v = g cl / (S + 1); outputs dense
__global__ void __launch_bounds__(256) cldice_norm_bwd_kernel(const ClGeom G, const Field cl, const Field ves,
                                                              const double* __restrict__ sums,
                                                              const float* __restrict__ gr, float* gcl, float* gv) {
  PDL_ENTER();
  const long long vox = (long long)G.D * G.H * G.W, tot = vox * G.N * G.C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    const int nc = (int)(i / vox), n = nc / G.C, c = nc % G.C;
    const long long e = i % vox;
    const int x = (int)(e % G.W), y = (int)((e / G.W) % G.H), z = (int)(e / ((long long)G.W * G.H));
    const double a = sums[2 * nc], s = sums[2 * nc + 1], k = (double)gr[nc] / (s + 1.0);
    if (gcl) gcl[i] = (float)(k * ((double)fetch(ves, G, n, c, z, y, x) - (a + 1.0) / (s + 1.0)));
    if (gv) gv[i] = (float)(k * (double)fetch(cl, G, n, c, z, y, x));
  }
}

int check_shape(int N, int C, int D, int H, int W) {
  B200_CHECK_ARG(N >= 1 && C >= 1 && D >= 1 && H >= 1 && W >= 1, "cldice: empty shape");
  B200_CHECK_ARG((long long)N * C <= 65535, "cldice: N*C = %lld exceeds the launch grid", (long long)N * C);
  B200_CHECK_ARG((long long)D * H * W < (1LL << 40), "cldice: volume too large");
  const ClGeom G = make_geom(N, C, D, H, W);
  B200_CHECK_ARG(ntiles(G) <= 2147483647LL, "cldice: volume too large");
  return B200SEG_OK;
}

Field field(const float* p, const int64_t* s, const int64_t* lab) {
  Field f;
  memset(&f, 0, sizeof(f));
  f.p = p;
  f.lab = reinterpret_cast<const long long*>(lab);
  if (s) {
    f.sn = s[0]; f.sc = s[1]; f.sd = s[2]; f.sh = s[3]; f.sw = s[4];
  }
  return f;
}

template <typename K>
int set_smem(K kernel, size_t bytes, int device) {
  if (bytes <= 48 * 1024) return B200SEG_OK;
  B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  (void)device;
  return B200SEG_OK;
}

}  // namespace

int64_t cldice_workspace(int N, int C, int D, int H, int W) {
  const ClGeom G = make_geom(N, C, D, H, W);
  return 2LL * N * C * ntiles(G) * kPart * (int64_t)sizeof(double);
}

int cldice_skeleton(const float* x, const int64_t* xs, const int64_t* xlab, int N, int C, int D, int H, int W,
                    int rounds, float* fields, int nfields, const float* other, const int64_t* os,
                    const int64_t* olab, int pass, void* ws, long long ws_bytes, int device, cudaStream_t st) {
  int rc = check_shape(N, C, D, H, W);
  if (rc != B200SEG_OK) return rc;
  B200_CHECK_ARG(rounds >= 1 && rounds <= kMaxRounds, "cldice_skeleton: rounds %d outside [1, %d]", rounds, kMaxRounds);
  B200_CHECK_ARG(fields && nfields >= (rounds < 2 ? rounds : 2), "cldice_skeleton: need min(rounds, 2) fields");
  B200_CHECK_ARG((x && xs && !xlab) || (!x && xlab), "cldice_skeleton: give x with strides, or labels");
  const bool sums = other || olab;
  B200_CHECK_ARG(!sums || (other && os && !olab) || (!other && olab), "cldice_skeleton: give other with strides, or labels");
  B200_CHECK_ARG(pass == 0 || pass == 1, "cldice_skeleton: pass must be 0 or 1");
  const ClGeom G = make_geom(N, C, D, H, W);
  B200_CHECK_ARG(!sums || (ws && ws_bytes >= cldice_workspace(N, C, D, H, W)), "cldice_skeleton: workspace too small");
  const size_t smem = fwd_smem(G);
  rc = set_smem(cldice_round_kernel<true>, smem, device);
  if (rc != B200SEG_OK) return rc;
  rc = set_smem(cldice_round_kernel<false>, smem, device);
  if (rc != B200SEG_OK) return rc;
  const long long fvox = (long long)N * C * D * H * W;
  const Field of = field(other, os, olab);
  double* part = sums ? static_cast<double*>(ws) + (long long)pass * N * C * ntiles(G) * kPart : nullptr;
  const dim3 grid((unsigned)ntiles(G), (unsigned)(N * C));
  for (int r = 0; r < rounds; ++r) {
    const Field in = r == 0 ? field(x, xs, xlab) : dense_field(fields + (long long)((r - 1) % nfields) * fvox, G);
    float* out = fields + (long long)(r % nfields) * fvox;
    const int bad = (xlab && r == 0 && sums) ? 1 : 0;
    if (sums && r == rounds - 1)
      launch_k(cldice_round_kernel<true>, grid, kThreads, smem, st, G, in, out, of, part, bad);
    else
      launch_k(cldice_round_kernel<false>, grid, kThreads, smem, st, G, in, out, of, part, bad);
    B200_LAUNCH_CHECK();
  }
  return B200SEG_OK;
}

int cldice_finalize(int N, int C, int D, int H, int W, int per_class, int labels, const float* alpha, double smooth,
                    double eps, int reduce, const void* ws, long long ws_bytes, double* stats, float* loss,
                    cudaStream_t st) {
  int rc = check_shape(N, C, D, H, W);
  if (rc != B200SEG_OK) return rc;
  B200_CHECK_ARG(!per_class || alpha, "cldice_finalize: the per-class loss needs alpha");
  B200_CHECK_ARG(!reduce || (ws && ws_bytes >= cldice_workspace(N, C, D, H, W)), "cldice_finalize: workspace too small");
  const ClGeom G = make_geom(N, C, D, H, W);
  launch_k(cldice_finalize_kernel, dim3(1), kThreads, 0, st, G, static_cast<const double*>(ws), per_class, labels,
           alpha, smooth, eps, reduce, stats, loss);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int cldice_bwd(const float* x, const int64_t* xs, int N, int C, int D, int H, int W, int rounds, const float* fields,
               const float* gsk, const float* t, const int64_t* ts, const int64_t* tlab, const float* skt,
               const double* stats, const float* gout, float* grad, float* scratch, int device, cudaStream_t st) {
  int rc = check_shape(N, C, D, H, W);
  if (rc != B200SEG_OK) return rc;
  B200_CHECK_ARG(rounds >= 1 && rounds <= kMaxRounds, "cldice_bwd: rounds %d outside [1, %d]", rounds, kMaxRounds);
  B200_CHECK_ARG(x && xs && grad && (rounds < 2 || (fields && scratch)), "cldice_bwd: null argument");
  B200_CHECK_ARG(gsk || (((t && ts && !tlab) || (!t && tlab)) && skt && stats && gout),
                 "cldice_bwd: give grad_skeleton, or the loss's target, target skeleton, stats and gout");
  const ClGeom G = make_geom(N, C, D, H, W);
  const size_t smem = bwd_smem(G);
  rc = set_smem(cldice_round_bwd_kernel, smem, device);
  if (rc != B200SEG_OK) return rc;
  const long long fvox = (long long)N * C * D * H * W;
  const Field tf = field(t, ts, tlab);
  const dim3 grid((unsigned)ntiles(G), (unsigned)(N * C));
  const float* gin = gsk;
  for (int r = rounds - 1; r >= 0; --r) {           // g_r goes to grad for even r, so g_0 lands there
    const Field in = r == 0 ? field(x, xs, nullptr) : dense_field(fields + (long long)(r - 1) * fvox, G);
    float* out = (r % 2 == 0) ? grad : scratch;
    launch_k(cldice_round_bwd_kernel, grid, kThreads, smem, st, G, in, gin, tf, stats, gout,
             (r == 0 && !gsk) ? skt : nullptr, out);
    B200_LAUNCH_CHECK();
    gin = out;
  }
  return B200SEG_OK;
}

int cldice_norm(const float* cl, const int64_t* cs, const float* v, const int64_t* vs, int N, int C, int D, int H,
                int W, double* sums, float* r, cudaStream_t st) {
  int rc = check_shape(N, C, D, H, W);
  if (rc != B200SEG_OK) return rc;
  B200_CHECK_ARG(cl && cs && v && vs && sums && r, "cldice_norm: null argument");
  const ClGeom G = make_geom(N, C, D, H, W);
  launch_k(cldice_norm_kernel, dim3(N * C), 1024, 0, st, G, field(cl, cs, nullptr), field(v, vs, nullptr), sums, r);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int cldice_norm_bwd(const float* cl, const int64_t* cs, const float* v, const int64_t* vs, int N, int C, int D, int H,
                    int W, const double* sums, const float* gr, float* gcl, float* gv, int device, cudaStream_t st) {
  int rc = check_shape(N, C, D, H, W);
  if (rc != B200SEG_OK) return rc;
  B200_CHECK_ARG(cl && cs && v && vs && sums && gr && (gcl || gv), "cldice_norm_bwd: null argument");
  const ClGeom G = make_geom(N, C, D, H, W);
  const long long tot = (long long)N * C * D * H * W;
  long long blocks = (tot + 255) / 256;
  const long long cap = 8LL * num_sms(device);
  if (blocks > cap) blocks = cap;
  launch_k(cldice_norm_bwd_kernel, dim3((unsigned)blocks), 256, 0, st, G, field(cl, cs, nullptr),
           field(v, vs, nullptr), sums, gr, gcl, gv);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
