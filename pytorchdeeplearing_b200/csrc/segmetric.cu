// The nine 3-D segmentation metrics of Seg_Metirc3d (model/metric.py:11-142) with exact surface distances (sm_90a).
//
//   1. segm_classify_kernel  one pass over both masks, tiled in shared memory with a one-voxel halo: foreground and
//                            18-neighbourhood surface bits of both masks (one byte per voxel), per-block int64 counts
//                            R, P, I, U, S_r, S_p and the count of values outside {0, 1}
//   2. segm_rowdist_kernel   along W, for both seed sets (real surface, pred surface): the integer distance to the
//                            nearest seed of the row, from a forward and a backward warp scan
//   3. segm_colenv_kernel    along H: the Felzenszwalb-Huttenlocher lower envelope of f + (dy*sy)^2, fp64
//   4. segm_depthenv_kernel  along D: the same, evaluated only at the other mask's surface voxels and reduced to
//                            per-block fp64 {sum d, sum d^2, max d}; nothing of the full fp64 volume is written
//   5. segm_finalize_kernel  per volume, the fixed-order sums of the partials -> counts [6], metrics [9], flag
// On demand (segmetric3d_points): pass 4 writes d in place at the surface voxels, then an ordered compaction
// (per-row counts, one scan over the rows, a warp-ballot write per row) emits the C-order linear indices of each
// surface together with the nn distance of each point.
//
// Transform t = 0 is seeded by the real surface and read at pred surface voxels (pred2real); t = 1 the reverse
// (real2pred).  H and D lines run one per thread with 32 consecutive x-columns per warp, so every load and store of a
// line step coalesces; the envelope of each line lives in workspace arrays laid out like the volume.  Lines without a
// seed stay +inf and never enter an envelope, so no inf - inf is formed.  Every reduction has a fixed order, so two
// runs give identical bits; nothing is allocated or synchronised.
#include <math.h>

#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kTX = 32, kTY = 8, kTZ = 4;                  // classification tile (x, y, z)
constexpr int kHX = kTX + 2, kHY = kTY + 2, kHZ = kTZ + 2;  // with the one-voxel halo
constexpr int kClsThreads = kTX * kTY;
constexpr int kLineThreads = 128;                          // H and D passes: 128 consecutive x-columns per block
constexpr int kRowWarps = 8;
constexpr int kNoSeed = 0x7fffffff;
constexpr int kCntWords = 8;                               // R, P, I, U, S_r, S_p, bad, (pad)

// cls byte bits
constexpr unsigned kRealFg = 1u, kPredFg = 2u, kRealSurf = 4u, kPredSurf = 8u;

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct SegLayout {
  long long V;                 // voxels per volume
  int nbc, nbd;                // blocks per volume of the classify / depth pass
  size_t cls, g, f, ev, efv, ez, cpart, dpart, rowcnt, bytes;
};

SegLayout seg_layout(int N, int D, int H, int W) {
  SegLayout L;
  L.V = (long long)D * H * W;
  L.nbc = ((W + kTX - 1) / kTX) * ((H + kTY - 1) / kTY) * ((D + kTZ - 1) / kTZ);
  L.nbd = ((W + kLineThreads - 1) / kLineThreads) * H;
  const size_t nv = (size_t)N * (size_t)L.V;
  size_t o = 0;
  L.cls = o; o += align256(nv);
  L.g = o; o += align256(2 * nv * 4);
  L.f = o; o += align256(2 * nv * 8);
  L.ev = o; o += align256(2 * nv * 4);
  L.efv = o; o += align256(2 * nv * 8);
  L.ez = o; o += align256(2 * nv * 8);
  L.cpart = o; o += align256((size_t)N * L.nbc * kCntWords * 8);
  L.dpart = o; o += align256((size_t)2 * N * L.nbd * 3 * 8);
  L.rowcnt = o; o += align256((size_t)2 * N * D * H * 8);
  L.bytes = o;
  return L;
}

__device__ __forceinline__ long long load_mask(const void* p, int dtype, long long i) {
  if (dtype == B200SEG_I64) return reinterpret_cast<const long long*>(p)[i];
  if (dtype == B200SEG_I32) return reinterpret_cast<const int*>(p)[i];
  return reinterpret_cast<const unsigned char*>(p)[i];
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ 1. classify + count
// grid (ceil(W/32), ceil(H/8), ceil(D/4) * N), block 256; thread (tx, ty) owns the kTZ voxels of its (x, y) column
__global__ void __launch_bounds__(kClsThreads) segm_classify_kernel(const void* __restrict__ real, int rdt,
                                                                    const void* __restrict__ pred, int pdt, int D,
                                                                    int H, int W, int zblocks,
                                                                    unsigned char* __restrict__ cls,
                                                                    long long* __restrict__ cpart) {
  PDL_ENTER();
  __shared__ unsigned char s_fg[kHZ][kHY][kHX];
  __shared__ unsigned long long s_red[kClsThreads / 32][kCntWords];
  const int n = blockIdx.z / zblocks;
  const int z0 = (blockIdx.z - n * zblocks) * kTZ, y0 = blockIdx.y * kTY, x0 = blockIdx.x * kTX;
  const long long V = (long long)D * H * W;
  const long long vbase = (long long)n * V;
  const int tid = threadIdx.x;
  unsigned long long bad = 0;
  for (int i = tid; i < kHZ * kHY * kHX; i += kClsThreads) {
    const int hx = i % kHX, hy = (i / kHX) % kHY, hz = i / (kHX * kHY);
    const int x = x0 + hx - 1, y = y0 + hy - 1, z = z0 + hz - 1;
    unsigned char b = 0;          // outside the volume is background (binary_erosion's border_value = 0)
    if (x >= 0 && x < W && y >= 0 && y < H && z >= 0 && z < D) {
      const long long j = vbase + ((long long)z * H + y) * W + x;
      const long long r = load_mask(real, rdt, j), p = load_mask(pred, pdt, j);
      b = (r != 0 ? kRealFg : 0u) | (p != 0 ? kPredFg : 0u);
      const bool inner = hx >= 1 && hx <= kTX && hy >= 1 && hy <= kTY && hz >= 1 && hz <= kTZ;
      if (inner && ((unsigned long long)r > 1ull || (unsigned long long)p > 1ull)) ++bad;
    }
    s_fg[hz][hy][hx] = b;
  }
  __syncthreads();
  const int tx = tid % kTX, ty = tid / kTX;
  const int x = x0 + tx, y = y0 + ty;
  unsigned long long c[6] = {0, 0, 0, 0, 0, 0};
  if (x < W && y < H) {
#pragma unroll
    for (int tz = 0; tz < kTZ; ++tz) {
      const int z = z0 + tz;
      if (z >= D) break;
      const unsigned ctr = s_fg[tz + 1][ty + 1][tx + 1];
      unsigned all = 0xffu;       // AND over the 18-neighbourhood (faces and edges, no corners)
#pragma unroll
      for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
          for (int dx = -1; dx <= 1; ++dx) {
            const int a = (dz != 0) + (dy != 0) + (dx != 0);
            if (a == 0 || a == 3) continue;
            all &= s_fg[tz + 1 + dz][ty + 1 + dy][tx + 1 + dx];
          }
      const unsigned rf = ctr & kRealFg, pf = ctr & kPredFg;
      const unsigned rs = (rf && !(all & kRealFg)) ? kRealSurf : 0u;
      const unsigned ps = (pf && !(all & kPredFg)) ? kPredSurf : 0u;
      cls[vbase + ((long long)z * H + y) * W + x] = (unsigned char)(ctr | rs | ps);
      c[0] += rf ? 1 : 0;
      c[1] += pf ? 1 : 0;
      c[2] += (rf && pf) ? 1 : 0;
      c[3] += (rf || pf) ? 1 : 0;
      c[4] += rs ? 1 : 0;
      c[5] += ps ? 1 : 0;
    }
  }
  const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
  for (int k = 0; k < 6; ++k) c[k] = warp_sum_u64(c[k]);
  bad = warp_sum_u64(bad);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 6; ++k) s_red[wid][k] = c[k];
    s_red[wid][6] = bad;
    s_red[wid][7] = 0;
  }
  __syncthreads();
  if (tid < kCntWords) {
    unsigned long long t = 0;
#pragma unroll
    for (int w = 0; w < kClsThreads / 32; ++w) t += s_red[w][tid];
    const long long blk = ((long long)(blockIdx.z - n * zblocks) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    cpart[((long long)n * ((long long)gridDim.x * gridDim.y * zblocks) + blk) * kCntWords + tid] = (long long)t;
  }
}

// ------------------------------------------------------------------------------------------------ 2. rows (W)
// g[t][n][z][y][x] = |x - nearest x' of the row with a seed of transform t| (kNoSeed if the row has none).
// One warp per row; a forward max-scan finds the nearest seed on the left, a backward min-scan the one on the right.
__global__ void __launch_bounds__(kRowWarps * 32) segm_rowdist_kernel(const unsigned char* __restrict__ cls,
                                                                      long long rows, int W, long long nv,
                                                                      int* __restrict__ g) {
  PDL_ENTER();
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * kRowWarps;
  for (long long row = (long long)blockIdx.x * kRowWarps + (threadIdx.x >> 5); row < rows; row += nwarps) {
    const unsigned char* c = cls + row * W;
    int* g0 = g + row * W;
    int* g1 = g0 + nv;
    int left0 = -1, left1 = -1;
    for (int x0 = 0; x0 < W; x0 += 32) {
      const int x = x0 + lane;
      const unsigned b = x < W ? c[x] : 0u;
      int l0 = (b & kRealSurf) ? x : -1, l1 = (b & kPredSurf) ? x : -1;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u0 = __shfl_up_sync(0xffffffffu, l0, o), u1 = __shfl_up_sync(0xffffffffu, l1, o);
        if (lane >= o) {
          l0 = max(l0, u0);
          l1 = max(l1, u1);
        }
      }
      l0 = max(l0, left0);
      l1 = max(l1, left1);
      if (x < W) {
        g0[x] = l0 >= 0 ? x - l0 : kNoSeed;
        g1[x] = l1 >= 0 ? x - l1 : kNoSeed;
      }
      left0 = __shfl_sync(0xffffffffu, l0, 31);
      left1 = __shfl_sync(0xffffffffu, l1, 31);
    }
    int right0 = kNoSeed, right1 = kNoSeed;
    for (int x0 = ((W - 1) / 32) * 32; x0 >= 0; x0 -= 32) {
      const int x = x0 + lane;
      const unsigned b = x < W ? c[x] : 0u;
      int r0 = (b & kRealSurf) ? x : kNoSeed, r1 = (b & kPredSurf) ? x : kNoSeed;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u0 = __shfl_down_sync(0xffffffffu, r0, o), u1 = __shfl_down_sync(0xffffffffu, r1, o);
        if (lane + o < 32) {
          r0 = min(r0, u0);
          r1 = min(r1, u1);
        }
      }
      r0 = min(r0, right0);
      r1 = min(r1, right1);
      if (x < W) {       // each lane re-reads only what it wrote itself in the forward sweep
        if (r0 != kNoSeed) g0[x] = min(g0[x], r0 - x);
        if (r1 != kNoSeed) g1[x] = min(g1[x], r1 - x);
      }
      right0 = __shfl_sync(0xffffffffu, r0, 0);
      right1 = __shfl_sync(0xffffffffu, r1, 0);
    }
  }
}

// ------------------------------------------------------------------------------------------------ lower envelope
// Felzenszwalb-Huttenlocher over one line of n samples at stride `st`: parabolas (p - q*s)^2 + f(q) for the finite
// f(q); env_v / env_f / env_z hold vertex index, vertex height and left boundary of each envelope segment at the
// same strided slots.  Returns the index of the last segment, -1 if every sample is +inf.
template <typename LoadF>
__device__ __forceinline__ int lower_envelope(LoadF load, int n, long long st, double s, int* __restrict__ env_v,
                                             double* __restrict__ env_f, double* __restrict__ env_z) {
  int k = -1;
  int vk = 0;
  double fk = 0.0, zk = 0.0;       // cached top of the stack
  for (int q = 0; q < n; ++q) {
    const double fq = load(q);
    if (isinf(fq)) continue;
    const double pq = (double)q * s;
    double sq = -INFINITY;
    while (k >= 0) {
      const double pv = (double)vk * s;
      sq = ((fq + pq * pq) - (fk + pv * pv)) / (2.0 * (pq - pv));
      if (k > 0 && sq <= zk) {
        --k;
        vk = env_v[k * st];
        fk = env_f[k * st];
        zk = env_z[k * st];
      } else {
        break;
      }
    }
    ++k;
    vk = q;
    fk = fq;
    zk = k == 0 ? -INFINITY : sq;
    env_v[k * st] = vk;
    env_f[k * st] = fk;
    env_z[k * st] = zk;
  }
  return k;
}

// ------------------------------------------------------------------------------------------------ 3. columns (H)
// f[t][n][z][y][x] = min_y' (g(y') sx)^2 + ((y - y') sy)^2.  grid (ceil(W/128), D, 2N)
__global__ void __launch_bounds__(kLineThreads) segm_colenv_kernel(const int* __restrict__ g,
                                                                   const double* __restrict__ spacing, int N, int D,
                                                                   int H, int W, double* __restrict__ f,
                                                                   int* __restrict__ env_v, double* __restrict__ env_f,
                                                                   double* __restrict__ env_z) {
  PDL_ENTER();
  const int x = blockIdx.x * kLineThreads + threadIdx.x;
  if (x >= W) return;
  const int tn = blockIdx.z, n = tn % N, z = blockIdx.y;
  const double sy = spacing[n * 3 + 1], sx = spacing[n * 3 + 2];
  const long long base = ((long long)tn * D + z) * H * W + x;
  const long long st = W;
  const int* gl = g + base;
  auto load = [&](int q) -> double {
    const int v = gl[q * st];
    if (v == kNoSeed) return INFINITY;
    const double d = (double)v * sx;
    return d * d;
  };
  int* ev = env_v + base;
  double* ef = env_f + base;
  double* ez = env_z + base;
  double* out = f + base;
  const int k = lower_envelope(load, H, st, sy, ev, ef, ez);
  if (k < 0) {
    for (int q = 0; q < H; ++q) out[q * st] = INFINITY;
    return;
  }
  int j = 0;
  int vj = ev[0];
  double fj = ef[0];
  double znext = k > 0 ? ez[st] : INFINITY;
  for (int q = 0; q < H; ++q) {
    const double pq = (double)q * sy;
    while (j < k && znext < pq) {
      ++j;
      vj = ev[j * st];
      fj = ef[j * st];
      znext = j < k ? ez[(j + 1) * st] : INFINITY;
    }
    const double d = (double)(q - vj) * sy;
    out[q * st] = d * d + fj;
  }
}

// ------------------------------------------------------------------------------------------------ 4. depth (D)
// the envelope of f along z, read where the other mask has a surface voxel: dpart[t][n][blk] = {sum d, sum d^2, max d}.
// write_d: also store d in place of f at those voxels (the points path).  grid (ceil(W/128), H, 2N)
__global__ void __launch_bounds__(kLineThreads) segm_depthenv_kernel(double* __restrict__ f,
                                                                     const unsigned char* __restrict__ cls,
                                                                     const double* __restrict__ spacing, int N, int D,
                                                                     int H, int W, int* __restrict__ env_v,
                                                                     double* __restrict__ env_f,
                                                                     double* __restrict__ env_z, int write_d,
                                                                     double* __restrict__ dpart) {
  PDL_ENTER();
  __shared__ double s_red[kLineThreads / 32][3];
  const int x = blockIdx.x * kLineThreads + threadIdx.x;
  const int tn = blockIdx.z, t = tn / N, n = tn % N, y = blockIdx.y;
  const unsigned evalbit = t == 0 ? kPredSurf : kRealSurf;
  const long long HW = (long long)H * W;
  double sum = 0.0, sum2 = 0.0, mx = 0.0;
  if (x < W) {
    const double sz = spacing[n * 3 + 0];
    const long long base = (long long)tn * D * HW + (long long)y * W + x;
    const unsigned char* cl = cls + (long long)n * D * HW + (long long)y * W + x;
    double* fl = f + base;
    int* ev = env_v + base;
    double* ef = env_f + base;
    double* ez = env_z + base;
    auto load = [&](int q) -> double { return fl[q * HW]; };
    const int k = lower_envelope(load, D, HW, sz, ev, ef, ez);
    int j = 0;
    int vj = k >= 0 ? ev[0] : 0;
    double fj = k >= 0 ? ef[0] : INFINITY;
    double znext = k > 0 ? ez[HW] : INFINITY;
    for (int q = 0; q < D; ++q) {
      if (!(cl[q * HW] & evalbit)) continue;
      const double pq = (double)q * sz;
      while (j < k && znext < pq) {
        ++j;
        vj = ev[j * HW];
        fj = ef[j * HW];
        znext = j < k ? ez[(j + 1) * HW] : INFINITY;
      }
      const double dd = (double)(q - vj) * sz;
      const double d = sqrt(dd * dd + fj);
      sum += d;
      sum2 += d * d;
      mx = fmax(mx, d);
      if (write_d) fl[q * HW] = d;
    }
  }
  sum = warp_sum(sum);
  sum2 = warp_sum(sum2);
  mx = warp_max(mx);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) {
    s_red[wid][0] = sum;
    s_red[wid][1] = sum2;
    s_red[wid][2] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0, m = 0.0;
#pragma unroll
    for (int w = 0; w < kLineThreads / 32; ++w) {
      a += s_red[w][0];
      b += s_red[w][1];
      m = fmax(m, s_red[w][2]);
    }
    const long long blk = (long long)blockIdx.y * gridDim.x + blockIdx.x;
    double* o = dpart + ((long long)tn * gridDim.x * gridDim.y + blk) * 3;
    o[0] = a;
    o[1] = b;
    o[2] = m;
  }
}

// ------------------------------------------------------------------------------------------------ 5. finalize
// one block per volume.  counts[n] = {R, P, I, U, S_r, S_p}; metrics[n] = {dice, jaccard, VOE, RVD, FNR, FPR, ASSD,
// RMSD, MSD} (model/metric.py:68-142); flags[n] = 1 if a mask holds a value outside {0, 1}
__global__ void __launch_bounds__(256) segm_finalize_kernel(const long long* __restrict__ cpart, int nbc,
                                                            const double* __restrict__ dpart, int nbd, int N,
                                                            long long* __restrict__ counts,
                                                            double* __restrict__ metrics, int* __restrict__ flags) {
  PDL_ENTER();
  __shared__ unsigned long long s_u[8][kCntWords];
  __shared__ double s_d[8][6];
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  unsigned long long c[kCntWords];
#pragma unroll
  for (int k = 0; k < kCntWords; ++k) c[k] = 0;
  for (int b = tid; b < nbc; b += 256) {
    const long long* p = cpart + ((long long)n * nbc + b) * kCntWords;
#pragma unroll
    for (int k = 0; k < kCntWords; ++k) c[k] += (unsigned long long)p[k];
  }
  // d[0..2] = pred2real {sum, sum^2, max}, d[3..5] = real2pred
  double d[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    for (int b = tid; b < nbd; b += 256) {
      const double* p = dpart + (((long long)t * N + n) * nbd + b) * 3;
      d[3 * t] += p[0];
      d[3 * t + 1] += p[1];
      d[3 * t + 2] = fmax(d[3 * t + 2], p[2]);
    }
  }
#pragma unroll
  for (int k = 0; k < kCntWords; ++k) c[k] = warp_sum_u64(c[k]);
#pragma unroll
  for (int k = 0; k < 6; ++k) d[k] = (k % 3 == 2) ? warp_max(d[k]) : warp_sum(d[k]);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < kCntWords; ++k) s_u[wid][k] = c[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) s_d[wid][k] = d[k];
  }
  __syncthreads();
  if (tid != 0) return;
  long long cnt[kCntWords];
  double dd[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < kCntWords; ++k) {
    unsigned long long s = 0;
    for (int w = 0; w < 8; ++w) s += s_u[w][k];
    cnt[k] = (long long)s;
  }
  for (int k = 0; k < 6; ++k)
    for (int w = 0; w < 8; ++w) dd[k] = (k % 3 == 2) ? fmax(dd[k], s_d[w][k]) : dd[k] + s_d[w][k];
  const long long R = cnt[0], P = cnt[1], I = cnt[2], U = cnt[3], Sr = cnt[4], Sp = cnt[5];
  for (int k = 0; k < 6; ++k) counts[(long long)n * 6 + k] = cnt[k];
  flags[n] = cnt[6] != 0 ? 1 : 0;
  double* m = metrics + (long long)n * 9;
  const double jac = (double)I / (double)U;
  m[0] = (double)(2 * I) / (double)(R + P);
  m[1] = jac;
  m[2] = 1.0 - jac;
  m[3] = (double)(P - R) / (double)R;
  m[4] = (double)(R - I) / (double)U;
  m[5] = (double)(P - I) / (double)U;
  if (Sr > 0 && Sp > 0) {
    const double S = (double)(Sr + Sp);
    m[6] = (dd[0] + dd[3]) / S;
    m[7] = sqrt((dd[1] + dd[4]) / S);
    m[8] = fmax(dd[2], dd[5]);
  } else {
    m[6] = m[7] = m[8] = NAN;
  }
}

// ------------------------------------------------------------------------------------------------ points path
// rowcnt[s][row] = surface voxels of surface s (0 real, 1 pred) in row (n, z, y); one warp per row
__global__ void __launch_bounds__(kRowWarps * 32) segm_rowcount_kernel(const unsigned char* __restrict__ cls,
                                                                       long long rows, int W,
                                                                       long long* __restrict__ rowcnt) {
  PDL_ENTER();
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * kRowWarps;
  for (long long row = (long long)blockIdx.x * kRowWarps + (threadIdx.x >> 5); row < rows; row += nwarps) {
    const unsigned char* c = cls + row * W;
    int a = 0, b = 0;
    for (int x = lane; x < W; x += 32) {
      const unsigned v = c[x];
      a += (v & kRealSurf) ? 1 : 0;
      b += (v & kPredSurf) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
      rowcnt[row] = a;
      rowcnt[rows + row] = b;
    }
  }
}

// in place: rowcnt[s] becomes its exclusive scan over all rows of all volumes.  grid 2 (one block per surface)
__global__ void __launch_bounds__(1024) segm_rowscan_kernel(long long* __restrict__ rowcnt, long long rows) {
  PDL_ENTER();
  __shared__ long long s_w[32];
  long long* r = rowcnt + blockIdx.x * rows;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  long long carry = 0;
  for (long long b = 0; b < rows; b += 1024) {
    const long long i = b + tid;
    const long long v = i < rows ? r[i] : 0;
    long long inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    long long before = 0, all = 0;
    for (int w = 0; w < 32; ++w) {
      const long long x = s_w[w];
      before += w < wid ? x : 0;
      all += x;
    }
    __syncthreads();
    if (i < rows) r[i] = carry + before + inc - v;
    carry += all;
  }
}

// ordered write of each surface: idx = linear index within the volume, nn = d of that voxel (written in place of f
// by the depth pass; real points read transform 1 = real2pred, pred points transform 0 = pred2real)
__global__ void __launch_bounds__(kRowWarps * 32) segm_compact_kernel(const unsigned char* __restrict__ cls,
                                                                      const long long* __restrict__ rowoff,
                                                                      const double* __restrict__ f, long long rows,
                                                                      int W, long long rows_per_vol, long long nv,
                                                                      long long cap_r, long long cap_p,
                                                                      long long* __restrict__ real_idx,
                                                                      long long* __restrict__ pred_idx,
                                                                      double* __restrict__ real_nn,
                                                                      double* __restrict__ pred_nn) {
  PDL_ENTER();
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  const long long nwarps = (long long)gridDim.x * kRowWarps;
  for (long long row = (long long)blockIdx.x * kRowWarps + (threadIdx.x >> 5); row < rows; row += nwarps) {
    const long long n = row / rows_per_vol;
    const long long vrow = (row - n * rows_per_vol) * W;      // linear index of (z, y, 0) within the volume
    long long oa = rowoff[row], ob = rowoff[rows + row];
    const unsigned char* c = cls + row * W;
    for (int x0 = 0; x0 < W; x0 += 32) {
      const int x = x0 + lane;
      const unsigned v = x < W ? c[x] : 0u;
      const unsigned ma = __ballot_sync(0xffffffffu, (v & kRealSurf) != 0);
      const unsigned mb = __ballot_sync(0xffffffffu, (v & kPredSurf) != 0);
      if (v & kRealSurf) {
        const long long s = oa + __popc(ma & lt);
        if (s < cap_r) {
          real_idx[s] = vrow + x;
          real_nn[s] = f[nv + row * W + x];
        }
      }
      if (v & kPredSurf) {
        const long long s = ob + __popc(mb & lt);
        if (s < cap_p) {
          pred_idx[s] = vrow + x;
          pred_nn[s] = f[row * W + x];
        }
      }
      oa += __popc(ma);
      ob += __popc(mb);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
int64_t segmetric3d_workspace(int N, int D, int H, int W) { return (int64_t)seg_layout(N, D, H, W).bytes; }

namespace {
struct SegBufs {
  unsigned char* cls;
  int* g;
  double* f;
  int* ev;
  double* efv;
  double* ez;
  long long* cpart;
  double* dpart;
  long long* rowcnt;
};

SegBufs seg_bufs(const SegLayout& L, void* ws) {
  char* w = static_cast<char*>(ws);
  return SegBufs{reinterpret_cast<unsigned char*>(w + L.cls), reinterpret_cast<int*>(w + L.g),
                 reinterpret_cast<double*>(w + L.f),          reinterpret_cast<int*>(w + L.ev),
                 reinterpret_cast<double*>(w + L.efv),        reinterpret_cast<double*>(w + L.ez),
                 reinterpret_cast<long long*>(w + L.cpart),   reinterpret_cast<double*>(w + L.dpart),
                 reinterpret_cast<long long*>(w + L.rowcnt)};
}

int seg_check(int rdt, int pdt, int N, int D, int H, int W, const SegLayout& L, void* ws, long long ws_bytes) {
  const auto dt_ok = [](int dt) { return dt == B200SEG_U8 || dt == B200SEG_I32 || dt == B200SEG_I64; };
  B200_CHECK_ARG(dt_ok(rdt) && dt_ok(pdt), "segmetric3d: mask dtypes %d / %d (bool/uint8, int32 or int64)", rdt, pdt);
  B200_CHECK_ARG(N >= 1 && D >= 1 && H >= 1 && W >= 1, "segmetric3d: empty shape");
  B200_CHECK_ARG(2 * N <= 65535 && D <= 65535 && H <= 65535 && (long long)((D + kTZ - 1) / kTZ) * N <= 65535,
                 "segmetric3d: shape (%d, %d, %d, %d) outside the launch grid", N, D, H, W);
  B200_CHECK_ARG(ws && (size_t)ws_bytes >= L.bytes, "segmetric3d: workspace too small");
  return B200SEG_OK;
}

// passes 1-4 (everything but the finalize)
void seg_run(const void* real, int rdt, const void* pred, int pdt, int N, int D, int H, int W, const double* spacing,
             const SegLayout& L, const SegBufs& B, int write_d, int device, cudaStream_t s) {
  const long long nv = (long long)N * L.V;
  const int zb = (D + kTZ - 1) / kTZ;
  launch_k(segm_classify_kernel, dim3((W + kTX - 1) / kTX, (H + kTY - 1) / kTY, zb * N), kClsThreads, 0, s, real, rdt,
           pred, pdt, D, H, W, zb, B.cls, B.cpart);
  const long long rows = (long long)N * D * H;
  long long rb = (rows + kRowWarps - 1) / kRowWarps;
  const long long cap = (long long)num_sms(device) * 16;
  if (rb > cap) rb = cap;
  launch_k(segm_rowdist_kernel, dim3((unsigned)rb), kRowWarps * 32, 0, s, (const unsigned char*)B.cls, rows, W, nv,
           B.g);
  const unsigned gx = (W + kLineThreads - 1) / kLineThreads;
  launch_k(segm_colenv_kernel, dim3(gx, D, 2 * N), kLineThreads, 0, s, (const int*)B.g, spacing, N, D, H, W, B.f,
           B.ev, B.efv, B.ez);
  launch_k(segm_depthenv_kernel, dim3(gx, H, 2 * N), kLineThreads, 0, s, B.f, (const unsigned char*)B.cls, spacing, N,
           D, H, W, B.ev, B.efv, B.ez, write_d, B.dpart);
}
}  // namespace

int segmetric3d(const void* real, int rdt, const void* pred, int pdt, int N, int D, int H, int W,
                const double* spacing, void* ws, long long ws_bytes, long long* counts, double* metrics, int* flags,
                int device, cudaStream_t s) {
  const SegLayout L = seg_layout(N, D, H, W);
  const int rc = seg_check(rdt, pdt, N, D, H, W, L, ws, ws_bytes);
  if (rc != B200SEG_OK) return rc;
  const SegBufs B = seg_bufs(L, ws);
  seg_run(real, rdt, pred, pdt, N, D, H, W, spacing, L, B, 0, device, s);
  launch_k(segm_finalize_kernel, dim3(N), 256, 0, s, (const long long*)B.cpart, L.nbc, (const double*)B.dpart, L.nbd,
           N, counts, metrics, flags);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int segmetric3d_points(const void* real, int rdt, const void* pred, int pdt, int N, int D, int H, int W,
                       const double* spacing, void* ws, long long ws_bytes, long long cap_r, long long cap_p,
                       long long* real_idx, long long* pred_idx, double* real_nn, double* pred_nn, int device,
                       cudaStream_t s) {
  const SegLayout L = seg_layout(N, D, H, W);
  const int rc = seg_check(rdt, pdt, N, D, H, W, L, ws, ws_bytes);
  if (rc != B200SEG_OK) return rc;
  B200_CHECK_ARG(cap_r >= 0 && cap_p >= 0, "segmetric3d_points: negative capacity");
  const SegBufs B = seg_bufs(L, ws);
  seg_run(real, rdt, pred, pdt, N, D, H, W, spacing, L, B, 1, device, s);
  const long long rows = (long long)N * D * H;
  long long rb = (rows + kRowWarps - 1) / kRowWarps;
  const long long cap = (long long)num_sms(device) * 16;
  if (rb > cap) rb = cap;
  launch_k(segm_rowcount_kernel, dim3((unsigned)rb), kRowWarps * 32, 0, s, (const unsigned char*)B.cls, rows, W,
           B.rowcnt);
  launch_k(segm_rowscan_kernel, dim3(2), 1024, 0, s, B.rowcnt, rows);
  launch_k(segm_compact_kernel, dim3((unsigned)rb), kRowWarps * 32, 0, s, (const unsigned char*)B.cls,
           (const long long*)B.rowcnt, (const double*)B.f, rows, W, (long long)D * H, (long long)N * L.V, cap_r, cap_p,
           real_idx, pred_idx, real_nn, pred_nn);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
