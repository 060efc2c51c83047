// Lovasz-Softmax loss (LovaszLoss, model/losses.py:462-473 -> model/lovasz.py:90-138) and the stable segmented radix
// sort it is built on (sm_90a).
//
// Forward, per class segment (class c over all voxels, or over one sample with per_image):
//   1. lovasz_keys_kernel   key = complemented order-preserving bits of e = |[t==c] - z_c| (ascending key order =
//                           descending e), value = index within the segment; ignored voxels get key 0xFFFFFFFF
//   2. radix sort           4 stable LSD passes of 8 bits: per-tile digit histogram, per-digit scan over the tiles,
//                           stable scatter (ranks within a tile from warp match + per-warp digit counts)
//   3. lovasz_tilecnt_kernel foreground count of every sorted tile
//   4. lovasz_grad_kernel   exact integer prefix counts of the sorted foreground, Jaccard J_i and grad_i = J_i - J_{i-1}
//                           in fp64 (lovasz.py:21-32), sum e_i grad_i per tile, grad_i scattered to coef[voxel][c]
//   5. lovasz_finalize_kernel the mean over present classes (and samples), per-segment weights
// Backward: one elementwise pass dz = gout * coef * sgn(z_c - [t==c]) * weight (torch's abs backward: sgn(0) = 0).
// Every reduction runs in a fixed order, so two runs give identical bits.  Nothing is synchronised or allocated, so
// the whole loss can sit inside a captured CUDA graph.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 16;
constexpr int kTile = kThreads * kItems;     // pairs per tile of the sort and of the gradient scan
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kIgnoredKey = 0xFFFFFFFFu;

inline long long tiles_of(long long len) { return (len + kTile - 1) / kTile; }
inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// exclusive scan of one value per thread over a 256-thread block; *total = sum of all
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    const uint32_t x = s_warp[w];
    before += w < wid ? x : 0u;
    all += x;
  }
  __syncthreads();
  *total = all;
  return before + inc - v;
}

// fixed-order block sum (deterministic)
__device__ __forceinline__ double block_sum(double v, double* s_tmp) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_tmp[wid] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) t += s_tmp[w];
  __syncthreads();
  return t;
}

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long* s_tmp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_tmp[wid] = v;
  __syncthreads();
  unsigned long long t = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) t += s_tmp[w];
  __syncthreads();
  return t;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ radix sort
// hist[(s*256 + digit)*ntiles + tile] = count of `digit` in tile `tile` of segment s; grid (ntiles, nseg)
__global__ void __launch_bounds__(kThreads) radix_hist_kernel(const uint32_t* __restrict__ keys, long long len,
                                                              int ntiles, int shift, uint32_t* __restrict__ hist) {
  PDL_ENTER();
  __shared__ uint32_t cnt[256];
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t* k = keys + (long long)blockIdx.y * len;
  const long long t0 = (long long)blockIdx.x * kTile;
#pragma unroll 4
  for (int i = threadIdx.x; i < kTile; i += kThreads) {
    const long long j = t0 + i;
    if (j < len) atomicAdd(&cnt[(k[j] >> shift) & 255u], 1u);
  }
  __syncthreads();
  hist[((long long)blockIdx.y * 256 + threadIdx.x) * ntiles + blockIdx.x] = cnt[threadIdx.x];
}

// in place: each (segment, digit) row of hist becomes its exclusive scan over the tiles; dtotal[s*256+d] = row sum.
// grid (256, nseg)
__global__ void __launch_bounds__(kThreads) radix_scan_kernel(uint32_t* __restrict__ hist, int ntiles,
                                                              uint32_t* __restrict__ dtotal) {
  PDL_ENTER();
  __shared__ uint32_t s_warp[kWarps];
  uint32_t* row = hist + ((long long)blockIdx.y * 256 + blockIdx.x) * ntiles;
  uint32_t carry = 0;
  for (int b = 0; b < ntiles; b += kThreads) {
    const int i = b + threadIdx.x;
    const uint32_t v = i < ntiles ? row[i] : 0u;
    uint32_t tot;
    const uint32_t ex = block_exclusive_scan(v, s_warp, &tot);
    if (i < ntiles) row[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) dtotal[(long long)blockIdx.y * 256 + blockIdx.x] = carry;
}

// stable scatter of one tile: destination = (pairs of smaller digits) + (this digit in earlier tiles) + rank within
// the tile.  Tile element order is (round, warp, lane), so ranks taken in that order keep the input order of ties.
// grid (ntiles, nseg)
__global__ void __launch_bounds__(kThreads) radix_scatter_kernel(const uint32_t* __restrict__ kin,
                                                                 const int32_t* __restrict__ vin,
                                                                 uint32_t* __restrict__ kout, int32_t* __restrict__ vout,
                                                                 long long len, int ntiles, int shift,
                                                                 const uint32_t* __restrict__ hist,
                                                                 const uint32_t* __restrict__ dtotal) {
  PDL_ENTER();
  __shared__ uint32_t s_warp[kWarps];
  __shared__ uint32_t dbase[256];
  __shared__ uint32_t wcnt[kWarps][256];     // this round's count of each digit per warp (zero between rounds)
  __shared__ uint32_t woff[kWarps][256];     // this round's destination of each digit's first pair per warp
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const long long seg = blockIdx.y;
  {
    uint32_t tot;
    const uint32_t ex = block_exclusive_scan(dtotal[seg * 256 + tid], s_warp, &tot);
    dbase[tid] = ex + hist[(seg * 256 + tid) * ntiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) wcnt[w][tid] = 0;
  }
  __syncthreads();
  const uint32_t* k = kin + seg * len;
  const int32_t* v = vin + seg * len;
  uint32_t* ko = kout + seg * len;
  int32_t* vo = vout + seg * len;
  const long long t0 = (long long)blockIdx.x * kTile;
  const unsigned lt_mask = (1u << lane) - 1u;
  for (int r = 0; r < kItems; ++r) {
    const long long j = t0 + (long long)r * kThreads + tid;
    const bool valid = j < len;
    uint32_t key = 0;
    int32_t val = 0;
    if (valid) {
      key = k[j];
      val = v[j];
    }
    const uint32_t digit = valid ? (key >> shift) & 255u : 256u;
    const unsigned peers = __match_any_sync(0xffffffffu, digit);
    const uint32_t rank = __popc(peers & lt_mask);
    if (valid && rank == 0) wcnt[wid][digit] = __popc(peers);
    __syncthreads();
    {
      uint32_t acc = dbase[tid];
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        const uint32_t c = wcnt[w][tid];
        woff[w][tid] = acc;
        acc += c;
        wcnt[w][tid] = 0;
      }
      dbase[tid] = acc;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = woff[wid][digit] + rank;
      ko[pos] = key;
      vo[pos] = val;
    }
  }
}

int64_t radix_sort_workspace(int nseg, long long len) {
  const long long nt = tiles_of(len);
  const size_t pairs = (size_t)nseg * (size_t)len;
  return (int64_t)(align256(pairs * 4) * 2 + align256((size_t)nseg * 256 * nt * 4) + align256((size_t)nseg * 256 * 4));
}

int radix_sort_pairs(const uint32_t* kin, const int32_t* vin, uint32_t* kout, int32_t* vout, int nseg, long long len,
                     void* ws, long long ws_bytes, cudaStream_t s) {
  B200_CHECK_ARG(nseg >= 1 && nseg <= 65535, "radix_sort: unsupported segment count %d", nseg);
  B200_CHECK_ARG(len >= 0 && len < (1LL << 31), "radix_sort: segment length %lld out of range", len);
  if (len == 0) return B200SEG_OK;
  B200_CHECK_ARG(ws && ws_bytes >= radix_sort_workspace(nseg, len), "radix_sort: workspace too small");
  const int nt = (int)tiles_of(len);
  const size_t pairs = (size_t)nseg * (size_t)len;
  char* p = static_cast<char*>(ws);
  uint32_t* ktmp = reinterpret_cast<uint32_t*>(p);
  p += align256(pairs * 4);
  int32_t* vtmp = reinterpret_cast<int32_t*>(p);
  p += align256(pairs * 4);
  uint32_t* hist = reinterpret_cast<uint32_t*>(p);
  p += align256((size_t)nseg * 256 * nt * 4);
  uint32_t* dtotal = reinterpret_cast<uint32_t*>(p);
  // in -> tmp -> out -> tmp -> out
  const uint32_t* ksrc[4] = {kin, ktmp, kout, ktmp};
  const int32_t* vsrc[4] = {vin, vtmp, vout, vtmp};
  uint32_t* kdst[4] = {ktmp, kout, ktmp, kout};
  int32_t* vdst[4] = {vtmp, vout, vtmp, vout};
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 8 * pass;
    launch_k(radix_hist_kernel, dim3(nt, nseg), kThreads, 0, s, ksrc[pass], len, nt, shift, hist);
    launch_k(radix_scan_kernel, dim3(256, nseg), kThreads, 0, s, hist, nt, dtotal);
    launch_k(radix_scatter_kernel, dim3(nt, nseg), kThreads, 0, s, ksrc[pass], vsrc[pass], kdst[pass], vdst[pass],
             len, nt, shift, (const uint32_t*)hist, (const uint32_t*)dtotal);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

// ------------------------------------------------------------------------------------------------ Lovasz-Softmax
// segment s: class c = s % C over voxels [b*len, (b+1)*len), b = s / C (b = 0 and len = N*vox without per_image)
__global__ void __launch_bounds__(kThreads) lovasz_keys_kernel(const float* __restrict__ z,
                                                               const long long* __restrict__ t, long long len, int C,
                                                               int has_ignore, long long ignore,
                                                               uint32_t* __restrict__ keys,
                                                               int32_t* __restrict__ vals) {
  PDL_ENTER();
  const int seg = blockIdx.y;
  const int c = seg % C;
  const long long p0 = (long long)(seg / C) * len;
  uint32_t* k = keys + (long long)seg * len;
  int32_t* v = vals + (long long)seg * len;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < len;
       j += (long long)gridDim.x * blockDim.x) {
    const long long P = p0 + j;
    const long long lbl = t[P];
    const float fg = lbl == c ? 1.f : 0.f;
    const float e = fabsf(fg - z[P * C + c]);            // lovasz.py:133, e >= 0 (or +NaN)
    k[j] = (has_ignore && lbl == ignore) ? kIgnoredKey : (~__float_as_uint(e)) & 0x7FFFFFFFu;
    v[j] = (int32_t)j;
  }
}

// tilecnt[s*ntiles + tile] = foreground pairs of the sorted tile
__global__ void __launch_bounds__(kThreads) lovasz_tilecnt_kernel(const uint32_t* __restrict__ keys,
                                                                  const int32_t* __restrict__ vals,
                                                                  const long long* __restrict__ t, long long len,
                                                                  int C, int ntiles, uint32_t* __restrict__ tilecnt) {
  PDL_ENTER();
  __shared__ unsigned long long s_tmp[kWarps];
  const int seg = blockIdx.y, c = seg % C;
  const long long p0 = (long long)(seg / C) * len;
  const uint32_t* k = keys + (long long)seg * len;
  const int32_t* v = vals + (long long)seg * len;
  const long long t0 = (long long)blockIdx.x * kTile;
  unsigned long long n = 0;
  for (int i = threadIdx.x; i < kTile; i += kThreads) {
    const long long j = t0 + i;
    if (j < len && k[j] != kIgnoredKey && t[p0 + v[j]] == c) ++n;
  }
  n = block_sum_u64(n, s_tmp);
  if (threadIdx.x == 0) tilecnt[(long long)seg * ntiles + blockIdx.x] = (uint32_t)n;
}

// Lovasz gradient of the sorted segment (lovasz.py:21-32) with exact integer counts: at sorted position i,
// cumfg = foreground in [0, i], cumbg = i + 1 - cumfg, J_i = 1 - (gts - cumfg) / (gts + cumbg), grad_i = J_i - J_{i-1}.
// Thread tid owns positions tile*kTile + tid*kItems + [0, kItems).
__global__ void __launch_bounds__(kThreads) lovasz_grad_kernel(const uint32_t* __restrict__ keys,
                                                               const int32_t* __restrict__ vals,
                                                               const long long* __restrict__ t, long long len, int C,
                                                               int ntiles, const uint32_t* __restrict__ tilecnt,
                                                               float* __restrict__ coef,
                                                               double* __restrict__ tileloss) {
  PDL_ENTER();
  __shared__ uint32_t s_warp[kWarps];
  __shared__ unsigned long long s_u[kWarps];
  __shared__ double s_d[kWarps];
  const int seg = blockIdx.y, c = seg % C;
  const long long p0 = (long long)(seg / C) * len;
  const uint32_t* k = keys + (long long)seg * len;
  const int32_t* v = vals + (long long)seg * len;
  const uint32_t* tc = tilecnt + (long long)seg * ntiles;
  unsigned long long before = 0, all = 0;
  for (int i = threadIdx.x; i < ntiles; i += kThreads) {
    const unsigned long long x = tc[i];
    all += x;
    if (i < (int)blockIdx.x) before += x;
  }
  before = block_sum_u64(before, s_u);
  const long long gts = (long long)block_sum_u64(all, s_u);
  const long long j0 = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kItems;
  uint32_t kk[kItems];
  int32_t vv[kItems];
  unsigned fgbits = 0;
  uint32_t mine = 0;
#pragma unroll
  for (int q = 0; q < kItems; ++q) {
    const long long j = j0 + q;
    kk[q] = kIgnoredKey;
    vv[q] = 0;
    if (j < len) {
      kk[q] = k[j];
      vv[q] = v[j];
      if (kk[q] != kIgnoredKey && t[p0 + vv[q]] == c) {
        fgbits |= 1u << q;
        ++mine;
      }
    }
  }
  uint32_t tot;
  const uint32_t ex = block_exclusive_scan(mine, s_warp, &tot);
  long long cum = (long long)before + ex;
  double acc = 0.0;
  const double g = (double)gts;
#pragma unroll
  for (int q = 0; q < kItems; ++q) {
    const long long j = j0 + q;
    if (j >= len) break;
    const int fg = (fgbits >> q) & 1;
    cum += fg;
    float grad = 0.f;
    if (kk[q] != kIgnoredKey && gts > 0) {
      const double cf = (double)cum, cp = (double)(cum - fg);
      const double Ji = 1.0 - (g - cf) / (g + ((double)(j + 1) - cf));
      const double Jp = 1.0 - (g - cp) / (g + ((double)j - cp));      // J_{-1} = 1 - gts/gts = 0
      const double gr = Ji - Jp;
      const float e = __uint_as_float(~kk[q] & 0x7FFFFFFFu);
      acc += (double)e * gr;
      grad = (float)gr;
    }
    coef[(p0 + vv[q]) * C + c] = grad;
  }
  acc = block_sum(acc, s_d);
  if (threadIdx.x == 0) tileloss[(long long)seg * ntiles + blockIdx.x] = acc;
}

// loss = mean over samples (nimg = N with per_image, else 1) of the mean over present classes; one block
__global__ void __launch_bounds__(kThreads) lovasz_finalize_kernel(const uint32_t* __restrict__ tilecnt,
                                                                   const double* __restrict__ tileloss, int nimg,
                                                                   int C, int ntiles, float* __restrict__ loss,
                                                                   float* __restrict__ seg_scale) {
  PDL_ENTER();
  __shared__ unsigned long long s_u[kWarps];
  __shared__ double s_d[kWarps];
  double total = 0.0;
  for (int b = 0; b < nimg; ++b) {
    double sum = 0.0;
    int K = 0;
    for (int c = 0; c < C; ++c) {
      const long long seg = (long long)b * C + c;
      unsigned long long n = 0;
      double l = 0.0;
      for (int i = threadIdx.x; i < ntiles; i += kThreads) {
        n += tilecnt[seg * ntiles + i];
        l += tileloss[seg * ntiles + i];
      }
      n = block_sum_u64(n, s_u);
      l = block_sum(l, s_d);
      if (n > 0) {
        sum += l;
        ++K;
      }
    }
    if (K > 0) total += sum / K;
    const float w = K > 0 ? (float)(1.0 / ((double)nimg * K)) : 0.f;
    for (int c = threadIdx.x; c < C; c += kThreads) {
      const long long seg = (long long)b * C + c;
      unsigned long long n = 0;
      for (int i = 0; i < ntiles; ++i) n += tilecnt[seg * ntiles + i];
      seg_scale[seg] = n > 0 ? w : 0.f;
    }
  }
  if (threadIdx.x == 0) loss[0] = (float)(total / nimg);
}

__global__ void __launch_bounds__(kThreads) lovasz_bwd_kernel(const float* __restrict__ z,
                                                              const long long* __restrict__ t, long long total, int C,
                                                              long long vox, int per_image,
                                                              const float* __restrict__ coef,
                                                              const float* __restrict__ seg_scale,
                                                              const float* __restrict__ gscale,
                                                              float* __restrict__ dz) {
  PDL_ENTER();
  const float gs = gscale[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long P = i / C;
    const int c = (int)(i - P * C);
    const long long seg = per_image ? (P / vox) * C + c : c;
    const float d = z[i] - (t[P] == c ? 1.f : 0.f);
    const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    dz[i] = gs * coef[i] * sg * seg_scale[seg];
  }
}

namespace {
struct LovaszLayout {
  int nseg, ntiles;
  long long len;
  size_t off_ka, off_va, off_kb, off_vb, off_sort, off_cnt, off_loss, bytes;
};

LovaszLayout lovasz_layout(int N, long long vox, int C, int per_image) {
  LovaszLayout L;
  L.nseg = per_image ? N * C : C;
  L.len = per_image ? vox : (long long)N * vox;
  L.ntiles = (int)tiles_of(L.len);
  const size_t pairs = (size_t)L.nseg * (size_t)L.len;
  size_t o = 0;
  L.off_ka = o; o += align256(pairs * 4);
  L.off_va = o; o += align256(pairs * 4);
  L.off_kb = o; o += align256(pairs * 4);
  L.off_vb = o; o += align256(pairs * 4);
  L.off_sort = o; o += (size_t)radix_sort_workspace(L.nseg, L.len);
  L.off_cnt = o; o += align256((size_t)L.nseg * L.ntiles * 4);
  L.off_loss = o; o += align256((size_t)L.nseg * L.ntiles * 8);
  L.bytes = o;
  return L;
}
}  // namespace

int64_t lovasz_workspace(int N, long long vox, int C, int per_image) {
  return (int64_t)lovasz_layout(N, vox, C, per_image).bytes;
}

int lovasz_fwd(const float* z, const long long* t, int N, long long vox, int C, int per_image, int has_ignore,
               long long ignore, void* ws, long long ws_bytes, float* loss, float* coef, float* seg_scale, int device,
               cudaStream_t s) {
  B200_CHECK_ARG(C >= 2 && C <= 1024, "lovasz: class count %d outside [2, 1024] (C == 1 is the sigmoid form)", C);
  B200_CHECK_ARG(N >= 1 && vox >= 1, "lovasz: empty batch");
  const LovaszLayout L = lovasz_layout(N, vox, C, per_image);
  B200_CHECK_ARG(L.len < (1LL << 31), "lovasz: a segment of %lld voxels (at most 2^31 - 1)", L.len);
  B200_CHECK_ARG(L.nseg <= 65535, "lovasz: %d class segments (at most 65535)", L.nseg);
  B200_CHECK_ARG(ws && (size_t)ws_bytes >= L.bytes, "lovasz: workspace too small");
  char* w = static_cast<char*>(ws);
  uint32_t* ka = reinterpret_cast<uint32_t*>(w + L.off_ka);
  int32_t* va = reinterpret_cast<int32_t*>(w + L.off_va);
  uint32_t* kb = reinterpret_cast<uint32_t*>(w + L.off_kb);
  int32_t* vb = reinterpret_cast<int32_t*>(w + L.off_vb);
  uint32_t* cnt = reinterpret_cast<uint32_t*>(w + L.off_cnt);
  double* tl = reinterpret_cast<double*>(w + L.off_loss);
  long long kb_x = (L.len + kThreads * 4 - 1) / (kThreads * 4);
  const long long cap = ((long long)num_sms(device) * 8 + L.nseg - 1) / L.nseg;
  if (kb_x > cap) kb_x = cap;
  if (kb_x < 1) kb_x = 1;
  launch_k(lovasz_keys_kernel, dim3((unsigned)kb_x, L.nseg), kThreads, 0, s, z, t, L.len, C, has_ignore, ignore, ka,
           va);
  B200_LAUNCH_CHECK();
  const int rc = radix_sort_pairs(ka, va, kb, vb, L.nseg, L.len, w + L.off_sort, (long long)(L.off_cnt - L.off_sort),
                                  s);
  if (rc != B200SEG_OK) return rc;
  const dim3 grid(L.ntiles, L.nseg);
  launch_k(lovasz_tilecnt_kernel, grid, kThreads, 0, s, (const uint32_t*)kb, (const int32_t*)vb, t, L.len, C, L.ntiles,
           cnt);
  launch_k(lovasz_grad_kernel, grid, kThreads, 0, s, (const uint32_t*)kb, (const int32_t*)vb, t, L.len, C, L.ntiles,
           (const uint32_t*)cnt, coef, tl);
  launch_k(lovasz_finalize_kernel, 1, kThreads, 0, s, (const uint32_t*)cnt, (const double*)tl, per_image ? N : 1, C,
           L.ntiles, loss, seg_scale);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int lovasz_bwd(const float* z, const long long* t, int N, long long vox, int C, int per_image, const float* coef,
               const float* seg_scale, const float* gscale, float* dz, int device, cudaStream_t s) {
  B200_CHECK_ARG(C >= 2 && N >= 1 && vox >= 1, "lovasz_bwd: bad shape");
  const long long total = (long long)N * vox * C;
  long long blocks = (total + kThreads * 4 - 1) / (kThreads * 4);
  const long long cap = (long long)num_sms(device) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_k(lovasz_bwd_kernel, (unsigned)blocks, kThreads, 0, s, z, t, total, C, vox, per_image, coef, seg_scale, gscale,
           dz);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
