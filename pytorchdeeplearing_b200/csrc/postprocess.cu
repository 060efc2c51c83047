// Mask post-processing of the reference's dataprocess/utils.py:7-66 (sm_90a): the largest face-connected component,
// binary morphology with ITK's ball, and the bounding box of label 1.  One (D, H, W) mask per call; a 2-D mask is
// D = 1.  Nothing is allocated or synchronised; every result is an integer, so reruns are bit-identical.
//
// Connected components (union-find; Playne & Hawick 2018, Allegretti, Bolelli & Grana 2019):
//   1. cc_local_kernel    one CTA per tile (32 x 4 x 4, or 32 x 16 when D == 1): union-find in shared memory over
//                         the tile's face neighbours; every foreground voxel gets the global linear index of the
//                         smallest voxel of its tile-local component, that root also the component's voxel count
//   2. cc_merge_kernel    the same tiles: each voxel on a low tile face joins the voxel across it in global memory
//                         (find, then an atomicMin that always hangs the larger root under the smaller)
//   3. cc_flatten_kernel  per voxel: label = final root; each tile-local root adds its count to the final root
//   4. cc_select_kernel   per block: max of (count, -root) over the roots and the number of roots
//   5. cc_finalize_kernel one block: the fixed-order reduction of the block partials -> {components, largest size}
//   6. cc_write_kernel    out = (label == chosen root)
// Links only ever point from a larger to a smaller index, so every root is its component's smallest linear index:
// the first voxel in C order, which is ITK's raster-order label and tie-break whatever order the atomics land in.
//
// Morphology: dilate(X) = {p : min over q in X of |p - q|^2 <= r^2 + r} (ITK's Ball of radius r has axes 2r + 1), as
// three separable passes over a uint16 squared distance: the nearest seed along x within r, then the windowed
// minimum of dy^2 + g along y and of dz^2 + g along z (|dy|, |dz| <= r; a window stops once d^2 reaches its best).
// Erosion is the complement of the dilation of the in-image background (outside the image is foreground);
// open = dilate(erode); close runs on a grid padded by r on each axis (outside is background), then crops.
//
// Box: per-block min / max / count over the voxels equal to 1, reduced by one block.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kTileVox = 512;            // voxels (= threads) per union-find tile
constexpr int kThreads = 256;            // per-voxel passes
constexpr int kSelectBlocks = 1024;      // block partials of the component selection and of the box
constexpr unsigned short kFar = 0xffffu; // no seed within r

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

__device__ __forceinline__ bool mask_nonzero(const void* p, int dt, long long i) {
  switch (dt) {
    case B200SEG_I64: return reinterpret_cast<const long long*>(p)[i] != 0;
    case B200SEG_I32: return reinterpret_cast<const int*>(p)[i] != 0;
    case B200SEG_I16: return reinterpret_cast<const short*>(p)[i] != 0;
    case B200SEG_F32: return reinterpret_cast<const float*>(p)[i] != 0.0f;     // NaN is nonzero, as in ITK's != 0
    default: return reinterpret_cast<const unsigned char*>(p)[i] != 0;
  }
}

__device__ __forceinline__ bool mask_is_one(const void* p, int dt, long long i) {
  switch (dt) {
    case B200SEG_I64: return reinterpret_cast<const long long*>(p)[i] == 1;
    case B200SEG_I32: return reinterpret_cast<const int*>(p)[i] == 1;
    case B200SEG_I16: return reinterpret_cast<const short*>(p)[i] == 1;
    default: return reinterpret_cast<const unsigned char*>(p)[i] == 1;
  }
}

// ---------------------------------------------------------------------------------------------- union-find helpers
__device__ __forceinline__ int find_s(const volatile int* s, int i) {
  int p = s[i];
  while (p != i) { i = p; p = s[i]; }
  return i;
}

__device__ __forceinline__ void union_s(int* s, int a, int b) {
  bool done = false;
  while (!done) {
    a = find_s(s, a);
    b = find_s(s, b);
    if (a < b) {
      const int old = atomicMin(&s[b], a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(&s[a], b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  }
}

// global forms: loads bypass L1, which other SMs' atomics do not keep coherent
__device__ __forceinline__ int find_g(const int* L, int i) {
  int p = __ldcg(L + i);
  while (p != i) { i = p; p = __ldcg(L + i); }
  return i;
}

__device__ __forceinline__ void union_g(int* L, int a, int b) {
  bool done = false;
  while (!done) {
    a = find_g(L, a);
    b = find_g(L, b);
    if (a < b) {
      const int old = atomicMin(&L[b], a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const int old = atomicMin(&L[a], b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  }
}

struct CcLayout {
  size_t label, size, part, best, bytes;
};

CcLayout cc_layout(long long V) {
  CcLayout L;
  size_t o = 0;
  L.label = o; o += align256((size_t)V * 4);
  L.size = o; o += align256((size_t)V * 4);
  L.part = o; o += align256((size_t)kSelectBlocks * 2 * 8);
  L.best = o; o += 256;
  L.bytes = o;
  return L;
}

struct Tile {
  int x, y, z;                   // voxel of this thread
  int x0, y0, z0;                // tile origin
};

template <int TY, int TZ>
__device__ __forceinline__ Tile tile_of(int H, int W) {
  const int tx = (W + 31) / 32, ty = (H + TY - 1) / TY;
  const int b = blockIdx.x;
  Tile t;
  t.x0 = (b % tx) * 32;
  t.y0 = ((b / tx) % ty) * TY;
  t.z0 = (b / tx / ty) * TZ;
  t.x = t.x0 + (threadIdx.x & 31);
  t.y = t.y0 + (threadIdx.x >> 5) % TY;
  t.z = t.z0 + threadIdx.x / (32 * TY);
  return t;
}

}  // namespace

// ------------------------------------------------------------------------------------------ 1. tile-local union-find
template <int TY, int TZ>
__global__ void __launch_bounds__(kTileVox) cc_local_kernel(const void* __restrict__ mask, int dt, int D, int H, int W,
                                                            int* __restrict__ label, int* __restrict__ size) {
  static_assert(32 * TY * TZ == kTileVox, "tile must hold kTileVox voxels");
  PDL_ENTER();
  __shared__ int s[kTileVox];
  __shared__ int cnt[kTileVox];
  const Tile t = tile_of<TY, TZ>(H, W);
  const int li = threadIdx.x;
  const bool in = t.x < W && t.y < H && t.z < D;
  const long long g = in ? ((long long)t.z * H + t.y) * W + t.x : 0;
  const bool fg = in && mask_nonzero(mask, dt, g);
  s[li] = fg ? li : -1;           // foreground entries stay >= 0, background stays -1
  cnt[li] = 0;
  __syncthreads();
  if (fg) {
    if ((li & 31) > 0 && s[li - 1] >= 0) union_s(s, li, li - 1);
    if ((li >> 5) % TY > 0 && s[li - 32] >= 0) union_s(s, li, li - 32);
    if (TZ > 1 && li >= 32 * TY && s[li - 32 * TY] >= 0) union_s(s, li, li - 32 * TY);
  }
  __syncthreads();
  const int r = fg ? find_s(s, li) : -1;
  if (fg) atomicAdd(&cnt[r], 1);
  __syncthreads();
  if (in) {
    int gl = -1;
    if (fg) {
      const int rx = t.x0 + (r & 31), ry = t.y0 + (r >> 5) % TY, rz = t.z0 + r / (32 * TY);
      gl = (int)(((long long)rz * H + ry) * W + rx);
    }
    label[g] = gl;
    size[g] = (fg && r == li) ? cnt[li] : 0;
  }
}

// ------------------------------------------------------------------------------------------ 2. merge across faces
template <int TY, int TZ>
__global__ void __launch_bounds__(kTileVox) cc_merge_kernel(int D, int H, int W, int* __restrict__ label) {
  PDL_ENTER();
  const Tile t = tile_of<TY, TZ>(H, W);
  if (t.x >= W || t.y >= H || t.z >= D) return;
  const bool fx = t.x == t.x0 && t.x > 0, fy = t.y == t.y0 && t.y > 0, fz = TZ > 1 && t.z == t.z0 && t.z > 0;
  if (!(fx || fy || fz)) return;
  const int g = (int)(((long long)t.z * H + t.y) * W + t.x);
  if (__ldcg(label + g) < 0) return;
  if (fx && __ldcg(label + g - 1) >= 0) union_g(label, g, g - 1);
  if (fy && __ldcg(label + g - W) >= 0) union_g(label, g, g - W);
  if (fz && __ldcg(label + g - H * W) >= 0) union_g(label, g, g - H * W);
}

// ------------------------------------------------------------------------------------------ 3. flatten + sizes
__global__ void __launch_bounds__(kThreads) cc_flatten_kernel(int V, int* __restrict__ label, int* __restrict__ size) {
  PDL_ENTER();
  for (long long j = (long long)blockIdx.x * kThreads + threadIdx.x; j < V; j += (long long)gridDim.x * kThreads) {
    const int i = (int)j;
    const int l = __ldcg(label + i);
    if (l < 0) continue;
    const int root = find_g(label, l);
    label[i] = root;                              // path compression to the final root: always an ancestor
    const int c = size[i];                        // nonzero only at tile-local roots; final roots receive, never give
    if (c > 0 && root != i) atomicAdd(&size[root], c);
  }
}

// ------------------------------------------------------------------------------------------ 4-5. choose the largest
__global__ void __launch_bounds__(kThreads) cc_select_kernel(int V, const int* __restrict__ label,
                                                             const int* __restrict__ size,
                                                             unsigned long long* __restrict__ part) {
  PDL_ENTER();
  __shared__ unsigned long long s_key[kThreads / 32], s_n[kThreads / 32];
  unsigned long long key = 0, n = 0;       // key = count << 32 | (2^31 - 1 - root): larger count, then smaller root
  for (long long j = (long long)blockIdx.x * kThreads + threadIdx.x; j < V; j += (long long)gridDim.x * kThreads) {
    const int i = (int)j;
    if (label[i] == i) {
      ++n;
      const unsigned long long k = ((unsigned long long)(unsigned)size[i] << 32) | (unsigned)(0x7fffffff - i);
      key = k > key ? k : key;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long k = __shfl_xor_sync(0xffffffffu, key, o);
    key = k > key ? k : key;
    n += __shfl_xor_sync(0xffffffffu, n, o);
  }
  if ((threadIdx.x & 31) == 0) { s_key[threadIdx.x >> 5] = key; s_n[threadIdx.x >> 5] = n; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) { key = s_key[w] > key ? s_key[w] : key; n += s_n[w]; }
    part[2 * blockIdx.x] = key;
    part[2 * blockIdx.x + 1] = n;
  }
}

__global__ void __launch_bounds__(32) cc_finalize_kernel(const unsigned long long* __restrict__ part, int nparts,
                                                         int* __restrict__ best, long long* __restrict__ stats) {
  PDL_ENTER();
  unsigned long long key = 0, n = 0;
  for (int b = threadIdx.x; b < nparts; b += 32) {
    key = part[2 * b] > key ? part[2 * b] : key;
    n += part[2 * b + 1];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long k = __shfl_xor_sync(0xffffffffu, key, o);
    key = k > key ? k : key;
    n += __shfl_xor_sync(0xffffffffu, n, o);
  }
  if (threadIdx.x == 0) {
    *best = n ? 0x7fffffff - (int)(key & 0xffffffffull) : -1;      // -1: no foreground, nothing is written as 1
    stats[0] = (long long)n;
    stats[1] = (long long)(key >> 32);
  }
}

__global__ void __launch_bounds__(kThreads) cc_write_kernel(int V, const int* __restrict__ label,
                                                            const int* __restrict__ best,
                                                            unsigned char* __restrict__ out) {
  PDL_ENTER();
  const int b = *best;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < V; i += (long long)gridDim.x * kThreads)
    out[i] = (b >= 0 && label[i] == b) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------ morphology
// pass x: g = (nearest seed along x within r)^2 over the domain (D, H, W); the source (sD, sH, sW) sits at offset
// (oz, oy, ox) inside it and is the only place seeds live; seed = (src != 0) != invert
__global__ void __launch_bounds__(kThreads) morph_row_kernel(const void* __restrict__ src, int dt, int sD, int sH,
                                                             int sW, int oz, int oy, int ox, int invert, int D, int H,
                                                             int W, int r, unsigned short* __restrict__ g) {
  PDL_ENTER();
  const long long V = (long long)D * H * W;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < V; i += (long long)gridDim.x * kThreads) {
    const int x = (int)(i % W);
    const long long zy = i / W;
    const int sy = (int)(zy % H) - oy, sz = (int)(zy / H) - oz;
    unsigned short v = kFar;
    if (sy >= 0 && sy < sH && sz >= 0 && sz < sD) {
      const long long row = ((long long)sz * sH + sy) * sW;
      const int sx = x - ox;
      for (int d = 0; d <= r; ++d) {
        const int a = sx - d, b = sx + d;
        if ((a >= 0 && a < sW && mask_nonzero(src, dt, row + a) != (invert != 0)) ||
            (b >= 0 && b < sW && mask_nonzero(src, dt, row + b) != (invert != 0))) {
          v = (unsigned short)(d * d);
          break;
        }
      }
    }
    g[i] = v;
  }
}

// passes y and z: g'(p) = min over |d| <= r of d^2 + g(p + d * step) along one axis of extent n at coordinate
// (i / step) % n.  FINAL: write out[(p - crop)] = (g' <= r^2 + r) != invert over the crop box (oD, oH, oW) at
// (cz, cy, cx) instead of g'.
template <bool FINAL>
__global__ void __launch_bounds__(kThreads) morph_line_kernel(const unsigned short* __restrict__ g, int D, int H,
                                                              int W, int axis, int r, unsigned short* __restrict__ gout,
                                                              int oD, int oH, int oW, int cz, int cy, int cx,
                                                              int invert, unsigned char* __restrict__ out) {
  PDL_ENTER();
  const long long step = axis == 1 ? (long long)W : (long long)W * H;
  const int n = axis == 1 ? H : D;
  const int lim = r * r + r;
  const long long V = (long long)oD * oH * oW;
  for (long long o = (long long)blockIdx.x * kThreads + threadIdx.x; o < V; o += (long long)gridDim.x * kThreads) {
    const int x = (int)(o % oW) + cx;
    const long long zy = o / oW;
    const int y = (int)(zy % oH) + cy, z = (int)(zy / oH) + cz;
    const long long i = ((long long)z * H + y) * W + x;
    const int c = axis == 1 ? y : z;
    int best = g[i];
    for (int d = 1; d <= r && d * d < best; ++d) {
      const int dd = d * d;
      if (c - d >= 0) { const int v = g[i - d * step]; if (v != kFar && v + dd < best) best = v + dd; }
      if (c + d < n) { const int v = g[i + d * step]; if (v != kFar && v + dd < best) best = v + dd; }
    }
    if (FINAL) out[o] = (unsigned char)((best <= lim) != (invert != 0));
    else gout[i] = (unsigned short)best;                 // <= 2 r^2 < kFar, or kFar
  }
}

// ------------------------------------------------------------------------------------------ box of label 1
__global__ void __launch_bounds__(kThreads) bbox_kernel(const void* __restrict__ mask, int dt, int D, int H, int W,
                                                        long long* __restrict__ part) {
  PDL_ENTER();
  __shared__ int s_lo[3], s_hi[3];
  __shared__ unsigned long long s_n;
  if (threadIdx.x < 3) { s_lo[threadIdx.x] = 0x7fffffff; s_hi[threadIdx.x] = -1; }
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  int lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1};       // x, y, z
  unsigned long long n = 0;
  const long long V = (long long)D * H * W;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < V; i += (long long)gridDim.x * kThreads) {
    if (!mask_is_one(mask, dt, i)) continue;
    const int c[3] = {(int)(i % W), (int)((i / W) % H), (int)(i / ((long long)W * H))};
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], c[a]); hi[a] = max(hi[a], c[a]); }
    ++n;
  }
  if (n) {
#pragma unroll
    for (int a = 0; a < 3; ++a) { atomicMin(&s_lo[a], lo[a]); atomicMax(&s_hi[a], hi[a]); }
    atomicAdd(&s_n, n);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long* p = part + 7 * blockIdx.x;
    for (int a = 0; a < 3; ++a) { p[a] = s_lo[a]; p[3 + a] = s_hi[a]; }
    p[6] = (long long)s_n;
  }
}

// box = {x0, y0, [z0,] sx, sy, [sz,] count}; all zero without a voxel equal to 1
__global__ void __launch_bounds__(32) bbox_finalize_kernel(const long long* __restrict__ part, int nparts, int dims,
                                                           long long* __restrict__ box) {
  PDL_ENTER();
  long long lo[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, hi[3] = {-1, -1, -1}, n = 0;
  for (int b = threadIdx.x; b < nparts; b += 32) {
    const long long* p = part + 7 * b;
#pragma unroll
    for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], p[a]); hi[a] = max(hi[a], p[3 + a]); }
    n += p[6];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
    n += __shfl_xor_sync(0xffffffffu, n, o);
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (a >= dims) break;
      box[a] = n ? lo[a] : 0;
      box[dims + a] = n ? hi[a] - lo[a] + 1 : 0;
    }
    box[2 * dims] = n;
  }
}

// ------------------------------------------------------------------------------------------ host side
namespace {

int grid_for(long long n, int dev) {
  const long long b = (n + kThreads - 1) / kThreads, cap = (long long)num_sms(dev) * 16;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

struct MorphLayout {
  int pD, pH, pW, pad;           // work domain (padded for close)
  size_t g1, g2, tmp, bytes;
};

MorphLayout morph_layout(int dims, int D, int H, int W, int r, int op) {
  MorphLayout L;
  L.pad = op == B200SEG_MORPH_CLOSE ? r : 0;
  L.pD = dims == 3 ? D + 2 * L.pad : D;
  L.pH = H + 2 * L.pad;
  L.pW = W + 2 * L.pad;
  const size_t nv = (size_t)L.pD * L.pH * L.pW;
  size_t o = 0;
  L.g1 = o; o += align256(nv * 2);
  L.g2 = o; o += align256(nv * 2);
  L.tmp = o; o += (op == B200SEG_MORPH_OPEN || op == B200SEG_MORPH_CLOSE) ? align256(nv) : 0;
  L.bytes = o;
  return L;
}

// one dilation of src's seeds over the domain (pD, pH, pW); the result (!= invert) lands on the crop box
// (oD, oH, oW) at (cz, cy, cx) of the domain, written densely to out
int dilate_pass(const void* src, int dt, int sD, int sH, int sW, int off, int dims, int invert, const MorphLayout& L,
                int r, unsigned short* g1, unsigned short* g2, int oD, int oH, int oW, int crop, unsigned char* out,
                int dev, cudaStream_t st) {
  const long long nv = (long long)L.pD * L.pH * L.pW, no = (long long)oD * oH * oW;
  const int oz = dims == 3 ? off : 0, cz = dims == 3 ? crop : 0;
  launch_k(morph_row_kernel, dim3(grid_for(nv, dev)), dim3(kThreads), 0, st, src, dt, sD, sH, sW, oz, off, off, invert,
           L.pD, L.pH, L.pW, r, g1);
  if (dims == 3) {
    launch_k(morph_line_kernel<false>, dim3(grid_for(nv, dev)), dim3(kThreads), 0, st, (const unsigned short*)g1,
             L.pD, L.pH, L.pW, 1, r, g2, L.pD, L.pH, L.pW, 0, 0, 0, 0, (unsigned char*)nullptr);
    launch_k(morph_line_kernel<true>, dim3(grid_for(no, dev)), dim3(kThreads), 0, st, (const unsigned short*)g2, L.pD,
             L.pH, L.pW, 2, r, (unsigned short*)nullptr, oD, oH, oW, cz, crop, crop, invert, out);
  } else {
    launch_k(morph_line_kernel<true>, dim3(grid_for(no, dev)), dim3(kThreads), 0, st, (const unsigned short*)g1, L.pD,
             L.pH, L.pW, 1, r, (unsigned short*)nullptr, oD, oH, oW, 0, crop, crop, invert, out);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace

long long components_workspace(int D, int H, int W) { return (long long)cc_layout((long long)D * H * W).bytes; }

int largest_component(const void* mask, int dt, int D, int H, int W, void* ws, unsigned char* out, long long* stats,
                      int dev, cudaStream_t st) {
  const long long V = (long long)D * H * W;
  const CcLayout L = cc_layout(V);
  char* base = static_cast<char*>(ws);
  int* label = reinterpret_cast<int*>(base + L.label);
  int* size = reinterpret_cast<int*>(base + L.size);
  unsigned long long* part = reinterpret_cast<unsigned long long*>(base + L.part);
  int* best = reinterpret_cast<int*>(base + L.best);
  const int tx = (W + 31) / 32;
  if (D == 1) {                  // 32 x 16 tiles
    const int nt = tx * ((H + 15) / 16);
    launch_k(cc_local_kernel<16, 1>, dim3(nt), dim3(kTileVox), 0, st, mask, dt, D, H, W, label, size);
    launch_k(cc_merge_kernel<16, 1>, dim3(nt), dim3(kTileVox), 0, st, D, H, W, label);
  } else {                       // 32 x 4 x 4 tiles
    const int nt = tx * ((H + 3) / 4) * ((D + 3) / 4);
    launch_k(cc_local_kernel<4, 4>, dim3(nt), dim3(kTileVox), 0, st, mask, dt, D, H, W, label, size);
    launch_k(cc_merge_kernel<4, 4>, dim3(nt), dim3(kTileVox), 0, st, D, H, W, label);
  }
  const int g = grid_for(V, dev), nsel = g < kSelectBlocks ? g : kSelectBlocks;
  launch_k(cc_flatten_kernel, dim3(g), dim3(kThreads), 0, st, (int)V, label, size);
  launch_k(cc_select_kernel, dim3(nsel), dim3(kThreads), 0, st, (int)V, (const int*)label, (const int*)size, part);
  launch_k(cc_finalize_kernel, dim3(1), dim3(32), 0, st, (const unsigned long long*)part, nsel, best, stats);
  launch_k(cc_write_kernel, dim3(g), dim3(kThreads), 0, st, (int)V, (const int*)label, (const int*)best, out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

long long morphology_workspace(int dims, int D, int H, int W, int r, int op) {
  return (long long)morph_layout(dims, D, H, W, r, op).bytes;
}

long long morphology_voxels(int dims, int D, int H, int W, int r, int op) {
  const MorphLayout L = morph_layout(dims, D, H, W, r, op);
  return (long long)L.pD * L.pH * L.pW;
}

int morphology(const void* mask, int dt, int dims, int D, int H, int W, int r, int op, void* ws, unsigned char* out,
               int dev, cudaStream_t st) {
  const MorphLayout L = morph_layout(dims, D, H, W, r, op);
  char* base = static_cast<char*>(ws);
  unsigned short* g1 = reinterpret_cast<unsigned short*>(base + L.g1);
  unsigned short* g2 = reinterpret_cast<unsigned short*>(base + L.g2);
  unsigned char* tmp = reinterpret_cast<unsigned char*>(base + L.tmp);
  switch (op) {
    case B200SEG_MORPH_DILATE:
      return dilate_pass(mask, dt, D, H, W, 0, dims, 0, L, r, g1, g2, D, H, W, 0, out, dev, st);
    case B200SEG_MORPH_ERODE:
      return dilate_pass(mask, dt, D, H, W, 0, dims, 1, L, r, g1, g2, D, H, W, 0, out, dev, st);
    case B200SEG_MORPH_OPEN: {
      const int rc = dilate_pass(mask, dt, D, H, W, 0, dims, 1, L, r, g1, g2, D, H, W, 0, tmp, dev, st);
      if (rc != B200SEG_OK) return rc;
      return dilate_pass(tmp, B200SEG_U8, D, H, W, 0, dims, 0, L, r, g1, g2, D, H, W, 0, out, dev, st);
    }
    default: {                   // close: dilate into the padded grid, erode it, keep the image's box
      const int rc = dilate_pass(mask, dt, D, H, W, L.pad, dims, 0, L, r, g1, g2, L.pD, L.pH, L.pW, 0, tmp, dev, st);
      if (rc != B200SEG_OK) return rc;
      return dilate_pass(tmp, B200SEG_U8, L.pD, L.pH, L.pW, 0, dims, 1, L, r, g1, g2, D, H, W, L.pad, out, dev, st);
    }
  }
}

long long label_bbox_workspace() { return (long long)kSelectBlocks * 7 * 8; }

int label_bbox(const void* mask, int dt, int dims, int D, int H, int W, void* ws, long long* box, int dev,
               cudaStream_t st) {
  const long long V = (long long)D * H * W;
  const int g = grid_for(V, dev), nb = g < kSelectBlocks ? g : kSelectBlocks;
  long long* part = static_cast<long long*>(ws);
  launch_k(bbox_kernel, dim3(nb), dim3(kThreads), 0, st, mask, dt, D, H, W, part);
  launch_k(bbox_finalize_kernel, dim3(1), dim3(32), 0, st, (const long long*)part, nb, dims, box);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
