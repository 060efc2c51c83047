// HBM-bound elementwise / reduction kernels of the hot path (sm_90a): weight (un)packing, the
// GroupNorm finalize / apply split, GroupNorm+ReLU+Dropout backward (two-pass: per-(n,c) sums,
// then dy = g*P + y*Q + R), bias column sums, 2x max-pooling, head sigmoid/softmax.
//
// All activation kernels use 128-bit accesses along the channel dimension of the NDHWC layout
// (VEC = 8 bf16 / 4 fp32 channels per thread); the grid is sized so that a thread's channel group
// never changes across its grid-stride loop, hence the per-(n,c) coefficients live in registers.
#include <string.h>

#include "common.cuh"
#include "gn_coef.cuh"

namespace b200seg {

// ---------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------
template <typename TO>
__global__ void pack_weight_kernel(const float* __restrict__ w, TO* __restrict__ out, int T, int K, int N2, int N1,
                                   long long st, long long sk, long long sn2, long long sn1, int flip) {
  PDL_ENTER();
  long long total = (long long)T * K * N2 * N1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int n1 = (int)(i % N1);
    long long r = i / N1;
    int n2 = (int)(r % N2);
    r /= N2;
    int k = (int)(r % K);
    int t = (int)(r / K);
    int ts = flip ? (T - 1 - t) : t;
    out[i] = from_f<TO>(w[ts * st + k * sk + n2 * sn2 + n1 * sn1]);
  }
}

__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, float* __restrict__ grad, int T, int K, int N,
                                    long long st, long long sk, long long sn) {
  PDL_ENTER();
  // iterate in DESTINATION order when the destination's fastest index is t (st == 1): coalesced writes
  long long total = (long long)T * K * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int n = (int)(i % N);
    long long r = i / N;
    int k = (int)(r % K);
    int t = (int)(r / K);
    grad[t * st + k * sk + n * sn] = dwp[i];
  }
}

// Multi-tensor forms: one launch (re)packs every conv operand of a network / unpacks every weight gradient.
// Each descriptor owns a contiguous range of thread blocks; a block finds its descriptor by binary search.
struct PackDesc {            // mirrors b200seg_pack_desc (include/b200seg.h)
  const float* src;
  void* dst;
  long long st, sk, sn2, sn1;
  int out_dtype, T, K, N2, N1, flip;
  int block_start, nblocks;
};

constexpr int kPackCols = 64;        // columns (k, n2, n1) staged per tile in the tap-contiguous paths
constexpr int kPackMaxT = 27;
constexpr int kPackIters = 8;        // column trips per warp and tile (8 warps, >= 1 column per trip)

// descriptor owning this block: the block_start column is staged in shared memory with one round of loads
__device__ __forceinline__ int pack_find_desc(const PackDesc* __restrict__ table, int count, int* s_start) {
  int lo = 0, hi = count - 1;
  if (count <= 1024) {
    for (int i = threadIdx.x; i < count; i += blockDim.x) s_start[i] = table[i].block_start;
    __syncthreads();
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_start[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    return lo;
  }
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].block_start <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(256) pack_multi_kernel(const PackDesc* __restrict__ table, int count) {
  PDL_ENTER();
  __shared__ float s_tile[kPackMaxT][kPackCols + 1];
  __shared__ long long s_col[kPackCols];
  __shared__ int s_start[1024];
  const PackDesc d = table[pack_find_desc(table, count, s_start)];
  const int b = blockIdx.x - d.block_start;
  if (d.st == 1 && d.T > 1 && d.T <= kPackMaxT) {
    // torch conv weights keep the taps contiguous ([co][ci][taps]): a warp reads whole tap runs (32/T columns per
    // trip, lane = (column, tap)), the tile is transposed through shared memory and the destination rows
    // [t][cols] are written with unit stride.  All index arithmetic is 32-bit and per column, not per element.
    const int T = d.T;
    const int J = d.K * d.N2 * d.N1;                                  // destination columns
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cpw = 32 / T;                                            // columns per warp trip
    const int sc = lane / T, ts = lane - sc * T;
    for (int j0 = b * kPackCols; j0 < J; j0 += d.nblocks * kPackCols) {
      const int ncol = J - j0 < kPackCols ? J - j0 : kPackCols;
      // source offset of every column of the tile: decoded once per column (the divisions), not once per element
      if ((int)threadIdx.x < ncol) {
        const int j = j0 + threadIdx.x;
        const int n1 = j % d.N1;
        const int r = j / d.N1;
        const int n2 = r % d.N2;
        const int k = r / d.N2;
        s_col[threadIdx.x] = k * d.sk + n2 * d.sn2 + n1 * d.sn1;
      }
      __syncthreads();
      // all of a warp's column trips are loaded before the first shared-memory store (one latency, not eight)
      float v[kPackIters];
#pragma unroll
      for (int i = 0; i < kPackIters; ++i) {
        const int jl = warp * cpw + sc + i * 8 * cpw;
        v[i] = 0.f;
        if (sc < cpw && jl < ncol) v[i] = d.src[ts + s_col[jl]];
      }
#pragma unroll
      for (int i = 0; i < kPackIters; ++i) {
        const int jl = warp * cpw + sc + i * 8 * cpw;
        if (sc < cpw && jl < ncol) s_tile[d.flip ? T - 1 - ts : ts][jl] = v[i];
      }
      __syncthreads();
      if (ncol == kPackCols) {
        for (int idx = threadIdx.x; idx < kPackCols * T; idx += blockDim.x) {
          const int t = idx / kPackCols, jl = idx % kPackCols;
          const float v = s_tile[t][jl];
          const long long o = (long long)t * J + j0 + jl;
          if (d.out_dtype == B200SEG_BF16) static_cast<bf16*>(d.dst)[o] = __float2bfloat16_rn(v);
          else static_cast<float*>(d.dst)[o] = v;
        }
      } else {
        for (int idx = threadIdx.x; idx < ncol * T; idx += blockDim.x) {
          const int t = idx / ncol, jl = idx - t * ncol;
          const float v = s_tile[t][jl];
          const long long o = (long long)t * J + j0 + jl;
          if (d.out_dtype == B200SEG_BF16) static_cast<bf16*>(d.dst)[o] = __float2bfloat16_rn(v);
          else static_cast<float*>(d.dst)[o] = v;
        }
      }
      __syncthreads();
    }
    return;
  }
  const long long total = (long long)d.T * d.K * d.N2 * d.N1;
  for (long long i = b * 256LL + threadIdx.x; i < total; i += (long long)d.nblocks * 256) {
    const int n1 = (int)(i % d.N1);
    long long r = i / d.N1;
    const int n2 = (int)(r % d.N2);
    r /= d.N2;
    const int k = (int)(r % d.K);
    const int t = (int)(r / d.K);
    const int ts = d.flip ? (d.T - 1 - t) : t;
    const float v = d.src[ts * d.st + k * d.sk + n2 * d.sn2 + n1 * d.sn1];
    if (d.out_dtype == B200SEG_BF16) static_cast<bf16*>(d.dst)[i] = __float2bfloat16_rn(v);
    else static_cast<float*>(d.dst)[i] = v;
  }
}

// unpack: dst[t*st + k*sk + n*sn2] = src[(t*K + k)*N2 + n]   (N1 unused = 1)
__global__ void __launch_bounds__(256) unpack_multi_kernel(const PackDesc* __restrict__ table, int count) {
  PDL_ENTER();
  __shared__ float s_tile[kPackMaxT][kPackCols + 1];
  __shared__ long long s_col[kPackCols];
  __shared__ int s_start[1024];
  const PackDesc d = table[pack_find_desc(table, count, s_start)];
  const int b = blockIdx.x - d.block_start;
  float* out = static_cast<float*>(d.dst);
  if (d.st == 1 && d.T > 1 && d.T <= kPackMaxT) {
    // source rows [t][cols] are read with unit stride; a warp then writes whole tap runs of the torch gradient
    const int T = d.T;
    const int J = d.K * d.N2;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cpw = 32 / T;
    const int sc = lane / T, ts = lane - sc * T;
    for (int j0 = b * kPackCols; j0 < J; j0 += d.nblocks * kPackCols) {
      const int ncol = J - j0 < kPackCols ? J - j0 : kPackCols;
      if (ncol == kPackCols) {
        constexpr int NR = (kPackCols * kPackMaxT + 255) / 256;      // 7 row trips, all loads first
        float v[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) {
          const int idx = threadIdx.x + i * 256;
          v[i] = idx < kPackCols * T ? d.src[(long long)(idx / kPackCols) * J + j0 + (idx % kPackCols)] : 0.f;
        }
#pragma unroll
        for (int i = 0; i < NR; ++i) {
          const int idx = threadIdx.x + i * 256;
          if (idx < kPackCols * T) s_tile[idx / kPackCols][idx % kPackCols] = v[i];
        }
      } else {
        for (int idx = threadIdx.x; idx < ncol * T; idx += blockDim.x) {
          const int t = idx / ncol, jl = idx - t * ncol;
          s_tile[t][jl] = d.src[(long long)t * J + j0 + jl];
        }
      }
      if ((int)threadIdx.x < ncol) {
        const int j = j0 + threadIdx.x;
        s_col[threadIdx.x] = (j / d.N2) * d.sk + (j % d.N2) * d.sn2;
      }
      __syncthreads();
      for (int jl = warp * cpw + sc; jl < ncol; jl += 8 * cpw)
        if (sc < cpw) out[ts + s_col[jl]] = s_tile[ts][jl];
      __syncthreads();
    }
    return;
  }
  const long long total = (long long)d.T * d.K * d.N2;
  for (long long i = b * 256LL + threadIdx.x; i < total; i += (long long)d.nblocks * 256) {
    const int n = (int)(i % d.N2);
    const long long r = i / d.N2;
    const int k = (int)(r % d.K);
    const int t = (int)(r / d.K);
    out[t * d.st + k * d.sk + n * d.sn2] = d.src[i];
  }
}

// Descriptor tables reach the device as KERNEL ARGUMENTS (<= 3968 bytes per launch), not through a host-to-device
// memcpy: a memcpy node inside the step's CUDA graph queues on the copy engine behind the application's own input
// prefetch (tens of MB per step) and stalls the whole graph for the duration of that transfer.
struct TableChunk {
  unsigned char b[3968];
};
__global__ void table_write_kernel(const __grid_constant__ TableChunk c, unsigned char* __restrict__ dst, int n) {
  PDL_ENTER();
  for (int i = threadIdx.x * 16; i < n; i += blockDim.x * 16)
    *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(c.b + i);
}

int ew_upload_table(const void* host, long long bytes, void* dev_dst, cudaStream_t s) {
  B200_CHECK_ARG((bytes % 16) == 0 && (reinterpret_cast<uintptr_t>(dev_dst) % 16) == 0,
                 "upload_table: size and destination must be multiples of 16 bytes");
  const unsigned char* src = static_cast<const unsigned char*>(host);
  unsigned char* dst = static_cast<unsigned char*>(dev_dst);
  for (long long off = 0; off < bytes; off += (long long)sizeof(TableChunk)) {
    const int n = (int)((bytes - off) < (long long)sizeof(TableChunk) ? (bytes - off) : (long long)sizeof(TableChunk));
    TableChunk c;
    memcpy(c.b, src + off, (size_t)n);
    launch_k(table_write_kernel, 1, 256, 0, s, c, dst + off, n);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_pack_multi(const void* table_dev, int count, int total_blocks, int unpack, cudaStream_t s) {
  if (count <= 0 || total_blocks <= 0) return B200SEG_OK;
  if (unpack) launch_k(unpack_multi_kernel, total_blocks, 256, 0, s, static_cast<const PackDesc*>(table_dev), count);
  else launch_k(pack_multi_kernel, total_blocks, 256, 0, s, static_cast<const PackDesc*>(table_dev), count);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

// ---------------------------------------------------------------------------------------------
// GroupNorm finalize: stats (double sum, sumsq per (n,c)) -> A,B per (n,c); mean,rstd per (n,g)
// ---------------------------------------------------------------------------------------------
__global__ void gn_finalize_kernel(const double* __restrict__ stats, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, const float* __restrict__ scale, int C, int groups,
                                   double m, float eps, float* __restrict__ coef, float* __restrict__ mr) {
  PDL_ENTER();
  const int n = blockIdx.x;
  const int cpg = C / groups;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    int g = c / cpg;
    double s = 0.0, q = 0.0;
    for (int j = 0; j < cpg; ++j) {
      const double* p = stats + ((long long)n * C + g * cpg + j) * 2;
      s += p[0];
      q += p[1];
    }
    double mean, rstd;
    gn_mean_rstd(s, q, m, eps, mean, rstd);
    double sc = scale ? (double)scale[(long long)n * C + c] : 1.0;
    double ga = gamma[c], be = beta[c];
    coef[((long long)n * C + c) * 2 + 0] = (float)gn_a(rstd, ga, sc);
    coef[((long long)n * C + c) * 2 + 1] = (float)gn_b(mean, rstd, ga, be, sc);
    if (c == g * cpg) {
      mr[((long long)n * groups + g) * 2 + 0] = (float)mean;
      mr[((long long)n * groups + g) * 2 + 1] = (float)rstd;
    }
  }
}


// ---------------------------------------------------------------------------------------------
// vector helpers: VEC channels of type T <-> float[VEC]
// ---------------------------------------------------------------------------------------------
template <typename T, int VEC> struct Vec;
template <> struct Vec<float, 4> {
  static __device__ __forceinline__ void load(const float* p, float* o) {
    float4 v = *reinterpret_cast<const float4*>(p);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct Vec<bf16, 8> {
  static __device__ __forceinline__ void load(const bf16* p, float* o) { load8(p, o); }
  static __device__ __forceinline__ void store(bf16* p, const float* v) { store8(p, v); }
};
template <typename T> struct Vec<T, 1> {
  static __device__ __forceinline__ void load(const T* p, float* o) { o[0] = to_f(*p); }
  static __device__ __forceinline__ void store(T* p, const float* v) { *p = from_f<T>(v[0]); }
};

// Common indexing: grid = (blocks, N); a thread walks "groups" (voxel, channel-group) of sample n with
// stride gridDim.x*blockDim.x, which the host makes a multiple of G = C/VEC.
#define EW_PROLOGUE(Cval)                                                        \
  const int n = blockIdx.y;                                                      \
  const int G = (Cval) / VEC;                                                    \
  const long long total = V * G;                                                 \
  const long long stride = (long long)gridDim.x * blockDim.x;                    \
  long long gi = blockIdx.x * (long long)blockDim.x + threadIdx.x;               \
  const int cg = (int)(gi % G);                                                  \
  const int c0 = cg * VEC;                                                       \
  long long vi = gi / G;            /* voxel of the first group of this thread */ \
  const long long vstep = stride / G; /* stride is a multiple of G */          \
  (void)total;

template <typename T, int VEC, int ACT>
__global__ void __launch_bounds__(256, 3) apply_kernel(const T* __restrict__ y1, long long ld1,
                                                    const float* __restrict__ coef1, const T* __restrict__ y2,
                                                    long long ld2, const float* __restrict__ coef2,
                                                    const T* __restrict__ res, long long ldr, T* __restrict__ out,
                                                    long long ldo, int C, long long V, const GnRef gn1,
                                                    const GnRef gn2) {
  PDL_ENTER();
  EW_PROLOGUE(C)
  float A1[VEC], B1[VEC], A2[VEC], B2[VEC];
  if (gn1.stats != nullptr) {
    // coefficients once per CTA (block-cooperative), then broadcast through shared memory
    extern __shared__ double s_dyn[];
    double* s_d = s_dyn;                                                  // scratch doubles
    float* s_f = reinterpret_cast<float*>(s_d + gn_cta_doubles(C, gn1.groups > gn2.groups ? gn1.groups : gn2.groups, false));
    float* s_cf = s_f + 3 * C;                                            // [4][C]: A1, B1, A2, B2
    gn_coefs<false, true, GnCta, ACT != B200SEG_ACT_RELU>(GnCta(), gn1, nullptr, n, C, s_d, s_f, s_cf, s_cf + C, nullptr, nullptr, nullptr);
    if (y2 != nullptr)
      gn_coefs<false, true, GnCta, ACT != B200SEG_ACT_RELU>(GnCta(), gn2, nullptr, n, C, s_d, s_f, s_cf + 2 * C, s_cf + 3 * C, nullptr, nullptr,
                            nullptr);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      A1[j] = s_cf[c0 + j];
      B1[j] = s_cf[C + c0 + j];
      A2[j] = y2 != nullptr ? s_cf[2 * C + c0 + j] : 0.f;
      B2[j] = y2 != nullptr ? s_cf[3 * C + c0 + j] : 0.f;
    }
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float* p = coef1 + ((long long)n * C + c0 + j) * 2;
      A1[j] = p[0];
      B1[j] = p[1];
      if (y2 != nullptr) {
        const float* q = coef2 + ((long long)n * C + c0 + j) * 2;
        A2[j] = q[0];
        B2[j] = q[1];
      } else {
        A2[j] = 0.f;
        B2[j] = 0.f;
      }
    }
  }
  // two trips of loads in flight per thread (the grid is sized to the resident CTAs, see ew_apply)
  const long long nb = (long long)n * V;
  for (; vi + vstep < V; vi += 2 * vstep) {
    const long long v0 = nb + vi, v1 = v0 + vstep;
    float a0[VEC], a1[VEC], o0[VEC], o1[VEC];
    Vec<T, VEC>::load(y1 + v0 * ld1 + c0, a0);
    Vec<T, VEC>::load(y1 + v1 * ld1 + c0, a1);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      o0[j] = gn_act<ACT>(fmaf(a0[j], A1[j], B1[j]));
      o1[j] = gn_act<ACT>(fmaf(a1[j], A1[j], B1[j]));
    }
    if (y2 != nullptr) {
      Vec<T, VEC>::load(y2 + v0 * ld2 + c0, a0);
      Vec<T, VEC>::load(y2 + v1 * ld2 + c0, a1);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        o0[j] += gn_act<ACT>(fmaf(a0[j], A2[j], B2[j]));
        o1[j] += gn_act<ACT>(fmaf(a1[j], A2[j], B2[j]));
      }
    }
    if (res != nullptr) {
      Vec<T, VEC>::load(res + v0 * ldr + c0, a0);
      Vec<T, VEC>::load(res + v1 * ldr + c0, a1);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        o0[j] += a0[j];
        o1[j] += a1[j];
      }
    }
    Vec<T, VEC>::store(out + v0 * ldo + c0, o0);
    Vec<T, VEC>::store(out + v1 * ldo + c0, o1);
  }
  if (vi < V) {
    const long long vox = nb + vi;
    float a[VEC], o[VEC];
    Vec<T, VEC>::load(y1 + vox * ld1 + c0, a);
#pragma unroll
    for (int j = 0; j < VEC; ++j) o[j] = gn_act<ACT>(fmaf(a[j], A1[j], B1[j]));
    if (y2 != nullptr) {
      Vec<T, VEC>::load(y2 + vox * ld2 + c0, a);
#pragma unroll
      for (int j = 0; j < VEC; ++j) o[j] += gn_act<ACT>(fmaf(a[j], A2[j], B2[j]));
    }
    if (res != nullptr) {
      Vec<T, VEC>::load(res + vox * ldr + c0, a);
#pragma unroll
      for (int j = 0; j < VEC; ++j) o[j] += a[j];
    }
    Vec<T, VEC>::store(out + vox * ldo + c0, o);
  }
}

// sums[n][c] += { sum g*m, sum g*m*y, sum y }, m = [y*A + B > 0]
// The projection coefficients of the GroupNorm backward are means of these sums.  A thread's own partial (a few
// dozen voxels) and the fold over the lanes of a warp that share its channel group run in fp32; everything after
// that -- across the 8 warps, across CTAs -- is accumulated in fp64 in a fixed order (one private shared-memory
// row per warp, then ONE fp64 global atomic per (channel, sum) per CTA).  The grid is sized to the resident CTAs
// (3 per SM) and the voxel loop keeps two trips of loads in flight: the kernel is a pure HBM stream.
template <typename T, int VEC, bool DEEP, int ACT>
__global__ void __launch_bounds__(256, DEEP ? 2 : 3) gn_bwd_reduce_kernel(const T* __restrict__ g, long long ldg,
                                                               const T* __restrict__ y, long long ldy,
                                                               const float* __restrict__ coef,
                                                               double* __restrict__ sums, int C, long long V,
                                                               const GnRef gn, const int staged) {
  PDL_ENTER();
  EW_PROLOGUE(C)
  // dynamic smem: doubles [3][C] accumulators (unstaged path) | coefficient scratch; then floats: scratch [3][C],
  // A/B [2][C], staging [8 warps][3][C] (if staged)
  extern __shared__ double s_redd[];
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) s_redd[i] = 0.0;
  double* s_cd = s_redd + 3 * C;
  float* s_cfl = reinterpret_cast<float*>(s_cd + gn_cta_doubles(C, gn.groups, false));
  float* s_ab = s_cfl + 3 * C;                                            // [2][C]
  float* s_part = s_ab + 2 * C;                                           // [8][3][C]
  float A[VEC], B[VEC];
  float f1[VEC], f2[VEC], f3[VEC];
  if (gn.stats != nullptr) {
    gn_coefs<false, true, GnCta, ACT != B200SEG_ACT_RELU>(GnCta(), gn, nullptr, n, C, s_cd, s_cfl, s_ab, s_ab + C, nullptr, nullptr, nullptr);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      A[j] = s_ab[c0 + j];
      B[j] = s_ab[C + c0 + j];
    }
  } else {
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    if (gn.stats == nullptr) {
      const float* p = coef + ((long long)n * C + c0 + j) * 2;
      A[j] = p[0];
      B[j] = p[1];
    }
    f1[j] = f2[j] = f3[j] = 0.f;
  }
  const T* yb = y + (long long)n * V * ldy + c0;
  const T* gb = g + (long long)n * V * ldg + c0;
  if constexpr (DEEP) {
    // four trips (eight 16-byte loads) in flight per thread: at two CTAs per SM that is 64 KB per SM on the wire,
    // which is what it takes to keep HBM busy at ~1 us latency (the two-trip loop alone stalls at ~3.3 TB/s)
    for (; vi + 3 * vstep < V; vi += 4 * vstep) {
      float ya[4][VEC], ga[4][VEC];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        Vec<T, VEC>::load(yb + (vi + u * vstep) * ldy, ya[u]);
        Vec<T, VEC>::load(gb + (vi + u * vstep) * ldg, ga[u]);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float d = gn_act_bwd<ACT>(fmaf(ya[u][j], A[j], B[j]), ga[u][j]);
          f1[j] += d;
          f2[j] = fmaf(d, ya[u][j], f2[j]);
          f3[j] += ya[u][j];
        }
    }
  }
  for (; vi + vstep < V; vi += 2 * vstep) {
    float y0[VEC], g0[VEC], y1[VEC], g1[VEC];
    Vec<T, VEC>::load(yb + vi * ldy, y0);
    Vec<T, VEC>::load(gb + vi * ldg, g0);
    Vec<T, VEC>::load(yb + (vi + vstep) * ldy, y1);
    Vec<T, VEC>::load(gb + (vi + vstep) * ldg, g1);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float d0 = gn_act_bwd<ACT>(fmaf(y0[j], A[j], B[j]), g0[j]);
      const float d1 = gn_act_bwd<ACT>(fmaf(y1[j], A[j], B[j]), g1[j]);
      f1[j] += d0 + d1;
      f2[j] = fmaf(d0, y0[j], fmaf(d1, y1[j], f2[j]));
      f3[j] += y0[j] + y1[j];
    }
  }
  if (vi < V) {
    float yv[VEC], gv[VEC];
    Vec<T, VEC>::load(yb + vi * ldy, yv);
    Vec<T, VEC>::load(gb + vi * ldg, gv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float d = gn_act_bwd<ACT>(fmaf(yv[j], A[j], B[j]), gv[j]);
      f1[j] += d;
      f2[j] = fmaf(d, yv[j], f2[j]);
      f3[j] += yv[j];
    }
  }
  // lanes l and l ^ off share the channel group when off is a multiple of G (G a power of two <= 16)
  const bool pow2 = (G & (G - 1)) == 0;
  const int lane_groups = (pow2 && G < 32) ? G : 32;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (staged) {
    if (lane_groups < 32) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        for (int off = 16; off >= lane_groups; off >>= 1) {
          f1[j] += __shfl_xor_sync(0xffffffffu, f1[j], off);
          f2[j] += __shfl_xor_sync(0xffffffffu, f2[j], off);
          f3[j] += __shfl_xor_sync(0xffffffffu, f3[j], off);
        }
      }
    }
    // every warp covers all C channels with its first G lanes: private rows, no atomics, fixed summation order
    if (lane < lane_groups) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        s_part[(wid * 3 + 0) * C + c0 + j] = f1[j];
        s_part[(wid * 3 + 1) * C + c0 + j] = f2[j];
        s_part[(wid * 3 + 2) * C + c0 + j] = f3[j];
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) {
      const int k = i / C, c = i - k * C;
      double t = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += (double)s_part[(w * 3 + k) * C + c];
      atomicAdd(sums + ((long long)n * C + c) * 3 + k, t);
    }
    return;
  }
  // general channel counts: fp64 shared-memory atomics
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    atomicAdd(&s_redd[0 * C + c0 + j], (double)f1[j]);
    atomicAdd(&s_redd[1 * C + c0 + j], (double)f2[j]);
    atomicAdd(&s_redd[2 * C + c0 + j], (double)f3[j]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) {
    int k = i / C, c = i - k * C;
    atomicAdd(sums + ((long long)n * C + c) * 3 + k, s_redd[i]);
  }
}

// one block; thread per channel.  See SURVEY.md App. G for the algebra.
__global__ void gn_bwd_finalize_kernel(const double* __restrict__ sums, const float* __restrict__ mr,
                                       const float* __restrict__ gamma, const float* __restrict__ scale, int N, int C,
                                       int groups, double vox, float* __restrict__ coef3,
                                       float* __restrict__ dgamma, float* __restrict__ dbeta,
                                       float* __restrict__ dbias) {
  PDL_ENTER();
  const int cpg = C / groups;
  const double m = (double)cpg * vox;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    const int g = c / cpg;
    double dg = 0.0, db = 0.0, dbi = 0.0;
    const double ga = gamma[c];
    for (int n = 0; n < N; ++n) {
      const double mu = mr[((long long)n * groups + g) * 2 + 0];
      const double r = mr[((long long)n * groups + g) * 2 + 1];
      double sa = 0.0, sax = 0.0;
      for (int j = 0; j < cpg; ++j) {
        const int cj = g * cpg + j;
        const double sj = scale ? (double)scale[(long long)n * C + cj] : 1.0;
        const double* p = sums + ((long long)n * C + cj) * 3;
        const double s1 = p[0] * sj, s2 = p[1] * sj;
        const double gj = gamma[cj];
        sa += gn_m1_term(gj, s1);
        sax += gn_m2_term(mu, r, gj, s1, s2);
      }
      const double m1 = sa / m, m2 = sax / m;
      const double sc = scale ? (double)scale[(long long)n * C + c] : 1.0;
      const double* p = sums + ((long long)n * C + c) * 3;
      const double s1 = p[0] * sc, s2 = p[1] * sc, s3 = p[2];
      const double P = gn_a(r, ga, sc);
      const double Q = gn_q(r, m2);
      const double R = gn_r(mu, r, m1, m2);
      float* o = coef3 + ((long long)n * C + c) * 3;
      o[0] = (float)P;
      o[1] = (float)Q;
      o[2] = (float)R;
      db += s1;
      dg += gn_dgamma(mu, r, s1, s2);
      dbi += gn_dbias(r, ga, s1, s3, Q, R, vox);
    }
    dgamma[c] += (float)dg;
    dbeta[c] += (float)db;
    if (dbias != nullptr) dbias[c] = (float)dbi;
  }
}


template <typename T, int VEC, int ACT>
__global__ void __launch_bounds__(256, 3) gn_bwd_apply_kernel(const T* __restrict__ g, long long ldg,
                                                           const T* __restrict__ y, long long ldy,
                                                           const float* __restrict__ coef,
                                                           const float* __restrict__ coef3, T* __restrict__ dy,
                                                           long long ldd, int C, long long V, const GnRef gn,
                                                           const double* __restrict__ sums, int N,
                                                           float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                           float* __restrict__ dbias) {
  PDL_ENTER();
  EW_PROLOGUE(C)
  float A[VEC], B[VEC], P[VEC], Q[VEC], R[VEC];
  if (gn.stats != nullptr) {
    extern __shared__ double s_dyn[];
    double* s_d = s_dyn;
    float* s_f = reinterpret_cast<float*>(s_d + gn_cta_doubles(C, gn.groups, true));
    float* s_c5 = s_f + 3 * C;                            // [5][C]: A, B, P, Q, R
    const double* grp = gn_coefs<true, true, GnCta, ACT != B200SEG_ACT_RELU>(GnCta(), gn, sums, n, C, s_d, s_f, s_c5, s_c5 + C, s_c5 + 2 * C,
                                             s_c5 + 3 * C, s_c5 + 4 * C);
    // parameter gradients (d gamma, d beta, d bias): ONE block per sample adds its sample's share from the
    // coefficients it has just derived (no serial loop over the batch at the tail of the grid); fp32 atomics over N
    if (blockIdx.x == gridDim.x - 1) param_grads_of_sample(gn, sums, grp, s_f, n, C, dgamma, dbeta, dbias);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      A[j] = s_c5[c0 + j];
      B[j] = s_c5[C + c0 + j];
      P[j] = s_c5[2 * C + c0 + j];
      Q[j] = s_c5[3 * C + c0 + j];
      R[j] = s_c5[4 * C + c0 + j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float* p = coef + ((long long)n * C + c0 + j) * 2;
      A[j] = p[0];
      B[j] = p[1];
      const float* q = coef3 + ((long long)n * C + c0 + j) * 3;
      P[j] = q[0];
      Q[j] = q[1];
      R[j] = q[2];
    }
  }
  const long long nb = (long long)n * V;
  for (; vi + vstep < V; vi += 2 * vstep) {
    const long long v0 = nb + vi, v1 = v0 + vstep;
    float y0[VEC], g0[VEC], y1[VEC], g1[VEC];
    Vec<T, VEC>::load(y + v0 * ldy + c0, y0);
    Vec<T, VEC>::load(g + v0 * ldg + c0, g0);
    Vec<T, VEC>::load(y + v1 * ldy + c0, y1);
    Vec<T, VEC>::load(g + v1 * ldg + c0, g1);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float d0 = gn_act_bwd_p<ACT>(fmaf(y0[j], A[j], B[j]), g0[j], P[j]);
      const float d1 = gn_act_bwd_p<ACT>(fmaf(y1[j], A[j], B[j]), g1[j], P[j]);
      g0[j] = d0 + fmaf(y0[j], Q[j], R[j]);
      g1[j] = d1 + fmaf(y1[j], Q[j], R[j]);
    }
    Vec<T, VEC>::store(dy + v0 * ldd + c0, g0);
    Vec<T, VEC>::store(dy + v1 * ldd + c0, g1);
  }
  if (vi < V) {
    const long long vox = nb + vi;
    float yv[VEC], gv[VEC], o[VEC];
    Vec<T, VEC>::load(y + vox * ldy + c0, yv);
    Vec<T, VEC>::load(g + vox * ldg + c0, gv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      float d = gn_act_bwd_p<ACT>(fmaf(yv[j], A[j], B[j]), gv[j], P[j]);
      o[j] = d + fmaf(yv[j], Q[j], R[j]);
    }
    Vec<T, VEC>::store(dy + vox * ldd + c0, o);
  }
}

// Fused GroupNorm+ReLU+Dropout backward for the SMALL pyramid levels: gn_bwd_reduce -> grid barrier -> gn_bwd_apply in
// ONE launch.  At 24^3 and below each of the two kernels is a few microseconds of launch + prologue around almost no
// data; the tensors stay in L2 between the phases.  Requirements (checked by the host): every CTA of the grid is
// resident at the same time (grid <= SMs x occupancy), channel groups are a power of two <= 256 (the staged
// reduction), fused coefficients.  `counter` is a zero-initialised word owned by this launch (one-shot barrier).
template <typename T, int VEC, int ACT>
__global__ void __launch_bounds__(256, 3) gn_bwd_fused_kernel(const T* __restrict__ g, long long ldg,
                                                              const T* __restrict__ y, long long ldy,
                                                              T* __restrict__ dy, long long ldd, double* sums,
                                                              unsigned int* counter, int C, long long V,
                                                              const GnRef gn, int N, float* __restrict__ dgamma,
                                                              float* __restrict__ dbeta, float* __restrict__ dbias) {
  PDL_ENTER();
  EW_PROLOGUE(C)
  extern __shared__ double s_dyn[];
  double* s_d = s_dyn;                                                    // coefficient scratch (backward size)
  float* s_f = reinterpret_cast<float*>(s_d + gn_cta_doubles(C, gn.groups, true));
  float* s_c5 = s_f + 3 * C;                                              // [5][C]: A, B, P, Q, R
  float* s_part = s_c5 + 5 * C;                                           // [8 warps][3][C]
  const T* yb = y + (long long)n * V * ldy + c0;
  const T* gb = g + (long long)n * V * ldg + c0;
  float A[VEC], B[VEC];
  // ---------------------------------------------------------------- phase 1: per-(n, c) sums
  gn_coefs<false, true, GnCta, ACT != B200SEG_ACT_RELU>(GnCta(), gn, nullptr, n, C, s_d, s_f, s_c5, s_c5 + C, nullptr, nullptr, nullptr);
  float f1[VEC], f2[VEC], f3[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    A[j] = s_c5[c0 + j];
    B[j] = s_c5[C + c0 + j];
    f1[j] = f2[j] = f3[j] = 0.f;
  }
  for (long long v = vi; v < V; v += vstep) {
    float yv[VEC], gv[VEC];
    Vec<T, VEC>::load(yb + v * ldy, yv);
    Vec<T, VEC>::load(gb + v * ldg, gv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float d = gn_act_bwd<ACT>(fmaf(yv[j], A[j], B[j]), gv[j]);
      f1[j] += d;
      f2[j] = fmaf(d, yv[j], f2[j]);
      f3[j] += yv[j];
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int lane_groups = G < 32 ? G : 32;
  if (G > 32) {     // a warp covers only part of the channels: rows it does not write stay zero
    for (int i = threadIdx.x; i < 24 * C; i += blockDim.x) s_part[i] = 0.f;
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    for (int off = 16; off >= lane_groups; off >>= 1) {
      f1[j] += __shfl_xor_sync(0xffffffffu, f1[j], off);
      f2[j] += __shfl_xor_sync(0xffffffffu, f2[j], off);
      f3[j] += __shfl_xor_sync(0xffffffffu, f3[j], off);
    }
  }
  if (lane < lane_groups) {
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      s_part[(wid * 3 + 0) * C + c0 + j] = f1[j];
      s_part[(wid * 3 + 1) * C + c0 + j] = f2[j];
      s_part[(wid * 3 + 2) * C + c0 + j] = f3[j];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) {
    const int k = i / C, c = i - k * C;
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += (double)s_part[(w * 3 + k) * C + c];
    atomicAdd(sums + ((long long)n * C + c) * 3 + k, t);
  }
  // ---------------------------------------------------------------- grid barrier (one shot)
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int total = gridDim.x * gridDim.y;
    atomicAdd(counter, 1u);
    while (*reinterpret_cast<volatile unsigned int*>(counter) < total) __nanosleep(20);
    __threadfence();
  }
  __syncthreads();
  // ---------------------------------------------------------------- phase 2: dy and the parameter gradients
  float P[VEC], Q[VEC], R[VEC];
  const double* grp = gn_coefs<true, true, GnCta, ACT != B200SEG_ACT_RELU>(GnCta(), gn, sums, n, C, s_d, s_f, s_c5, s_c5 + C, s_c5 + 2 * C,
                                           s_c5 + 3 * C, s_c5 + 4 * C);
  if (blockIdx.x == gridDim.x - 1) param_grads_of_sample(gn, sums, grp, s_f, n, C, dgamma, dbeta, dbias);
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    A[j] = s_c5[c0 + j];
    B[j] = s_c5[C + c0 + j];
    P[j] = s_c5[2 * C + c0 + j];
    Q[j] = s_c5[3 * C + c0 + j];
    R[j] = s_c5[4 * C + c0 + j];
  }
  T* db_ = dy + (long long)n * V * ldd + c0;
  for (long long v = vi; v < V; v += vstep) {
    float yv[VEC], gv[VEC], o[VEC];
    Vec<T, VEC>::load(yb + v * ldy, yv);
    Vec<T, VEC>::load(gb + v * ldg, gv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float d = gn_act_bwd_p<ACT>(fmaf(yv[j], A[j], B[j]), gv[j], P[j]);
      o[j] = d + fmaf(yv[j], Q[j], R[j]);
    }
    Vec<T, VEC>::store(db_ + v * ldd, o);
  }
}

// out[c] += sum over all voxels of all samples
template <typename T, int VEC>
__global__ void __launch_bounds__(256) colsum_kernel(const T* __restrict__ x, long long ld, float* __restrict__ out,
                                                     int C, long long V) {
  PDL_ENTER();
  EW_PROLOGUE(C)
  extern __shared__ float s_red[];   // [C]
  for (int i = threadIdx.x; i < C; i += blockDim.x) s_red[i] = 0.f;
  __syncthreads();
  float s[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) s[j] = 0.f;
  for (; vi < V; vi += vstep) {
    const long long vox = (long long)n * V + vi;
    float v[VEC];
    Vec<T, VEC>::load(x + vox * ld + c0, v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) s[j] += v[j];
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) atomicAdd(&s_red[c0 + j], s[j]);
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(out + i, s_red[i]);
}

// ---------------------------------------------------------------------------------------------
// 2x max pooling (window kd x 2 x 2, kd = 2 for 3-D, 1 for 2-D)
// ---------------------------------------------------------------------------------------------
template <typename T, int VEC>
__global__ void __launch_bounds__(256) pool_fwd_kernel(const T* __restrict__ x, long long ldx, T* __restrict__ out,
                                                       long long ldo, int C, int OD, int OH, int OW, int kd) {
  PDL_ENTER();
  const long long V = (long long)OD * OH * OW;
  EW_PROLOGUE(C)
  const int XH = OH * 2, XW = OW * 2, XD = OD * kd;
  for (; gi < total; gi += stride) {
    long long o = gi / G;
    int ow = (int)(o % OW);
    long long t2 = o / OW;
    int oh = (int)(t2 % OH);
    int od = (int)(t2 / OH);
    float best[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) best[j] = -INFINITY;
    for (int a = 0; a < kd; ++a)
      for (int b = 0; b < 2; ++b)
        for (int c = 0; c < 2; ++c) {
          long long vox = (((long long)n * XD + od * kd + a) * XH + oh * 2 + b) * XW + ow * 2 + c;
          float v[VEC];
          Vec<T, VEC>::load(x + vox * ldx + c0, v);
#pragma unroll
          for (int j = 0; j < VEC; ++j) best[j] = fmaxf(best[j], v[j]);
        }
    Vec<T, VEC>::store(out + ((long long)n * V + o) * ldo + c0, best);
  }
}

// thread per (coarse voxel, channel group): g_x[window] = addend[window] + (first arg-max ? g_out : 0)
template <typename T, int VEC>
__global__ void __launch_bounds__(256) pool_bwd_kernel(const T* __restrict__ x, long long ldx,
                                                       const T* __restrict__ go, long long ldg,
                                                       const T* __restrict__ addend, long long lda,
                                                       T* __restrict__ gx, long long ldo, int C, int OD, int OH,
                                                       int OW, int kd) {
  PDL_ENTER();
  const long long V = (long long)OD * OH * OW;
  EW_PROLOGUE(C)
  const int XH = OH * 2, XW = OW * 2, XD = OD * kd;
  for (; gi < total; gi += stride) {
    long long o = gi / G;
    int ow = (int)(o % OW);
    long long t2 = o / OW;
    int oh = (int)(t2 % OH);
    int od = (int)(t2 / OH);
    float best[VEC];
    int arg[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      best[j] = -INFINITY;
      arg[j] = 0;
    }
    int widx = 0;
    for (int a = 0; a < kd; ++a)
      for (int b = 0; b < 2; ++b)
        for (int c = 0; c < 2; ++c, ++widx) {
          long long vox = (((long long)n * XD + od * kd + a) * XH + oh * 2 + b) * XW + ow * 2 + c;
          float v[VEC];
          Vec<T, VEC>::load(x + vox * ldx + c0, v);
#pragma unroll
          for (int j = 0; j < VEC; ++j)
            if (v[j] > best[j]) {
              best[j] = v[j];
              arg[j] = widx;
            }
        }
    float gv[VEC];
    Vec<T, VEC>::load(go + ((long long)n * V + o) * ldg + c0, gv);
    widx = 0;
    for (int a = 0; a < kd; ++a)
      for (int b = 0; b < 2; ++b)
        for (int c = 0; c < 2; ++c, ++widx) {
          long long vox = (((long long)n * XD + od * kd + a) * XH + oh * 2 + b) * XW + ow * 2 + c;
          float r[VEC];
          if (addend != nullptr) {
            Vec<T, VEC>::load(addend + vox * lda + c0, r);
          } else {
#pragma unroll
            for (int j = 0; j < VEC; ++j) r[j] = 0.f;
          }
#pragma unroll
          for (int j = 0; j < VEC; ++j)
            if (arg[j] == widx) r[j] += gv[j];
          Vec<T, VEC>::store(gx + vox * ldo + c0, r);
        }
  }
}

// ---------------------------------------------------------------------------------------------
// head: sigmoid (C == 1) / softmax over channels (C > 1), fp32 channels-last
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) head_probs_kernel(const float* __restrict__ z, float* __restrict__ p,
                                                         long long nvox, int C) {
  PDL_ENTER();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox;
       i += (long long)gridDim.x * blockDim.x) {
    const float* zi = z + i * C;
    float* pi = p + i * C;
    if (C == 1) {
      pi[0] = 1.f / (1.f + expf(-zi[0]));
    } else if (C == 2) {
      float2 v = *reinterpret_cast<const float2*>(zi);
      float mx = fmaxf(v.x, v.y);
      float e0 = expf(v.x - mx), e1 = expf(v.y - mx);
      float inv = 1.f / (e0 + e1);
      *reinterpret_cast<float2*>(pi) = make_float2(e0 * inv, e1 * inv);
    } else {
      float mx = zi[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, zi[c]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(zi[c] - mx);
      float inv = 1.f / s;
      for (int c = 0; c < C; ++c) pi[c] = expf(zi[c] - mx) * inv;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host-side launch helpers
// ---------------------------------------------------------------------------------------------
static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

// can tensor t be accessed with 16-byte channel vectors?
static bool vec_ok(const b200seg_tensor* t) {
  if (t == nullptr) return true;
  const int vec = t->dtype == B200SEG_BF16 ? 8 : 4;
  return (t->c % vec == 0) && (t->ld % vec == 0) && al16(t->ptr);
}

// blocks per sample such that gridDim.x*256 is a multiple of G and the grid fills the chip
static int ew_blocks(long long V, int G, int N, int device, int per_sm = 8) {
  long long total = V * G;
  long long want = (total + 256 * 4 - 1) / (256 * 4);        // ~4 groups per thread
  long long cap = ((long long)num_sms(device) * per_sm + N - 1) / N;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  // 256 % G == 0 for every power-of-two G <= 256; otherwise round blocks so that blocks*256 % G == 0
  if (256 % G != 0) {
    long long k = G;   // blocks multiple of G always works
    want = ((want + k - 1) / k) * k;
  }
  return (int)want;
}

#define EW_DISPATCH(TENSOR_FOR_DTYPE, ALL_VEC_OK, ...)                          \
  do {                                                                           \
    if ((TENSOR_FOR_DTYPE)->dtype == B200SEG_BF16) {                             \
      typedef bf16 T;                                                            \
      if (ALL_VEC_OK) { constexpr int VEC = 8; __VA_ARGS__; } else { constexpr int VEC = 1; __VA_ARGS__; } \
    } else {                                                                     \
      typedef float T;                                                           \
      if (ALL_VEC_OK) { constexpr int VEC = 4; __VA_ARGS__; } else { constexpr int VEC = 1; __VA_ARGS__; } \
    }                                                                            \
  } while (0)

int ew_pack_weight(const float* w, void* out, int out_dtype, int T, int K, int N2, int N1, long long st,
                   long long sk, long long sn2, long long sn1, int flip, cudaStream_t s) {
  long long total = (long long)T * K * N2 * N1;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  if (blocks < 1) blocks = 1;
  if (out_dtype == B200SEG_BF16)
    launch_k(pack_weight_kernel<bf16>, blocks, 256, 0, s, w, static_cast<bf16*>(out), T, K, N2, N1, st, sk, sn2, sn1, flip);
  else
    launch_k(pack_weight_kernel<float>, blocks, 256, 0, s, w, static_cast<float*>(out), T, K, N2, N1, st, sk, sn2, sn1, flip);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_unpack_wgrad(const float* dwp, float* grad, int T, int K, int N, long long st, long long sk, long long sn,
                    cudaStream_t s) {
  long long total = (long long)T * K * N;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  if (blocks < 1) blocks = 1;
  launch_k(unpack_wgrad_kernel, blocks, 256, 0, s, dwp, grad, T, K, N, st, sk, sn);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_gn_finalize(const double* stats, const float* gamma, const float* beta, const float* scale, int N, int C,
                   int groups, long long vox, float eps, float* coef, float* mr, cudaStream_t s) {
  B200_CHECK_ARG(C % groups == 0, "gn_finalize: C=%d not divisible by groups=%d", C, groups);
  double m = (double)(C / groups) * (double)vox;
  launch_k(gn_finalize_kernel, N, 256, 0, s, stats, gamma, beta, scale, C, groups, m, eps, coef, mr);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_apply(const b200seg_tensor* y1, const float* c1, const b200seg_gn* g1, const b200seg_tensor* y2,
             const float* c2, const b200seg_gn* g2, const b200seg_tensor* res, const b200seg_tensor* out, int device,
             cudaStream_t s) {
  B200_CHECK_ARG(same_geom(y1, out) && (!y2 || same_geom(y2, out)) && (!res || same_geom(res, out)),
                 "apply: shape mismatch");
  B200_CHECK_ARG(y1->dtype == out->dtype && (!y2 || y2->dtype == out->dtype) && (!res || res->dtype == out->dtype),
                 "apply: dtype mismatch");
  const bool vok = vec_ok(y1) && vec_ok(y2) && vec_ok(res) && vec_ok(out);
  const long long V = nvox(out);
  const int C = out->c;
  EW_DISPATCH(out, vok, {
    const int G = C / VEC;
    dim3 grid(ew_blocks(V, G, out->n, device, 3), out->n);
    const int mg = (g1 && g2 && g2->groups > g1->groups) ? g2->groups : (g1 ? g1->groups : 1);
    // (precomputed-coefficient form: no coefficient scratch -- any channel count fits)
    const size_t smem = (g1 && g1->stats) ? gn_cta_doubles(C, mg, false) * sizeof(double) + (size_t)7 * C * sizeof(float) : 0;
    auto go = [&](auto kernel) {
      launch_k(kernel, grid, 256, smem, s, static_cast<const T*>(y1->ptr), y1->ld, c1, y2 ? static_cast<const T*>(y2->ptr) : nullptr, y2 ? y2->ld : 0, c2,
          res ? static_cast<const T*>(res->ptr) : nullptr, res ? res->ld : 0, static_cast<T*>(out->ptr), out->ld, C, V,
          gn_ref(g1, C), gn_ref(g2, C));
    };
    if (g1 && g1->act == B200SEG_ACT_LEAKY) go(apply_kernel<T, VEC, B200SEG_ACT_LEAKY>);
    else go(apply_kernel<T, VEC, B200SEG_ACT_RELU>);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_gn_bwd_reduce(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, const b200seg_gn* gn,
                     double* sums, int device, cudaStream_t s) {
  B200_CHECK_ARG(same_geom(g, y) && g->dtype == y->dtype, "gn_bwd_reduce: g/y mismatch");
  const bool vok = vec_ok(g) && vec_ok(y);
  const long long V = nvox(y);
  const int C = y->c;
  EW_DISPATCH(y, vok, {
    const int G = C / VEC;
    // large streams: deeper load pipeline, two CTAs per SM
    const bool deep = V * G >= (long long)num_sms(device) * 2 * 256 * 8;
    dim3 grid(ew_blocks(V, G, y->n, device, deep ? 2 : 3), y->n);
    const bool pow2g = (G & (G - 1)) == 0;
    const int groups = (gn && gn->stats) ? gn->groups : 1;
    const size_t full = (3 * C + gn_cta_doubles(C, groups, false)) * sizeof(double) + (size_t)5 * C * sizeof(float);
    const size_t staged_bytes = full + (size_t)8 * 3 * C * sizeof(float);
    const int staged = (pow2g && G <= 32 && staged_bytes <= 46 * 1024) ? 1 : 0;
    // precomputed-coefficient form without staging: only the [3][C] fp64 accumulators are touched (wide nets)
    const size_t base = (gn && gn->stats) ? full : (size_t)3 * C * sizeof(double);
    auto go = [&](auto kernel) {
      launch_k(kernel, grid, 256, staged ? staged_bytes : base, s, static_cast<const T*>(g->ptr), g->ld, static_cast<const T*>(y->ptr), y->ld, coef, sums, C, V,
          gn_ref(gn, C), staged);
    };
    const bool leaky = gn && gn->act == B200SEG_ACT_LEAKY;
    if (deep)
      leaky ? go(gn_bwd_reduce_kernel<T, VEC, true, B200SEG_ACT_LEAKY>) : go(gn_bwd_reduce_kernel<T, VEC, true, B200SEG_ACT_RELU>);
    else
      leaky ? go(gn_bwd_reduce_kernel<T, VEC, false, B200SEG_ACT_LEAKY>) : go(gn_bwd_reduce_kernel<T, VEC, false, B200SEG_ACT_RELU>);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_gn_bwd_finalize(const double* sums, const float* mr, const float* gamma, const float* scale, int N, int C,
                       int groups, long long vox, float* coef3, float* dgamma, float* dbeta, float* dbias,
                       cudaStream_t s) {
  B200_CHECK_ARG(C % groups == 0, "gn_bwd_finalize: C=%d not divisible by groups=%d", C, groups);
  int blocks = (C + 63) / 64;
  launch_k(gn_bwd_finalize_kernel, blocks, 64, 0, s, sums, mr, gamma, scale, N, C, groups, (double)vox, coef3, dgamma,
                                               dbeta, dbias);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_gn_bwd_apply(const b200seg_tensor* g, const b200seg_tensor* y, const float* coef, const float* coef3,
                    const b200seg_gn* gn, const double* sums, float* dgamma, float* dbeta, float* dbias,
                    const b200seg_tensor* dy, int device, cudaStream_t s, int sum_y_from_stats) {
  B200_CHECK_ARG(same_geom(g, y) && same_geom(dy, y) && g->dtype == y->dtype && dy->dtype == y->dtype,
                 "gn_bwd_apply: tensor mismatch");
  const bool vok = vec_ok(g) && vec_ok(y) && vec_ok(dy);
  const long long V = nvox(y);
  const int C = y->c;
  B200_CHECK_ARG(!(gn && gn->stats) || C <= 512, "gn_bwd_apply: fused coefficients support C <= 512 (got %d)", C);
  EW_DISPATCH(y, vok, {
    const int G = C / VEC;
    dim3 grid(ew_blocks(V, G, y->n, device, 3), y->n);
    const int groups = (gn && gn->stats) ? gn->groups : 1;
    const size_t smem = (gn && gn->stats) ? gn_cta_doubles(C, groups, true) * sizeof(double) + (size_t)8 * C * sizeof(float) : 0;
    GnRef gref = gn_ref(gn, C);
    gref.sum_y_from_stats = sum_y_from_stats;
    auto go = [&](auto kernel) {
      launch_k(kernel, grid, 256, smem, s, static_cast<const T*>(g->ptr), g->ld, static_cast<const T*>(y->ptr), y->ld,
               coef, coef3, static_cast<T*>(dy->ptr), dy->ld, C, V, gref, sums, y->n, dgamma, dbeta, dbias);
    };
    if (gn && gn->act == B200SEG_ACT_LEAKY) go(gn_bwd_apply_kernel<T, VEC, B200SEG_ACT_LEAKY>);
    else go(gn_bwd_apply_kernel<T, VEC, B200SEG_ACT_RELU>);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

// 1 if the fused backward can take this layer (small tensor, vectorised access, staged reduction applicable)
int ew_gn_bwd_fused_supported(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_tensor* dy) {
  if (!(vec_ok(g) && vec_ok(y) && vec_ok(dy))) return 0;
  const int vec = y->dtype == B200SEG_BF16 ? 8 : 4;
  const int G = y->c / vec;
  if (G < 1 || G > 256 || (G & (G - 1)) != 0 || y->c > 512) return 0;
  const long long elems = nvox(y) * y->c * (long long)y->n;
  return elems <= (4ll << 20) ? 1 : 0;          // <= 4 Mi elements: the 24^3 x 64 level and below
}

int ew_gn_bwd_fused(const b200seg_tensor* g, const b200seg_tensor* y, const b200seg_gn* gn, double* sums,
                    unsigned int* counter, float* dgamma, float* dbeta, float* dbias, const b200seg_tensor* dy,
                    int device, cudaStream_t s) {
  B200_CHECK_ARG(same_geom(g, y) && same_geom(dy, y) && g->dtype == y->dtype && dy->dtype == y->dtype,
                 "gn_bwd_fused: tensor mismatch");
  B200_CHECK_ARG(ew_gn_bwd_fused_supported(g, y, dy), "gn_bwd_fused: unsupported shape");
  const long long V = nvox(y);
  const int C = y->c;
  const int sms = num_sms(device);
  EW_DISPATCH(y, true, {
    const int G = C / VEC;
    const size_t smem = gn_cta_doubles(C, gn->groups, true) * sizeof(double) + (size_t)(8 + 24) * C * sizeof(float);
    const bool leaky = gn->act == B200SEG_ACT_LEAKY;
    auto kernel = leaky ? gn_bwd_fused_kernel<T, VEC, B200SEG_ACT_LEAKY> : gn_bwd_fused_kernel<T, VEC, B200SEG_ACT_RELU>;
    if (smem > 48 * 1024) {
      static int attr_done[2][64] = {{0}};
      if (device >= 0 && device < 64 && !attr_done[leaky][device]) {
        B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr_done[leaky][device] = 1;
      }
    }
    // all CTAs must be co-resident: cap the grid at one CTA per SM (the tensors are small)
    int bx = ew_blocks(V, G, y->n, device, 1);
    while (bx > 1 && (long long)bx * y->n > sms) --bx;
    if ((256 % G) != 0) bx = (bx / G) * G;
    B200_CHECK_ARG(bx >= 1 && (long long)bx * y->n <= sms, "gn_bwd_fused: batch too large for a resident grid");
    dim3 grid(bx, y->n);
    launch_k(kernel, grid, 256, smem, s, static_cast<const T*>(g->ptr), g->ld, static_cast<const T*>(y->ptr), y->ld, static_cast<T*>(dy->ptr), dy->ld,
        sums, counter, C, V, gn_ref(gn, C), y->n, dgamma, dbeta, dbias);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_colsum(const b200seg_tensor* dy, float* out, int device, cudaStream_t s) {
  const bool vok = vec_ok(dy);
  const long long V = nvox(dy);
  const int C = dy->c;
  EW_DISPATCH(dy, vok, {
    const int G = C / VEC;
    dim3 grid(ew_blocks(V, G, dy->n, device), dy->n);
    launch_k(colsum_kernel<T, VEC>, grid, 256, C * sizeof(float), s, static_cast<const T*>(dy->ptr), dy->ld, out, C, V);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_pool_fwd(const b200seg_tensor* x, const b200seg_tensor* out, int dims, int device, cudaStream_t s) {
  const int kd = dims == 3 ? 2 : 1;
  B200_CHECK_ARG(x->n == out->n && x->c == out->c && x->d == out->d * kd && x->h == out->h * 2 &&
                     x->w == out->w * 2 && x->dtype == out->dtype,
                 "pool_fwd: shape mismatch");
  const bool vok = vec_ok(x) && vec_ok(out);
  const long long V = nvox(out);
  const int C = out->c;
  EW_DISPATCH(out, vok, {
    const int G = C / VEC;
    dim3 grid(ew_blocks(V, G, out->n, device), out->n);
    launch_k(pool_fwd_kernel<T, VEC>, grid, 256, 0, s, static_cast<const T*>(x->ptr), x->ld, static_cast<T*>(out->ptr),
                                                 out->ld, C, out->d, out->h, out->w, kd);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_pool_bwd(const b200seg_tensor* x, const b200seg_tensor* go, const b200seg_tensor* addend,
                const b200seg_tensor* gx, int dims, int device, cudaStream_t s) {
  const int kd = dims == 3 ? 2 : 1;
  B200_CHECK_ARG(same_geom(x, gx) && (!addend || same_geom(addend, gx)) && x->n == go->n && x->c == go->c &&
                     x->d == go->d * kd && x->h == go->h * 2 && x->w == go->w * 2,
                 "pool_bwd: shape mismatch");
  B200_CHECK_ARG(x->dtype == gx->dtype && go->dtype == gx->dtype && (!addend || addend->dtype == gx->dtype),
                 "pool_bwd: dtype mismatch");
  const bool vok = vec_ok(x) && vec_ok(go) && vec_ok(addend) && vec_ok(gx);
  const long long V = nvox(go);
  const int C = go->c;
  EW_DISPATCH(gx, vok, {
    const int G = C / VEC;
    dim3 grid(ew_blocks(V, G, go->n, device), go->n);
    launch_k(pool_bwd_kernel<T, VEC>, grid, 256, 0, s, static_cast<const T*>(x->ptr), x->ld, static_cast<const T*>(go->ptr), go->ld,
        addend ? static_cast<const T*>(addend->ptr) : nullptr, addend ? addend->ld : 0, static_cast<T*>(gx->ptr),
        gx->ld, C, go->d, go->h, go->w, kd);
  });
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ew_head_probs(const float* logits, float* probs, long long nvox_, int C, int device, cudaStream_t s) {
  long long blocks = (nvox_ + 255) / 256;
  long long cap = (long long)num_sms(device) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_k(head_probs_kernel, (int)blocks, 256, 0, s, logits, probs, nvox_, C);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
