// SSIM / SSIM3D of model/lossesSSIM.py:49-93 with separable Gaussian windows, forward and backward (sm_90a).
//
// The reference filters five fields (x, y, x^2, y^2, xy) with a dense depthwise k^2 / k^3 window (F.conv2d /
// F.conv3d, groups = channel), and autograd runs five more dense convolutions backward.  The window is the outer
// product of one 1-D Gaussian, so here every field is filtered along W, H and (3-D) D in turn: 3k taps instead of k^3.
//
//   ssim_filter_kernel<false>  forward.  One CTA per (n*c, W tile of 32, H tile of TH, D chunk) walks the D chunk.
//                              Each input slice is staged in shared memory with its zero-padded halo, filtered along W
//                              and then H (fp64), and the result goes into a ring of the last kd filtered slices; the
//                              D taps are a gather over that ring (each thread reads only its own column, so the ring
//                              needs no barrier).  The epilogue forms the SSIM map S per output voxel, adds it to a
//                              per-thread fp64 sum and, when a gradient is wanted, writes the four backward
//                              coefficients dS/dmu1, dS/dmu2, dS/dm11 = dS/dm22 = -S/R and dS/dm12 = 2A/(QR) (fp64).
//                              At the end of the chunk the column sums are written, one fp64 partial per (CTA, column).
//   ssim_finalize_kernel       fixed-order sums of the partials: the mean (with the element count, so a data-parallel
//                              caller can all-reduce the pair), or per sample (2-D), or per (sample, W column) (3-D).
//   ssim_filter_kernel<true>   backward.  The same body applied with the adjoint filter (flipped taps, padding
//                              k - 1 - P) to the four coefficient fields scaled by d loss / d S, and combined
//                              pointwise: dx = F0 + 2x F2 + y F3, dy = F1 + 2y F2 + x F3.
// Everything accumulates in fp64; every reduction has a fixed order, so reruns are bit-identical.  Nothing is
// allocated or synchronised.
#include "common.cuh"

namespace b200seg {

namespace {

constexpr int kTW = 32;                     // output columns per CTA (one warp wide)
constexpr int kMaxK = 31;
constexpr int kTargetCtas = 256;            // D chunks are added until a launch has about this many CTAs
constexpr size_t kSmemPreferred = 113 * 1024;   // two CTAs per SM
constexpr size_t kSmemMax = 226 * 1024;        // the 227 KB opt-in less the static taps
constexpr double kC1 = 0.0001, kC2 = 0.0009;    // 0.01 ** 2, 0.03 ** 2 (lossesSSIM.py:61-62)

struct SsimGeom {
  int N, C;
  int Din, Hin, Win;       // extents the filter reads (forward: the image; backward: the map)
  int Dout, Hout, Wout;    // extents it writes
  int k, kd;               // taps along H and W / along D (1 for 2-D)
  int p, pd;               // zero padding along H and W / along D
  int TH, nWT, nHT, nDC, Dc;
  int mode;                // 0: mean, 1: per sample (2-D), 2: per (sample, W column) (3-D)
  float g[kMaxK + 1];      // 1-D taps (flipped for the adjoint)
};

struct Strides {
  long long n, c, d, h, w;
};

struct SsimIo {
  const float* x;
  const float* y;
  Strides sx, sy;
  double* coef;            // forward: written (or NULL); backward: read.  [4][N*C*D'*H'*W']
  double* part;            // forward: partials [CTA][32]
  const float* gout;       // backward: d loss / d value (mode 0: [1], 1: [N], 2: [N][W'])
  const double* count;     // backward, mode 0: the element count (global under data parallelism)
  float* dx;
  float* dy;
};

int nfields(bool bwd) { return bwd ? 4 : 5; }

size_t smem_bytes(bool bwd, int k, int kd, int TH) {
  const size_t R = TH + k - 1, SW = kTW + k - 1, nf = nfields(bwd);
  const size_t stage = bwd ? 4 * R * SW * sizeof(double) : 2 * R * SW * sizeof(float);
  return stage + nf * R * kTW * sizeof(double) + (size_t)kd * nf * TH * kTW * sizeof(double);
}

int pick_th(bool bwd, int k, int kd) {
  for (size_t lim : {kSmemPreferred, kSmemMax})
    for (int th = 8; th >= 1; th /= 2)
      if (smem_bytes(bwd, k, kd, th) <= lim) return th;
  return 1;
}

// tiling of one pass; the forward's fixes the partial layout
void tile(SsimGeom& G, bool bwd) {
  G.TH = pick_th(bwd, G.k, G.kd);
  G.nWT = (G.Wout + kTW - 1) / kTW;
  G.nHT = (G.Hout + G.TH - 1) / G.TH;
  const long long base = (long long)G.nWT * G.nHT * G.N * G.C;
  long long ndc = (kTargetCtas + base - 1) / base;
  const long long most = (G.Dout + G.kd - 1) / G.kd;      // chunks at least kd slices long
  if (ndc > most) ndc = most;
  if (ndc < 1) ndc = 1;
  G.Dc = (int)((G.Dout + ndc - 1) / ndc);
  G.nDC = (G.Dout + G.Dc - 1) / G.Dc;
}

// geometry of the forward (bwd = false) or the adjoint (bwd = true) filter
SsimGeom make_geom(int dims, int N, int C, int D, int H, int W, int k, const float* taps, int size_average, bool bwd) {
  SsimGeom G;
  memset(&G, 0, sizeof(G));
  const int P = k / 2;
  const int Dm = dims == 3 ? D + 2 * P - k + 1 : 1;
  const int Hm = H + 2 * P - k + 1, Wm = W + 2 * P - k + 1;
  G.N = N;
  G.C = C;
  G.k = k;
  G.kd = dims == 3 ? k : 1;
  if (!bwd) {
    G.Din = dims == 3 ? D : 1; G.Hin = H; G.Win = W;
    G.Dout = Dm; G.Hout = Hm; G.Wout = Wm;
    G.p = P;
    for (int j = 0; j < k; ++j) G.g[j] = taps[j];
  } else {
    G.Din = Dm; G.Hin = Hm; G.Win = Wm;
    G.Dout = dims == 3 ? D : 1; G.Hout = H; G.Wout = W;
    G.p = k - 1 - P;
    for (int j = 0; j < k; ++j) G.g[j] = taps[k - 1 - j];
  }
  G.pd = dims == 3 ? G.p : 0;
  G.mode = size_average ? 0 : (dims == 2 ? 1 : 2);
  tile(G, bwd);
  return G;
}

__host__ __device__ long long num_partials(const SsimGeom& G) {
  return (long long)G.N * G.C * G.nDC * G.nHT * G.nWT * kTW;
}

template <bool BWD>
__global__ void __launch_bounds__(256) ssim_filter_kernel(const SsimGeom G, const SsimIo io) {
  PDL_ENTER();
  constexpr int NF = BWD ? 4 : 5;
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ double gs[kMaxK + 1];
  const int TH = G.TH, k = G.k, kd = G.kd;
  const int R = TH + k - 1, SW = kTW + k - 1;
  const int nthr = TH * kTW;
  const int tid = threadIdx.x, th = tid >> 5, tw = tid & 31;
  const int wt = blockIdx.x, ht = blockIdx.y % G.nHT, dc = blockIdx.y / G.nHT, nc = blockIdx.z;
  const int n = nc / G.C, c = nc % G.C;
  const int h0 = ht * TH, w0 = wt * kTW;
  const int o0 = dc * G.Dc, o1 = min(G.Dout, o0 + G.Dc);

  size_t stage_bytes = BWD ? (size_t)4 * R * SW * sizeof(double) : (size_t)2 * R * SW * sizeof(float);
  float* xs = reinterpret_cast<float*>(smem);          // forward: x, y
  float* ys = xs + R * SW;
  double* cs = reinterpret_cast<double*>(smem);        // backward: four scaled coefficient fields
  double* wbuf = reinterpret_cast<double*>(smem + stage_bytes);     // [NF][R][32]
  double* ring = wbuf + (size_t)NF * R * kTW;                       // [kd][NF][TH*32]
  if (tid < kMaxK + 1) gs[tid] = tid < k ? (double)G.g[tid] : 0.0;

  // backward: d loss / d S per map element = gout * 1/count
  const long long vmap = (long long)G.Din * G.Hin * G.Win;
  double s_cta = 0.0;
  if (BWD) {
    if (G.mode == 0) s_cta = (double)io.gout[0] / io.count[0];
    else if (G.mode == 1) s_cta = (double)io.gout[n] / ((double)G.C * G.Hin * G.Win);
    else s_cta = 1.0 / ((double)G.C * G.Din * G.Hin);
  }

  double sacc = 0.0;

  auto process_slice = [&](int z, int slot) {
    __syncthreads();                                    // the previous slice's W pass has read the stage
    for (int i = tid; i < R * SW; i += nthr) {
      const int r = i / SW, cc = i - r * SW;
      const int h = h0 - G.p + r, w = w0 - G.p + cc;
      const bool in = h >= 0 && h < G.Hin && w >= 0 && w < G.Win;
      if (!BWD) {
        float xv = 0.f, yv = 0.f;
        if (in) {
          xv = io.x[n * io.sx.n + c * io.sx.c + z * io.sx.d + h * io.sx.h + w * io.sx.w];
          yv = io.y[n * io.sy.n + c * io.sy.c + z * io.sy.d + h * io.sy.h + w * io.sy.w];
        }
        xs[i] = xv;
        ys[i] = yv;
      } else {
        double v[4] = {0.0, 0.0, 0.0, 0.0};
        if (in) {
          double s = s_cta;
          if (G.mode == 2) s *= (double)io.gout[(long long)n * G.Win + w];
          const long long e = (((long long)nc * G.Din + z) * G.Hin + h) * G.Win + w;
          const long long tot = (long long)G.N * G.C * vmap;
#pragma unroll
          for (int f = 0; f < 4; ++f) v[f] = s * io.coef[f * tot + e];
        }
#pragma unroll
        for (int f = 0; f < 4; ++f) cs[(size_t)f * R * SW + i] = v[f];
      }
    }
    __syncthreads();
    for (int i = tid; i < R * kTW; i += nthr) {         // along W
      const int r = i >> 5, cc = i & 31;
      double a[NF];
#pragma unroll
      for (int f = 0; f < NF; ++f) a[f] = 0.0;
      for (int j = 0; j < k; ++j) {
        const double t = gs[j];
        const int e = r * SW + cc + j;
        if (!BWD) {
          const double xv = xs[e], yv = ys[e];
          a[0] = fma(t, xv, a[0]);
          a[1] = fma(t, yv, a[1]);
          a[2] = fma(t, xv * xv, a[2]);
          a[3] = fma(t, yv * yv, a[3]);
          a[4] = fma(t, xv * yv, a[4]);
        } else {
#pragma unroll
          for (int f = 0; f < NF; ++f) a[f] = fma(t, cs[(size_t)f * R * SW + e], a[f]);
        }
      }
#pragma unroll
      for (int f = 0; f < NF; ++f) wbuf[((size_t)f * R + r) * kTW + cc] = a[f];
    }
    __syncthreads();
    double a[NF];                                       // along H, into this thread's column of the ring
#pragma unroll
    for (int f = 0; f < NF; ++f) a[f] = 0.0;
    for (int j = 0; j < k; ++j) {
      const double t = gs[j];
#pragma unroll
      for (int f = 0; f < NF; ++f) a[f] = fma(t, wbuf[((size_t)f * R + th + j) * kTW + tw], a[f]);
    }
#pragma unroll
    for (int f = 0; f < NF; ++f) ring[((size_t)slot * NF + f) * nthr + tid] = a[f];
  };

  for (int z = o0 - G.pd; z < o0 - G.pd + kd - 1; ++z)
    if (z >= 0 && z < G.Din) process_slice(z, (z + G.pd) % kd);
  for (int o = o0; o < o1; ++o) {
    const int zn = o - G.pd + kd - 1;
    if (zn >= 0 && zn < G.Din) process_slice(zn, (zn + G.pd) % kd);
    double m[NF];                                       // along D: gather over the ring
#pragma unroll
    for (int f = 0; f < NF; ++f) m[f] = 0.0;
    for (int j = 0; j < kd; ++j) {
      const int z = o - G.pd + j;
      if (z < 0 || z >= G.Din) continue;
      const double t = kd == 1 ? 1.0 : gs[j];
      const int slot = (o + j) % kd;
#pragma unroll
      for (int f = 0; f < NF; ++f) m[f] = fma(t, ring[((size_t)slot * NF + f) * nthr + tid], m[f]);
    }
    const int h = h0 + th, w = w0 + tw;
    if (h >= G.Hout || w >= G.Wout) continue;
    const long long e = (((long long)nc * G.Dout + o) * G.Hout + h) * G.Wout + w;
    if (!BWD) {
      const double mu1 = m[0], mu2 = m[1];
      const double s11 = m[2] - mu1 * mu1, s22 = m[3] - mu2 * mu2, s12 = m[4] - mu1 * mu2;
      const double A = 2.0 * mu1 * mu2 + kC1, B = 2.0 * s12 + kC2;
      const double Q = mu1 * mu1 + mu2 * mu2 + kC1, Rr = s11 + s22 + kC2;
      const double QR = Q * Rr, S = A * B / QR;
      sacc += S;
      if (io.coef) {
        const long long tot = (long long)G.N * G.C * G.Dout * G.Hout * G.Wout;
        const double sq = S / Q, sr = S / Rr, bq = B / QR, aq = A / QR;
        io.coef[e] = 2.0 * mu2 * (bq - aq) + 2.0 * mu1 * (sr - sq);
        io.coef[tot + e] = 2.0 * mu1 * (bq - aq) + 2.0 * mu2 * (sr - sq);
        io.coef[2 * tot + e] = -sr;
        io.coef[3 * tot + e] = 2.0 * aq;
      }
    } else {
      const double xv = io.x[n * io.sx.n + c * io.sx.c + o * io.sx.d + h * io.sx.h + w * io.sx.w];
      const double yv = io.y[n * io.sy.n + c * io.sy.c + o * io.sy.d + h * io.sy.h + w * io.sy.w];
      if (io.dx) io.dx[e] = (float)(m[0] + 2.0 * xv * m[2] + yv * m[3]);
      if (io.dy) io.dy[e] = (float)(m[1] + 2.0 * yv * m[2] + xv * m[3]);
    }
  }
  if (!BWD) {                                           // column sums of S: fixed order over the TH rows
    __syncthreads();
    wbuf[tid] = sacc;
    __syncthreads();
    if (tid < kTW) {
      double s = 0.0;
      for (int r = 0; r < TH; ++r) s += wbuf[r * kTW + tid];
      const long long blk = (((long long)nc * G.nDC + dc) * G.nHT + ht) * G.nWT + wt;
      io.part[blk * kTW + tid] = s;
    }
  }
}

// one CTA per output value; reduce != 0: acc <- fixed-order sums of the partials (mode 0: acc = {sum, count}),
// then value = acc / count
__global__ void __launch_bounds__(256) ssim_finalize_kernel(const SsimGeom G, const double* __restrict__ part,
                                                            int reduce, double* acc, float* value) {
  PDL_ENTER();
  __shared__ double red[256];
  const int i = blockIdx.x;
  const long long per_n = num_partials(G) / G.N;
  double cnt;
  if (G.mode == 0) cnt = (double)G.N * G.C * G.Dout * G.Hout * G.Wout;
  else if (G.mode == 1) cnt = (double)G.C * G.Hout * G.Wout;
  else cnt = (double)G.C * G.Dout * G.Hout;
  if (reduce) {
    long long base, stride, num;
    if (G.mode == 0) { base = 0; stride = 1; num = per_n * G.N; }
    else if (G.mode == 1) { base = i * per_n; stride = 1; num = per_n; }
    else {
      const int n = i / G.Wout, w = i % G.Wout;
      base = n * per_n + w; stride = (long long)G.nWT * kTW; num = (long long)G.C * G.nDC * G.nHT;
    }
    double s = 0.0;
    for (long long r = threadIdx.x; r < num; r += blockDim.x) s += part[base + r * stride];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      acc[i] = red[0];
      if (G.mode == 0) acc[1] = cnt;
      value[i] = (float)(red[0] / cnt);
    }
  } else if (threadIdx.x == 0) {
    value[i] = (float)(acc[i] / (G.mode == 0 ? acc[1] : cnt));
  }
}

int check_common(int dims, int N, int C, int D, int H, int W, int k, const float* taps) {
  B200_CHECK_ARG(dims == 2 || dims == 3, "ssim: dims must be 2 or 3, got %d", dims);
  B200_CHECK_ARG(k >= 1 && k <= kMaxK, "ssim: window_size %d outside [1, %d]", k, kMaxK);
  B200_CHECK_ARG(taps, "ssim: null taps");
  B200_CHECK_ARG(N >= 1 && C >= 1 && H >= 1 && W >= 1 && (dims == 2 || D >= 1), "ssim: empty shape");
  const int P = k / 2;
  B200_CHECK_ARG(H + 2 * P - k + 1 >= 1 && W + 2 * P - k + 1 >= 1, "ssim: empty map");
  B200_CHECK_ARG((long long)N * C <= 65535, "ssim: N*C = %lld exceeds the launch grid", (long long)N * C);
  return B200SEG_OK;
}

Strides strides(const int64_t* s) { return Strides{(long long)s[0], (long long)s[1], (long long)s[2], (long long)s[3], (long long)s[4]}; }

template <bool BWD>
int launch_filter(const SsimGeom& G, const SsimIo& io, int device, cudaStream_t st) {
  B200_CHECK_ARG((long long)G.nHT * G.nDC <= 65535, "ssim: shape outside the launch grid");
  const size_t smem = smem_bytes(BWD, G.k, G.kd, G.TH);
  static int attr_done[64] = {0};
  if (device >= 0 && device < 64 && !attr_done[device]) {
    B200_CUDA(cudaFuncSetAttribute(ssim_filter_kernel<BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax));
    attr_done[device] = 1;
  }
  launch_k(ssim_filter_kernel<BWD>, dim3(G.nWT, G.nHT * G.nDC, G.N * G.C), G.TH * kTW, smem, st, G, io);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace

int64_t ssim_workspace(int dims, int N, int C, int D, int H, int W, int k) {
  float taps[kMaxK + 1] = {0.f};
  const SsimGeom G = make_geom(dims, N, C, D, H, W, k, taps, 1, false);
  return num_partials(G) * (int64_t)sizeof(double);
}

int ssim_fwd(int dims, const float* x, const int64_t* xs, const float* y, const int64_t* ys, int N, int C, int D,
             int H, int W, int k, const float* taps, double* coef, void* ws, long long ws_bytes, int device,
             cudaStream_t st) {
  int rc = check_common(dims, N, C, D, H, W, k, taps);
  if (rc != B200SEG_OK) return rc;
  const SsimGeom G = make_geom(dims, N, C, D, H, W, k, taps, 1, false);
  B200_CHECK_ARG(ws && ws_bytes >= num_partials(G) * (long long)sizeof(double), "ssim_fwd: workspace too small");
  SsimIo io;
  memset(&io, 0, sizeof(io));
  io.x = x; io.y = y; io.sx = strides(xs); io.sy = strides(ys);
  io.coef = coef;
  io.part = static_cast<double*>(ws);
  return launch_filter<false>(G, io, device, st);
}

int ssim_finalize(int dims, int N, int C, int D, int H, int W, int k, int size_average, int reduce, const void* ws,
                  long long ws_bytes, double* acc, float* value, cudaStream_t st) {
  float taps[kMaxK + 1] = {0.f};
  int rc = check_common(dims, N, C, D, H, W, k, taps);
  if (rc != B200SEG_OK) return rc;
  const SsimGeom G = make_geom(dims, N, C, D, H, W, k, taps, size_average, false);
  B200_CHECK_ARG(!reduce || (ws && ws_bytes >= num_partials(G) * (long long)sizeof(double)),
                 "ssim_finalize: workspace too small");
  const long long nout = G.mode == 0 ? 1 : G.mode == 1 ? N : (long long)N * G.Wout;
  B200_CHECK_ARG(nout <= 2147483647LL, "ssim_finalize: too many outputs");
  launch_k(ssim_finalize_kernel, dim3((unsigned)nout), 256, 0, st, G, static_cast<const double*>(ws), reduce, acc,
           value);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int ssim_bwd(int dims, const float* x, const int64_t* xs, const float* y, const int64_t* ys, int N, int C, int D,
             int H, int W, int k, const float* taps, const double* coef, int size_average, const float* gout,
             const double* acc, float* dx, float* dy, int device, cudaStream_t st) {
  int rc = check_common(dims, N, C, D, H, W, k, taps);
  if (rc != B200SEG_OK) return rc;
  const SsimGeom G = make_geom(dims, N, C, D, H, W, k, taps, size_average, true);
  B200_CHECK_ARG(!(G.mode == 0 && !acc), "ssim_bwd: the mean needs acc");
  SsimIo io;
  memset(&io, 0, sizeof(io));
  io.x = x; io.y = y; io.sx = strides(xs); io.sy = strides(ys);
  io.coef = const_cast<double*>(coef);
  io.gout = gout;
  io.count = acc ? acc + 1 : nullptr;
  io.dx = dx; io.dy = dy;
  return launch_filter<true>(G, io, device, st);
}

}  // namespace b200seg
