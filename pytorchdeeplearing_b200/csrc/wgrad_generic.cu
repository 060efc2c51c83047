// Generic weight-gradient kernel on CUDA cores (fp32 FFMA) for sm_90a.
//
//   dwp[t][ka][kb] += sum_{n,o} a[n, o*s + t - p, ka] * b[n, o, kb]
//
// GEMM view: rows R = (tap, ka) flattened (taps*Ka rows), cols = kb, reduction over all output
// voxels of all samples, split across gridDim.z chunks (split-K) with fp32 atomics at the end.
// Used for every layer in PARITY mode and for the non-MMA-shaped layers in PERF mode
// (DESIGN.md section 4).  256 threads, 4x4 micro-tile, BA x BB = 4096 tile, 16 voxels per step.
#include "common.cuh"

namespace b200seg {

template <typename TA, typename TB>
struct WgradArgs {
  const TA* a;
  const TB* b;
  float* dwp;
  int AD, AH, AW;   // spatial dims of a (gathered side)
  long long ald;
  int OD, OH, OW;   // spatial dims of b (dense side)
  long long bld;
  int N, Ka, Kb, Rtot;
  long long NV;     // N * OD*OH*OW
  int steps_per_chunk;
  ConvGeom g;
  int avec, bvec;
};

template <typename TA, typename TB, int BB>
__global__ void __launch_bounds__(256) wgrad_ffma_kernel(const WgradArgs<TA, TB> w) {
  PDL_ENTER();
  constexpr int BA = 4096 / BB;
  constexpr int BV = 16;
  constexpr int AQ = BA / 4;           // A quads per voxel row
  constexpr int APASS = (BV * AQ) / 256;
  constexpr int AVSTEP = 256 / AQ;     // voxel stride between passes
  constexpr int BQ = BB / 4;
  __shared__ __align__(16) float As[BV][BA];
  __shared__ __align__(16) float Bs[BV][BB];

  const int tid = threadIdx.x;
  const int tx = tid % BQ, ty = tid / BQ;
  const int r0 = blockIdx.x * BA;
  const int c0 = blockIdx.y * BB;
  const long long V = (long long)w.OD * w.OH * w.OW;

  // A loader: fixed row quad, varying voxel
  const int arq = tid % AQ;
  const int av0 = tid / AQ;
  const int R = r0 + arq * 4;
  const bool fast = (w.Ka % 4) == 0;
  int kd_[4], kh_[4], kw_[4], ka_[4];
  bool rvalid[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    int Re = R + e;
    rvalid[e] = Re < w.Rtot;
    int Rc = rvalid[e] ? Re : 0;
    int t = Rc / w.Ka;
    ka_[e] = Rc - t * w.Ka;
    kw_[e] = t % w.g.kw;
    int t2 = t / w.g.kw;
    kh_[e] = t2 % w.g.kh;
    kd_[e] = t2 / w.g.kh;
  }
  // B loader
  const bool bload = tid < BV * BQ;
  const int bv = tid / BQ, bq = tid % BQ;

  float4 ra[APASS];
  float4 rb;

  auto load_step = [&](long long g0) {
#pragma unroll
    for (int p = 0; p < APASS; ++p) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      long long gv = g0 + av0 + p * AVSTEP;
      if (gv < w.NV) {
        int n = (int)(gv / V);
        int o = (int)(gv - (long long)n * V);
        int ow = o % w.OW;
        int t2 = o / w.OW;
        int oh = t2 % w.OH;
        int od = t2 / w.OH;
        const TA* abase = w.a + (long long)n * w.AD * w.AH * w.AW * w.ald;
        if (fast) {
          if (rvalid[0]) {
            int id = od * w.g.sd + kd_[0] - w.g.pd;
            int ih = oh * w.g.sh + kh_[0] - w.g.ph;
            int iw = ow * w.g.sw + kw_[0] - w.g.pw;
            if ((unsigned)id < (unsigned)w.AD && (unsigned)ih < (unsigned)w.AH && (unsigned)iw < (unsigned)w.AW) {
              const TA* pa = abase + (((long long)id * w.AH + ih) * w.AW + iw) * w.ald + ka_[0];
              if (w.avec) {
                v = load4(pa);
              } else {
                v.x = to_f(pa[0]); v.y = to_f(pa[1]); v.z = to_f(pa[2]); v.w = to_f(pa[3]);
              }
            }
          }
        } else {
          float vv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (!rvalid[e]) continue;
            int id = od * w.g.sd + kd_[e] - w.g.pd;
            int ih = oh * w.g.sh + kh_[e] - w.g.ph;
            int iw = ow * w.g.sw + kw_[e] - w.g.pw;
            if ((unsigned)id < (unsigned)w.AD && (unsigned)ih < (unsigned)w.AH && (unsigned)iw < (unsigned)w.AW)
              vv[e] = to_f(abase[(((long long)id * w.AH + ih) * w.AW + iw) * w.ald + ka_[e]]);
          }
          v = make_float4(vv[0], vv[1], vv[2], vv[3]);
        }
      }
      ra[p] = v;
    }
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bload) {
      long long gv = g0 + bv;
      int col = c0 + bq * 4;
      if (gv < w.NV && col < w.Kb) {
        const TB* pb = w.b + gv * w.bld + col;
        if (w.bvec && col + 3 < w.Kb) {
          rb = load4(pb);
        } else {
          rb.x = to_f(pb[0]);
          if (col + 1 < w.Kb) rb.y = to_f(pb[1]);
          if (col + 2 < w.Kb) rb.z = to_f(pb[2]);
          if (col + 3 < w.Kb) rb.w = to_f(pb[3]);
        }
      }
    }
  };
  auto store_step = [&]() {
#pragma unroll
    for (int p = 0; p < APASS; ++p)
      *reinterpret_cast<float4*>(&As[av0 + p * AVSTEP][arq * 4]) = ra[p];
    if (bload) *reinterpret_cast<float4*>(&Bs[bv][bq * 4]) = rb;
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const long long total_steps = (w.NV + BV - 1) / BV;
  long long s_begin = (long long)blockIdx.z * w.steps_per_chunk;
  long long s_end = s_begin + w.steps_per_chunk;
  if (s_end > total_steps) s_end = total_steps;
  if (s_begin >= s_end) return;

  load_step(s_begin * BV);
  store_step();
  __syncthreads();
  for (long long s = s_begin; s < s_end; ++s) {
    if (s + 1 < s_end) load_step((s + 1) * BV);
#pragma unroll
    for (int v = 0; v < BV; ++v) {
      float4 a4 = *reinterpret_cast<const float4*>(&As[v][ty * 4]);
      float4 b4 = *reinterpret_cast<const float4*>(&Bs[v][tx * 4]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
      const float bvv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bvv[j], acc[i][j]);
    }
    __syncthreads();
    if (s + 1 < s_end) {
      store_step();
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int Ri = r0 + ty * 4 + i;
    if (Ri >= w.Rtot) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int col = c0 + tx * 4 + j;
      if (col < w.Kb) atomicAdd(w.dwp + (long long)Ri * w.Kb + col, acc[i][j]);
    }
  }
}

static bool aligned_w(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

template <typename TA, typename TB>
static int wgrad_typed(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                       cudaStream_t st) {
  WgradArgs<TA, TB> w;
  if (conv_geometry(kind, dims, &w.g) != 0 || w.g.up) {
    set_error("b200seg_wgrad: kind must be K3, K1 or DOWN (got %d)", kind);
    return B200SEG_EINVAL;
  }
  B200_CHECK_ARG(a->n == b->n && a->d == b->d * w.g.sd && a->h == b->h * w.g.sh && a->w == b->w * w.g.sw,
                 "b200seg_wgrad: a/b spatial dims do not match kind %d", kind);
  w.a = static_cast<const TA*>(a->ptr);
  w.b = static_cast<const TB*>(b->ptr);
  w.dwp = dwp;
  w.AD = a->d; w.AH = a->h; w.AW = a->w; w.ald = a->ld;
  w.OD = b->d; w.OH = b->h; w.OW = b->w; w.bld = b->ld;
  w.N = a->n; w.Ka = a->c; w.Kb = b->c;
  const int taps = w.g.kd * w.g.kh * w.g.kw;
  w.Rtot = taps * w.Ka;
  w.NV = (long long)b->n * b->d * b->h * b->w;
  w.avec = (w.Ka % 4 == 0) && (a->ld % 4 == 0) && aligned_w(a->ptr, sizeof(TA) * 4);
  w.bvec = (w.Kb % 4 == 0) && (b->ld % 4 == 0) && aligned_w(b->ptr, sizeof(TB) * 4);
  const int BB = w.Kb <= 16 ? 16 : (w.Kb <= 32 ? 32 : 64);
  const int BA = 4096 / BB;
  const int gx = (w.Rtot + BA - 1) / BA, gy = (w.Kb + BB - 1) / BB;
  const long long total_steps = (w.NV + 15) / 16;
  long long want = (4LL * num_sms(device) + (long long)gx * gy - 1) / ((long long)gx * gy);
  if (want < 1) want = 1;
  long long min_steps = 8;                      // keep >= 128 voxels per CTA
  long long chunks = want;
  if (chunks > (total_steps + min_steps - 1) / min_steps) chunks = (total_steps + min_steps - 1) / min_steps;
  if (chunks < 1) chunks = 1;
  if (chunks > 65535) chunks = 65535;
  w.steps_per_chunk = (int)((total_steps + chunks - 1) / chunks);
  chunks = (total_steps + w.steps_per_chunk - 1) / w.steps_per_chunk;
  dim3 grid(gx, gy, (unsigned)chunks), block(256);
  if (BB == 16) launch_k(wgrad_ffma_kernel<TA, TB, 16>, grid, block, 0, st, w);
  else if (BB == 32) launch_k(wgrad_ffma_kernel<TA, TB, 32>, grid, block, 0, st, w);
  else launch_k(wgrad_ffma_kernel<TA, TB, 64>, grid, block, 0, st, w);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int wgrad_generic(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                  cudaStream_t st) {
  B200_CHECK_ARG(a && b && dwp, "b200seg_wgrad: null argument");
  if (a->dtype == B200SEG_F32 && b->dtype == B200SEG_F32) return wgrad_typed<float, float>(kind, dims, a, b, dwp, device, st);
  if (a->dtype == B200SEG_BF16 && b->dtype == B200SEG_BF16) return wgrad_typed<bf16, bf16>(kind, dims, a, b, dwp, device, st);
  if (a->dtype == B200SEG_F32 && b->dtype == B200SEG_BF16) return wgrad_typed<float, bf16>(kind, dims, a, b, dwp, device, st);
  return wgrad_typed<bf16, float>(kind, dims, a, b, dwp, device, st);
}

}  // namespace b200seg
