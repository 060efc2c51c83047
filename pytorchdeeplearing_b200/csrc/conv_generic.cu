// Generic implicit-GEMM convolution on CUDA cores (fp32 FFMA, fp32 accumulate) for sm_90a.
//
// Role (DESIGN.md section 4): (1) the whole conv family in PARITY mode (fp32 storage; fp32
// products are what the 1e-3 / identical-argmax bar needs, SURVEY.md section 0.8), (2) in PERF
// mode the layers that are not dense-MMA shaped: the stem (Cin = image channels, K = 27),
// the head (Cout = numclass) and any shape the tensor-core path does not cover.
//
// GEMM view: rows = output positions of one sample (BM per CTA), cols = output channels
// (BN per CTA), K = taps x Cin walked in chunks of 16 channels of one tap.  The A tile is
// gathered on the fly (zero padding = predicated loads), the B tile comes from the packed
// [tap][Cin][Cout] weights.  256 threads, 4x4 register micro-tile, register-staged double
// buffering.  Epilogue: +bias, GroupNorm sum / sum-of-squares partials (smem atomics -> one
// fp64 atomic per column per CTA), optional residual addend, 128-bit coalesced NDHWC stores.
// The transposed conv (UP) is the same GEMM with cols = (tap, Cout) and a depth-to-space store.
#include "common.cuh"

namespace b200seg {

template <typename TX, typename TW, typename TY>
struct ConvArgs {
  const TX* x;
  const TW* w;
  const float* bias;
  TY* y;
  const TY* addend;
  double* stats;
  int XD, XH, XW;        // input spatial dims
  long long xld;
  int OD, OH, OW;        // row space dims (output dims for gather kinds, input dims for UP)
  long long yld, ald;
  int Cin, Cout, Ncols;  // Ncols = Cout (gather) or taps*Cout (UP)
  int Mrows;             // OD*OH*OW
  ConvGeom g;
  int xvec, wvec, yvec, avec;
};

template <typename TX, typename TW, typename TY, int BN>
__global__ void __launch_bounds__(256) conv_ffma_kernel(const ConvArgs<TX, TW, TY> a) {
  PDL_ENTER();
  constexpr int BM = 4096 / BN;
  constexpr int BK = 16;
  constexpr int PASSES = BM / 64;
  constexpr int TXN = BN / 4;   // threads along columns
  // one buffer: [As | Bs] during the main loop, reused as the (deterministic) statistics scratch
  constexpr int AS_FLOATS = BK * (BM + 4);
  constexpr int BS_FLOATS = BK * BN;
  constexpr int ST_FLOATS = 2 * (BM / 4) * BN;          // per (row-thread, column) sum and sum of squares
  constexpr int SM_FLOATS = (AS_FLOATS + BS_FLOATS) > ST_FLOATS ? (AS_FLOATS + BS_FLOATS) : ST_FLOATS;
  __shared__ __align__(16) float smem_f[SM_FLOATS];
  float (*As)[BM + 4] = reinterpret_cast<float (*)[BM + 4]>(smem_f);
  float (*Bs)[BN] = reinterpret_cast<float (*)[BN]>(smem_f + AS_FLOATS);

  const int tid = threadIdx.x;
  const int tx = tid % TXN, ty = tid / TXN;
  const int n = blockIdx.z;
  const int m0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- A loader mapping: row lr = tid/4 (+64 per pass), channel quad q = tid%4
  const int lq = tid & 3;
  int rd[PASSES], rh[PASSES], rw[PASSES];
  bool rv[PASSES];
#pragma unroll
  for (int p = 0; p < PASSES; ++p) {
    int m = m0 + (tid >> 2) + 64 * p;
    rv[p] = m < a.Mrows;
    int mm = rv[p] ? m : 0;
    rw[p] = mm % a.OW;
    int t2 = mm / a.OW;
    rh[p] = t2 % a.OH;
    rd[p] = t2 / a.OH;
  }
  // ---- B loader mapping: element e = tid*4 of the BK x BN tile
  const bool bload = tid * 4 < BK * BN;
  const int bk = (tid * 4) / BN, bc = (tid * 4) % BN;

  const int cchunks = (a.Cin + BK - 1) / BK;
  const int taps = a.g.kd * a.g.kh * a.g.kw;
  const int nchunks = taps * cchunks;
  const TX* xbase = a.x + (long long)n * a.XD * a.XH * a.XW * a.xld;

  float4 ra[PASSES];
  float4 rb;

  auto load_tiles = [&](int chunk) {
    const int t = chunk / cchunks;
    const int c0 = (chunk - t * cchunks) * BK;
    const int kw_ = t % a.g.kw;
    const int t2 = t / a.g.kw;
    const int kh_ = t2 % a.g.kh;
    const int kd_ = t2 / a.g.kh;
    const int ch = c0 + lq * 4;
#pragma unroll
    for (int p = 0; p < PASSES; ++p) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rv[p]) {
        int id = rd[p] * a.g.sd + kd_ - a.g.pd;
        int ih = rh[p] * a.g.sh + kh_ - a.g.ph;
        int iw = rw[p] * a.g.sw + kw_ - a.g.pw;
        if ((unsigned)id < (unsigned)a.XD && (unsigned)ih < (unsigned)a.XH && (unsigned)iw < (unsigned)a.XW &&
            ch < a.Cin) {
          const TX* px = xbase + (((long long)id * a.XH + ih) * a.XW + iw) * a.xld + ch;
          if (a.xvec && ch + 3 < a.Cin) {
            v = load4(px);
          } else {
            v.x = to_f(px[0]);
            if (ch + 1 < a.Cin) v.y = to_f(px[1]);
            if (ch + 2 < a.Cin) v.z = to_f(px[2]);
            if (ch + 3 < a.Cin) v.w = to_f(px[3]);
          }
        }
      }
      ra[p] = v;
    }
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bload) {
      int ci = c0 + bk;
      int col = n0 + bc;
      if (ci < a.Cin && col < a.Ncols) {
        const TW* pw = a.w + ((long long)t * a.Cin + ci) * a.Ncols + col;
        if (a.wvec && col + 3 < a.Ncols) {
          rb = load4(pw);
        } else {
          rb.x = to_f(pw[0]);
          if (col + 1 < a.Ncols) rb.y = to_f(pw[1]);
          if (col + 2 < a.Ncols) rb.z = to_f(pw[2]);
          if (col + 3 < a.Ncols) rb.w = to_f(pw[3]);
        }
      }
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int p = 0; p < PASSES; ++p) {
      int lr = (tid >> 2) + 64 * p;
      As[lq * 4 + 0][lr] = ra[p].x;
      As[lq * 4 + 1][lr] = ra[p].y;
      As[lq * 4 + 2][lr] = ra[p].z;
      As[lq * 4 + 3][lr] = ra[p].w;
    }
    if (bload) *reinterpret_cast<float4*>(&Bs[bk][bc]) = rb;
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  load_tiles(0);
  store_tiles();
  __syncthreads();
  for (int chunk = 0; chunk < nchunks; ++chunk) {
    if (chunk + 1 < nchunks) load_tiles(chunk + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
      const float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
    if (chunk + 1 < nchunks) {
      store_tiles();
      __syncthreads();
    }
  }

  // ------------------------------------------------------------------ epilogue
  const int col0 = n0 + tx * 4;
  float bvals[4] = {0.f, 0.f, 0.f, 0.f};
  if (a.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (col0 + j < a.Ncols) bvals[j] = a.bias[(col0 + j) % a.Cout];
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] += bvals[j];

  if (a.stats != nullptr) {
    // fixed-order reduction (bit-reproducible): thread (ty, tx) publishes its 4-row partials, then one
    // thread per column adds the BM/4 partials in fp64; one fp64 atomic per column per CTA follows.
    __syncthreads();                                   // main loop done: As/Bs can be overwritten
    float* s_part = smem_f;                            // [2][BM/4][BN]
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float s = 0.f, q = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (m0 + ty * 4 + i < a.Mrows) {
          float v = acc[i][j];
          s += v;
          q = fmaf(v, v, q);
        }
      }
      s_part[ty * BN + tx * 4 + j] = s;
      s_part[(BM / 4) * BN + ty * BN + tx * 4 + j] = q;
    }
    __syncthreads();
    if (tid < 2 * BN) {
      const int which = tid / BN, c = tid - which * BN;
      if (n0 + c < a.Ncols) {
        double t = 0.0;
        const float* pp = s_part + which * (BM / 4) * BN + c;
#pragma unroll 4
        for (int r = 0; r < BM / 4; ++r) t += (double)pp[r * BN];
        const int co = (n0 + c) % a.Cout;
        atomicAdd(a.stats + ((long long)n * a.Cout + co) * 2 + which, t);
      }
    }
  }

  if (col0 >= a.Ncols) return;
  int tcol = 0, co0 = col0;
  int fa = 0, fb = 0, fc = 0;
  if (a.g.up) {
    tcol = col0 / a.Cout;
    co0 = col0 - tcol * a.Cout;
    fc = tcol % a.g.uw;
    int t2 = tcol / a.g.uw;
    fb = t2 % a.g.uh;
    fa = t2 / a.g.uh;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= a.Mrows) continue;
    long long ovox;
    if (a.g.up) {
      int w_ = m % a.OW;
      int t2 = m / a.OW;
      int h_ = t2 % a.OH;
      int d_ = t2 / a.OH;
      ovox = (((long long)n * (a.OD * a.g.ud) + (d_ * a.g.ud + fa)) * (a.OH * a.g.uh) + (h_ * a.g.uh + fb)) *
                 (a.OW * a.g.uw) + (w_ * a.g.uw + fc);
    } else {
      ovox = (long long)n * a.Mrows + m;
    }
    float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    if (a.addend != nullptr) {
      const TY* pa = a.addend + ovox * a.ald + co0;
      if (a.avec && col0 + 3 < a.Ncols) {
        float4 r = load4(pa);
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      } else {
        v.x += to_f(pa[0]);
        if (col0 + 1 < a.Ncols) v.y += to_f(pa[1]);
        if (col0 + 2 < a.Ncols) v.z += to_f(pa[2]);
        if (col0 + 3 < a.Ncols) v.w += to_f(pa[3]);
      }
    }
    TY* py = a.y + ovox * a.yld + co0;
    if (a.yvec && col0 + 3 < a.Ncols) {
      store4(py, v);
    } else {
      py[0] = from_f<TY>(v.x);
      if (col0 + 1 < a.Ncols) py[1] = from_f<TY>(v.y);
      if (col0 + 2 < a.Ncols) py[2] = from_f<TY>(v.z);
      if (col0 + 3 < a.Ncols) py[3] = from_f<TY>(v.w);
    }
  }
}

template <typename TX, typename TW, typename TY>
static int launch_conv(const ConvArgs<TX, TW, TY>& a, int nbatch, cudaStream_t st) {
  dim3 block(256);
  if (a.Ncols <= 16) {
    dim3 grid((a.Mrows + 255) / 256, 1, nbatch);
    launch_k(conv_ffma_kernel<TX, TW, TY, 16>, grid, block, 0, st, a);
  } else if (a.Ncols <= 32) {
    dim3 grid((a.Mrows + 127) / 128, 1, nbatch);
    launch_k(conv_ffma_kernel<TX, TW, TY, 32>, grid, block, 0, st, a);
  } else {
    dim3 grid((a.Mrows + 63) / 64, (a.Ncols + 63) / 64, nbatch);
    launch_k(conv_ffma_kernel<TX, TW, TY, 64>, grid, block, 0, st, a);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

static bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

int conv_geometry(int kind, int dims, ConvGeom* g) {
  ConvGeom z = {1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 1, 1, 1};
  const int k3d = dims == 3 ? 3 : 1, k2d = dims == 3 ? 2 : 1;
  switch (kind) {
    case B200SEG_K3: z.kd = k3d; z.kh = 3; z.kw = 3; z.pd = dims == 3 ? 1 : 0; z.ph = 1; z.pw = 1; break;
    case B200SEG_K1: break;
    case B200SEG_DOWN: z.kd = k2d; z.kh = 2; z.kw = 2; z.sd = k2d; z.sh = 2; z.sw = 2; break;
    case B200SEG_UP: z.up = 1; z.ud = k2d; z.uh = 2; z.uw = 2; break;
    default: return -1;
  }
  *g = z;
  return 0;
}

template <typename TX, typename TW, typename TY>
static int conv_typed(int kind, int dims, const b200seg_tensor* x, const void* wpk, const float* bias,
                      const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, cudaStream_t st) {
  ConvArgs<TX, TW, TY> a;
  if (conv_geometry(kind, dims, &a.g) != 0) {
    set_error("b200seg_conv: bad kind %d", kind);
    return B200SEG_EINVAL;
  }
  a.x = static_cast<const TX*>(x->ptr);
  a.w = static_cast<const TW*>(wpk);
  a.bias = bias;
  a.y = static_cast<TY*>(y->ptr);
  a.addend = addend ? static_cast<const TY*>(addend->ptr) : nullptr;
  a.stats = stats;
  a.XD = x->d; a.XH = x->h; a.XW = x->w; a.xld = x->ld;
  a.yld = y->ld;
  a.ald = addend ? addend->ld : 0;
  a.Cin = x->c;
  a.Cout = y->c;
  if (a.g.up) {
    a.OD = x->d; a.OH = x->h; a.OW = x->w;
    a.Ncols = a.g.ud * a.g.uh * a.g.uw * a.Cout;
    B200_CHECK_ARG(y->d == x->d * a.g.ud && y->h == x->h * 2 && y->w == x->w * 2,
                   "b200seg_conv(UP): output dims must be 2x the input dims");
  } else {
    a.OD = y->d; a.OH = y->h; a.OW = y->w;
    a.Ncols = a.Cout;
    B200_CHECK_ARG(x->d == y->d * a.g.sd && x->h == y->h * a.g.sh && x->w == y->w * a.g.sw,
                   "b200seg_conv: input/output spatial dims do not match kind %d", kind);
  }
  a.Mrows = a.OD * a.OH * a.OW;
  a.xvec = (a.Cin % 4 == 0) && (x->ld % 4 == 0) && aligned(x->ptr, sizeof(TX) * 4);
  a.wvec = (a.Ncols % 4 == 0) && aligned(wpk, sizeof(TW) * 4);
  a.yvec = (a.Cout % 4 == 0) && (y->ld % 4 == 0) && aligned(y->ptr, sizeof(TY) * 4);
  a.avec = addend ? ((a.Cout % 4 == 0) && (addend->ld % 4 == 0) && aligned(addend->ptr, sizeof(TY) * 4)) : 0;
  return launch_conv(a, x->n, st);
}

int conv_generic(int kind, int dims, const b200seg_tensor* x, const void* wpk, int w_dtype, const float* bias,
                 const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, cudaStream_t st) {
  B200_CHECK_ARG(x && y && wpk, "b200seg_conv: null tensor");
  B200_CHECK_ARG(x->n == y->n, "b200seg_conv: batch mismatch");
  if (addend) {
    B200_CHECK_ARG(same_geom(addend, y) && addend->dtype == y->dtype, "b200seg_conv: addend must match y");
  }
  const int xd = x->dtype, yd = y->dtype;
  if (w_dtype == B200SEG_F32) {
    B200_CHECK_ARG(xd == B200SEG_F32 && yd == B200SEG_F32, "b200seg_conv: fp32 weights need fp32 x and y");
    return conv_typed<float, float, float>(kind, dims, x, wpk, bias, y, stats, addend, st);
  }
  if (xd == B200SEG_BF16 && yd == B200SEG_BF16)
    return conv_typed<bf16, bf16, bf16>(kind, dims, x, wpk, bias, y, stats, addend, st);
  if (xd == B200SEG_F32 && yd == B200SEG_BF16)
    return conv_typed<float, bf16, bf16>(kind, dims, x, wpk, bias, y, stats, addend, st);
  if (xd == B200SEG_BF16 && yd == B200SEG_F32)
    return conv_typed<bf16, bf16, float>(kind, dims, x, wpk, bias, y, stats, addend, st);
  return conv_typed<float, bf16, float>(kind, dims, x, wpk, bias, y, stats, addend, st);
}

}  // namespace b200seg
