// CUDA-core kernels for the layers that are NOT dense MMAs (sm_90a): the stem (Cin = image channels, 1..4)
// and the head (Cout = number of classes, 1..8).  These layers move full-resolution tensors with a
// handful of FLOPs per byte, so they are written as HBM-streaming stencil / pointwise kernels:
// one thread per voxel, 128-bit channel-vector stores/loads, weights in shared memory.
//
//   conv_smallcin_kernel   : 3x3x3 / 3x3 / 1x1 conv, Cin <= 4 -> Cout in {8,16,24,32}; fused bias + GroupNorm
//                            statistics (VNet3d.py:28-29 in_tr.conv1/conv2; Unet3d.py:67 enc1conv1)
//   wgrad_smallcin_kernel  : its weight gradient, dwp[t][ci][co] += sum_v x[v+t][ci] * dy[v][co]
//   head_fwd_kernel        : 1x1 conv Cin -> numclass + bias + sigmoid / softmax in one pass
//                            (VNet3d.py:94-98 out_tr; Unet3d.py:56-61)
//   head_bwd_kernel        : dX = dlogits * W, dW += dlogits^T * X, db += sum dlogits in one pass
#include "common.cuh"

namespace b200seg {

// ------------------------------------------------------------------------------------------------
// stem forward
// ------------------------------------------------------------------------------------------------
template <typename TX, typename TW, typename TY, int COUT>
__global__ void __launch_bounds__(256) conv_smallcin_kernel(const TX* __restrict__ x, long long xld,
                                                            const TW* __restrict__ w, const float* __restrict__ bias,
                                                            TY* __restrict__ y, long long yld,
                                                            double* __restrict__ stats, int D, int H, int W, int Cin,
                                                            int kd, int kh, int kw, int pd, int ph, int pw) {
  PDL_ENTER();
  extern __shared__ float s_w[];                  // [taps*Cin][COUT] + [COUT] bias + stats scratch
  const int taps = kd * kh * kw;
  const int nw = taps * Cin * COUT;
  float* s_b = s_w + nw;
  float* s_red = s_b + COUT;                      // [8 warps][2*COUT]
  for (int i = threadIdx.x; i < nw; i += blockDim.x) s_w[i] = to_f(w[i]);
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) s_b[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int n = blockIdx.y;
  const long long V = (long long)D * H * W;
  const TX* xb = x + (long long)n * V * xld;
  float ssum[COUT], ssq[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) ssum[c] = ssq[c] = 0.f;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < V; v += (long long)gridDim.x * blockDim.x) {
    const int vi = (int)v;                 // voxels per sample < 2^31: 32-bit decode
    const int ow = vi % W;
    const int t2 = vi / W;
    const int oh = t2 % H;
    const int od = t2 / H;
    float acc[COUT];
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = s_b[c];
    int tap = 0;
    for (int a = 0; a < kd; ++a) {
      const int id = od + a - pd;
      for (int b = 0; b < kh; ++b) {
        const int ih = oh + b - ph;
        for (int cc = 0; cc < kw; ++cc, ++tap) {
          const int iw = ow + cc - pw;
          if ((unsigned)id >= (unsigned)D || (unsigned)ih >= (unsigned)H || (unsigned)iw >= (unsigned)W) continue;
          const TX* px = xb + (((long long)id * H + ih) * W + iw) * xld;
          for (int ci = 0; ci < Cin; ++ci) {
            const float xv = to_f(px[ci]);
            const float4* wr = reinterpret_cast<const float4*>(s_w + (tap * Cin + ci) * COUT);
#pragma unroll
            for (int c4 = 0; c4 < COUT / 4; ++c4) {
              const float4 wv = wr[c4];
              acc[4 * c4 + 0] = fmaf(xv, wv.x, acc[4 * c4 + 0]);
              acc[4 * c4 + 1] = fmaf(xv, wv.y, acc[4 * c4 + 1]);
              acc[4 * c4 + 2] = fmaf(xv, wv.z, acc[4 * c4 + 2]);
              acc[4 * c4 + 3] = fmaf(xv, wv.w, acc[4 * c4 + 3]);
            }
          }
        }
      }
    }
    TY* py = y + ((long long)n * V + v) * yld;
#pragma unroll
    for (int c4 = 0; c4 < COUT / 4; ++c4)
      store4(py + 4 * c4, make_float4(acc[4 * c4], acc[4 * c4 + 1], acc[4 * c4 + 2], acc[4 * c4 + 3]));
    if (stats != nullptr) {
#pragma unroll
      for (int c = 0; c < COUT; ++c) {
        ssum[c] += acc[c];
        ssq[c] = fmaf(acc[c], acc[c], ssq[c]);
      }
    }
  }
  if (stats != nullptr) {
    // fixed-order: warp shuffle, one row per warp in smem, then fp64 over the warps
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < COUT; ++c) {
      const float a = warp_sum(ssum[c]);
      const float b = warp_sum(ssq[c]);
      if (lane == 0) {
        s_red[wid * 2 * COUT + c] = a;
        s_red[wid * 2 * COUT + COUT + c] = b;
      }
    }
    __syncthreads();
    if (threadIdx.x < 2 * COUT) {
      double t = 0.0;
      for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += (double)s_red[k * 2 * COUT + threadIdx.x];
      const int which = threadIdx.x / COUT, c = threadIdx.x - which * COUT;
      atomicAdd(stats + ((long long)n * COUT + c) * 2 + which, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// stem weight gradient.  dwp[t][ci][co] += sum_v x[v+t][ci] * dy[v][co]  with Cin <= 4.
// Lane <-> role r = (tap, ci); one voxel per group of ceil(R/32) warps at a time: all lanes of a warp read the
// SAME dy row (one broadcast transaction of COUT channels) and each its own shifted x element, so every
// thread keeps COUT accumulators for its (tap, ci) pair; nothing is staged, the reads stream through L1.
// ------------------------------------------------------------------------------------------------
template <typename TA, typename TB, int COUT>
__global__ void __launch_bounds__(256) wgrad_smallcin_kernel(const TA* __restrict__ a, long long ald,
                                                             const TB* __restrict__ b, long long bld,
                                                             float* __restrict__ dwp, int N, int D, int H, int W,
                                                             int Cin, int kd, int kh, int kw, int pd, int ph, int pw) {
  PDL_ENTER();
  __shared__ float s_red[8][32][COUT + 1];
  const int taps = kd * kh * kw;
  const int R = taps * Cin;
  const int wpv = (R + 31) / 32;                  // warps cooperating on one voxel
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int vslot = wid / wpv;                    // voxel slot of this warp inside the block
  const int slots = 8 / wpv;                      // voxels processed per block iteration
  const int r = (wid % wpv) * 32 + lane;          // role
  const bool active = r < R && vslot < slots;
  const int tap = active ? r / Cin : 0, ci = active ? r - tap * Cin : 0;
  const int cw = tap % kw - pw, ch_ = (tap / kw) % kh - ph, cd = tap / (kw * kh) - pd;
  const long long V = (long long)D * H * W;
  const long long NV = (long long)N * V;
  float acc[COUT];
#pragma unroll
  for (int c = 0; c < COUT; ++c) acc[c] = 0.f;
  if (vslot < slots) {
    // each voxel slot walks a contiguous chunk: coordinates advance incrementally (no per-voxel division)
    const long long nslots = (long long)gridDim.x * slots;
    const long long chunk = (NV + nslots - 1) / nslots;
    long long gv = ((long long)blockIdx.x * slots + vslot) * chunk;
    long long gend = gv + chunk < NV ? gv + chunk : NV;
    if (gv < gend) {
      int n = (int)(gv / V);
      long long o = gv - (long long)n * V;
      int ow = (int)(o % W), oh = (int)((o / W) % H), od = (int)(o / ((long long)W * H));
      const TB* pb = b + gv * bld;
      // 4 voxels per trip: their x / dy loads are all issued before the first FMA (latency overlap)
      while (gv < gend) {
        float xv[4];
        float4 dv[4][COUT / 4];
        int cnt = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          xv[u] = 0.f;
          if (gv + u < gend) {
            const int id = od + cd, ih = oh + ch_, iw = ow + cw;
            if (active && (unsigned)id < (unsigned)D && (unsigned)ih < (unsigned)H && (unsigned)iw < (unsigned)W)
              xv[u] = to_f(a[((((long long)n * D + id) * H + ih) * W + iw) * ald + ci]);
#pragma unroll
            for (int c4 = 0; c4 < COUT / 4; ++c4) dv[u][c4] = load4(pb + (long long)u * bld + 4 * c4);
            ++cnt;
            if (++ow == W) {
              ow = 0;
              if (++oh == H) {
                oh = 0;
                if (++od == D) {
                  od = 0;
                  ++n;
                }
              }
            }
          } else {
#pragma unroll
            for (int c4 = 0; c4 < COUT / 4; ++c4) dv[u][c4] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
          for (int c4 = 0; c4 < COUT / 4; ++c4) {
            acc[4 * c4 + 0] = fmaf(xv[u], dv[u][c4].x, acc[4 * c4 + 0]);
            acc[4 * c4 + 1] = fmaf(xv[u], dv[u][c4].y, acc[4 * c4 + 1]);
            acc[4 * c4 + 2] = fmaf(xv[u], dv[u][c4].z, acc[4 * c4 + 2]);
            acc[4 * c4 + 3] = fmaf(xv[u], dv[u][c4].w, acc[4 * c4 + 3]);
          }
        }
        gv += cnt;
        pb += (long long)cnt * bld;
      }
    }
  }
  // fold the voxel slots: role r of every slot -> one atomic per (role, channel) per block
#pragma unroll
  for (int c = 0; c < COUT; ++c) s_red[wid][lane][c] = active ? acc[c] : 0.f;
  __syncthreads();
  for (int i = threadIdx.x; i < wpv * 32 * COUT; i += blockDim.x) {
    const int c = i % COUT;
    const int rr = i / COUT;                      // role
    if (rr >= R) continue;
    const int w_in = rr / 32, l = rr % 32;
    float t = 0.f;
    for (int sl = 0; sl < slots; ++sl) t += s_red[sl * wpv + w_in][l][c];
    atomicAdd(dwp + (long long)rr * COUT + c, t);
  }
}

// ------------------------------------------------------------------------------------------------
// head forward: logits = W x + b (fp32), probs = sigmoid / softmax(logits)
// ------------------------------------------------------------------------------------------------
template <typename TX, int NC>
__global__ void __launch_bounds__(256) head_fwd_kernel(const TX* __restrict__ x, long long xld, int Cin,
                                                       const float* __restrict__ w /*[NC][Cin]*/,
                                                       const float* __restrict__ bias, float* __restrict__ logits,
                                                       float* __restrict__ probs, long long NV) {
  PDL_ENTER();
  extern __shared__ float s_hw[];                 // [NC][Cin] + [NC]
  for (int i = threadIdx.x; i < NC * Cin; i += blockDim.x) s_hw[i] = w[i];
  for (int i = threadIdx.x; i < NC; i += blockDim.x) s_hw[NC * Cin + i] = bias ? bias[i] : 0.f;
  __syncthreads();
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < NV; v += (long long)gridDim.x * blockDim.x) {
    float z[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) z[c] = s_hw[NC * Cin + c];
    const TX* px = x + v * xld;
    for (int k = 0; k < Cin; k += 4) {
      const float4 xv = load4(px + k);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const float4 wv = *reinterpret_cast<const float4*>(s_hw + c * Cin + k);
        z[c] = fmaf(xv.x, wv.x, z[c]);
        z[c] = fmaf(xv.y, wv.y, z[c]);
        z[c] = fmaf(xv.z, wv.z, z[c]);
        z[c] = fmaf(xv.w, wv.w, z[c]);
      }
    }
    float p[NC];
    if (NC == 1) {
      p[0] = 1.f / (1.f + expf(-z[0]));
    } else {
      float mx = z[0];
#pragma unroll
      for (int c = 1; c < NC; ++c) mx = fmaxf(mx, z[c]);
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        p[c] = expf(z[c] - mx);
        s += p[c];
      }
      const float inv = 1.f / s;
#pragma unroll
      for (int c = 0; c < NC; ++c) p[c] *= inv;
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) logits[v * NC + c] = z[c];
    if (probs != nullptr) {           // a captured training step that reads the accuracy from the loss pass skips it
#pragma unroll
      for (int c = 0; c < NC; ++c) probs[v * NC + c] = p[c];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// head backward: dX[v][k] = sum_c dl[v][c] W[c][k];  dW[c][k] += sum_v dl[v][c] X[v][k];  db[c] += sum_v dl[v][c]
// ------------------------------------------------------------------------------------------------
template <typename TX, int NC, int CIN>
__global__ void __launch_bounds__(256) head_bwd_kernel(const TX* __restrict__ x, long long xld,
                                                       const float* __restrict__ dl, const float* __restrict__ w,
                                                       TX* __restrict__ dx, long long dxld, float* __restrict__ dw,
                                                       float* __restrict__ db, long long NV) {
  PDL_ENTER();
  __shared__ float s_hw[NC * CIN];
  __shared__ float s_acc[8][NC * CIN + NC];
  for (int i = threadIdx.x; i < NC * CIN; i += blockDim.x) s_hw[i] = w[i];
  __syncthreads();
  float aw[NC][CIN];
  float ab[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    ab[c] = 0.f;
#pragma unroll
    for (int k = 0; k < CIN; ++k) aw[c][k] = 0.f;
  }
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < NV; v += (long long)gridDim.x * blockDim.x) {
    float g[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      g[c] = dl[v * NC + c];
      ab[c] += g[c];
    }
    const TX* px = x + v * xld;
    TX* pd = dx + v * dxld;
#pragma unroll
    for (int k = 0; k < CIN; k += 4) {
      const float4 xv = load4(px + k);
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
      float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < NC; ++c) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          aw[c][k + j] = fmaf(g[c], xs[j], aw[c][k + j]);
          o[j] = fmaf(g[c], s_hw[c * CIN + k + j], o[j]);
        }
      }
      store4(pd + k, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
#pragma unroll
    for (int k = 0; k < CIN; ++k) {
      const float t = warp_sum(aw[c][k]);
      if (lane == 0) s_acc[wid][c * CIN + k] = t;
    }
    const float t = warp_sum(ab[c]);
    if (lane == 0) s_acc[wid][NC * CIN + c] = t;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NC * CIN + NC; i += blockDim.x) {
    float t = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += s_acc[k][i];
    if (i < NC * CIN) atomicAdd(dw + i, t);
    else atomicAdd(db + (i - NC * CIN), t);
  }
}

// ------------------------------------------------------------------------------------------------
// host dispatch
// ------------------------------------------------------------------------------------------------
static bool al16s(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

int smallcin_conv_supported(int kind, const b200seg_tensor* x, const b200seg_tensor* y, const b200seg_tensor* addend) {
  if (kind != B200SEG_K3 && kind != B200SEG_K1) return 0;
  if (addend != nullptr) return 0;
  if (x->c > 4) return 0;
  if (y->c != 8 && y->c != 16 && y->c != 24 && y->c != 32) return 0;
  if ((y->ld % 8) || !al16s(y->ptr)) return 0;
  if (x->d != y->d || x->h != y->h || x->w != y->w) return 0;
  return 1;
}

template <typename TX, typename TW, typename TY>
static int smallcin_conv_typed(const ConvGeom& g, const b200seg_tensor* x, const void* w, const float* bias,
                               const b200seg_tensor* y, double* stats, int device, cudaStream_t st) {
  const long long V = (long long)x->d * x->h * x->w;
  const int taps = g.kd * g.kh * g.kw;
  long long blocks = (V + 255) / 256;
  const long long cap = ((long long)num_sms(device) * 8 + x->n - 1) / x->n;
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks, x->n);
#define LAUNCH_SC(CO)                                                                                              \
  launch_k(conv_smallcin_kernel<TX, TW, TY, CO>, grid, 256, (taps * x->c * CO + CO + 8 * 2 * CO) * sizeof(float), st, \
      static_cast<const TX*>(x->ptr), x->ld, static_cast<const TW*>(w), bias, static_cast<TY*>(y->ptr), y->ld,     \
      stats, x->d, x->h, x->w, x->c, g.kd, g.kh, g.kw, g.pd, g.ph, g.pw)
  switch (y->c) {
    case 8: LAUNCH_SC(8); break;
    case 16: LAUNCH_SC(16); break;
    case 24: LAUNCH_SC(24); break;
    default: LAUNCH_SC(32); break;
  }
#undef LAUNCH_SC
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int smallcin_conv(int kind, int dims, const b200seg_tensor* x, const void* w, int w_dtype, const float* bias,
                  const b200seg_tensor* y, double* stats, int device, cudaStream_t st) {
  ConvGeom g;
  conv_geometry(kind, dims, &g);
  const int xd = x->dtype, yd = y->dtype;
  if (w_dtype == B200SEG_F32) {
    B200_CHECK_ARG(xd == B200SEG_F32 && yd == B200SEG_F32, "smallcin_conv: fp32 weights need fp32 tensors");
    return smallcin_conv_typed<float, float, float>(g, x, w, bias, y, stats, device, st);
  }
  B200_CHECK_ARG(yd == B200SEG_BF16, "smallcin_conv: bf16 weights need a bf16 output");
  if (xd == B200SEG_F32) return smallcin_conv_typed<float, bf16, bf16>(g, x, w, bias, y, stats, device, st);
  return smallcin_conv_typed<bf16, bf16, bf16>(g, x, w, bias, y, stats, device, st);
}

int smallcin_wgrad_supported(int kind, const b200seg_tensor* a, const b200seg_tensor* b) {
  if (kind != B200SEG_K3 && kind != B200SEG_K1) return 0;
  if (a->c > 4) return 0;
  if (b->c != 8 && b->c != 16 && b->c != 24 && b->c != 32) return 0;
  if ((b->ld % 4) || !al16s(b->ptr)) return 0;
  if (b->dtype == B200SEG_BF16 && (b->ld % 8)) return 0;
  if (a->d != b->d || a->h != b->h || a->w != b->w) return 0;
  return 1;
}

template <typename TA, typename TB>
static int smallcin_wgrad_typed(const ConvGeom& g, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp,
                                int device, cudaStream_t st) {
  const long long NV = (long long)b->n * b->d * b->h * b->w;
  long long grid = (long long)num_sms(device) * 8;
  if (grid > NV) grid = NV;
#define LAUNCH_SW(CO)                                                                                        \
  launch_k(wgrad_smallcin_kernel<TA, TB, CO>, (unsigned)grid, 256, 0, st, \
      static_cast<const TA*>(a->ptr), a->ld, static_cast<const TB*>(b->ptr), b->ld, dwp, b->n, b->d, b->h,   \
      b->w, a->c, g.kd, g.kh, g.kw, g.pd, g.ph, g.pw)
  switch (b->c) {
    case 8: LAUNCH_SW(8); break;
    case 16: LAUNCH_SW(16); break;
    case 24: LAUNCH_SW(24); break;
    default: LAUNCH_SW(32); break;
  }
#undef LAUNCH_SW
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int smallcin_wgrad(int kind, int dims, const b200seg_tensor* a, const b200seg_tensor* b, float* dwp, int device,
                   cudaStream_t st) {
  ConvGeom g;
  conv_geometry(kind, dims, &g);
  if (a->dtype == B200SEG_F32 && b->dtype == B200SEG_F32) return smallcin_wgrad_typed<float, float>(g, a, b, dwp, device, st);
  if (a->dtype == B200SEG_F32 && b->dtype == B200SEG_BF16) return smallcin_wgrad_typed<float, bf16>(g, a, b, dwp, device, st);
  if (a->dtype == B200SEG_BF16 && b->dtype == B200SEG_BF16) return smallcin_wgrad_typed<bf16, bf16>(g, a, b, dwp, device, st);
  return smallcin_wgrad_typed<bf16, float>(g, a, b, dwp, device, st);
}

static int head_blocks(long long NV, int device) {
  long long blocks = (NV + 255) / 256;
  const long long cap = (long long)num_sms(device) * 8;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

template <typename TX>
static int head_fwd_typed(const b200seg_tensor* x, const float* w, const float* bias, float* logits, float* probs,
                          int nc, int device, cudaStream_t st) {
  const long long NV = (long long)x->n * x->d * x->h * x->w;
  const int blocks = head_blocks(NV, device);
  const size_t sm = (size_t)(nc * x->c + nc) * sizeof(float);
#define LAUNCH_HF(NC) \
  launch_k(head_fwd_kernel<TX, NC>, blocks, 256, sm, st, static_cast<const TX*>(x->ptr), x->ld, x->c, w, bias, logits, probs, NV)
  switch (nc) {
    case 1: LAUNCH_HF(1); break;
    case 2: LAUNCH_HF(2); break;
    case 3: LAUNCH_HF(3); break;
    case 4: LAUNCH_HF(4); break;
    case 5: LAUNCH_HF(5); break;
    case 6: LAUNCH_HF(6); break;
    case 7: LAUNCH_HF(7); break;
    default: LAUNCH_HF(8); break;
  }
#undef LAUNCH_HF
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int head_fwd(const b200seg_tensor* x, const float* w, const float* bias, float* logits, float* probs, int nc,
             int device, cudaStream_t st) {
  B200_CHECK_ARG(nc >= 1 && nc <= 8, "b200seg_head_fwd: 1..8 classes supported (got %d)", nc);
  B200_CHECK_ARG((x->c % 4) == 0 && (x->ld % 4) == 0 && al16s(x->ptr) && (x->dtype == B200SEG_F32 || (x->ld % 8) == 0),
                 "b200seg_head_fwd: input channels must be a multiple of 4 and 16-byte aligned");
  if (x->dtype == B200SEG_BF16) return head_fwd_typed<bf16>(x, w, bias, logits, probs, nc, device, st);
  return head_fwd_typed<float>(x, w, bias, logits, probs, nc, device, st);
}

template <typename TX, int CIN>
static int head_bwd_cin(const b200seg_tensor* x, const float* dl, const float* w, const b200seg_tensor* dx, float* dw,
                        float* db, int nc, int device, cudaStream_t st) {
  const long long NV = (long long)x->n * x->d * x->h * x->w;
  const int blocks = head_blocks(NV, device) / 2 + 1;
#define LAUNCH_HB(NC)                                                                                          \
  launch_k(head_bwd_kernel<TX, NC, CIN>, blocks, 256, 0, st, static_cast<const TX*>(x->ptr), x->ld, dl, w,           \
                                                       static_cast<TX*>(dx->ptr), dx->ld, dw, db, NV)
  switch (nc) {
    case 1: LAUNCH_HB(1); break;
    case 2: LAUNCH_HB(2); break;
    case 3: LAUNCH_HB(3); break;
    case 4: LAUNCH_HB(4); break;
    default:
      set_error("b200seg_head_bwd: fused path supports 1..4 classes");
      return B200SEG_EINVAL;
  }
#undef LAUNCH_HB
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int head_bwd_supported(const b200seg_tensor* x, int nc) { return nc >= 1 && nc <= 4 && (x->c == 16 || x->c == 32); }

int head_bwd(const b200seg_tensor* x, const float* dl, const float* w, const b200seg_tensor* dx, float* dw, float* db,
             int nc, int device, cudaStream_t st) {
  B200_CHECK_ARG(head_bwd_supported(x, nc), "b200seg_head_bwd: unsupported shape (Cin=%d, classes=%d)", x->c, nc);
  B200_CHECK_ARG(same_geom(x, dx) && x->dtype == dx->dtype, "b200seg_head_bwd: x/dx mismatch");
  B200_CHECK_ARG((x->ld % 4) == 0 && (dx->ld % 4) == 0 && al16s(x->ptr) && al16s(dx->ptr) &&
                     (x->dtype == B200SEG_F32 || ((x->ld % 8) == 0 && (dx->ld % 8) == 0)),
                 "b200seg_head_bwd: tensors must be 16-byte aligned");
  if (x->dtype == B200SEG_BF16) {
    if (x->c == 16) return head_bwd_cin<bf16, 16>(x, dl, w, dx, dw, db, nc, device, st);
    return head_bwd_cin<bf16, 32>(x, dl, w, dx, dw, db, nc, device, st);
  }
  if (x->c == 16) return head_bwd_cin<float, 16>(x, dl, w, dx, dw, db, nc, device, st);
  return head_bwd_cin<float, 32>(x, dl, w, dx, dw, db, nc, device, st);
}

}  // namespace b200seg
