// Fused segmentation losses (sm_90a): ONE reduction pass over logits + labels producing every
// partial sum the Dice / BCE / CE / focal family needs, a scalar finalize, and ONE elementwise
// backward pass writing d loss / d logits (closed forms: SURVEY.md App. C; reference formulas:
// model/losses.py:43-53,141-147,160-181,252-260,273-285,301-325).
// logits: fp32 channels-last [N][vox][C]; labels: int64 [N][vox] (read as-is, 8 B/voxel); the binary losses also
// take fp32 soft targets (``y_true.float()``, model/losses.py:47,144).
// The same pass also produces (optionally) the per-sample sums of the reference's per-step accuracy
// (model/metric.py:146-181 dice_coeff / iou_coeff / multiclass_dice_coeff on the thresholded probabilities), so the
// training step needs no separate read of ``probs`` for it, and counts labels outside [0, C) (the reference raises
// in F.one_hot / F.cross_entropy; here the count lands in ``part`` and the host raises).
#include "common.cuh"

namespace b200seg {


__device__ __forceinline__ double block_reduce_to_global(double v, double* dst, double* s_tmp) {
  // warp shuffle -> one smem slot per warp -> thread 0 adds to global
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_tmp[wid] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += s_tmp[i];
    atomicAdd(dst, t);
  }
  __syncthreads();
  return v;
}

__device__ __forceinline__ float softplus_neg_abs(float z) { return log1pf(expf(-fabsf(z))); }

// ---- binary (C == 1): I = sum p t, P = sum p, T = sum t, sum bce, sum alpha (1-pt)^gamma bce, V, bad
// grid = (blocks per sample, N); metric[n][0] = {sum [p>.5] t, sum [p>.5], sum t}
template <typename TL>
__global__ void __launch_bounds__(256) loss_partials_binary_kernel(const float* __restrict__ z,
                                                                   const TL* __restrict__ t, long long vox,
                                                                   float gamma, float alpha_f,
                                                                   double* __restrict__ part,
                                                                   double* __restrict__ metric) {
  PDL_ENTER();
  __shared__ double s_tmp[8];
  const long long base = (long long)blockIdx.y * vox;
  float aI = 0.f, aP = 0.f, aT = 0.f, aB = 0.f, aF = 0.f, mI = 0.f, mA = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < vox;
       i += (long long)gridDim.x * blockDim.x) {
    float zi = z[base + i];
    float ti = (float)t[base + i];
    float p = 1.f / (1.f + expf(-zi));
    float b = fmaxf(zi, 0.f) - zi * ti + softplus_neg_abs(zi);
    float pt = expf(-b);
    aI = fmaf(p, ti, aI);
    aP += p;
    aT += ti;
    aB += b;
    aF += alpha_f * powf(1.f - pt, gamma) * b;
    if (p > 0.5f) {
      mI += ti;
      mA += 1.f;
    }
  }
  block_reduce_to_global((double)aI, part + 0, s_tmp);
  block_reduce_to_global((double)aP, part + 1, s_tmp);
  block_reduce_to_global((double)aT, part + 2, s_tmp);
  block_reduce_to_global((double)aB, part + 3, s_tmp);
  block_reduce_to_global((double)aF, part + 4, s_tmp);
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(part + 5, (double)vox);
  if (metric != nullptr) {
    double* m = metric + (long long)blockIdx.y * 3;
    block_reduce_to_global((double)mI, m + 0, s_tmp);
    block_reduce_to_global((double)mA, m + 1, s_tmp);
    block_reduce_to_global((double)aT, m + 2, s_tmp);
  }
}

// ---- multi-class, C <= kMaxC in registers; grid = (blocks per sample, N)
// metric[n][c] = {sum [p_c>.5][t==c], sum [p_c>.5], sum [t==c]}; part[3C+3] += labels outside [0, C)
template <int C>
__global__ void __launch_bounds__(256) loss_partials_multi_kernel(const float* __restrict__ z,
                                                                  const long long* __restrict__ t, long long vox,
                                                                  float gamma, double* __restrict__ part,
                                                                  double* __restrict__ metric) {
  PDL_ENTER();
  __shared__ double s_tmp[8];
  const long long base = (long long)blockIdx.y * vox;
  float aI[C], aP[C], aN[C], mI[C], mA[C];
  float aNll = 0.f, aF = 0.f, aBad = 0.f;
#pragma unroll
  for (int c = 0; c < C; ++c) aI[c] = aP[c] = aN[c] = mI[c] = mA[c] = 0.f;
  for (long long ii = blockIdx.x * (long long)blockDim.x + threadIdx.x; ii < vox;
       ii += (long long)gridDim.x * blockDim.x) {
    const long long i = base + ii;
    float v[C];
    if (C == 2) {
      float2 q = *reinterpret_cast<const float2*>(z + i * 2);
      v[0] = q.x; v[1] = q.y;
    } else if (C == 4) {
      float4 q = *reinterpret_cast<const float4*>(z + i * 4);
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) v[c] = z[i * C + c];
    }
    const long long tl = t[i];
    if (tl < 0 || tl >= C) {          // the reference raises (F.one_hot / F.cross_entropy); flagged for the host
      aBad += 1.f;
      continue;
    }
    const int ti = (int)tl;
    float mx = v[0];
#pragma unroll
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, v[c]);
    float s = 0.f, e[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      e[c] = expf(v[c] - mx);
      s += e[c];
    }
    const float inv = 1.f / s;
    const float lse = mx + logf(s);
    float zt = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float p = e[c] * inv;
      const bool hit = (c == ti);
      const bool on = p > 0.5f;
      aP[c] += p;
      if (on) mA[c] += 1.f;
      if (hit) {
        aI[c] += p;
        aN[c] += 1.f;
        zt = v[c];
        if (on) mI[c] += 1.f;
      }
    }
    const float nll = lse - zt;
    const float ptt = expf(-nll);
    aNll += nll;
    aF += powf(1.f - ptt, gamma) * nll;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    block_reduce_to_global((double)aI[c], part + c, s_tmp);
    block_reduce_to_global((double)aP[c], part + C + c, s_tmp);
    block_reduce_to_global((double)aN[c], part + 2 * C + c, s_tmp);
  }
  block_reduce_to_global((double)aNll, part + 3 * C, s_tmp);
  block_reduce_to_global((double)aF, part + 3 * C + 1, s_tmp);
  block_reduce_to_global((double)aBad, part + 3 * C + 3, s_tmp);
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(part + 3 * C + 2, (double)vox);
  if (metric != nullptr) {
    double* m = metric + (long long)blockIdx.y * C * 3;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      block_reduce_to_global((double)mI[c], m + 3 * c + 0, s_tmp);
      block_reduce_to_global((double)mA[c], m + 3 * c + 1, s_tmp);
      block_reduce_to_global((double)aN[c], m + 3 * c + 2, s_tmp);
    }
  }
}

// ---- multi-class, any C (<= 1024): per-class sums through shared-memory atomics
__global__ void __launch_bounds__(256) loss_partials_multi_generic_kernel(const float* __restrict__ z,
                                                                          const long long* __restrict__ t,
                                                                          long long vox, int C, float gamma,
                                                                          double* __restrict__ part,
                                                                          double* __restrict__ metric) {
  PDL_ENTER();
  extern __shared__ float s_acc[];   // [3*C + 2] loss sums, [1] bad labels, [2*C] metric
  const int NS = 5 * C + 3;
  for (int i = threadIdx.x; i < NS; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  float* s_bad = s_acc + 3 * C + 2;
  float* s_mI = s_bad + 1;
  float* s_mA = s_mI + C;
  const long long base = (long long)blockIdx.y * vox;
  for (long long ii = blockIdx.x * (long long)blockDim.x + threadIdx.x; ii < vox;
       ii += (long long)gridDim.x * blockDim.x) {
    const long long i = base + ii;
    const float* zi = z + i * C;
    const long long tl = t[i];
    if (tl < 0 || tl >= C) {
      atomicAdd(s_bad, 1.f);
      continue;
    }
    const int ti = (int)tl;
    float mx = zi[0];
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, zi[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(zi[c] - mx);
    const float inv = 1.f / s, lse = mx + logf(s);
    for (int c = 0; c < C; ++c) {
      const float p = expf(zi[c] - mx) * inv;
      atomicAdd(&s_acc[C + c], p);
      if (p > 0.5f) atomicAdd(&s_mA[c], 1.f);
      if (c == ti) {
        atomicAdd(&s_acc[c], p);
        atomicAdd(&s_acc[2 * C + c], 1.f);
        if (p > 0.5f) atomicAdd(&s_mI[c], 1.f);
      }
    }
    const float nll = lse - zi[ti];
    atomicAdd(&s_acc[3 * C], nll);
    atomicAdd(&s_acc[3 * C + 1], powf(1.f - expf(-nll), gamma) * nll);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * C + 2; i += blockDim.x) atomicAdd(part + i, (double)s_acc[i]);
  if (threadIdx.x == 0 && s_bad[0] != 0.f) atomicAdd(part + 3 * C + 3, (double)s_bad[0]);
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(part + 3 * C + 2, (double)vox);
  if (metric != nullptr) {
    double* m = metric + (long long)blockIdx.y * C * 3;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      atomicAdd(m + 3 * c + 0, (double)s_mI[c]);
      atomicAdd(m + 3 * c + 1, (double)s_mA[c]);
      atomicAdd(m + 3 * c + 2, (double)s_acc[2 * C + c]);
    }
  }
}

// ---- per-step accuracy from the per-sample sums (model/metric.py:146-181): out[0] = dice_coeff (C == 1) or
// multiclass_dice_coeff (mean over classes 1..C-1 of the per-sample-mean Dice), out[1] = the iou_coeff analogue
__global__ void metric_finalize_kernel(const double* __restrict__ metric, int N, int C, float* __restrict__ out) {
  PDL_ENTER();
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const double s = 1e-5;
  double dice = 0.0, iou = 0.0;
  const int c0 = C == 1 ? 0 : 1;
  for (int c = c0; c < C; ++c) {
    double dc = 0.0, ic = 0.0;
    for (int n = 0; n < N; ++n) {
      const double* m = metric + ((long long)n * C + c) * 3;
      dc += (2.0 * m[0] + s) / (m[1] + m[2] + s);
      ic += (m[0] + s) / (m[1] + m[2] - m[0] + s);
    }
    dice += dc / N;
    iou += ic / N;
  }
  const int nc = C == 1 ? 1 : C - 1;
  out[0] = (float)(dice / nc);
  out[1] = (float)(iou / nc);
}

// ---- the same per-sample sums from materialised probabilities (drop-in dice_coeff(probs, y) etc.): probs fp32
// channels-last [N][vox][C]; labels int64 or fp32 (C == 1 only)
template <typename TL>
__global__ void __launch_bounds__(256) metric_partials_kernel(const float* __restrict__ p, const TL* __restrict__ t,
                                                              long long vox, int C, float thr,
                                                              double* __restrict__ metric) {
  PDL_ENTER();
  extern __shared__ float s_m[];     // [3*C]
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) s_m[i] = 0.f;
  __syncthreads();
  const long long base = (long long)blockIdx.y * vox;
  for (long long ii = blockIdx.x * (long long)blockDim.x + threadIdx.x; ii < vox;
       ii += (long long)gridDim.x * blockDim.x) {
    const long long i = base + ii;
    if (C == 1) {
      const float ti = (float)t[i];
      const bool on = p[i] > thr;
      if (on) {
        atomicAdd(&s_m[0], ti);
        atomicAdd(&s_m[1], 1.f);
      }
      if (ti != 0.f) atomicAdd(&s_m[2], ti);
    } else {
      const long long tl = (long long)t[i];
      for (int c = 0; c < C; ++c) {
        const bool on = p[i * C + c] > thr;
        const bool hit = tl == c;
        if (on) atomicAdd(&s_m[3 * c + 1], 1.f);
        if (hit) atomicAdd(&s_m[3 * c + 2], 1.f);
        if (on && hit) atomicAdd(&s_m[3 * c + 0], 1.f);
      }
    }
  }
  __syncthreads();
  double* m = metric + (long long)blockIdx.y * C * 3;
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x)
    if (s_m[i] != 0.f) atomicAdd(m + i, (double)s_m[i]);
}

// ---- finalize: one thread
__global__ void loss_finalize_kernel(const double* __restrict__ part, int C, int terms,
                                     const float* __restrict__ alpha, float gamma, float alpha_f,
                                     float* __restrict__ loss, float* __restrict__ lcoef) {
  PDL_ENTER();
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const double s = 1e-5, eps = 1e-7;
  double val = 0.0;
  if (C == 1) {
    const double I = part[0], P = part[1], T = part[2], sb = part[3], sf = part[4], V = part[5];
    double a = 0.0, b = 0.0;
    const double den = P + T + s;
    if (terms & B200SEG_LOSS_DICE) {
      const double dcl = den < eps ? eps : den;
      val += 1.0 - (2.0 * I + s) / dcl;
      a = -2.0 / den;
      b = (2.0 * I + s) / (den * den);
    }
    if (terms & B200SEG_LOSS_CE) val += sb / V;
    if (terms & B200SEG_LOSS_FOCAL) val += sf / V;
    lcoef[0] = (float)a;
    lcoef[1] = (float)b;
    lcoef[2] = (terms & B200SEG_LOSS_CE) ? (float)(1.0 / V) : 0.f;
    lcoef[3] = (terms & B200SEG_LOSS_FOCAL) ? (float)((double)alpha_f / V) : 0.f;
    lcoef[4] = gamma;
  } else {
    const double* I = part;
    const double* Ps = part + C;
    const double* Cn = part + 2 * C;
    const double snll = part[3 * C], sfoc = part[3 * C + 1], V = part[3 * C + 2];
    double K = 0.0;
    for (int c = 0; c < C; ++c) K += Cn[c] > 0.0 ? 1.0 : 0.0;
    for (int c = 0; c < C; ++c) {
      double a = 0.0, b = 0.0;
      if (terms & B200SEG_LOSS_DICE) {
        const double present = Cn[c] > 0.0 ? 1.0 : 0.0;
        const double D = Cn[c] + Ps[c];
        const double draw = (2.0 * I[c] + s) / (D + s);
        const double d = draw < eps ? eps : draw;
        const double al = alpha[c];
        val += -(d * present * al) / K;
        const double w = (draw >= eps) ? al * present / K : 0.0;
        a = -2.0 * w / (D + s);
        b = w * (2.0 * I[c] + s) / ((D + s) * (D + s));
      }
      lcoef[c] = (float)a;
      lcoef[C + c] = (float)b;
    }
    if (terms & B200SEG_LOSS_CE) val += snll / V;
    if (terms & B200SEG_LOSS_FOCAL) val += sfoc / V;
    lcoef[2 * C] = (terms & B200SEG_LOSS_CE) ? (float)(1.0 / V) : 0.f;
    lcoef[2 * C + 1] = (terms & B200SEG_LOSS_FOCAL) ? (float)(1.0 / V) : 0.f;
    lcoef[2 * C + 2] = gamma;
    if (part[3 * C + 3] > 0.0) val = __longlong_as_double(0x7ff8000000000000LL);   // labels outside [0, C)
  }
  loss[0] = (float)val;
}

// d/dce of (1-pt)^gamma * ce with pt = exp(-ce):  (1-pt)^gamma + gamma (1-pt)^(gamma-1) pt ce
// At om = 0 the limit is 1 for gamma = 0 ((1-pt)^0 = 1), pt ce for gamma = 1 and 0 for every other gamma > 0.
__device__ __forceinline__ float focal_factor(float ce, float gamma) {
  const float pt = expf(-ce);
  const float om = 1.f - pt;
  if (gamma == 2.f) return om * om + 2.f * om * pt * ce;
  if (om <= 0.f) return gamma == 0.f ? 1.f : (gamma == 1.f ? pt * ce : 0.f);
  return powf(om, gamma) + gamma * powf(om, gamma - 1.f) * pt * ce;
}

template <typename TL>
__global__ void __launch_bounds__(256) loss_bwd_binary_kernel(const float* __restrict__ z,
                                                              const TL* __restrict__ t, long long nvox,
                                                              const float* __restrict__ lcoef,
                                                              const float* __restrict__ gscale,
                                                              float* __restrict__ dz) {
  PDL_ENTER();
  const float a = lcoef[0], b = lcoef[1], cs = lcoef[2], fs = lcoef[3], gamma = lcoef[4];
  const float gs = gscale[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox;
       i += (long long)gridDim.x * blockDim.x) {
    const float zi = z[i];
    const float ti = (float)t[i];
    const float p = 1.f / (1.f + expf(-zi));
    float g = (ti * a + b) * p * (1.f - p) + cs * (p - ti);
    if (fs != 0.f) {
      const float bce = fmaxf(zi, 0.f) - zi * ti + softplus_neg_abs(zi);
      g += fs * focal_factor(bce, gamma) * (p - ti);
    }
    dz[i] = g * gs;
  }
}

template <int C>
__global__ void __launch_bounds__(256) loss_bwd_multi_kernel(const float* __restrict__ z,
                                                             const long long* __restrict__ t, long long nvox,
                                                             const float* __restrict__ lcoef,
                                                             const float* __restrict__ gscale,
                                                             float* __restrict__ dz) {
  PDL_ENTER();
  float a[C], b[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    a[c] = lcoef[c];
    b[c] = lcoef[C + c];
  }
  const float cs = lcoef[2 * C], fs = lcoef[2 * C + 1], gamma = lcoef[2 * C + 2];
  const float gs = gscale[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox;
       i += (long long)gridDim.x * blockDim.x) {
    float v[C], p[C], o[C];
#pragma unroll
    for (int c = 0; c < C; ++c) v[c] = z[i * C + c];
    const int ti = (int)t[i];
    float mx = v[0];
#pragma unroll
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, v[c]);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      p[c] = expf(v[c] - mx);
      s += p[c];
    }
    const float inv = 1.f / s;
    float dot = 0.f, zt = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      p[c] *= inv;
      const float gd = (c == ti ? a[c] : 0.f) + b[c];
      o[c] = gd;
      dot = fmaf(gd, p[c], dot);
      if (c == ti) zt = v[c];
    }
    float k = cs;
    if (fs != 0.f) {
      const float nll = mx + logf(s) - zt;
      k += fs * focal_factor(nll, gamma);
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float oh = (c == ti) ? 1.f : 0.f;
      dz[i * C + c] = (p[c] * (o[c] - dot) + k * (p[c] - oh)) * gs;
    }
  }
}

__global__ void __launch_bounds__(256) loss_bwd_multi_generic_kernel(const float* __restrict__ z,
                                                                     const long long* __restrict__ t,
                                                                     long long nvox, int C,
                                                                     const float* __restrict__ lcoef,
                                                                     const float* __restrict__ gscale,
                                                                     float* __restrict__ dz) {
  PDL_ENTER();
  const float cs = lcoef[2 * C], fs = lcoef[2 * C + 1], gamma = lcoef[2 * C + 2];
  const float gs = gscale[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox;
       i += (long long)gridDim.x * blockDim.x) {
    const float* zi = z + i * C;
    const long long tl = t[i];
    if (tl < 0 || tl >= C) {             // flagged by loss_partials (the host raises): no out-of-bounds read
      for (int c = 0; c < C; ++c) dz[i * C + c] = 0.f;
      continue;
    }
    const int ti = (int)tl;
    float mx = zi[0];
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, zi[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(zi[c] - mx);
    const float inv = 1.f / s;
    float dot = 0.f;
    for (int c = 0; c < C; ++c) {
      const float p = expf(zi[c] - mx) * inv;
      dot = fmaf((c == ti ? lcoef[c] : 0.f) + lcoef[C + c], p, dot);
    }
    float k = cs;
    if (fs != 0.f) k += fs * focal_factor(mx + logf(s) - zi[ti], gamma);
    for (int c = 0; c < C; ++c) {
      const float p = expf(zi[c] - mx) * inv;
      const float gd = (c == ti ? lcoef[c] : 0.f) + lcoef[C + c];
      dz[i * C + c] = (p * (gd - dot) + k * (p - (c == ti ? 1.f : 0.f))) * gs;
    }
  }
}

// ---- binary sensitivity-specificity (BinarySSLoss, model/losses.py:87-99): the binary sums with the two squared-error
// sums in place of the cross-entropy ones.  part = {I, P, T, sum (p-t)^2 t, sum (p-t)^2 (1-t), V, 0}; metric as above
template <typename TL>
__global__ void __launch_bounds__(256) loss_partials_ss_kernel(const float* __restrict__ z, const TL* __restrict__ t,
                                                               long long vox, double* __restrict__ part,
                                                               double* __restrict__ metric) {
  PDL_ENTER();
  __shared__ double s_tmp[8];
  const long long base = (long long)blockIdx.y * vox;
  float aI = 0.f, aP = 0.f, aT = 0.f, aF = 0.f, aB = 0.f, mI = 0.f, mA = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < vox;
       i += (long long)gridDim.x * blockDim.x) {
    const float zi = z[base + i];
    const float ti = (float)t[base + i];
    const float p = 1.f / (1.f + expf(-zi));
    const float d = p - ti;
    const float d2 = d * d;
    aI = fmaf(p, ti, aI);
    aP += p;
    aT += ti;
    aF = fmaf(d2, ti, aF);
    aB = fmaf(d2, 1.f - ti, aB);
    if (p > 0.5f) {
      mI += ti;
      mA += 1.f;
    }
  }
  block_reduce_to_global((double)aI, part + 0, s_tmp);
  block_reduce_to_global((double)aP, part + 1, s_tmp);
  block_reduce_to_global((double)aT, part + 2, s_tmp);
  block_reduce_to_global((double)aF, part + 3, s_tmp);
  block_reduce_to_global((double)aB, part + 4, s_tmp);
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(part + 5, (double)vox);
  if (metric != nullptr) {
    double* m = metric + (long long)blockIdx.y * 3;
    block_reduce_to_global((double)mI, m + 0, s_tmp);
    block_reduce_to_global((double)mA, m + 1, s_tmp);
    block_reduce_to_global((double)aT, m + 2, s_tmp);
  }
}

// torch.clamp(x, 0, 2): the value, and whether the gradient passes (clamp backward keeps it for 0 <= x <= 2)
__device__ __forceinline__ double clamp02(double x, bool* pass) {
  *pass = x >= 0.0 && x <= 2.0;
  return x < 0.0 ? 0.0 : (x > 2.0 ? 2.0 : x);
}

// ---- finalize of the Jaccard / exponential-log Dice / Tversky / sensitivity-specificity losses (one term bit each):
// the value and the lcoef layout of loss_finalize_kernel, so loss_bwd_*_kernel serve all but SS unchanged.
// TVERSKY: alpha_f = alpha, gamma = beta; SS: alpha_f = r.
__global__ void loss_finalize_ext_kernel(const double* __restrict__ part, int C, int terms,
                                         const float* __restrict__ alpha, float gamma, float alpha_f,
                                         float* __restrict__ loss, float* __restrict__ lcoef) {
  PDL_ENTER();
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const double s = 1e-5, eps = 1e-7;
  double val = 0.0;
  if (C == 1) {
    const double I = part[0], P = part[1], T = part[2];
    double a = 0.0, b = 0.0;
    bool pass = true;
    if (terms == B200SEG_LOSS_JACCARD) {                  // losses.py:26-30: 1 - (I+s) / max(P+T-I+s, eps)
      const double U = P + T - I + s;
      if (U >= eps) {
        val = 1.0 - (I + s) / U;
        a = -1.0 / U - (I + s) / (U * U);
        b = (I + s) / (U * U);
      } else {
        val = 1.0 - (I + s) / eps;
        a = -1.0 / eps;
      }
    } else if (terms == B200SEG_LOSS_ELDICE) {            // losses.py:72-74: clamp((-log(dsc+s))^0.3, 0, 2)
      const double D = P + T + s;
      const double Dc = D < eps ? eps : D;
      const double dsc = (2.0 * I + s) / Dc;
      const double u = -log(dsc + s);
      val = clamp02(pow(u, 0.3), &pass);
      if (pass) {
        const double k = -0.3 * pow(u, -0.7) / (dsc + s);      // d loss / d dsc
        a = 2.0 * k / Dc;
        b = D >= eps ? -k * (2.0 * I + s) / (D * D) : 0.0;
      }
    } else if (terms == B200SEG_LOSS_TVERSKY) {           // losses.py:120-126, fp = P-I, fn = T-I
      const double al = alpha_f, be = gamma;
      const double Dt = I + al * (P - I) + be * (T - I) + s;
      val = clamp02(1.0 - (I + s) / Dt, &pass);
      if (pass) {
        a = -1.0 / Dt + (I + s) * (1.0 - al - be) / (Dt * Dt);
        b = (I + s) * al / (Dt * Dt);
      }
    } else {                                              // SS, losses.py:94-99
      const double Sf = part[3], Sb = part[4], V = part[5], r = alpha_f;
      val = r * Sf / (s + T) + (1.0 - r) * Sb / (s + V - T);
      a = r / (s + T);                                    // loss_bwd_ss_kernel: fg and bg weights
      b = (1.0 - r) / (s + V - T);
    }
    lcoef[0] = (float)a;
    lcoef[1] = (float)b;
    lcoef[2] = 0.f;
    lcoef[3] = 0.f;
    lcoef[4] = 0.f;
  } else {                                                // ELDICE, losses.py:372-382
    const double* I = part;
    const double* Ps = part + C;
    const double* Cn = part + 2 * C;
    double K = 0.0, S = 0.0;
    for (int c = 0; c < C; ++c) {
      K += Cn[c] > 0.0 ? 1.0 : 0.0;
      const double draw = (2.0 * I[c] + s) / (Cn[c] + Ps[c] + s);
      const double d = draw < eps ? eps : draw;
      const double dice = Cn[c] > 0.0 ? d * (double)alpha[c] : 0.0;
      S += pow(-log(dice + s), 0.3);                      // absent classes add (-log s)^0.3
    }
    bool pass;
    val = clamp02(S / K, &pass);
    for (int c = 0; c < C; ++c) {
      double a = 0.0, b = 0.0;
      const double D = Cn[c] + Ps[c];
      const double draw = (2.0 * I[c] + s) / (D + s);
      if (pass && Cn[c] > 0.0 && draw >= eps) {
        const double al = alpha[c];
        const double dice = draw * al;
        const double k = -0.3 * pow(-log(dice + s), -0.7) / (dice + s) * al / K;    // d loss / d d_c
        a = 2.0 * k / (D + s);
        b = -k * (2.0 * I[c] + s) / ((D + s) * (D + s));
      }
      lcoef[c] = (float)a;
      lcoef[C + c] = (float)b;
    }
    lcoef[2 * C] = 0.f;
    lcoef[2 * C + 1] = 0.f;
    lcoef[2 * C + 2] = 0.f;
    if (part[3 * C + 3] > 0.0) val = __longlong_as_double(0x7ff8000000000000LL);   // labels outside [0, C)
  }
  loss[0] = (float)val;
}

// ---- BinarySSLoss backward: 2 (p-t) (r t / (s+T) + (1-r)(1-t) / (s+V-T)) p (1-p); lcoef[0..1] from the finalize
template <typename TL>
__global__ void __launch_bounds__(256) loss_bwd_ss_kernel(const float* __restrict__ z, const TL* __restrict__ t,
                                                          long long nvox, const float* __restrict__ lcoef,
                                                          const float* __restrict__ gscale, float* __restrict__ dz) {
  PDL_ENTER();
  const float wf = lcoef[0], wb = lcoef[1], gs = gscale[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox;
       i += (long long)gridDim.x * blockDim.x) {
    const float ti = (float)t[i];
    const float p = 1.f / (1.f + expf(-z[i]));
    const float g = 2.f * (p - ti) * (wf * ti + wb * (1.f - ti)) * p * (1.f - p);
    dz[i] = g * gs;
  }
}

static int loss_blocks(long long nvox_, int device) {
  long long blocks = (nvox_ + 256 * 4 - 1) / (256 * 4);
  long long cap = (long long)num_sms(device) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// blocks per sample for the (blocks, N) grids of the partial-sum kernels
static dim3 sample_grid(long long vox, int N, int device) {
  // blocks per SM over the whole grid: every block ends in one fp64 atomic per partial sum (15 for two classes) on
  // the SAME few addresses, so more blocks buy load parallelism and pay in serialised atomics
  const int bps = 4;
  long long per = (vox + 256 * 4 - 1) / (256 * 4);
  long long cap = ((long long)num_sms(device) * bps + N - 1) / N;
  if (per > cap) per = cap;
  if (per < 1) per = 1;
  return dim3((unsigned)per, (unsigned)N, 1);
}

int loss_partials(const float* logits, const void* labels, int label_dtype, int N, long long vox, int C, float gamma,
                  float alpha_f, double* part, double* metric, int device, cudaStream_t s) {
  B200_CHECK_ARG(C >= 1 && C <= 1024, "loss_partials: unsupported class count %d", C);
  B200_CHECK_ARG(N >= 1 && N <= 65535, "loss_partials: unsupported batch size %d", N);
  B200_CHECK_ARG(label_dtype == B200SEG_I64 || (label_dtype == B200SEG_F32 && C == 1),
                 "loss_partials: labels must be int64 (fp32 soft targets only for the binary losses)");
  const dim3 grid = sample_grid(vox, N, device);
  const long long* tl = static_cast<const long long*>(labels);
  switch (C) {
    case 1:
      if (label_dtype == B200SEG_F32)
        launch_k(loss_partials_binary_kernel<float>, grid, 256, 0, s, logits, static_cast<const float*>(labels), vox, gamma,
                                                                alpha_f, part, metric);
      else
        launch_k(loss_partials_binary_kernel<long long>, grid, 256, 0, s, logits, tl, vox, gamma, alpha_f, part, metric);
      break;
    case 2: launch_k(loss_partials_multi_kernel<2>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    case 3: launch_k(loss_partials_multi_kernel<3>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    case 4: launch_k(loss_partials_multi_kernel<4>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    case 5: launch_k(loss_partials_multi_kernel<5>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    case 6: launch_k(loss_partials_multi_kernel<6>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    case 7: launch_k(loss_partials_multi_kernel<7>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    case 8: launch_k(loss_partials_multi_kernel<8>, grid, 256, 0, s, logits, tl, vox, gamma, part, metric); break;
    default:
      launch_k(loss_partials_multi_generic_kernel, grid, 256, (5 * C + 3) * sizeof(float), s, logits, tl, vox, C, gamma,
                                                                                        part, metric);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int metric_partials(const float* probs, const void* labels, int label_dtype, int N, long long vox, int C, float thr,
                    double* metric, int device, cudaStream_t s) {
  B200_CHECK_ARG(C >= 1 && C <= 1024 && N >= 1 && N <= 65535, "metric_partials: unsupported shape");
  const dim3 grid = sample_grid(vox, N, device);
  if (label_dtype == B200SEG_F32)
    launch_k(metric_partials_kernel<float>, grid, 256, 3 * C * sizeof(float), s, probs, static_cast<const float*>(labels),
                                                                           vox, C, thr, metric);
  else
    launch_k(metric_partials_kernel<long long>, grid, 256, 3 * C * sizeof(float), s, probs, static_cast<const long long*>(labels), vox, C, thr, metric);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int metric_finalize(const double* metric, int N, int C, float* out, cudaStream_t s) {
  launch_k(metric_finalize_kernel, 1, 32, 0, s, metric, N, C, out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int loss_finalize(const double* part, int C, int terms, const float* alpha, float gamma, float alpha_f, float* loss,
                  float* lcoef, cudaStream_t s) {
  if (terms & B200SEG_LOSS_EXT_MASK)
    launch_k(loss_finalize_ext_kernel, 1, 32, 0, s, part, C, terms, alpha, gamma, alpha_f, loss, lcoef);
  else
    launch_k(loss_finalize_kernel, 1, 32, 0, s, part, C, terms, alpha, gamma, alpha_f, loss, lcoef);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int loss_bwd(const float* logits, const void* labels_, int label_dtype, long long nvox_, int C, const float* lcoef,
             const float* gscale, float* dlogits, int device, cudaStream_t s) {
  B200_CHECK_ARG(C >= 1 && C <= 1024, "loss_bwd: unsupported class count %d", C);
  B200_CHECK_ARG(label_dtype == B200SEG_I64 || (label_dtype == B200SEG_F32 && C == 1),
                 "loss_bwd: labels must be int64 (fp32 soft targets only for the binary losses)");
  const int blocks = loss_blocks(nvox_, device);
  const long long* labels = static_cast<const long long*>(labels_);
  switch (C) {
    case 1:
      if (label_dtype == B200SEG_F32)
        launch_k(loss_bwd_binary_kernel<float>, blocks, 256, 0, s, logits, static_cast<const float*>(labels_), nvox_, lcoef,
                                                             gscale, dlogits);
      else
        launch_k(loss_bwd_binary_kernel<long long>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits);
      break;
    case 2: launch_k(loss_bwd_multi_kernel<2>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    case 3: launch_k(loss_bwd_multi_kernel<3>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    case 4: launch_k(loss_bwd_multi_kernel<4>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    case 5: launch_k(loss_bwd_multi_kernel<5>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    case 6: launch_k(loss_bwd_multi_kernel<6>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    case 7: launch_k(loss_bwd_multi_kernel<7>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    case 8: launch_k(loss_bwd_multi_kernel<8>, blocks, 256, 0, s, logits, labels, nvox_, lcoef, gscale, dlogits); break;
    default:
      launch_k(loss_bwd_multi_generic_kernel, blocks, 256, 0, s, logits, labels, nvox_, C, lcoef, gscale, dlogits);
  }
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int loss_partials_ss(const float* logits, const void* labels, int label_dtype, int N, long long vox, double* part,
                     double* metric, int device, cudaStream_t s) {
  B200_CHECK_ARG(N >= 1 && N <= 65535, "loss_partials_ss: unsupported batch size %d", N);
  const dim3 grid = sample_grid(vox, N, device);
  if (label_dtype == B200SEG_F32)
    launch_k(loss_partials_ss_kernel<float>, grid, 256, 0, s, logits, static_cast<const float*>(labels), vox, part,
             metric);
  else
    launch_k(loss_partials_ss_kernel<long long>, grid, 256, 0, s, logits, static_cast<const long long*>(labels), vox,
             part, metric);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int loss_bwd_ss(const float* logits, const void* labels, int label_dtype, long long nvox_, const float* lcoef,
                const float* gscale, float* dlogits, int device, cudaStream_t s) {
  const int blocks = loss_blocks(nvox_, device);
  if (label_dtype == B200SEG_F32)
    launch_k(loss_bwd_ss_kernel<float>, blocks, 256, 0, s, logits, static_cast<const float*>(labels), nvox_, lcoef,
             gscale, dlogits);
  else
    launch_k(loss_bwd_ss_kernel<long long>, blocks, 256, 0, s, logits, static_cast<const long long*>(labels), nvox_,
             lcoef, gscale, dlogits);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
