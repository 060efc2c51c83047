// GroupNorm coefficients for every kernel that applies the norm: the elementwise GroupNorm kernels and finalize
// kernels (elementwise.cu), the fused input-block and up_tr32 kernels (stem_gn.cu, up_gn.cu) and the backward-sums
// epilogues of the halo convolutions (conv_halo.cu, conv_halo_ws.cu).  A ReLU mask taken in the forward pass is
// the one the backward pass sees only while both derive their coefficients with the same expressions, in the same
// order and precision: each expression is written once, below.
#pragma once

#include "common.cuh"

namespace b200seg {

// ---------------------------------------------------------------------------------------------
// Fused GroupNorm coefficients: instead of separate finalize launches, every kernel that applies the
// norm (forward apply, backward mask / dy) derives A, B (and mean, rstd) for its own channels straight
// from the fp64 statistics.
// ---------------------------------------------------------------------------------------------
struct GnRef {
  const double* stats;     // [N][C][2]  (null -> use the precomputed coefficient array instead)
  const float* gamma;
  const float* beta;
  const float* scale;      // [N][C] dropout scale or null
  int groups;
  double m;                // elements per group = (C/groups) * voxels
  float eps;
  int sum_y_from_stats;    // backward: sum of y per (n,c) = stats[n][c][0] (the backward sums came from a conv epilogue)
};

// The GnRef of one GroupNorm application over C channels; null (or no statistics) gives the empty reference.
// (static: a host helper of each launcher, not a symbol of the library)
static inline GnRef gn_ref(const b200seg_gn* g, int C) {
  GnRef r;
  if (g == nullptr || g->stats == nullptr) {
    r.stats = nullptr; r.gamma = nullptr; r.beta = nullptr; r.scale = nullptr; r.groups = 1; r.m = 1.0; r.eps = 0.f;
    r.sum_y_from_stats = 0;
    return r;
  }
  r.stats = g->stats; r.gamma = g->gamma; r.beta = g->beta; r.scale = g->scale; r.groups = g->groups;
  r.m = (double)(C / g->groups) * (double)g->vox;
  r.eps = g->eps;
  r.sum_y_from_stats = 0;
  return r;
}

// ---------------------------------------------------------------------------------------------
// The expressions (SURVEY.md App. G).  ga, be = gamma, beta and sc = dropout scale of the channel, all widened
// from fp32; s1 = sum g*m * sc, s2 = sum g*m*y * sc, s3 = sum y over the channel's vox voxels of one sample.
// ---------------------------------------------------------------------------------------------
// mean and 1/sqrt(var + eps) of a group from the sums of y (s) and y^2 (q) over its m elements (rsqrt: device only)
__device__ __forceinline__ void gn_mean_rstd(double s, double q, double m, float eps, double& mean, double& rstd) {
  mean = s / m;
  double var = q / m - mean * mean;
  if (var < 0.0) var = 0.0;
  rstd = rsqrt(var + (double)eps);
}
// forward y*A + B; A is also P, the factor of g*m in the backward dy = g*m*P + y*Q + R
__host__ __device__ __forceinline__ double gn_a(double rstd, double ga, double sc) { return rstd * ga * sc; }
__host__ __device__ __forceinline__ double gn_b(double mean, double rstd, double ga, double be, double sc) {
  return (be - mean * rstd * ga) * sc;
}
// one channel's terms of the group means m1 = sum(m1_term) / m and m2 = sum(m2_term) / m
__host__ __device__ __forceinline__ double gn_m1_term(double ga, double s1) { return ga * s1; }
__host__ __device__ __forceinline__ double gn_m2_term(double mean, double rstd, double ga, double s1, double s2) {
  return ga * rstd * (s2 - mean * s1);
}
__host__ __device__ __forceinline__ double gn_q(double rstd, double m2) { return -rstd * rstd * m2; }
__host__ __device__ __forceinline__ double gn_r(double mean, double rstd, double m1, double m2) {
  return -rstd * m1 + rstd * rstd * mean * m2;
}
// one sample's share of the parameter gradients: d beta += s1, d gamma += gn_dgamma, d bias += gn_dbias
__host__ __device__ __forceinline__ double gn_dgamma(double mean, double rstd, double s1, double s2) {
  return rstd * (s2 - mean * s1);
}
__host__ __device__ __forceinline__ double gn_dbias(double rstd, double ga, double s1, double s3, double q, double r,
                                                    double vox) {
  return rstd * ga * s1 + q * s3 + r * vox;
}

// The activation after the norm and dropout (B200SEG_ACT_*, a template parameter of the kernels that apply it), on the
// pre-activation v = y*A + B: the forward value, and the backward factor on the incoming gradient g (torch's
// threshold_backward / leaky_relu_backward, both keyed on the sign of v).  gn_act_bwd_p is g' * P with the ReLU form
// written as the kernels always wrote it.  The LeakyReLU products are __fmul_rn: each is one rounding, never fused
// into a neighbouring add.
template <int ACT>
__device__ __forceinline__ float gn_act(float v) {
  if constexpr (ACT == B200SEG_ACT_LEAKY) return v > 0.f ? v : __fmul_rn(v, 0.01f);
  else return fmaxf(v, 0.f);
}
template <int ACT>
__device__ __forceinline__ float gn_act_bwd(float v, float g) {
  if constexpr (ACT == B200SEG_ACT_LEAKY) return v > 0.f ? g : __fmul_rn(g, 0.01f);
  else return v > 0.f ? g : 0.f;
}
template <int ACT>
__device__ __forceinline__ float gn_act_bwd_p(float v, float g, float P) {
  if constexpr (ACT == B200SEG_ACT_LEAKY) return __fmul_rn(v > 0.f ? g : __fmul_rn(g, 0.01f), P);
  else return v > 0.f ? g * P : 0.f;
}

// The threads that derive the coefficients together, thread tid() of count(), and the barrier they meet at: the
// whole CTA ...
struct GnCta {
  __device__ __forceinline__ int tid() const { return threadIdx.x; }
  __device__ __forceinline__ unsigned count() const { return blockDim.x; }
  __device__ __forceinline__ void sync() const { __syncthreads(); }
};
// ... or threads t = 0 .. COUNT-1 at named barrier ID (the epilogue warpgroup of the halo convolutions)
template <int ID, int COUNT>
struct GnNamedBarrier {
  int t;
  __device__ __forceinline__ int tid() const { return t; }
  __device__ __forceinline__ int count() const { return COUNT; }
  __device__ __forceinline__ void sync() const { asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(COUNT) : "memory"); }
};

// Block-cooperative form used by the kernels: the coefficients of ALL C channels of sample n at once, derived by
// the threads of th, which all call it.  Every global operand (statistics, backward sums and, with
// STAGE, gamma, beta, dropout scale) is fetched in ONE round of independent loads, one thread per channel; the
// per-group sums then run over shared memory in fixed channel order.  (Walking a group's channels with dependent
// global loads costs ~cpg L2 latencies per CTA, which is the whole run time of the kernels of the small pyramid
// levels.)
//   s_d : double scratch, (BWD ? 4 : 2) * (C + groups) (within gn_cta_doubles); on return
//         grp = s_d + (BWD ? 4 : 2) * C holds {mean, rstd} per group, {mean, rstd, m1, m2} when BWD
//   s_f : STAGE: float scratch, 3 * C (scale, gamma, beta).  Without STAGE (forward only: callers without the
//         shared memory) the last pass reads gamma, beta and the scale from global memory.
//   A, B (and P, Q, R when BWD): outputs, C floats each (shared memory)
// The channel loops take one or two trips per thread: they are not unrolled, which would only cost the callers
// registers.
__host__ __device__ inline size_t gn_cta_doubles(int C, int groups, bool bwd) { return (size_t)(bwd ? 4 : 2) * C + 4 * groups; }

template <bool BWD, bool STAGE, class Threads, bool WIDE = false>
__device__ __forceinline__ double* gn_coefs(Threads th, const GnRef& r, const double* __restrict__ sums, int n, int C,
                                            double* s_d, float* s_f, float* A, float* B, float* P, float* Q,
                                            float* R) {
  static_assert(STAGE || !BWD, "the backward form stages gamma and the scale for param_grads_of_sample");
  constexpr int GS = BWD ? 4 : 2;     // doubles per group in grp
  const int cpg = C / r.groups;
  double* d0 = s_d;
  double* d1 = s_d + C;
  double* d2 = s_d + 2 * C;           // BWD only
  double* d3 = s_d + 3 * C;           // BWD only
  double* grp = s_d + GS * C;
  float* f_sc = s_f;                  // STAGE only
  float* f_ga = s_f + C;
  float* f_be = s_f + 2 * C;
#pragma unroll 1
  for (int c = th.tid(); c < C; c += th.count()) {
    const double* p = r.stats + ((long long)n * C + c) * 2;
    d0[c] = p[0];
    d1[c] = p[1];
    if (STAGE) {
      f_sc[c] = r.scale ? r.scale[(long long)n * C + c] : 1.f;
      f_ga[c] = r.gamma[c];
      f_be[c] = r.beta[c];
    }
    if (BWD) {
      const double* q = sums + ((long long)n * C + c) * 3;
      d2[c] = q[0];
      d3[c] = q[1];
    }
  }
  th.sync();
  // one group per thread (the group loops are written twice so that the one-per-thread form, which every ReLU kernel
  // uses, compiles exactly as it always has); WIDE: any number of groups (InstanceNorm has one per channel, more than
  // a CTA has threads)
  if constexpr (WIDE) {
#pragma unroll 1
    for (int g = th.tid(); g < r.groups; g += th.count()) {
      double s = 0.0, q = 0.0;
      for (int k = 0; k < cpg; ++k) {
        s += d0[g * cpg + k];
        q += d1[g * cpg + k];
      }
      double mean, rstd;
      gn_mean_rstd(s, q, r.m, r.eps, mean, rstd);
      grp[g * GS + 0] = mean;
      grp[g * GS + 1] = rstd;
    }
  } else if (th.tid() < r.groups) {
    const int g = th.tid();
    double s = 0.0, q = 0.0;
    for (int k = 0; k < cpg; ++k) {
      s += d0[g * cpg + k];
      q += d1[g * cpg + k];
    }
    double mean, rstd;
    gn_mean_rstd(s, q, r.m, r.eps, mean, rstd);
    grp[g * GS + 0] = mean;
    grp[g * GS + 1] = rstd;
  }
  th.sync();
#pragma unroll 1
  for (int c = th.tid(); c < C; c += th.count()) {
    const int g = c / cpg;
    const double mean = grp[g * GS + 0], rstd = grp[g * GS + 1];
    double sc, ga, be;
    if (STAGE) {
      sc = (double)f_sc[c], ga = (double)f_ga[c], be = (double)f_be[c];
    } else {
      sc = r.scale ? (double)r.scale[(long long)n * C + c] : 1.0;
      ga = (double)r.gamma[c], be = (double)r.beta[c];
    }
    A[c] = (float)gn_a(rstd, ga, sc);
    B[c] = (float)gn_b(mean, rstd, ga, be, sc);
    if (BWD) {
      const double s1 = d2[c] * sc, s2 = d3[c] * sc;
      d2[c] = gn_m1_term(ga, s1);
      d3[c] = gn_m2_term(mean, rstd, ga, s1, s2);
    }
  }
  if (BWD) {
    th.sync();
    if constexpr (WIDE) {
#pragma unroll 1
      for (int g = th.tid(); g < r.groups; g += th.count()) {
        double sa = 0.0, sax = 0.0;
        for (int k = 0; k < cpg; ++k) {
          sa += d2[g * cpg + k];
          sax += d3[g * cpg + k];
        }
        grp[g * 4 + 2] = sa / r.m;
        grp[g * 4 + 3] = sax / r.m;
      }
    } else if (th.tid() < r.groups) {
      const int g = th.tid();
      double sa = 0.0, sax = 0.0;
      for (int k = 0; k < cpg; ++k) {
        sa += d2[g * cpg + k];
        sax += d3[g * cpg + k];
      }
      grp[g * 4 + 2] = sa / r.m;
      grp[g * 4 + 3] = sax / r.m;
    }
    th.sync();
#pragma unroll 1
    for (int c = th.tid(); c < C; c += th.count()) {
      const int g = c / cpg;
      const double mu = grp[g * 4 + 0], rs = grp[g * 4 + 1], m1 = grp[g * 4 + 2], m2 = grp[g * 4 + 3];
      P[c] = (float)gn_a(rs, (double)f_ga[c], (double)f_sc[c]);
      Q[c] = (float)gn_q(rs, m2);
      R[c] = (float)gn_r(mu, rs, m1, m2);
    }
  }
  th.sync();
  return grp;
}

// d gamma, d beta, d bias of ONE sample from the coefficients a CTA has just derived for it with
// gn_coefs<true, ...> (grp = {mean, rstd, m1, m2} per group; s_f = scale, gamma, beta per channel): the three
// parameter gradients are sums over the batch, added with fp32 atomics (the gradient bucket is zero on entry).
__device__ __forceinline__ void param_grads_of_sample(const GnRef& gn, const double* __restrict__ sums,
                                                      const double* grp, const float* s_f, int n, int C,
                                                      float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                      float* __restrict__ dbias) {
  const int cpg = C / gn.groups;
  const double vox = gn.m / (double)cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double mu = grp[g * 4 + 0], rs = grp[g * 4 + 1], m1 = grp[g * 4 + 2], m2 = grp[g * 4 + 3];
    const double sc = (double)s_f[c], ga = (double)s_f[C + c];
    const double* sp = sums + ((long long)n * C + c) * 3;
    const double s1 = sp[0] * sc, s2 = sp[1] * sc;
    const double s3 = gn.sum_y_from_stats ? gn.stats[((long long)n * C + c) * 2] : sp[2];
    atomicAdd(dbeta + c, (float)s1);
    atomicAdd(dgamma + c, (float)gn_dgamma(mu, rs, s1, s2));
    if (dbias != nullptr) atomicAdd(dbias + c, (float)gn_dbias(rs, ga, s1, s3, gn_q(rs, m2), gn_r(mu, rs, m1, m2), vox));
  }
}

}  // namespace b200seg
