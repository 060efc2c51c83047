// Fused GroupNorm coefficients shared by the elementwise GroupNorm kernels (elementwise.cu) and the fused
// input-block kernels (stem_gn.cu): the same expressions, in the same precision, wherever the norm is applied.
#pragma once

#include "common.cuh"

namespace b200seg {

// ---------------------------------------------------------------------------------------------
// Fused GroupNorm coefficients: instead of separate finalize launches, every kernel that applies the
// norm (forward apply, backward mask / dy) derives A, B (and mean, rstd) for its own channels straight
// from the fp64 statistics -- same code everywhere, so forward and backward see bit-identical values.
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

// Block-cooperative form used by the kernels: the coefficients of ALL C channels of sample n at once.
// Every global operand (statistics, backward sums, gamma, beta, dropout scale) is fetched in ONE round of
// independent loads, one thread per channel; the per-group sums then run over shared memory in fixed channel
// order.  (The per-thread forms above walk the group's channels with dependent global loads -- ~cpg L2
// latencies per CTA, which is the whole run time of the kernels of the small pyramid levels.)
//   s_d : double scratch, (BWD ? 4 : 2) * C + 4 * groups;  on return s_d[GRP..] = {mean, rstd, m1, m2} per group
//   s_f : float scratch, 3 * C  (scale, gamma, beta)
//   A, B (and P, Q, R when BWD): outputs, C floats each (shared memory)
__host__ __device__ inline size_t gn_cta_doubles(int C, int groups, bool bwd) { return (size_t)(bwd ? 4 : 2) * C + 4 * groups; }

template <bool BWD>
__device__ __forceinline__ double* gn_cta_coefs(const GnRef& r, const double* __restrict__ sums, int n, int C,
                                                double* s_d, float* s_f, float* A, float* B, float* P, float* Q,
                                                float* R) {
  const int cpg = C / r.groups;
  double* d0 = s_d;
  double* d1 = s_d + C;
  double* d2 = s_d + 2 * C;           // BWD only
  double* d3 = s_d + 3 * C;           // BWD only
  double* grp = s_d + (BWD ? 4 : 2) * C;
  float* f_sc = s_f;
  float* f_ga = s_f + C;
  float* f_be = s_f + 2 * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const double* p = r.stats + ((long long)n * C + c) * 2;
    d0[c] = p[0];
    d1[c] = p[1];
    f_sc[c] = r.scale ? r.scale[(long long)n * C + c] : 1.f;
    f_ga[c] = r.gamma[c];
    f_be[c] = r.beta[c];
    if (BWD) {
      const double* q = sums + ((long long)n * C + c) * 3;
      d2[c] = q[0];
      d3[c] = q[1];
    }
  }
  __syncthreads();
  if ((int)threadIdx.x < r.groups) {
    const int g = threadIdx.x;
    double s = 0.0, q = 0.0;
    for (int k = 0; k < cpg; ++k) {
      s += d0[g * cpg + k];
      q += d1[g * cpg + k];
    }
    const double mean = s / r.m;
    double var = q / r.m - mean * mean;
    if (var < 0.0) var = 0.0;
    grp[g * 4 + 0] = mean;
    grp[g * 4 + 1] = rsqrt(var + (double)r.eps);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double mean = grp[g * 4 + 0], rstd = grp[g * 4 + 1];
    const double sc = (double)f_sc[c], ga = (double)f_ga[c], be = (double)f_be[c];
    A[c] = (float)(rstd * ga * sc);
    B[c] = (float)((be - mean * rstd * ga) * sc);
    if (BWD) {
      const double s1 = d2[c] * sc, s2 = d3[c] * sc;
      d2[c] = ga * s1;
      d3[c] = ga * rstd * (s2 - mean * s1);
    }
  }
  if (BWD) {
    __syncthreads();
    if ((int)threadIdx.x < r.groups) {
      const int g = threadIdx.x;
      double sa = 0.0, sax = 0.0;
      for (int k = 0; k < cpg; ++k) {
        sa += d2[g * cpg + k];
        sax += d3[g * cpg + k];
      }
      grp[g * 4 + 2] = sa / r.m;
      grp[g * 4 + 3] = sax / r.m;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / cpg;
      const double mu = grp[g * 4 + 0], rs = grp[g * 4 + 1], m1 = grp[g * 4 + 2], m2 = grp[g * 4 + 3];
      P[c] = (float)(rs * (double)f_ga[c] * (double)f_sc[c]);
      Q[c] = (float)(-rs * rs * m2);
      R[c] = (float)(-rs * m1 + rs * rs * mu * m2);
    }
  }
  __syncthreads();
  return grp;
}

// d gamma, d beta, d bias of ONE sample from the coefficients a CTA has just derived for it with
// gn_cta_coefs<true> (grp = {mean, rstd, m1, m2} per group; s_f = scale, gamma, beta per channel): the three
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
    const double qd = -rs * rs * m2, rd = -rs * m1 + rs * rs * mu * m2;
    atomicAdd(dbeta + c, (float)s1);
    atomicAdd(dgamma + c, (float)(rs * (s2 - mu * s1)));
    if (dbias != nullptr) atomicAdd(dbias + c, (float)(rs * ga * s1 + qd * s3 + rd * vox));
  }
}

}  // namespace b200seg
