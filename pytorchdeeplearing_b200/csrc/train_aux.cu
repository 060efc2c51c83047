// Kernels around the conv path of one training / inference step (sm_90a):
//   adam_tick + adam_step   : fused Adam / AdamW over FLAT fp32 parameter / gradient / moment buffers
//                             (optim.AdamW(lr) model/modelVNet.py:548; optim.Adam model/modelUnet.py:849) -- SURVEY 8f-1
//   dropout_masks_kernel    : ALL nn.Dropout3d/2d(p) channel masks of one forward in one launch, reproducing the
//                             Philox stream of the per-module torch draws (networks/VNet3d.py:11,31,51,67;
//                             Unet3d.py:74,83; SURVEY 0.5) -- replaces 34 bernoulli_ launches
//   head_mask / mask_logits : forward-only head: 1x1 conv -> (sigmoid > threshold)*255 or argmax -> uint8 mask, no
//                             logits / probs materialised (predict, model/modelVNet.py:655-676) -- SURVEY 8f-3
#include <curand_kernel.h>

#include "common.cuh"

namespace b200seg {

// ------------------------------------------------------------------------------------------------
// Adam / AdamW (torch.optim semantics, single-tensor form):
//   AdamW: p *= 1 - lr*wd           Adam: g += wd*p
//   m = m + (g - m)(1 - b1) ; v = b2 v + (1 - b2) g g
//   p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// state[0] = t (step count, fp32 like torch's step tensor), state[1] = lr / (1 - b1^t), state[2] = sqrt(1 - b2^t)
// The step count lives on the device so that the update can be replayed from a CUDA graph.
// Like torch, every constant (1 - b1, 1 - b2, 1 - lr wd, b^t, lr / bc1) is computed in double from the double
// hyper-parameters and rounded to fp32 once: 1.f - 0.999f is 111 fp32 ulps away from (float)(1 - 0.999).
// ------------------------------------------------------------------------------------------------
__global__ void adam_tick_kernel(float* __restrict__ state, double lr, double beta1, double beta2) {
  PDL_ENTER();
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const double t = (double)state[0] + 1.0;
  state[0] = (float)t;
  const double bc1 = 1.0 - pow(beta1, t);
  const double bc2 = 1.0 - pow(beta2, t);
  state[1] = (float)(lr / bc1);
  state[2] = (float)sqrt(bc2);
}

// w1 = 1 - b1, w2 = 1 - b2, decay = 1 - lr wd: each the fp32 rounding of the double value
__global__ void __launch_bounds__(256) adam_step_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                        float* __restrict__ m, float* __restrict__ v, long long n,
                                                        const float* __restrict__ state, float w1, float w2,
                                                        float beta2, float eps, float wd, float decay, int decoupled,
                                                        const float* __restrict__ gscale, long long n4) {
  PDL_ENTER();
  const float step_size = state[1], bc2s = state[2];
  const float gs = gscale ? gscale[0] : 1.f;
  const long long stride = (long long)gridDim.x * blockDim.x;      // n4: float4 groups (0 when a buffer is unaligned)
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    const float4 gv4 = reinterpret_cast<const float4*>(g)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float pa[4] = {pv.x, pv.y, pv.z, pv.w}, ga[4] = {gv4.x, gv4.y, gv4.z, gv4.w};
    float ma[4] = {mv.x, mv.y, mv.z, mv.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float gg = ga[k] * gs;
      if (decoupled) pa[k] *= decay; else gg = fmaf(wd, pa[k], gg);
      ma[k] = fmaf(gg - ma[k], w1, ma[k]);
      va[k] = fmaf(va[k], beta2, w2 * gg * gg);
      const float denom = sqrtf(va[k]) / bc2s + eps;
      pa[k] = fmaf(-step_size, ma[k] / denom, pa[k]);
    }
    reinterpret_cast<float4*>(p)[i] = make_float4(pa[0], pa[1], pa[2], pa[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(ma[0], ma[1], ma[2], ma[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(va[0], va[1], va[2], va[3]);
  }
  // tail (n % 4 elements)
  for (long long i = (n4 << 2) + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += stride) {
    float gg = g[i] * gs, pp = p[i];
    if (decoupled) pp *= decay; else gg = fmaf(wd, pp, gg);
    const float mm = fmaf(gg - m[i], w1, m[i]);
    const float vv = fmaf(v[i], beta2, w2 * gg * gg);
    m[i] = mm;
    v[i] = vv;
    p[i] = fmaf(-step_size, mm / (sqrtf(vv) / bc2s + eps), pp);
  }
}

int adam_step(float* p, const float* g, float* m, float* v, long long n, float* state, double lr, double beta1,
              double beta2, float eps, double wd, int decoupled, const float* gscale, int tick, int device,
              cudaStream_t s) {
  const bool al = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                    reinterpret_cast<uintptr_t>(v)) % 16) == 0;
  if (tick) launch_k(adam_tick_kernel, 1, 32, 0, s, state, lr, beta1, beta2);
  const long long n4 = al ? (n >> 2) : 0;         // unaligned slices (per-parameter calls) take the scalar loop
  long long blocks = ((al ? n / 4 : n) + 255) / 256;
  const long long cap = (long long)num_sms(device) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_k(adam_step_kernel, (int)blocks, 256, 0, s, p, g, m, v, n, state, (float)(1.0 - beta1),
           (float)(1.0 - beta2), (float)beta2, eps, (float)wd, (float)(1.0 - lr * wd), decoupled, gscale, n4);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

// ------------------------------------------------------------------------------------------------
// Dropout channel masks.  torch draws mask k of a forward as
//   x.new_empty((N, C_k, 1, ..)).bernoulli_(1 - p)         (then .div_(1 - p))
// and its CUDA bernoulli_ kernel gives element j (numel = N*C_k <= 256 * grid) the first value of
//   curand_uniform4(Philox4_32_10(seed, subsequence = j, offset = offset_k)),  offset_k = offset_0 + 4 k
// (every such call advances the generator's offset by 4) compared in double against 1 - p.  One thread per mask
// element here; rng = {seed, offset_0} is read from device memory so a captured launch follows the generator.
// table[k] = {first output element, element count, j0}: output element i of mask k is element j0 + (i - first) of the
// draw (j0 = rank * N_local * C_k when a data-parallel rank takes its slice of the global-batch draw, SURVEY 8e);
// out[i] = keep ? 1/(1-p) : 0.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dropout_masks_kernel(const long long* __restrict__ rng,
                                                            const int* __restrict__ table, int nmasks, int total,
                                                            double keep, float scale, float* __restrict__ out) {
  PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int k = 0;
  // masks are few (<= 64): linear search of the owning mask
  while (k + 1 < nmasks && i >= table[3 * (k + 1)]) ++k;
  const int j = i - table[3 * k] + table[3 * k + 2];
  curandStatePhilox4_32_10_t st;
  curand_init((unsigned long long)rng[0], (unsigned long long)j, (unsigned long long)(rng[1] + 4LL * k), &st);
  const float4 u = curand_uniform4(&st);
  out[i] = ((double)u.x < keep) ? scale : 0.f;
}

int dropout_masks(const long long* rng, const int* table, int nmasks, int total, double p_drop, float* out,
                  cudaStream_t s) {
  B200_CHECK_ARG(nmasks >= 1 && total >= 1 && p_drop >= 0.0 && p_drop < 1.0, "b200seg_dropout_masks: bad argument");
  const double keep = 1.0 - p_drop;
  launch_k(dropout_masks_kernel, (total + 255) / 256, 256, 0, s, rng, table, nmasks, total, keep, (float)(1.0 / keep), out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

// ------------------------------------------------------------------------------------------------
// inference head
// ------------------------------------------------------------------------------------------------
template <int NC>
__device__ __forceinline__ unsigned char mask_of(const float* z, float thr) {
  if (NC == 1) {
    const float p = 1.f / (1.f + expf(-z[0]));            // same expression as head_fwd: probs > out_threshold
    return p > thr ? 255 : 0;
  }
  int best = 0;
  float bv = z[0];
#pragma unroll
  for (int c = 1; c < NC; ++c)
    if (z[c] > bv) {                                       // np.argmax: first maximum
      bv = z[c];
      best = c;
    }
  return (unsigned char)best;
}

template <typename TX, int NC>
__global__ void __launch_bounds__(256) head_mask_kernel(const TX* __restrict__ x, long long xld, int Cin,
                                                        const float* __restrict__ w, const float* __restrict__ bias,
                                                        unsigned char* __restrict__ mask, long long NV, float thr) {
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
    mask[v] = mask_of<NC>(z, thr);
  }
}

__global__ void __launch_bounds__(256) mask_logits_kernel(const float* __restrict__ z, long long NV, int C, float thr,
                                                          unsigned char* __restrict__ mask) {
  PDL_ENTER();
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < NV; v += (long long)gridDim.x * blockDim.x) {
    const float* zi = z + v * C;
    if (C == 1) {
      mask[v] = mask_of<1>(zi, thr);
    } else {
      int best = 0;
      float bv = zi[0];
      for (int c = 1; c < C; ++c)
        if (zi[c] > bv) {
          bv = zi[c];
          best = c;
        }
      mask[v] = (unsigned char)best;
    }
  }
}

static int mask_blocks(long long nv, int device) {
  long long b = (nv + 255) / 256;
  const long long cap = (long long)num_sms(device) * 8;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

template <typename TX>
static int head_mask_typed(const b200seg_tensor* x, const float* w, const float* bias, unsigned char* mask, int nc,
                           float thr, int device, cudaStream_t st) {
  const long long NV = (long long)x->n * x->d * x->h * x->w;
  const int blocks = mask_blocks(NV, device);
  const size_t smem = (size_t)(nc * x->c + nc) * sizeof(float);
#define LAUNCH_HM(NC)                                                                                              \
  launch_k(head_mask_kernel<TX, NC>, blocks, 256, smem, st, static_cast<const TX*>(x->ptr), x->ld, x->c, w, bias, mask, \
                                                      NV, thr)
  switch (nc) {
    case 1: LAUNCH_HM(1); break;
    case 2: LAUNCH_HM(2); break;
    case 3: LAUNCH_HM(3); break;
    case 4: LAUNCH_HM(4); break;
    case 5: LAUNCH_HM(5); break;
    case 6: LAUNCH_HM(6); break;
    case 7: LAUNCH_HM(7); break;
    default: LAUNCH_HM(8); break;
  }
#undef LAUNCH_HM
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int head_mask(const b200seg_tensor* x, const float* w, const float* bias, unsigned char* mask, int nc, float thr,
              int device, cudaStream_t st) {
  B200_CHECK_ARG(nc >= 1 && nc <= 8, "b200seg_head_mask: 1..8 classes supported (got %d)", nc);
  B200_CHECK_ARG((x->c % 4) == 0 && (x->ld % 4) == 0 && (reinterpret_cast<uintptr_t>(x->ptr) % 16) == 0 &&
                     (x->dtype == B200SEG_F32 || (x->ld % 8) == 0) && x->c <= 1024,
                 "b200seg_head_mask: input channels must be a multiple of 4 and 16-byte aligned");
  if (x->dtype == B200SEG_BF16) return head_mask_typed<bf16>(x, w, bias, mask, nc, thr, device, st);
  return head_mask_typed<float>(x, w, bias, mask, nc, thr, device, st);
}

int mask_logits(const float* logits, long long nv, int C, float thr, unsigned char* mask, int device, cudaStream_t st) {
  launch_k(mask_logits_kernel, mask_blocks(nv, device), 256, 0, st, logits, nv, C, thr, mask);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
