// Device-side input staging (sm_90a): what the reference's datasets do to a batch on the host before the step,
// done on the GPU from the raw 8-bit images so that a step moves 1 byte per voxel over PCIe instead of 4 + 8.
//   stage_u8_sums / stage_u8_normalize : datasetModelSegwithopencv.__getitem__ (model/dataset.py:138-142):
//       image = (image - image.mean()) / image.std()   on the resized 8-bit image (numpy: float64, population std)
//       images_tensor = torch.as_tensor(image).float()
//     The per-image sums of x and x*x are accumulated as INTEGERS (exact); mean and the variance numerator
//     n*sum(x^2) - sum(x)^2 are therefore exact (128-bit), and each output is ((double)x - mean) / std rounded once to
//     fp32 -- numpy rounds its variance a few more times on the way, so the two agree to ~1 ulp of fp32, not bitwise.
//     A constant image gives 0/0 = NaN everywhere, as numpy does.
//   stage_labels_u8 : label_tensor = torch.as_tensor(label).long() (dataset.py:150-157) with the trainer's
//       y[y != 0] = 1 (model/modelUnet.py:130) folded in when `binarize` is set.
// SURVEY.md 8(f) row 4.
#include "common.cuh"

namespace b200seg {

__global__ void __launch_bounds__(256) stage_u8_sums_kernel(const unsigned char* __restrict__ img, long long per,
                                                            unsigned long long* __restrict__ sums) {
  PDL_ENTER();
  const int n = blockIdx.y;
  const unsigned char* base = img + (long long)n * per;
  unsigned long long s1 = 0, s2 = 0;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthr = (long long)gridDim.x * blockDim.x;
  // 16 pixels per load where the sample is 16-byte aligned; per-thread partials fit 32 bits for 2^16 pixels per trip
  const bool vec = ((reinterpret_cast<uintptr_t>(base) | (uintptr_t)per) & 15) == 0;
  if (vec) {
    const uint4* b4 = reinterpret_cast<const uint4*>(base);
    const long long n16 = per >> 4;
    for (long long i = tid; i < n16; i += nthr) {
      const uint4 q = __ldg(b4 + i);
      const unsigned int w[4] = {q.x, q.y, q.z, q.w};
      unsigned int a1 = 0, a2 = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const unsigned int v = (w[k] >> (8 * b)) & 0xffu;
          a1 += v;
          a2 += v * v;
        }
      s1 += a1;
      s2 += a2;
    }
  } else {
    for (long long i = tid; i < per; i += nthr) {
      const unsigned int v = base[i];
      s1 += v;
      s2 += v * v;
    }
  }
  // warp fold, then one pair of 64-bit atomics per warp (integer: order does not matter)
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(sums + 2 * n, s1);
    atomicAdd(sums + 2 * n + 1, s2);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) stage_u8_normalize_kernel(const unsigned char* __restrict__ img, long long per,
                                                                 const unsigned long long* __restrict__ sums,
                                                                 T* __restrict__ out) {
  PDL_ENTER();
  const int n = blockIdx.y;
  const unsigned long long s1 = sums[2 * n], s2 = sums[2 * n + 1];
  const double cnt = (double)per;
  const double mean = (double)s1 / cnt;
  // population variance = (n*S2 - S1^2) / n^2, numerator exact in 128 bits
  const unsigned __int128 num = (unsigned __int128)(unsigned long long)per * s2 - (unsigned __int128)s1 * s1;
  const double var = ((double)(unsigned long long)(num >> 64) * 18446744073709551616.0 + (double)(unsigned long long)num) /
                     (cnt * cnt);
  const double sd = sqrt(var);
  const unsigned char* base = img + (long long)n * per;
  T* ob = out + (long long)n * per;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthr = (long long)gridDim.x * blockDim.x;
  for (long long i = tid; i < per; i += nthr) {
    const float f = (float)(((double)base[i] - mean) / sd);
    if constexpr (sizeof(T) == 4) ob[i] = f;
    else ob[i] = __float2bfloat16_rn(f);
  }
}

__global__ void __launch_bounds__(256) stage_labels_u8_kernel(const unsigned char* __restrict__ lab, long long count,
                                                              int binarize, long long* __restrict__ out) {
  PDL_ENTER();
  const long long nthr = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += nthr) {
    const unsigned int v = lab[i];
    out[i] = binarize ? (v != 0u ? 1ll : 0ll) : (long long)v;
  }
}

static int stage_blocks(long long work, int device, int per_sm) {
  long long b = (work + 255) / 256;
  const long long cap = (long long)num_sms(device) * per_sm;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

int stage_u8_sums(const unsigned char* img, int n, long long per, unsigned long long* sums, int device, cudaStream_t st) {
  int bx = stage_blocks((per + 15) / 16, device, 8) / n;
  if (bx < 1) bx = 1;
  launch_k(stage_u8_sums_kernel, dim3(bx, n), 256, 0, st, img, per, sums);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int stage_u8_normalize(const unsigned char* img, int n, long long per, const unsigned long long* sums, void* out,
                       int out_dtype, int device, cudaStream_t st) {
  int bx = stage_blocks(per, device, 8) / n;
  if (bx < 1) bx = 1;
  if (out_dtype == B200SEG_F32)
    launch_k(stage_u8_normalize_kernel<float>, dim3(bx, n), 256, 0, st, img, per, sums, static_cast<float*>(out));
  else
    launch_k(stage_u8_normalize_kernel<bf16>, dim3(bx, n), 256, 0, st, img, per, sums, static_cast<bf16*>(out));
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int stage_labels_u8(const unsigned char* lab, long long count, int binarize, long long* out, int device, cudaStream_t st) {
  launch_k(stage_labels_u8_kernel, stage_blocks(count, device, 8), 256, 0, st, lab, count, binarize, out);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // namespace b200seg
