// 1x1x1 convolutions at 16..64 channels on mma.sync (sm_90a, bf16): VNet3d.py:64 up-path `conv` (2C -> C after the
// skip concat) and its data gradient.
//
// These layers do 32..128 MACs per byte: they are HBM streams with a small GEMM attached.  On the wgmma/TMA path
// (conv_tc.cu) every 128-voxel tile pays a TMA issue, an mbarrier round trip into the MMA warpgroup and an
// accumulator hand-over through shared memory before a single byte is stored.  Here the GEMM stays in registers:
//   * a CTA copies 512 consecutive voxels x Cin (one contiguous run of the NDHWC tensor, or pitched rows of a
//     concat buffer) into shared memory with 16-byte cp.async, double buffered;
//   * each of the 8 warps multiplies four 16-voxel row groups: A fragments by ldmatrix (rows padded by 16 B: no bank
//     conflicts), B fragments = the whole weight matrix, held in registers for the kernel's lifetime
//     (m16n8k16, fp32 accumulators);
//   * epilogue on the accumulator fragments: + bias, GroupNorm statistics (per-lane column partials, folded once per
//     sample), + addend, bf16x2 stores.
#include "pw_mma.cuh"

namespace b200seg {

// UP = false: 1x1x1 conv.  UP = true: k2s2 transposed conv (VNet3d.py:62 up_conv and the data gradient of the k2s2
// down conv): the same A fragments are multiplied by the 8 (4 in 2-D) tap matrices and every product row is stored
// to its own fine voxel (2d+a, 2h+b, 2w+c); a 16-row group is 16 consecutive coarse voxels of one w-row.
template <int CIN, int COUT, bool UP>
__global__ void __launch_bounds__(PW_THREADS, UP ? 1 : 2)
    pw_conv_mma_kernel(const bf16* __restrict__ x, long long xld, const bf16* __restrict__ w /*[tap][COUT][CIN]*/,
                       const float* __restrict__ bias, bf16* __restrict__ y, long long yld,
                       const bf16* __restrict__ addend, long long ald, double* __restrict__ stats, long long NV,
                       long long V, int D, int H, int W, int ud) {
  PDL_ENTER();
  constexpr int XP = CIN * 2 + 16;                 // smem row pitch (bytes)
  constexpr int KS = CIN / 16, NT = COUT / 8;
  constexpr int XCH = CIN / 8;                     // 16-byte chunks per voxel
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_red = reinterpret_cast<float*>(smem_raw + 2 * PW_TILE * XP);        // [8 warps][2 * COUT]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, tq = lane & 3;

  // weights -> B fragments (held in registers for the kernel's lifetime)
  constexpr int TAPS = UP ? 8 : 1;
  const int taps = UP ? 4 * ud : 1;                 // 2-D transposed conv: 4 taps
  uint32_t wb[TAPS][KS][NT][2];
#pragma unroll
  for (int tp = 0; tp < TAPS; ++tp)
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
        pw_b_frag<CIN, COUT>(w, tp < taps ? tp : 0, ks, nt, gq, tq, wb[tp][ks][nt][0], wb[tp][ks][nt][1]);
  float bv[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bv[nt][0] = bias ? bias[nt * 8 + 2 * tq] : 0.f;
    bv[nt][1] = bias ? bias[nt * 8 + 2 * tq + 1] : 0.f;
  }
  float ssum[NT][2], ssq[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) ssum[nt][0] = ssum[nt][1] = ssq[nt][0] = ssq[nt][1] = 0.f;

  auto flush_stats = [&](long long n) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float a = ssum[nt][j], b = ssq[nt][j];
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
        }
        if (gq == 0) {
          s_red[warp * 2 * COUT + nt * 8 + 2 * tq + j] = a;
          s_red[warp * 2 * COUT + COUT + nt * 8 + 2 * tq + j] = b;
        }
        ssum[nt][j] = 0.f;
        ssq[nt][j] = 0.f;
      }
    __syncthreads();
    if (threadIdx.x < 2 * COUT) {
      double t = 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += (double)s_red[k * 2 * COUT + threadIdx.x];
      const int which = threadIdx.x / COUT, c = threadIdx.x - which * COUT;
      atomicAdd(stats + (n * COUT + c) * 2 + which, t);
    }
    __syncthreads();
  };

  auto load_tile = [&](int buf, long long tile) {
    const uint32_t xs = (uint32_t)__cvta_generic_to_shared(smem_raw + (size_t)buf * PW_TILE * XP);
    const bf16* src = x + tile * PW_TILE * xld;
    for (int q = threadIdx.x; q < PW_TILE * XCH; q += PW_THREADS) {
      const int v = q / XCH, part = q - v * XCH;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(xs + (uint32_t)(v * XP + part * 16)),
                   "l"(src + (long long)v * xld + part * 8)
                   : "memory");
    }
  };

  const long long tiles = NV / PW_TILE;
  const long long tpc = (tiles + gridDim.x - 1) / gridDim.x;
  const long long first = blockIdx.x * tpc;
  const long long last = first + tpc < tiles ? first + tpc : tiles;
  if (first >= last) return;
  load_tile(0, first);
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  const int a_lane = pw_a_lane(lane, XP);
  long long cur_n = first * PW_TILE / V;
  for (long long tile = first; tile < last; ++tile) {
    const int buf = (int)((tile - first) & 1);
    if (tile + 1 < last) load_tile(buf ^ 1, tile + 1);
    const long long n = tile * PW_TILE / V;
    if (n != cur_n) {
      if (stats != nullptr) flush_stats(cur_n);
      cur_n = n;
    }
    const uint32_t xs = (uint32_t)__cvta_generic_to_shared(smem_raw + (size_t)buf * PW_TILE * XP);
#pragma unroll
    for (int mi = 0; mi < PW_TILE / (8 * 16); ++mi) {
      const int r0 = (warp * (PW_TILE / 8) + mi * 16);          // first voxel row of this 16-row group in the tile
      uint32_t a[KS][4];
      pw_a_frags<KS>(a, xs, r0 * XP + a_lane);
      const long long v0 = tile * PW_TILE + r0;        // first (coarse) voxel of the group
      long long ob = v0;                               // UP: fine voxel of coarse voxel v0 at tap (0,0,0)
      int fw = 0, fh = 0;
      if (UP) ob = pw_up_base(v0, V, D, H, W, ud, fw, fh);
#pragma unroll
      for (int tp = 0; tp < TAPS; ++tp) {
        if (UP && tp >= taps) break;
        float acc[NT][4];
        pw_chain<KS, NT>(acc, a, wb[tp], bv);
        if (stats != nullptr) {
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            ssum[nt][0] += acc[nt][0] + acc[nt][2];
            ssum[nt][1] += acc[nt][1] + acc[nt][3];
            ssq[nt][0] = fmaf(acc[nt][0], acc[nt][0], fmaf(acc[nt][2], acc[nt][2], ssq[nt][0]));
            ssq[nt][1] = fmaf(acc[nt][1], acc[nt][1], fmaf(acc[nt][3], acc[nt][3], ssq[nt][1]));
          }
        }
        // output voxel of fragment row g (and g + 8)
        long long o0, o1;
        if (UP) {
          const int fc = tp & 1, fb = (tp >> 1) & 1, fa = tp >> 2;        // tap = (a, b, c), c fastest
          const long long t0 = ob + ((long long)fa * fh + fb) * fw + fc;
          o0 = t0 + 2 * gq;
          o1 = o0 + 16;
        } else {
          o0 = v0 + gq;
          o1 = o0 + 8;
        }
        if (addend != nullptr) {
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const float2 r0v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(addend + o0 * ald + nt * 8 + 2 * tq));
            const float2 r1v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(addend + o1 * ald + nt * 8 + 2 * tq));
            acc[nt][0] += r0v.x; acc[nt][1] += r0v.y;
            acc[nt][2] += r1v.x; acc[nt][3] += r1v.y;
          }
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          *reinterpret_cast<__nv_bfloat162*>(y + o0 * yld + nt * 8 + 2 * tq) = __floats2bfloat162_rn(acc[nt][0], acc[nt][1]);
          *reinterpret_cast<__nv_bfloat162*>(y + o1 * yld + nt * 8 + 2 * tq) = __floats2bfloat162_rn(acc[nt][2], acc[nt][3]);
        }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
  }
  if (stats != nullptr) flush_stats(cur_n);
}

// ------------------------------------------------------------------------------------------------
static bool al16pw(const void* p) { return (reinterpret_cast<uintptr_t>(p) % 16) == 0; }

static bool pw_ch(int c) { return c == 16 || c == 32 || c == 64; }

int pw_mma_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                     const b200seg_tensor* addend) {
  if ((kind != B200SEG_K1 && kind != B200SEG_UP) || w_dtype != B200SEG_BF16_TC) return 0;
  if (!pw_ch(x->c) || !pw_ch(y->c)) return 0;
  if (x->c * y->c > (kind == B200SEG_UP ? 512 : 2048)) return 0;      // the weight fragments live in registers
  if (x->dtype != B200SEG_BF16 || y->dtype != B200SEG_BF16) return 0;
  if (addend && addend->dtype != B200SEG_BF16) return 0;
  if ((x->ld % 8) || (y->ld % 8) || !al16pw(x->ptr) || !al16pw(y->ptr)) return 0;
  if (addend && ((addend->ld % 8) || !al16pw(addend->ptr))) return 0;
  if (x->n != y->n) return 0;
  if (kind == B200SEG_UP) {
    const int ud = dims == 3 ? 2 : 1;
    if (y->d != x->d * ud || y->h != x->h * 2 || y->w != x->w * 2) return 0;
    if (x->w % 16 != 0) return 0;                 // a 16-row fragment group = 16 coarse voxels of one w-row
  } else if (x->d != y->d || x->h != y->h || x->w != y->w) {
    return 0;
  }
  const long long V = (long long)x->d * x->h * x->w;
  if (V % PW_TILE != 0) return 0;
  if ((long long)y->d * y->h * y->w * y->n < 65536) return 0;         // small levels stay on the wgmma kernel
  return 1;
}

template <int CIN, int COUT, bool UP>
static int pw_launch(int dims, const b200seg_tensor* x, const void* w, const float* bias, const b200seg_tensor* y,
                     double* stats, const b200seg_tensor* addend, int device, cudaStream_t st) {
  const long long V = (long long)x->d * x->h * x->w;
  const long long NV = V * x->n;
  const size_t smem = (size_t)2 * PW_TILE * (CIN * 2 + 16) + (size_t)8 * 2 * COUT * sizeof(float);
  static int attr_done[64] = {0};
  if (smem > 48 * 1024 && device >= 0 && device < 64 && !attr_done[device]) {
    B200_CUDA(cudaFuncSetAttribute(pw_conv_mma_kernel<CIN, COUT, UP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   160 * 1024));
    attr_done[device] = 1;
  }
  const long long tiles = NV / PW_TILE;
  long long grid = (long long)num_sms(device) * (UP ? 1 : 2);
  if (grid > tiles) grid = tiles;
  launch_k(pw_conv_mma_kernel<CIN, COUT, UP>, (unsigned)grid, PW_THREADS, smem, st, static_cast<const bf16*>(x->ptr), x->ld, static_cast<const bf16*>(w), bias, static_cast<bf16*>(y->ptr), y->ld,
      addend ? static_cast<const bf16*>(addend->ptr) : nullptr, addend ? addend->ld : 0, stats, NV, V, x->d, x->h,
      x->w, dims == 3 ? 2 : 1);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int pw_mma_conv(int kind, int dims, const b200seg_tensor* x, const void* w, const float* bias,
                const b200seg_tensor* y, double* stats, const b200seg_tensor* addend, int device, cudaStream_t st) {
#define PW_CASE(CI, CO, U) \
  if (x->c == CI && y->c == CO) return pw_launch<CI, CO, U>(dims, x, w, bias, y, stats, addend, device, st)
  if (kind == B200SEG_UP) {
    PW_CASE(16, 16, true); PW_CASE(16, 32, true); PW_CASE(32, 16, true);
  } else {
    PW_CASE(16, 16, false); PW_CASE(16, 32, false); PW_CASE(16, 64, false);
    PW_CASE(32, 16, false); PW_CASE(32, 32, false); PW_CASE(32, 64, false);
    PW_CASE(64, 16, false); PW_CASE(64, 32, false);
  }
#undef PW_CASE
  set_error("pw_mma_conv: unsupported channel counts %d -> %d", x->c, y->c);
  return B200SEG_EINVAL;
}

}  // namespace b200seg
