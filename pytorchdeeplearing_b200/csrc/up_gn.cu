// Fused first layer of VNet3d's up_tr32 (VNet3d.py:62-72): up_conv, a 2x2x2 stride-2 transposed convolution from 32
// channels at the coarse grid to 16 at the fine grid, then GroupNorm(8, 16), Dropout and ReLU into the left half of
// the skip-concat buffer.  Each coarse voxel (64 B) makes 8 fine voxels (256 B): the raw output y is 4x the bytes of
// what it is computed from, so these kernels never store it.  Every pass recomputes y from the coarse input x with
// pw_conv_mma_kernel<32, 16, true>'s fragments and mma chain (pw_mma.cuh), so the recomputed values are bit-identical
// to what the stored tensor held.
//
//   STATS   per-(n, c) sum y, sum y^2: the PW_MMA epilogue's order and partials (same tile walk, lanes -> warps -> one
//           fp64 atomic per CTA and sample)
//   APPLY   out = relu(y*A + B), A/B from the statistics, gamma, beta and dropout scale (gn_coefs), written into a
//           pitched buffer
//   BSUMS   per-(n, c) sum g*m, sum g*m*y, sum y (m = ReLU mask), the layout gn_bwd_apply_gn reads
//   BWD     dy = g*m*P + y*Q + R, rounded to bf16 as the stored dy is, kept on chip: it feeds the data gradient to the
//           coarse grid (the DOWN-kind convolution, K = 8 taps x 16 channels per coarse voxel) and the weight gradient
//           [tap][16][32]; d gamma, d beta and d bias come from the sums (param_grads_of_sample)
//
// STATS / APPLY / BSUMS walk pw_conv_mma_kernel's 512-voxel tiles.  BWD takes 128-voxel tiles in two phases: first
// every warp recomputes y of its 16-voxel group at all 8 taps, forms dy, runs the data gradient and parks dy in
// shared memory; then warp t reduces the weight gradient of tap t over the tile's 8 groups (dy^T x X, both operands
// by ldmatrix.trans), so its accumulators are 16 registers instead of 128.  The fine-grid operands (APPLY's output,
// the gradient g of BSUMS and BWD) pass through a per-warp shared-memory stage in whole 16-byte chunks, and g of a
// warp's next group is loaded (cp.async) while the current one is computed.
#include "pw_mma.cuh"
#include "gn_coef.cuh"

namespace b200seg {

enum { UG_STATS = 0, UG_APPLY = 1, UG_BSUMS = 2 };

constexpr int UG_CI = 32, UG_C = 16, UG_GROUPS = 8, UG_TAPS = 8;
constexpr int UG_KS = UG_CI / 16, UG_NT = UG_C / 8;
constexpr int UG_XP = UG_CI * 2 + 16;           // x tile row pitch (bytes), as pw_conv_mma_kernel
constexpr int UB_TILE = 128;                    // BWD: coarse voxels per tile = 8 groups, one per warp
constexpr int UB_DYP = 24;                      // BWD: dy row pitch (bf16): 48-byte rows, conflict-free ldmatrix

struct UpGnParams {
  const bf16* x;                                // coarse input [N][D][H][W][32], pitch xld
  long long xld;
  const bf16* w;                                // packed forward operand [8][16][32]
  const float* bias;                            // [16] or null
  GnRef gn;                                     // APPLY / BSUMS / BWD
  double* stats;                                // STATS out [N][16][2] (zero on entry)
  bf16* out;                                    // APPLY out, fine grid, pitch ldo
  long long ldo;
  const bf16* g;                                // BSUMS / BWD: activation gradient, fine grid, pitch ldg
  long long ldg;
  double* sums;                                 // BSUMS out (zero on entry) / BWD in, [N][16][3]
  float* dw;                                    // BWD: += [8][16][32]
  bf16* dx;                                     // BWD: data gradient, coarse grid, pitch ldx
  long long ldx;
  float* dgamma;                                // BWD: += [16]
  float* dbeta;
  float* dbias;                                 // may be null
  long long NV, V;                              // coarse voxels in all / per sample
  int N, D, H, W;                               // coarse grid
};

__device__ __forceinline__ float ug_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__device__ __forceinline__ uint32_t ug_pack(__nv_bfloat162 v) { return *reinterpret_cast<uint32_t*>(&v); }

__device__ __forceinline__ float2 ug_ld2(const bf16* p) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}

// 16-byte cp.async of `rows` voxel rows of x starting at coarse voxel v into a shared tile of UG_XP-byte rows
__device__ __forceinline__ void ug_load_tile(unsigned char* dst, const bf16* x, long long xld, long long v, int rows) {
  const uint32_t xs = (uint32_t)__cvta_generic_to_shared(dst);
  constexpr int XCH = UG_CI / 8;
  const bf16* src = x + v * xld;
  for (int q = threadIdx.x; q < rows * XCH; q += PW_THREADS) {
    const int r = q / XCH, part = q - r * XCH;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(xs + (uint32_t)(r * UG_XP + part * 16)),
                 "l"(src + (long long)r * xld + part * 8)
                 : "memory");
  }
}

// Fine-grid traffic of one 16-voxel group goes through a per-warp shared-memory stage, so global memory sees whole
// 16-byte chunks: the group's 8 taps cover 4 runs (tap rows (a, b)) of 32 consecutive fine voxels x 16 channels.
// A lane's fragment values, 4 bytes at every other fine voxel, are only ever read or written in the stage.
constexpr int UG_SP = 24;                       // stage row pitch (bf16): 48-byte rows, at most 2-way bank conflicts
constexpr int UG_STAGE = 4 * 32 * UG_SP;        // bf16 elements per stage

// element offset in a stage of the lane's fragment pair (tap tp, fragment row gq + 8 h, n-tile nt)
__device__ __forceinline__ int ug_frag(int tp, int h, int nt, int gq, int tq) {
  return ((tp >> 1) * 32 + 2 * (gq + 8 * h) + (tp & 1)) * UG_SP + nt * 8 + 2 * tq;
}

// chunk k (0..7) of the lane: run r, fine voxel j of the run, channel half hc; t + returned offset is its global address
__device__ __forceinline__ long long ug_chunk(int k, int lane, long long ob, int fw, int fh, long long ld, int& soff) {
  const int q = lane + 32 * k, r = q >> 6, j = (q >> 1) & 31, hc = q & 1;
  soff = (r * 32 + j) * UG_SP + hc * 8;
  return (ob + ((long long)(r >> 1) * fh + (r & 1)) * fw + j) * ld + hc * 8;
}

// cp.async the group's fine-grid runs of t (16 channels, pitch ld) into a stage
__device__ __forceinline__ void ug_stage_load(bf16* stage, const bf16* t, long long ld, long long ob, int fw, int fh,
                                              int lane) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(stage);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int so;
    const long long go = ug_chunk(k, lane, ob, fw, fh, ld, so);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s + (uint32_t)so * 2), "l"(t + go) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// the stage's runs -> t (16 channels, pitch ld), 16-byte stores
__device__ __forceinline__ void ug_stage_store(const bf16* stage, bf16* t, long long ld, long long ob, int fw, int fh,
                                               int lane) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int so;
    const long long go = ug_chunk(k, lane, ob, fw, fh, ld, so);
    *reinterpret_cast<uint4*>(t + go) = *reinterpret_cast<const uint4*>(stage + so);
  }
}

// shared memory of the STATS / APPLY / BSUMS kernel: x tiles, stages (APPLY one per warp, BSUMS two), coefficients
__host__ __device__ inline size_t ug_stage_off() { return (size_t)2 * PW_TILE * UG_XP; }
__host__ __device__ inline size_t ug_coef_off(int mode) {
  return ug_stage_off() + (size_t)(mode == UG_BSUMS ? 2 : mode == UG_APPLY ? 1 : 0) * 8 * UG_STAGE * 2;
}
__host__ __device__ inline size_t ug_smem(int mode) {
  return ug_coef_off(mode) + gn_cta_doubles(UG_C, UG_GROUPS, false) * sizeof(double) +
         (size_t)(3 + 2 + 8 * 3) * UG_C * sizeof(float);
}

template <int MODE>
__global__ void __launch_bounds__(PW_THREADS, 1) up_gn_kernel(const __grid_constant__ UpGnParams p) {
  PDL_ENTER();
  constexpr int KS = UG_KS, NT = UG_NT, C = UG_C, XP = UG_XP;
  constexpr int K = MODE == UG_BSUMS ? 3 : 2;   // sums per (n, c) folded at a sample boundary
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* s_d = reinterpret_cast<double*>(smem_raw + ug_coef_off(MODE));
  float* s_f = reinterpret_cast<float*>(s_d + gn_cta_doubles(C, UG_GROUPS, false));
  float* s_cf = s_f + 3 * C;                    // A, B
  float* s_red = s_cf + 2 * C;                  // [8 warps][K][C]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, tq = lane & 3;
  bf16* stage0 = reinterpret_cast<bf16*>(smem_raw + ug_stage_off()) + (size_t)warp * (MODE == UG_BSUMS ? 2 : 1) * UG_STAGE;
  constexpr int GPT = PW_TILE / (8 * 16);       // 16-voxel groups per warp and tile
  // fine voxel (tap (0,0,0), fragment row 0) of group mi of the warp in a tile
  auto group_base = [&](long long tile, int mi, int& fw, int& fh) {
    return pw_up_base(tile * PW_TILE + warp * (PW_TILE / 8) + mi * 16, p.V, p.D, p.H, p.W, 2, fw, fh);
  };

  uint32_t wb[UG_TAPS][KS][NT][2];
#pragma unroll
  for (int tp = 0; tp < UG_TAPS; ++tp)
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) pw_b_frag<UG_CI, C>(p.w, tp, ks, nt, gq, tq, wb[tp][ks][nt][0], wb[tp][ks][nt][1]);
  float bv[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bv[nt][0] = p.bias ? p.bias[nt * 8 + 2 * tq] : 0.f;
    bv[nt][1] = p.bias ? p.bias[nt * 8 + 2 * tq + 1] : 0.f;
  }
  float f1[NT][2], f2[NT][2], f3[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) f1[nt][0] = f1[nt][1] = f2[nt][0] = f2[nt][1] = f3[nt][0] = f3[nt][1] = 0.f;

  // lanes -> per-warp rows -> fp64 over the 8 warps in order -> one atomic per CTA, sample and value
  auto flush = [&](long long n) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float v[3] = {f1[nt][j], f2[nt][j], f3[nt][j]};
#pragma unroll
        for (int k = 0; k < K; ++k) {
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
          if (gq == 0) s_red[(warp * K + k) * C + nt * 8 + 2 * tq + j] = v[k];
        }
        f1[nt][j] = f2[nt][j] = f3[nt][j] = 0.f;
      }
    __syncthreads();
    if ((int)threadIdx.x < K * C) {
      double t = 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += (double)s_red[k * K * C + threadIdx.x];
      const int which = threadIdx.x / C, c = threadIdx.x - which * C;
      double* dst = MODE == UG_STATS ? p.stats : p.sums;
      atomicAdd(dst + (n * C + c) * K + which, t);
    }
    __syncthreads();
  };
  auto coefs = [&](long long n) {
    gn_coefs<false, true>(GnCta(), p.gn, nullptr, (int)n, C, s_d, s_f, s_cf, s_cf + C, nullptr, nullptr, nullptr);
  };

  const long long tiles = p.NV / PW_TILE;
  const long long tpc = (tiles + gridDim.x - 1) / gridDim.x;
  const long long first = blockIdx.x * tpc;
  const long long last = first + tpc < tiles ? first + tpc : tiles;
  if (first >= last) return;
  ug_load_tile(smem_raw, p.x, p.xld, first * PW_TILE, PW_TILE);
  if constexpr (MODE == UG_BSUMS) {
    int fw, fh;
    const long long ob = group_base(first, 0, fw, fh);
    ug_stage_load(stage0, p.g, p.ldg, ob, fw, fh, lane);
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  const int a_lane = pw_a_lane(lane, XP);
  int sb = 0;                                   // BSUMS: the stage holding the current group's g
  long long cur_n = first * PW_TILE / p.V;
  if (MODE != UG_STATS) coefs(cur_n);
  for (long long tile = first; tile < last; ++tile) {
    const int buf = (int)((tile - first) & 1);
    if (tile + 1 < last) ug_load_tile(smem_raw + (size_t)(buf ^ 1) * PW_TILE * XP, p.x, p.xld, (tile + 1) * PW_TILE, PW_TILE);
    const long long n = tile * PW_TILE / p.V;
    if (n != cur_n) {
      if (MODE != UG_APPLY) flush(cur_n);
      if (MODE != UG_STATS) coefs(n);
      cur_n = n;
    }
    const uint32_t xs = (uint32_t)__cvta_generic_to_shared(smem_raw + (size_t)buf * PW_TILE * XP);
#pragma unroll 1
    for (int mi = 0; mi < GPT; ++mi) {
      const int r0 = warp * (PW_TILE / 8) + mi * 16;
      uint32_t a[KS][4];
      pw_a_frags<KS>(a, xs, r0 * XP + a_lane);
      int fw, fh;
      const long long ob = group_base(tile, mi, fw, fh);
      bf16* stage = stage0 + sb * UG_STAGE;
      __syncwarp();                             // every lane is done with the stage it is about to refill
      if constexpr (MODE == UG_BSUMS) {
        // g of the warp's next group streams in while this one is computed
        const long long nt_ = mi + 1 < GPT ? tile : tile + 1;
        if (nt_ < last) {
          int nfw, nfh;
          const long long nob = group_base(nt_, (mi + 1) % GPT, nfw, nfh);
          ug_stage_load(stage0 + (sb ^ 1) * UG_STAGE, p.g, p.ldg, nob, nfw, nfh, lane);
        } else {
          asm volatile("cp.async.commit_group;" ::: "memory");
        }
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncwarp();
        sb ^= 1;
      }
#pragma unroll
      for (int tp = 0; tp < UG_TAPS; ++tp) {
        float acc[NT][4];
        pw_chain<KS, NT>(acc, a, wb[tp], bv);
        if constexpr (MODE == UG_STATS) {
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            f1[nt][0] += acc[nt][0] + acc[nt][2];
            f1[nt][1] += acc[nt][1] + acc[nt][3];
            f2[nt][0] = fmaf(acc[nt][0], acc[nt][0], fmaf(acc[nt][2], acc[nt][2], f2[nt][0]));
            f2[nt][1] = fmaf(acc[nt][1], acc[nt][1], fmaf(acc[nt][3], acc[nt][3], f2[nt][1]));
          }
        } else {
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const float2 A = *reinterpret_cast<const float2*>(s_cf + nt * 8 + 2 * tq);
            const float2 B = *reinterpret_cast<const float2*>(s_cf + C + nt * 8 + 2 * tq);
            float y[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) y[k] = ug_round(acc[nt][k]);
            bf16* s0 = stage + ug_frag(tp, 0, nt, gq, tq);
            bf16* s1 = stage + ug_frag(tp, 1, nt, gq, tq);
            if constexpr (MODE == UG_APPLY) {
              *reinterpret_cast<__nv_bfloat162*>(s0) =
                  __floats2bfloat162_rn(fmaxf(fmaf(y[0], A.x, B.x), 0.f), fmaxf(fmaf(y[1], A.y, B.y), 0.f));
              *reinterpret_cast<__nv_bfloat162*>(s1) =
                  __floats2bfloat162_rn(fmaxf(fmaf(y[2], A.x, B.x), 0.f), fmaxf(fmaf(y[3], A.y, B.y), 0.f));
            } else {
              const float2 glo = ug_ld2(s0), ghi = ug_ld2(s1);
              const float gv[4] = {glo.x, glo.y, ghi.x, ghi.y};
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const int j = k & 1;
                const float d = fmaf(y[k], j ? A.y : A.x, j ? B.y : B.x) > 0.f ? gv[k] : 0.f;
                f1[nt][j] += d;
                f2[nt][j] = fmaf(d, y[k], f2[nt][j]);
                f3[nt][j] += y[k];
              }
            }
          }
        }
      }
      if constexpr (MODE == UG_APPLY) {
        __syncwarp();
        ug_stage_store(stage, p.out, p.ldo, ob, fw, fh, lane);
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
  }
  if (MODE != UG_APPLY) flush(cur_n);
}

// ------------------------------------------------------------------------------------------------
// BWD
// ------------------------------------------------------------------------------------------------
struct UbSmem {
  size_t x, wf, wd, dys, stage, coef, total;
};
__host__ __device__ inline UbSmem ub_smem() {
  UbSmem s;
  s.x = 0;
  s.wf = s.x + (size_t)2 * UB_TILE * UG_XP;
  s.wd = s.wf + (size_t)UG_TAPS * UG_KS * UG_NT * 32 * sizeof(uint2);
  s.dys = s.wd + (size_t)UG_TAPS * (UG_CI / 8) * 32 * sizeof(uint2);
  s.stage = s.dys + (size_t)(UB_TILE / 16) * UG_TAPS * 16 * UB_DYP * 2;
  s.coef = s.stage + (size_t)8 * 2 * UG_STAGE * 2;
  s.total = s.coef + gn_cta_doubles(UG_C, UG_GROUPS, true) * sizeof(double) + (size_t)(3 + 5) * UG_C * sizeof(float);
  return s;
}

__global__ void __launch_bounds__(PW_THREADS, 1) up_gn_bwd_kernel(const __grid_constant__ UpGnParams p) {
  PDL_ENTER();
  constexpr int KS = UG_KS, NT = UG_NT, C = UG_C, XP = UG_XP, CT = UG_CI / 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const UbSmem L = ub_smem();
  uint2* s_wf = reinterpret_cast<uint2*>(smem_raw + L.wf);       // [tap][ks][nt][lane]: forward B fragments
  uint2* s_wd = reinterpret_cast<uint2*>(smem_raw + L.wd);       // [tap][ci tile][lane]: data-gradient B fragments
  bf16* s_dy = reinterpret_cast<bf16*>(smem_raw + L.dys);        // [group][tap][16 voxels][UB_DYP]
  double* s_d = reinterpret_cast<double*>(smem_raw + L.coef);
  float* s_f = reinterpret_cast<float*>(s_d + gn_cta_doubles(C, UG_GROUPS, true));
  float* s_cf = s_f + 3 * C;                                     // A, B, P, Q, R
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gq = lane >> 2, tq = lane & 3;
  bf16* stage0 = reinterpret_cast<bf16*>(smem_raw + L.stage) + (size_t)warp * 2 * UG_STAGE;   // two per warp
  // fine voxel (tap (0,0,0), fragment row 0) of the warp's group in a tile
  auto group_base = [&](long long tile, int& fw, int& fh) {
    return pw_up_base(tile * UB_TILE + warp * 16, p.V, p.D, p.H, p.W, 2, fw, fh);
  };

  // B fragments from the forward operand w[tap][co][ci]: the forward chain's (k = ci, n = co) and the data
  // gradient's (k = co, n = ci) = W^T of each tap, so no separate data-gradient pack is needed
  for (int i = threadIdx.x; i < UG_TAPS * KS * NT * 32; i += PW_THREADS) {
    const int ln = i & 31, nt = (i >> 5) % NT, ks = (i >> 5) / NT % KS, tp = (i >> 5) / (NT * KS);
    uint2 b;
    pw_b_frag<UG_CI, C>(p.w, tp, ks, nt, ln >> 2, ln & 3, b.x, b.y);
    s_wf[i] = b;
  }
  for (int i = threadIdx.x; i < UG_TAPS * CT * 32; i += PW_THREADS) {
    const int ln = i & 31, ct = (i >> 5) % CT, tp = (i >> 5) / CT;
    const int ci = ct * 8 + (ln >> 2), co = 2 * (ln & 3);
    const unsigned short* wt = reinterpret_cast<const unsigned short*>(p.w) + (size_t)tp * C * UG_CI + ci;
    uint2 b;
    b.x = (uint32_t)wt[co * UG_CI] | ((uint32_t)wt[(co + 1) * UG_CI] << 16);
    b.y = (uint32_t)wt[(co + 8) * UG_CI] | ((uint32_t)wt[(co + 9) * UG_CI] << 16);
    s_wd[i] = b;
  }
  float bv[NT][2];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    bv[nt][0] = p.bias ? p.bias[nt * 8 + 2 * tq] : 0.f;
    bv[nt][1] = p.bias ? p.bias[nt * 8 + 2 * tq + 1] : 0.f;
  }
  float accw[CT][4];                            // dW[tap = warp][co][ci] of this CTA
#pragma unroll
  for (int ct = 0; ct < CT; ++ct) accw[ct][0] = accw[ct][1] = accw[ct][2] = accw[ct][3] = 0.f;
  auto coefs = [&](long long n) {
    gn_coefs<true, true>(GnCta(), p.gn, p.sums, (int)n, C, s_d, s_f, s_cf, s_cf + C, s_cf + 2 * C, s_cf + 3 * C,
                         s_cf + 4 * C);
  };
  auto cf = [&](int k, int nt) { return *reinterpret_cast<const float2*>(s_cf + k * C + nt * 8 + 2 * tq); };

  const long long tiles = p.NV / UB_TILE;
  const long long tpc = (tiles + gridDim.x - 1) / gridDim.x;
  const long long first = blockIdx.x * tpc;
  const long long last = first + tpc < tiles ? first + tpc : tiles;
  const int a_lane = pw_a_lane(lane, XP);
  const int vrow = (lane >> 4) * 8 + (lane & 7);                 // ldmatrix.trans row of the dy^T fragments
  const uint32_t dys0 = (uint32_t)__cvta_generic_to_shared(s_dy);
  long long cur_n = -1;
  int sb = 0;                                                    // the stage holding the current group's g
  if (first < last) {
    ug_load_tile(smem_raw, p.x, p.xld, first * UB_TILE, UB_TILE);
    int fw, fh;
    const long long ob = group_base(first, fw, fh);
    ug_stage_load(stage0, p.g, p.ldg, ob, fw, fh, lane);
    asm volatile("cp.async.wait_all;" ::: "memory");
  }
  __syncthreads();
  for (long long tile = first; tile < last; ++tile) {
    const int buf = (int)((tile - first) & 1);
    const bool more = tile + 1 < last;
    if (more) ug_load_tile(smem_raw + (size_t)(buf ^ 1) * UB_TILE * XP, p.x, p.xld, (tile + 1) * UB_TILE, UB_TILE);
    const long long n = tile * UB_TILE / p.V;
    if (n != cur_n) {
      coefs(n);
      cur_n = n;
    }
    const uint32_t xs = (uint32_t)__cvta_generic_to_shared(smem_raw + (size_t)buf * UB_TILE * XP);
    // ---- phase 1: the warp's 16-voxel group, all taps: y -> dy -> data gradient; dy parked for phase 2
    {
      const int grp = warp, r0 = grp * 16;
      uint32_t a[KS][4];
      pw_a_frags<KS>(a, xs, r0 * XP + a_lane);
      const long long v0 = tile * UB_TILE + r0;
      const bf16* stage = stage0 + sb * UG_STAGE;
      __syncwarp();                             // every lane is done with the stage it is about to refill
      if (more) {                               // g of the next tile's group streams in while this one is computed
        int nfw, nfh;
        const long long nob = group_base(tile + 1, nfw, nfh);
        ug_stage_load(stage0 + (sb ^ 1) * UG_STAGE, p.g, p.ldg, nob, nfw, nfh, lane);
      } else {
        asm volatile("cp.async.commit_group;" ::: "memory");
      }
      asm volatile("cp.async.wait_group 1;" ::: "memory");
      __syncwarp();
      sb ^= 1;
      float dxa[CT][4];
#pragma unroll
      for (int ct = 0; ct < CT; ++ct) dxa[ct][0] = dxa[ct][1] = dxa[ct][2] = dxa[ct][3] = 0.f;
#pragma unroll
      for (int tp = 0; tp < UG_TAPS; ++tp) {
        uint32_t wb[KS][NT][2];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) {
            const uint2 b = s_wf[((tp * KS + ks) * NT + nt) * 32 + lane];
            wb[ks][nt][0] = b.x;
            wb[ks][nt][1] = b.y;
          }
        float acc[NT][4];
        pw_chain<KS, NT>(acc, a, wb, bv);
        uint32_t af[4];                         // dy as the A operand (rows = coarse voxels, k = 16 channels)
        bf16* dq = s_dy + ((size_t)(grp * UG_TAPS + tp) * 16 + gq) * UB_DYP + 2 * tq;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const float2 A = cf(0, nt), B = cf(1, nt), P = cf(2, nt), Q = cf(3, nt), R = cf(4, nt);
          const float2 glo = ug_ld2(stage + ug_frag(tp, 0, nt, gq, tq));
          const float2 ghi = ug_ld2(stage + ug_frag(tp, 1, nt, gq, tq));
          const float gv[4] = {glo.x, glo.y, ghi.x, ghi.y};
          float o[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const bool j = k & 1;
            const float y = ug_round(acc[nt][k]);
            const float dm = fmaf(y, j ? A.y : A.x, j ? B.y : B.x) > 0.f ? gv[k] * (j ? P.y : P.x) : 0.f;
            o[k] = dm + fmaf(y, j ? Q.y : Q.x, j ? R.y : R.x);
          }
          const __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], o[3]);
          *reinterpret_cast<__nv_bfloat162*>(dq + nt * 8) = lo;
          *reinterpret_cast<__nv_bfloat162*>(dq + 8 * UB_DYP + nt * 8) = hi;
          af[2 * nt] = ug_pack(lo);
          af[2 * nt + 1] = ug_pack(hi);
        }
#pragma unroll
        for (int ct = 0; ct < CT; ++ct) {
          const uint2 b = s_wd[(tp * CT + ct) * 32 + lane];
          pw_mma(dxa[ct], af, b.x, b.y);
        }
      }
      bf16* px = p.dx + (v0 + gq) * p.ldx + 2 * tq;
#pragma unroll
      for (int ct = 0; ct < CT; ++ct) {
        *reinterpret_cast<__nv_bfloat162*>(px + ct * 8) = __floats2bfloat162_rn(dxa[ct][0], dxa[ct][1]);
        *reinterpret_cast<__nv_bfloat162*>(px + 8 * p.ldx + ct * 8) = __floats2bfloat162_rn(dxa[ct][2], dxa[ct][3]);
      }
    }
    __syncthreads();
    // ---- phase 2: warp = tap; dW[tap][co][ci] += sum over the tile's voxels of dy[co] x[ci]
#pragma unroll 1
    for (int grp = 0; grp < UB_TILE / 16; ++grp) {
      uint32_t af[4], bx[KS][4];
      const uint32_t da = dys0 + (uint32_t)(((grp * UG_TAPS + warp) * 16 + vrow) * UB_DYP + ((lane >> 3) & 1) * 8) * 2;
      asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                   : "=r"(af[0]), "=r"(af[1]), "=r"(af[2]), "=r"(af[3])
                   : "r"(da));
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                     : "=r"(bx[ks][0]), "=r"(bx[ks][1]), "=r"(bx[ks][2]), "=r"(bx[ks][3])
                     : "r"(xs + (uint32_t)(grp * 16 * XP + a_lane + ks * 32)));
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        pw_mma(accw[2 * ks], af, bx[ks][0], bx[ks][1]);
        pw_mma(accw[2 * ks + 1], af, bx[ks][2], bx[ks][3]);
      }
    }
    if (more) asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
  }
  if (first < last) {
    float* dwt = p.dw + (size_t)warp * C * UG_CI;
#pragma unroll
    for (int ct = 0; ct < CT; ++ct) {
      const int ci = ct * 8 + 2 * tq;
      atomicAdd(dwt + gq * UG_CI + ci, accw[ct][0]);
      atomicAdd(dwt + gq * UG_CI + ci + 1, accw[ct][1]);
      atomicAdd(dwt + (gq + 8) * UG_CI + ci, accw[ct][2]);
      atomicAdd(dwt + (gq + 8) * UG_CI + ci + 1, accw[ct][3]);
    }
  }
  // d gamma, d beta, d bias: one CTA per sample, from the sums (as gn_bwd_apply_kernel)
  for (int s = blockIdx.x; s < p.N; s += gridDim.x) {
    __syncthreads();
    const double* grp = gn_coefs<true, true>(GnCta(), p.gn, p.sums, s, C, s_d, s_f, s_cf, s_cf + C, s_cf + 2 * C,
                                             s_cf + 3 * C, s_cf + 4 * C);
    param_grads_of_sample(p.gn, p.sums, grp, s_f, s, C, p.dgamma, p.dbeta, p.dbias);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int pw_mma_supported(int kind, int dims, const b200seg_tensor* x, int w_dtype, const b200seg_tensor* y,
                     const b200seg_tensor* addend);

// the fine-grid tensor the transposed convolution of x would write
static b200seg_tensor ug_fine(const b200seg_tensor* x) {
  b200seg_tensor y = *x;
  y.d *= 2; y.h *= 2; y.w *= 2;
  y.c = UG_C;
  y.ld = UG_C;
  y.dtype = B200SEG_BF16;
  return y;
}

int up_gn_supported(const b200seg_tensor* x, int cout, int dims) {
  if (x == nullptr || dims != 3 || cout != UG_C || x->c != UG_CI || x->dtype != B200SEG_BF16) return 0;
  // exactly the shapes b200seg_conv runs on pw_conv_mma_kernel<32, 16, true>: the recompute is bit-identical to it
  const b200seg_tensor y = ug_fine(x);
  return pw_mma_supported(B200SEG_UP, 3, x, B200SEG_BF16_TC, &y, nullptr);
}

static bool ug_fine_ok(const b200seg_tensor* t, const b200seg_tensor* x) {
  return t && t->ptr && t->dtype == B200SEG_BF16 && t->c == UG_C && t->n == x->n && t->d == 2 * x->d &&
         t->h == 2 * x->h && t->w == 2 * x->w && (t->ld % 8) == 0 && (reinterpret_cast<uintptr_t>(t->ptr) % 16) == 0;
}

static bool ug_gn_ok(const b200seg_gn* gn, const b200seg_tensor* x) {
  return gn && gn->stats && gn->gamma && gn->beta && gn->groups == UG_GROUPS &&
         gn->vox == 8LL * x->d * x->h * x->w;
}

template <typename Kern>
static int ug_launch(Kern kernel, const UpGnParams& p, size_t smem, long long tiles, int device, cudaStream_t st,
                     int* attr_done) {
  if (smem > 48 * 1024 && device >= 0 && device < 64 && !attr_done[device]) {
    B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done[device] = 1;
  }
  long long grid = num_sms(device);
  if (grid > tiles) grid = tiles;
  launch_k(kernel, (unsigned)grid, PW_THREADS, smem, st, p);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int up_gn(int mode, const b200seg_tensor* x, const void* w, const float* bias, const b200seg_gn* gn, double* stats,
          const b200seg_tensor* out, const b200seg_tensor* gr, double* sums, float* dw, const b200seg_tensor* dx,
          float* dgamma, float* dbeta, float* dbias, int device, cudaStream_t st) {
  B200_CHECK_ARG(up_gn_supported(x, UG_C, 3), "b200seg_up_gn: unsupported input (bf16, 32 channels, 3-D, the shapes "
                 "of the pointwise mma.sync transposed convolution)");
  B200_CHECK_ARG(w != nullptr, "b200seg_up_gn: null weights");
  UpGnParams p;
  memset(&p, 0, sizeof(p));
  p.x = static_cast<const bf16*>(x->ptr);
  p.xld = x->ld;
  p.w = static_cast<const bf16*>(w);
  p.bias = bias;
  p.V = (long long)x->d * x->h * x->w;
  p.NV = p.V * x->n;
  p.N = x->n; p.D = x->d; p.H = x->h; p.W = x->w;
  const long long tiles = p.NV / PW_TILE;
  if (mode == 0) {
    B200_CHECK_ARG(stats != nullptr, "b200seg_up_gn_stats: null statistics");
    p.stats = stats;
    static int attr[64] = {0};
    return ug_launch(up_gn_kernel<UG_STATS>, p, ug_smem(UG_STATS), tiles, device, st, attr);
  }
  B200_CHECK_ARG(ug_gn_ok(gn, x), "b200seg_up_gn: bad GroupNorm reference (8 groups, vox = the fine grid's D*H*W)");
  p.gn = gn_ref(gn, UG_C);
  if (mode == 1) {
    B200_CHECK_ARG(ug_fine_ok(out, x), "b200seg_up_gn_apply: bad output tensor (bf16, 16 channels, the fine grid, 16-byte aligned rows)");
    p.out = static_cast<bf16*>(out->ptr);
    p.ldo = out->ld;
    static int attr[64] = {0};
    return ug_launch(up_gn_kernel<UG_APPLY>, p, ug_smem(UG_APPLY), tiles, device, st, attr);
  }
  B200_CHECK_ARG(ug_fine_ok(gr, x), "b200seg_up_gn: bad gradient tensor (bf16, 16 channels, the fine grid, 16-byte aligned rows)");
  B200_CHECK_ARG(sums != nullptr, "b200seg_up_gn: null backward sums");
  p.g = static_cast<const bf16*>(gr->ptr);
  p.ldg = gr->ld;
  p.sums = sums;
  if (mode == 2) {
    static int attr[64] = {0};
    return ug_launch(up_gn_kernel<UG_BSUMS>, p, ug_smem(UG_BSUMS), tiles, device, st, attr);
  }
  B200_CHECK_ARG(mode == 3 && dw && dgamma && dbeta, "b200seg_up_gn_bwd: null gradient");
  B200_CHECK_ARG(dx && dx->ptr && dx->dtype == B200SEG_BF16 && dx->c == UG_CI && dx->n == x->n && dx->d == x->d &&
                 dx->h == x->h && dx->w == x->w && (dx->ld % 2) == 0 && (reinterpret_cast<uintptr_t>(dx->ptr) % 4) == 0,
                 "b200seg_up_gn_bwd: bad data-gradient tensor (bf16, 32 channels, the coarse grid)");
  p.dw = dw;
  p.dx = static_cast<bf16*>(dx->ptr);
  p.ldx = dx->ld;
  p.dgamma = dgamma;
  p.dbeta = dbeta;
  p.dbias = dbias;
  static int attr[64] = {0};
  return ug_launch(up_gn_bwd_kernel, p, ub_smem().total, p.NV / UB_TILE, device, st, attr);
}

}  // namespace b200seg
