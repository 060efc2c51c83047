// Fragment code of the pointwise / k2s2-transposed mma.sync convolution (pw_mma.cu), shared with the fused up_tr32
// layer (up_gn.cu): both build the same A fragments (ldmatrix from a voxel-major tile), the same B fragments from the
// packed [tap][COUT][CIN] weights and run the same m16n8k16 chain, so a recomputed transposed-conv output is
// bit-identical to the one pw_conv_mma_kernel stores.
#pragma once

#include "common.cuh"

namespace b200seg {

constexpr int PW_TILE = 512;            // voxels per CTA step
constexpr int PW_THREADS = 256;

__device__ __forceinline__ void pw_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// B fragment of (tap tp, k-step ks, n-tile nt): b0 = (k = 2t, 2t+1 ; n = g), b1 = (k = 2t+8, 2t+9 ; n = g);
// w is [tap][n][k], k contiguous
template <int CIN, int COUT>
__device__ __forceinline__ void pw_b_frag(const bf16* w, int tp, int ks, int nt, int gq, int tq,
                                          uint32_t& b0, uint32_t& b1) {
  const bf16* wr = w + (tp * COUT + nt * 8 + gq) * CIN + ks * 16 + 2 * tq;
  b0 = *reinterpret_cast<const uint32_t*>(wr);
  b1 = *reinterpret_cast<const uint32_t*>(wr + 8);
}

// ldmatrix (non-transposed) lane address in a tile of XP-byte voxel rows: matrix m = lane >> 3 -> (voxel half m & 1,
// channel half m >> 1)
__device__ __forceinline__ int pw_a_lane(int lane, int XP) {
  return (((lane >> 3) & 1) * 8 + (lane & 7)) * XP + (lane >> 4) * 16;
}

// A fragments of the 16-voxel row group starting at byte offset `row` of the shared tile xs
template <int KS>
__device__ __forceinline__ void pw_a_frags(uint32_t (&a)[KS][4], uint32_t xs, int row) {
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(a[ks][0]), "=r"(a[ks][1]), "=r"(a[ks][2]), "=r"(a[ks][3])
                 : "r"(xs + (uint32_t)(row + ks * 32)));
}

// acc[nt] = bias + A x B(tap): the k-steps in order, per n-tile
template <int KS, int NT>
__device__ __forceinline__ void pw_chain(float (&acc)[NT][4], const uint32_t (&a)[KS][4],
                                         const uint32_t (&wb)[KS][NT][2], const float (&bv)[NT][2]) {
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    acc[nt][0] = acc[nt][2] = bv[nt][0];
    acc[nt][1] = acc[nt][3] = bv[nt][1];
  }
#pragma unroll
  for (int ks = 0; ks < KS; ++ks)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) pw_mma(acc[nt], a[ks], wb[ks][nt][0], wb[ks][nt][1]);
}

// k2s2 transposed conv: fine voxel of coarse voxel v0 (the first of a 16-voxel w-row group) at tap (0,0,0), and the
// fine row pitches fw (= 2W) and fh (= 2H)
__device__ __forceinline__ long long pw_up_base(long long v0, long long V, int D, int H, int W, int ud, int& fw,
                                                int& fh) {
  const long long vs = v0 % V;
  const long long ns = v0 / V;
  const int cw = (int)(vs % W), ch = (int)((vs / W) % H), cd = (int)(vs / ((long long)W * H));
  fw = 2 * W;
  fh = 2 * H;
  return ((ns * (D * ud) + (long long)cd * ud) * fh + 2 * ch) * fw + 2 * cw;
}

}  // namespace b200seg
