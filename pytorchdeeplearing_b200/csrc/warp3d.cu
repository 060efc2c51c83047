// voxelmorph's SpatialTransformer as VNet3dRegistration uses it (networks/VNet3dregistration.py:6-45,171-206): the
// reference builds sampling locations from the predicted displacement field and calls
// F.grid_sample(src, new_locs, align_corners=True) once with mode='bilinear' (trilinear on 5-D input) for the moving
// image and once with mode='nearest' for the moving label.  Both run here in one launch; the backward gives d loss /
// d ddf through the image path (nearest sampling has no gradient, and the moving volumes are inputs).
//
// Positions follow torch's arithmetic exactly (ATen GridSampler: grid_sampler_unnormalize, then the floor cell and
// the eight corner weights for trilinear, nearbyint for nearest), so the nearest labels are bit-identical to torch's
// and the trilinear weights are the same fp32 numbers.
#include "common.cuh"

namespace b200seg {

namespace {

// The sampling position along one axis of extent s (> 1) for grid index gi and displacement f, in the reference's
// fp32 order: loc = grid + flow; 2 * (loc / (s - 1) - 0.5); then ((n + 1) / 2) * (s - 1).  Every step is one
// rounded operation (__fadd_rn / __fdiv_rn / __fmul_rn cannot be contracted into FMAs).
__device__ __forceinline__ float warp_coord(int gi, float f, int s) {
  const float sm1 = (float)(s - 1);
  const float loc = __fadd_rn((float)gi, f);
  const float nrm = __fmul_rn(2.f, __fsub_rn(__fdiv_rn(loc, sm1), 0.5f));
  return __fmul_rn(__fdiv_rn(__fadd_rn(nrm, 1.f), 2.f), sm1);
}

// Corner indices (floor cell) and trilinear weights of one sample; ok[k] marks the corners inside the volume.
// Corners in grid_sample's order: tnw, tne, tsw, tse, bnw, bne, bsw, bse (t/b = z, n/s = y, w/e = x).
struct Cell {
  long long off[8];
  bool ok[8];
  float w[8];
  int x0, y0, z0;
  float ix, iy, iz;
  bool any;       // every coordinate passes coord_in_range: the weights are finite and some corners may be inside
};

// |coordinate| far beyond the volume: every corner is outside (and floor() stays within int range)
__device__ __forceinline__ bool coord_in_range(float u, int s) { return u > -2.f && u < (float)s + 1.f; }

__device__ __forceinline__ void make_cell(float ix, float iy, float iz, int D, int H, int W, Cell& c) {
  c.ix = ix; c.iy = iy; c.iz = iz;
  const bool any = coord_in_range(ix, W) && coord_in_range(iy, H) && coord_in_range(iz, D);
  c.any = any;
  const int x0 = any ? (int)floorf(ix) : -4, y0 = any ? (int)floorf(iy) : -4, z0 = any ? (int)floorf(iz) : -4;
  c.x0 = x0; c.y0 = y0; c.z0 = z0;
  const float fx0 = (float)x0, fy0 = (float)y0, fz0 = (float)z0;
  const float fx1 = (float)(x0 + 1), fy1 = (float)(y0 + 1), fz1 = (float)(z0 + 1);
  // torch: tnw = (ix_bse - ix) * (iy_bse - iy) * (iz_bse - iz), ... products left to right
  const float ex = __fsub_rn(fx1, ix), wx = __fsub_rn(ix, fx0);
  const float ey = __fsub_rn(fy1, iy), wy = __fsub_rn(iy, fy0);
  const float ez = __fsub_rn(fz1, iz), wz = __fsub_rn(iz, fz0);
  c.w[0] = __fmul_rn(__fmul_rn(ex, ey), ez);   // tnw (x0, y0, z0)
  c.w[1] = __fmul_rn(__fmul_rn(wx, ey), ez);   // tne (x1, y0, z0)
  c.w[2] = __fmul_rn(__fmul_rn(ex, wy), ez);   // tsw (x0, y1, z0)
  c.w[3] = __fmul_rn(__fmul_rn(wx, wy), ez);   // tse (x1, y1, z0)
  c.w[4] = __fmul_rn(__fmul_rn(ex, ey), wz);   // bnw (x0, y0, z1)
  c.w[5] = __fmul_rn(__fmul_rn(wx, ey), wz);   // bne (x1, y0, z1)
  c.w[6] = __fmul_rn(__fmul_rn(ex, wy), wz);   // bsw (x0, y1, z1)
  c.w[7] = __fmul_rn(__fmul_rn(wx, wy), wz);   // bse (x1, y1, z1)
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int x = x0 + (k & 1), y = y0 + ((k >> 1) & 1), z = z0 + (k >> 2);
    c.ok[k] = x >= 0 && x < W && y >= 0 && y < H && z >= 0 && z < D;
    c.off[k] = c.ok[k] ? ((long long)z * H + y) * W + x : 0;
  }
}

__global__ void __launch_bounds__(256) warp3d_kernel(const float* __restrict__ ddf, const float* __restrict__ image,
                                                     int ci, const float* __restrict__ label, int cl, int N, int D,
                                                     int H, int W, float* __restrict__ moved_image,
                                                     float* __restrict__ moved_label) {
  PDL_ENTER();
  const long long V = (long long)D * H * W;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)N * V) return;
  const int n = (int)(i / V);
  const long long v = i - (long long)n * V;
  const int w = (int)(v % W), h = (int)((v / W) % H), d = (int)(v / ((long long)W * H));
  const float* f = ddf + i * 3;
  // channel 0 of the field moves along D (grid_sample's z), 1 along H (y), 2 along W (x)
  const float iz = warp_coord(d, f[0], D), iy = warp_coord(h, f[1], H), ix = warp_coord(w, f[2], W);
  if (ci > 0) {
    Cell c;
    make_cell(ix, iy, iz, D, H, W, c);
    for (int ch = 0; ch < ci; ++ch) {
      const float* src = image + ((long long)n * ci + ch) * V;
      float o = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (c.ok[k]) o = fmaf(src[c.off[k]], c.w[k], o);     // out += v * w, in corner order (as torch's CUDA kernel)
      moved_image[((long long)n * ci + ch) * V + v] = o;
    }
  }
  if (cl > 0) {
    const bool in = coord_in_range(ix, W) && coord_in_range(iy, H) && coord_in_range(iz, D);
    const int x = in ? (int)nearbyintf(ix) : -1, y = in ? (int)nearbyintf(iy) : -1, z = in ? (int)nearbyintf(iz) : -1;
    const bool ok = x >= 0 && x < W && y >= 0 && y < H && z >= 0 && z < D;
    const long long off = ok ? ((long long)z * H + y) * W + x : 0;
    for (int ch = 0; ch < cl; ++ch) {
      const float* src = label + ((long long)n * cl + ch) * V;
      moved_label[((long long)n * cl + ch) * V + v] = ok ? src[off] : 0.f;
    }
  }
}

__global__ void __launch_bounds__(256) warp3d_bwd_kernel(const float* __restrict__ ddf, const float* __restrict__ image,
                                                         int ci, const float* __restrict__ gmoved,
                                                         const float* __restrict__ addend, int N, int D, int H, int W,
                                                         float* __restrict__ gddf) {
  PDL_ENTER();
  const long long V = (long long)D * H * W;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)N * V) return;
  const int n = (int)(i / V);
  const long long v = i - (long long)n * V;
  const int w = (int)(v % W), h = (int)((v / W) % H), d = (int)(v / ((long long)W * H));
  const float* f = ddf + i * 3;
  const float iz = warp_coord(d, f[0], D), iy = warp_coord(h, f[1], H), ix = warp_coord(w, f[2], W);
  Cell c;
  make_cell(ix, iy, iz, D, H, W, c);
  const float fx0 = (float)c.x0, fy0 = (float)c.y0, fz0 = (float)c.z0;
  const float ex = __fsub_rn((float)(c.x0 + 1), ix), wx = __fsub_rn(ix, fx0);
  const float ey = __fsub_rn((float)(c.y0 + 1), iy), wy = __fsub_rn(iy, fy0);
  const float ez = __fsub_rn((float)(c.z0 + 1), iz), wz = __fsub_rn(iz, fz0);
  // d weight / d x, y, z of each corner (sign folded in below), grid_sample's gix / giy / giz accumulation.  A corner
  // outside the volume adds val = 0 times finite factors, i.e. nothing, as torch skips it -- but only while every
  // coordinate is in range: beyond it (|ddf| = inf, NaN) the factors are not finite and 0 * inf would be NaN, and
  // every corner is outside, so the sample adds nothing at all.
  float gix = 0.f, giy = 0.f, giz = 0.f;
  const int nch = c.any ? ci : 0;
  for (int ch = 0; ch < nch; ++ch) {
    const float* src = image + ((long long)n * ci + ch) * V;
    const float go = gmoved[((long long)n * ci + ch) * V + v];
    float val[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) val[k] = c.ok[k] ? src[c.off[k]] : 0.f;
    // x: the west corners (k even) lose, the east corners (k odd) gain
    gix -= val[0] * ey * ez * go;  giy -= val[0] * ex * ez * go;  giz -= val[0] * ex * ey * go;
    gix += val[1] * ey * ez * go;  giy -= val[1] * wx * ez * go;  giz -= val[1] * wx * ey * go;
    gix -= val[2] * wy * ez * go;  giy += val[2] * ex * ez * go;  giz -= val[2] * ex * wy * go;
    gix += val[3] * wy * ez * go;  giy += val[3] * wx * ez * go;  giz -= val[3] * wx * wy * go;
    gix -= val[4] * ey * wz * go;  giy -= val[4] * ex * wz * go;  giz += val[4] * ex * ey * go;
    gix += val[5] * ey * wz * go;  giy -= val[5] * wx * wz * go;  giz += val[5] * wx * ey * go;
    gix -= val[6] * wy * wz * go;  giy += val[6] * ex * wz * go;  giz += val[6] * ex * wy * go;
    gix += val[7] * wy * wz * go;  giy += val[7] * wx * wz * go;  giz += val[7] * wx * wy * go;
  }
  // grid_sample's grid gradient is gi * (s - 1) / 2; the normalisation 2 * (loc / (s - 1) - 0.5) contributes
  // 2 / (s - 1): d loss / d ddf along D, H, W
  const float gz = __fdiv_rn(__fmul_rn(__fmul_rn(giz, __fdiv_rn((float)(D - 1), 2.f)), 2.f), (float)(D - 1));
  const float gy = __fdiv_rn(__fmul_rn(__fmul_rn(giy, __fdiv_rn((float)(H - 1), 2.f)), 2.f), (float)(H - 1));
  const float gx = __fdiv_rn(__fmul_rn(__fmul_rn(gix, __fdiv_rn((float)(W - 1), 2.f)), 2.f), (float)(W - 1));
  float* o = gddf + i * 3;
  if (addend != nullptr) {
    const float* a = addend + i * 3;
    o[0] = __fadd_rn(gz, a[0]);
    o[1] = __fadd_rn(gy, a[1]);
    o[2] = __fadd_rn(gx, a[2]);
  } else {
    o[0] = gz;
    o[1] = gy;
    o[2] = gx;
  }
}

}  // namespace

static int warp_blocks(int N, int D, int H, int W) { return (int)(((long long)N * D * H * W + 255) / 256); }

static bool warp_dims_ok(int N, int D, int H, int W) {
  return N > 0 && D > 1 && H > 1 && W > 1 && (long long)N * D * H * W < (1ll << 31);
}

}  // namespace b200seg

using namespace b200seg;

extern "C" {

int b200seg_warp3d(const float* ddf, const float* image, int ci, const float* label, int cl, int N, int D, int H, int W,
                   float* moved_image, float* moved_label, int device, b200seg_stream stream) {
  B200_CHECK_ARG(ddf != nullptr && warp_dims_ok(N, D, H, W), "b200seg_warp3d: bad field or shape");
  B200_CHECK_ARG(ci >= 0 && cl >= 0 && ci + cl > 0, "b200seg_warp3d: nothing to warp");
  B200_CHECK_ARG(ci == 0 || (image != nullptr && moved_image != nullptr), "b200seg_warp3d: null image");
  B200_CHECK_ARG(cl == 0 || (label != nullptr && moved_label != nullptr), "b200seg_warp3d: null label");
  B200_DEVICE(device);
  launch_k(warp3d_kernel, warp_blocks(N, D, H, W), 256, 0, static_cast<cudaStream_t>(stream), ddf, image, ci, label,
           cl, N, D, H, W, moved_image, moved_label);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

int b200seg_warp3d_bwd(const float* ddf, const float* image, int ci, const float* gmoved, const float* addend, int N,
                       int D, int H, int W, float* gddf, int device, b200seg_stream stream) {
  B200_CHECK_ARG(ddf != nullptr && gddf != nullptr && warp_dims_ok(N, D, H, W), "b200seg_warp3d_bwd: bad field or shape");
  B200_CHECK_ARG(ci > 0 && image != nullptr && gmoved != nullptr, "b200seg_warp3d_bwd: null image or gradient");
  B200_DEVICE(device);
  launch_k(warp3d_bwd_kernel, warp_blocks(N, D, H, W), 256, 0, static_cast<cudaStream_t>(stream), ddf, image, ci,
           gmoved, addend, N, D, H, W, gddf);
  B200_LAUNCH_CHECK();
  return B200SEG_OK;
}

}  // extern "C"
