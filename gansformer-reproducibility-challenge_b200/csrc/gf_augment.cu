// gf_augment.cu -- adaptive discriminator augmentation (include/gf_ops.h, SURVEY A.4 item 15): the integer "pixel blitting"
// geometry and the per-image colour matrix in one pass over an NCHW fp32 image, and its adjoint.
//
// Both kernels walk 32 x 8 pixel tiles of the OUTPUT of their direction (the augmented image forward, the source image in the
// adjoint) with a tile-stride loop, so any batch fits one grid.  A tile of a transposing dihedral map (rotation by 90 or 270
// degrees) reads 8 source columns of 32 rows: four 32-byte sectors per row, which L1 serves to the block's 8 warps.
#include "gf_common.cuh"
#include "../../include/gf_ops.h"

namespace gf {

constexpr int AUG_TX = 32, AUG_TY = 8;

struct AugGeom { int code, tx, ty; };

// The per-image parameters as the kernels define them for ANY stored value (the host cannot check device data): the dihedral code
// masked to 3 bits, and on a non-square grid with bit 1 cleared (the transposing rotations by 90 / 270 degrees fall back to 0 / 180);
// |t| clamped to N - 1, so that one reflection brings every index back onto the grid.
__device__ __forceinline__ AugGeom aug_geom(const int* __restrict__ geom, int b, int H, int W) {
  AugGeom g;
  g.code = __ldg(geom + 4 * b) & 7;
  if (H != W) g.code &= ~2;
  g.tx = min(max(__ldg(geom + 4 * b + 1), -(W - 1)), W - 1);
  g.ty = min(max(__ldg(geom + 4 * b + 2), -(H - 1)), H - 1);
  return g;
}

// R_N: mirror without repeating the edge pixel; valid for i in [-(N-1), 2(N-1)]
__device__ __forceinline__ int aug_mirror(int i, int N) { return i < 0 ? -i : (i >= N ? 2 * (N - 1) - i : i); }

// D(x, y) = rotation by k * 90 degrees (k = code >> 1) after an x flip (code bit 0); a bijection of the grid onto itself
__device__ __forceinline__ void aug_dihedral(int code, int x, int y, int H, int W, int& u, int& v) {
  if (code & 1) x = W - 1 - x;
  switch (code >> 1) {
    case 0: u = x; v = y; break;
    case 1: u = y; v = W - 1 - x; break;              // H == W
    case 2: u = W - 1 - x; v = H - 1 - y; break;
    default: u = H - 1 - y; v = x; break;             // H == W
  }
}

// D^-1(u, v)
__device__ __forceinline__ void aug_dihedral_inv(int code, int u, int v, int H, int W, int& x, int& y) {
  switch (code >> 1) {
    case 0: x = u; y = v; break;
    case 1: x = W - 1 - v; y = u; break;
    case 2: x = W - 1 - u; y = H - 1 - v; break;
    default: x = v; y = H - 1 - u; break;
  }
  if (code & 1) x = W - 1 - x;
}

// The preimages s (s - t in the blit's sense: s = d - t for an output coordinate d in [0, N)) of source index q under R_N, in a
// fixed order: q itself, then its one mirror that can be reached (-q for t > 0, 2(N-1) - q for t < 0).  Returns the count (0..2).
__device__ __forceinline__ int aug_preimages(int q, int t, int N, int s[2]) {
  int n = 0;
  if (q >= -t && q <= N - 1 - t) s[n++] = q;
  if (q > 0 && q <= t) s[n++] = -q;                                   // -q >= -t
  if (q < N - 1 && q >= N - 1 + t) s[n++] = 2 * (N - 1) - q;          // 2(N-1) - q <= N - 1 - t
  return n;
}

__global__ void __launch_bounds__(AUG_TX * AUG_TY) augment_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                  const int* __restrict__ geom, const float* __restrict__ color,
                                                                  int C, int H, int W, long long tiles, int tiles_x, int tiles_y) {
  const size_t HW = (size_t)H * W;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int b = (int)(tile / ((long long)tiles_x * tiles_y));
    const int rem = (int)(tile % ((long long)tiles_x * tiles_y));
    const int px = (rem % tiles_x) * AUG_TX + threadIdx.x, py = (rem / tiles_x) * AUG_TY + threadIdx.y;
    if (px >= W || py >= H) continue;
    const AugGeom g = aug_geom(geom, b, H, W);
    int u, v;
    aug_dihedral(g.code, px, py, H, W, u, v);
    const int sx = aug_mirror(u - g.tx, W), sy = aug_mirror(v - g.ty, H);
    const float* src = x + (size_t)b * C * HW + (size_t)sy * W + sx;
    float* dst = y + (size_t)b * C * HW + (size_t)py * W + px;
    if (color) {                                                      // C == 3: out_c = M[c][0] r + M[c][1] g + M[c][2] b + M[c][3]
      const float* M = color + 12 * b;
      const float r = __ldg(src), gr = __ldg(src + HW), bl = __ldg(src + 2 * HW);
#pragma unroll
      for (int c = 0; c < 3; ++c)
        dst[c * HW] = fmaf(__ldg(M + 4 * c + 2), bl, fmaf(__ldg(M + 4 * c + 1), gr, fmaf(__ldg(M + 4 * c), r, __ldg(M + 4 * c + 3))));
    } else {
      for (int c = 0; c < C; ++c) dst[c * HW] = __ldg(src + c * HW);
    }
  }
}

// gx = A^T gy: at every source pixel q, the sum over the output pixels p that read q (at most 2 per axis, gathered in a fixed
// order: no atomics, the same bits on every run) of M3^T gy[p], M3 the colour matrix without its offset column.
__global__ void __launch_bounds__(AUG_TX * AUG_TY) augment_adjoint_kernel(const float* __restrict__ gy, float* __restrict__ gx,
                                                                          const int* __restrict__ geom, const float* __restrict__ color,
                                                                          int C, int H, int W, long long tiles, int tiles_x, int tiles_y) {
  const size_t HW = (size_t)H * W;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int b = (int)(tile / ((long long)tiles_x * tiles_y));
    const int rem = (int)(tile % ((long long)tiles_x * tiles_y));
    const int qx = (rem % tiles_x) * AUG_TX + threadIdx.x, qy = (rem / tiles_x) * AUG_TY + threadIdx.y;
    if (qx >= W || qy >= H) continue;
    const AugGeom g = aug_geom(geom, b, H, W);
    int sxs[2], sys[2];
    const int nx = aug_preimages(qx, g.tx, W, sxs), ny = aug_preimages(qy, g.ty, H, sys);
    const float* src = gy + (size_t)b * C * HW;
    float* dst = gx + (size_t)b * C * HW + (size_t)qy * W + qx;
    if (color) {
      const float* M = color + 12 * b;
      float m[3][3];
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < 3; ++j) m[c][j] = __ldg(M + 4 * c + j);
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      for (int iy = 0; iy < ny; ++iy)
        for (int ix = 0; ix < nx; ++ix) {
          int px, py;
          aug_dihedral_inv(g.code, sxs[ix] + g.tx, sys[iy] + g.ty, H, W, px, py);
          const float* s = src + (size_t)py * W + px;
          const float g0 = __ldg(s), g1 = __ldg(s + HW), g2 = __ldg(s + 2 * HW);
          a0 += fmaf(m[2][0], g2, fmaf(m[1][0], g1, m[0][0] * g0));
          a1 += fmaf(m[2][1], g2, fmaf(m[1][1], g1, m[0][1] * g0));
          a2 += fmaf(m[2][2], g2, fmaf(m[1][2], g1, m[0][2] * g0));
        }
      dst[0] = a0; dst[HW] = a1; dst[2 * HW] = a2;
    } else {
      int off[4], n = 0;
      for (int iy = 0; iy < ny; ++iy)
        for (int ix = 0; ix < nx; ++ix) {
          int px, py;
          aug_dihedral_inv(g.code, sxs[ix] + g.tx, sys[iy] + g.ty, H, W, px, py);
          off[n++] = py * W + px;
        }
      for (int c = 0; c < C; ++c) {
        float a = 0.f;
        for (int i = 0; i < n; ++i) a += __ldg(src + c * HW + off[i]);
        dst[c * HW] = a;
      }
    }
  }
}

// Shared argument checks of both entry points; fills the tile grid.
static int augment_check(const char* name, const float* in, const float* out, const int* geom, const float* color, int B, int C, int H,
                         int W, long long* tiles, int* tiles_x, int* tiles_y) {
  if (!in || !out || !geom) { set_error("%s: null pointer", name); return GF_ERR_INVALID; }
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("%s: bad sizes B=%d C=%d H=%d W=%d", name, B, C, H, W); return GF_ERR_INVALID; }
  if (H < 2 || W < 2) { set_error("%s: H and W must be at least 2 (H=%d W=%d)", name, H, W); return GF_ERR_UNSUPPORTED; }
  if (color && C != 3) { set_error("%s: a colour matrix needs C == 3 (C=%d)", name, C); return GF_ERR_UNSUPPORTED; }
  if (H > 32768 || W > 32768 || (long long)C * H * W > 0x7fffffffLL) {
    set_error("%s: image too large (C=%d H=%d W=%d): H, W <= 32768 and C*H*W < 2^31", name, C, H, W); return GF_ERR_UNSUPPORTED;
  }
  *tiles_x = (W + AUG_TX - 1) / AUG_TX;
  *tiles_y = (H + AUG_TY - 1) / AUG_TY;
  *tiles = (long long)B * *tiles_x * *tiles_y;
  return GF_OK;
}

static inline int augment_grid(long long tiles) {
  const long long cap = (long long)num_sms() * 8;                     // 8 CTAs of 256 threads per SM; larger batches loop
  return (int)(tiles < cap ? tiles : cap);
}

}  // namespace gf

using namespace gf;

extern "C" {

int gf_augment_nchw(const float* x, float* y, const int* geom, const float* color, int B, int C, int H, int W, void* stream) {
  long long tiles; int tx, ty;
  const int rc = augment_check("gf_augment_nchw", x, y, geom, color, B, C, H, W, &tiles, &tx, &ty);
  if (rc != GF_OK) return rc;
  augment_kernel<<<augment_grid(tiles), dim3(AUG_TX, AUG_TY), 0, (cudaStream_t)stream>>>(x, y, geom, color, C, H, W, tiles, tx, ty);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_augment_adjoint_nchw(const float* gy, float* gx, const int* geom, const float* color, int B, int C, int H, int W, void* stream) {
  long long tiles; int tx, ty;
  const int rc = augment_check("gf_augment_adjoint_nchw", gy, gx, geom, color, B, C, H, W, &tiles, &tx, &ty);
  if (rc != GF_OK) return rc;
  augment_adjoint_kernel<<<augment_grid(tiles), dim3(AUG_TX, AUG_TY), 0, (cudaStream_t)stream>>>(gy, gx, geom, color, C, H, W, tiles, tx, ty);
  GF_LAUNCH_OK();
  return GF_OK;
}

}  // extern "C"
