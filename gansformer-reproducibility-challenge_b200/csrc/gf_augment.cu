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

// ================================================================================================ fractional geometry (item 16)
// ADA's band-limited resampler: mirror extension E, 2x upsampling with sym6 (U), bilinear sampling at nu = L q + e on the 2x output
// grid (V), 2x downsampling with sym6.  Per axis: U[nu] = 2 sum_m E[m] f[nu + 5 - 2m] for nu in [-2(N-1), 4N-3] (zero beyond), and
// out[o] = sum_k f[k] V[2o + k + 1], V[q] read at nu(q).  Both kernels walk 16 x 16 tiles of their output with a tile-stride loop.
constexpr int RS_T = 16, RS_Q = 2 * RS_T + 10;                       // tile edge; 2x-grid points a tile's down filter reads per axis
constexpr int RS_CAP = 10240;                                         // floats per shared region (two regions: 80 KB per CTA)
constexpr int RS_QC = 64;                                             // adjoint: 2x output points per axis of one staged chunk
constexpr int RS_GU = RS_CAP - RS_Q * RS_Q;                           // adjoint: offset of the gU accumulator in the second region

constexpr double RS_SYM6[12] = {0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633,
                                0.4910559419267466, 0.787641141030194, 0.3379294217276218, -0.07263752278646252,
                                -0.021060292512300564, 0.04472490177066578, 0.0017677118642428036, -0.007800708325034148};
constexpr double RS_SUM = RS_SYM6[0] + RS_SYM6[1] + RS_SYM6[2] + RS_SYM6[3] + RS_SYM6[4] + RS_SYM6[5] + RS_SYM6[6] + RS_SYM6[7] +
                          RS_SYM6[8] + RS_SYM6[9] + RS_SYM6[10] + RS_SYM6[11];
#define RS_TAP(i) (float)(RS_SYM6[i] / RS_SUM)
__constant__ float rs_f[12] = {RS_TAP(0), RS_TAP(1), RS_TAP(2), RS_TAP(3), RS_TAP(4), RS_TAP(5),
                               RS_TAP(6), RS_TAP(7), RS_TAP(8), RS_TAP(9), RS_TAP(10), RS_TAP(11)};
#undef RS_TAP

__device__ __forceinline__ int fdiv2(int a) { return a >> 1; }        // floor(a / 2)
__device__ __forceinline__ int cdiv2(int a) { return -((-a) >> 1); }  // ceil(a / 2)

// The per-image map nu(q) = L q + e (2x output grid -> 2x source grid), composed of frac[b] = F^-1 and the blit of geom[b]; with
// `ident` (F^-1 exactly the identity: the blit) and `ok` (inside the domain: finite, singular values in [1/16, 16], |t| <= 64 max(H, W)).
struct ResMap { float l00, l01, l10, l11, e0, e1; bool ident, ok; };

__device__ ResMap res_map(const int* __restrict__ geom, const float* __restrict__ frac, int b, int H, int W) {
  ResMap m;
  float a[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = __ldg(frac + 6 * b + i);
  m.ident = a[0] == 1.f && a[1] == 0.f && a[2] == 0.f && a[3] == 0.f && a[4] == 1.f && a[5] == 0.f;
  const float s2 = a[0] * a[0] + a[1] * a[1] + a[3] * a[3] + a[4] * a[4], det = fabsf(a[0] * a[4] - a[1] * a[3]);
  const float smax2 = 0.5f * (s2 + sqrtf(fmaxf(s2 * s2 - 4.f * det * det, 0.f))), smin2 = det * det / smax2;
  const float tmax = 64.f * (float)max(H, W);
  bool fin = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) fin = fin && isfinite(a[i]);
  m.ok = fin && smax2 <= 256.f && smin2 >= 1.f / 256.f && fabsf(a[2]) <= tmax && fabsf(a[5]) <= tmax;
  if (!m.ok) { a[0] = 1.f; a[1] = 0.f; a[2] = 0.f; a[3] = 0.f; a[4] = 1.f; a[5] = 0.f; }
  const AugGeom g = aug_geom(geom, b, H, W);
  const float fl = (g.code & 1) ? -1.f : 1.f;
  const int k = g.code >> 1;
  const float cs = k == 0 ? 1.f : (k == 2 ? -1.f : 0.f), sn = k == 1 ? 1.f : (k == 3 ? -1.f : 0.f);
  const float d00 = cs * fl, d01 = sn, d10 = -sn * fl, d11 = cs;     // D = R_k diag(flip, 1)
  m.l00 = d00 * a[0] + d01 * a[3]; m.l01 = d00 * a[1] + d01 * a[4];
  m.l10 = d10 * a[0] + d11 * a[3]; m.l11 = d10 * a[1] + d11 * a[4];
  const float cx = 0.5f * (W - 1), cy = 0.5f * (H - 1);
  const float w0 = a[2] - (a[0] * cx + a[1] * cy), w1 = a[5] - (a[3] * cx + a[4] * cy);
  const float o0 = d00 * w0 + d01 * w1 - g.tx + cx, o1 = d10 * w0 + d11 * w1 - g.ty + cy;
  m.e0 = 2.f * o0 - 6.f * (m.l00 + m.l01);
  m.e1 = 2.f * o1 - 6.f * (m.l10 + m.l11);
  return m;
}

__device__ __forceinline__ float2 res_nu(const ResMap& m, float qx, float qy) {
  return make_float2(fmaf(m.l00, qx, fmaf(m.l01, qy, m.e0)), fmaf(m.l10, qx, fmaf(m.l11, qy, m.e1)));
}

// Integer 2x-source box [u0, u1] (per axis) holding both bilinear taps of nu(q) for every q of a box, padded by one for rounding and
// clipped to U's extent [-2(N-1), 4N-3]; empty when u0 > u1.
__device__ void res_nu_box(const ResMap& m, int qx0, int qx1, int qy0, int qy1, int H, int W, int& ux0, int& ux1, int& uy0, int& uy1) {
  const float2 c0 = res_nu(m, qx0, qy0), c1 = res_nu(m, qx1, qy0), c2 = res_nu(m, qx0, qy1), c3 = res_nu(m, qx1, qy1);
  const float xmin = fminf(fminf(c0.x, c1.x), fminf(c2.x, c3.x)), xmax = fmaxf(fmaxf(c0.x, c1.x), fmaxf(c2.x, c3.x));
  const float ymin = fminf(fminf(c0.y, c1.y), fminf(c2.y, c3.y)), ymax = fmaxf(fmaxf(c0.y, c1.y), fmaxf(c2.y, c3.y));
  ux0 = max((int)floorf(xmin) - 1, -2 * (W - 1)); ux1 = min((int)floorf(xmax) + 2, 4 * W - 3);
  uy0 = max((int)floorf(ymin) - 1, -2 * (H - 1)); uy1 = min((int)floorf(ymax) + 2, 4 * H - 3);
}

// Weights of the 2x-upsampled, bilinearly sampled source at nu along one axis: wt[j] on extended index m0 + j (j < 7), zero where a
// bilinear tap lies outside U's extent or m outside [-(N-1), 2(N-1)].  Returns m0.
__device__ __forceinline__ int res_axis_weights(float nu, int N, float wt[7]) {
  const float f0 = floorf(nu);
  const int n0 = (int)f0;
  const float a = nu - f0;
  const int m0 = cdiv2(n0 - 6);
  const bool v0 = n0 >= -2 * (N - 1) && n0 <= 4 * N - 3, v1 = n0 + 1 >= -2 * (N - 1) && n0 + 1 <= 4 * N - 3;
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    const int mm = m0 + j, k0 = n0 + 5 - 2 * mm, k1 = k0 + 1;
    float w = 0.f;
    if (v0 && k0 >= 0 && k0 < 12) w = (1.f - a) * rs_f[k0];
    if (v1 && k1 >= 0 && k1 < 12) w = fmaf(a, rs_f[k1], w);
    wt[j] = (mm >= -(N - 1) && mm <= 2 * (N - 1)) ? 2.f * w : 0.f;
  }
  return m0;
}

// V at nu, straight from the source through L2 (the fallback path): 7 x 7 extended taps.
__device__ float res_sample_direct(const float* __restrict__ src, float2 nu, int H, int W) {
  float wx[7], wy[7];
  const int mx0 = res_axis_weights(nu.x, W, wx), my0 = res_axis_weights(nu.y, H, wy);
  float acc = 0.f;
  for (int jy = 0; jy < 7; ++jy) {
    if (wy[jy] == 0.f) continue;
    const float* row = src + (size_t)aug_mirror(my0 + jy, H) * W;
    float r = 0.f;
#pragma unroll
    for (int jx = 0; jx < 7; ++jx)
      if (wx[jx] != 0.f) r = fmaf(wx[jx], __ldg(row + aug_mirror(mx0 + jx, W)), r);
    acc = fmaf(wy[jy], r, acc);
  }
  return acc;
}

__device__ __forceinline__ void res_write_nan(float* dst, size_t HW, int C) {
  for (int c = 0; c < C; ++c) dst[c * HW] = __int_as_float(0x7fc00000);
}

// Forward.  Per tile: the blit (F^-1 the identity, gf_augment_nchw's arithmetic), NaN (outside the domain), the shared-memory plan
// (E -> U rows -> U -> V -> V rows -> out, one channel at a time) when the tile's footprint fits two RS_CAP regions, else the direct
// per-pixel path.  Colour after the geometry, from registers.
__global__ void __launch_bounds__(RS_T * RS_T) augment_resample_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                         const int* __restrict__ geom, const float* __restrict__ frac,
                                                                         const float* __restrict__ color, int C, int H, int W,
                                                                         long long tiles, int tiles_x, int tiles_y) {
  extern __shared__ float rs_smem[];
  float* sA = rs_smem;
  float* sB = rs_smem + RS_CAP;
  const size_t HW = (size_t)H * W;
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * RS_T + tx;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int b = (int)(tile / ((long long)tiles_x * tiles_y));
    const int rem = (int)(tile % ((long long)tiles_x * tiles_y));
    const int ox0 = (rem % tiles_x) * RS_T, oy0 = (rem / tiles_x) * RS_T;
    const int nox = min(RS_T, W - ox0), noy = min(RS_T, H - oy0);
    const bool mine = tx < nox && ty < noy;
    const int px = ox0 + tx, py = oy0 + ty;
    const ResMap m = res_map(geom, frac, b, H, W);
    float* dst = y + (size_t)b * C * HW + (size_t)py * W + px;
    if (m.ident) {                                                    // the blit, as augment_kernel computes it
      if (!mine) continue;
      const AugGeom g = aug_geom(geom, b, H, W);
      int u, v;
      aug_dihedral(g.code, px, py, H, W, u, v);
      const float* src = x + (size_t)b * C * HW + (size_t)aug_mirror(v - g.ty, H) * W + aug_mirror(u - g.tx, W);
      if (color) {
        const float* M = color + 12 * b;
        const float r = __ldg(src), gr = __ldg(src + HW), bl = __ldg(src + 2 * HW);
#pragma unroll
        for (int c = 0; c < 3; ++c)
          dst[c * HW] = fmaf(__ldg(M + 4 * c + 2), bl, fmaf(__ldg(M + 4 * c + 1), gr, fmaf(__ldg(M + 4 * c), r, __ldg(M + 4 * c + 3))));
      } else {
        for (int c = 0; c < C; ++c) dst[c * HW] = __ldg(src + c * HW);
      }
      continue;
    }
    if (!m.ok) {
      if (mine) res_write_nan(dst, HW, C);
      continue;
    }
    const int qx0 = 2 * ox0 + 1, qy0 = 2 * oy0 + 1, nqx = 2 * nox + 10, nqy = 2 * noy + 10;
    int ux0, ux1, uy0, uy1;
    res_nu_box(m, qx0, qx0 + nqx - 1, qy0, qy0 + nqy - 1, H, W, ux0, ux1, uy0, uy1);
    const int ex0 = max(cdiv2(ux0 - 6), -(W - 1)), ex1 = min(fdiv2(ux1 + 5), 2 * (W - 1));
    const int ey0 = max(cdiv2(uy0 - 6), -(H - 1)), ey1 = min(fdiv2(uy1 + 5), 2 * (H - 1));
    const int nux = ux1 - ux0 + 1, nuy = uy1 - uy0 + 1, nex = ex1 - ex0 + 1, ney = ey1 - ey0 + 1;
    const bool empty = nux <= 0 || nuy <= 0 || nex <= 0 || ney <= 0;  // the tile reads only zeros
    const bool fits = empty || ((long long)nex * ney <= RS_CAP && (long long)ney * nux <= RS_CAP && (long long)nuy * nux <= RS_CAP);
    const float* xb = x + (size_t)b * C * HW;
    float v3[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < C; ++c) {
      const float* xc = xb + (size_t)c * HW;
      float out = 0.f;
      if (empty) {
      } else if (fits) {
        for (int i = tid; i < nex * ney; i += RS_T * RS_T) {
          const int iy = i / nex, ix = i - iy * nex;
          sA[i] = __ldg(xc + (size_t)aug_mirror(ey0 + iy, H) * W + aug_mirror(ex0 + ix, W));
        }
        __syncthreads();
        for (int i = tid; i < ney * nux; i += RS_T * RS_T) {          // up-filter along x: rows of E -> rows at 2x columns
          const int iy = i / nux, jx = i - iy * nux, nu = ux0 + jx, mlo = cdiv2(nu - 6);
          float acc = 0.f;
#pragma unroll
          for (int t = 0; t < 6; ++t) {
            const int mx = mlo + t;
            if (mx >= ex0 && mx <= ex1) acc = fmaf(rs_f[nu + 5 - 2 * mx], sA[iy * nex + mx - ex0], acc);
          }
          sB[i] = 2.f * acc;
        }
        __syncthreads();
        for (int i = tid; i < nuy * nux; i += RS_T * RS_T) {          // up-filter along y: U
          const int jy = i / nux, jx = i - jy * nux, nu = uy0 + jy, mlo = cdiv2(nu - 6);
          float acc = 0.f;
#pragma unroll
          for (int t = 0; t < 6; ++t) {
            const int my = mlo + t;
            if (my >= ey0 && my <= ey1) acc = fmaf(rs_f[nu + 5 - 2 * my], sB[(my - ey0) * nux + jx], acc);
          }
          sA[i] = 2.f * acc;
        }
        __syncthreads();
        for (int i = tid; i < nqy * nqx; i += RS_T * RS_T) {          // bilinear: V on the tile's 2x output points
          const int iy = i / nqx, ix = i - iy * nqx;
          const float2 nu = res_nu(m, (float)(qx0 + ix), (float)(qy0 + iy));
          const float fx = floorf(nu.x), fy = floorf(nu.y), ax = nu.x - fx, ay = nu.y - fy;
          const int jx = (int)fx - ux0, jy = (int)fy - uy0;
          auto at = [&](int yy, int xx) { return (xx >= 0 && xx < nux && yy >= 0 && yy < nuy) ? sA[yy * nux + xx] : 0.f; };
          const float top = fmaf(ax, at(jy, jx + 1), (1.f - ax) * at(jy, jx));
          const float bot = fmaf(ax, at(jy + 1, jx + 1), (1.f - ax) * at(jy + 1, jx));
          sB[iy * RS_Q + ix] = fmaf(ay, bot, (1.f - ay) * top);
        }
        __syncthreads();
        for (int i = tid; i < nqy * RS_T; i += RS_T * RS_T) {         // down-filter along x
          const int iy = i / RS_T, ox = i - iy * RS_T;
          float acc = 0.f;
          if (ox < nox) {
#pragma unroll
            for (int k = 0; k < 12; ++k) acc = fmaf(rs_f[k], sB[iy * RS_Q + 2 * ox + k], acc);
          }
          sA[i] = acc;
        }
        __syncthreads();
        if (mine) {                                                   // down-filter along y
#pragma unroll
          for (int k = 0; k < 12; ++k) out = fmaf(rs_f[k], sA[(2 * ty + k) * RS_T + tx], out);
        }
        __syncthreads();
      } else if (mine) {                                              // direct per-pixel path
        for (int ky = 0; ky < 12; ++ky) {
          float r = 0.f;
          for (int kx = 0; kx < 12; ++kx)
            r = fmaf(rs_f[kx], res_sample_direct(xc, res_nu(m, (float)(2 * px + kx + 1), (float)(2 * py + ky + 1)), H, W), r);
          out = fmaf(rs_f[ky], r, out);
        }
      }
      if (!mine) continue;
      if (color) v3[c] = out;
      else dst[c * HW] = out;
    }
    if (color && mine) {
      const float* M = color + 12 * b;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        dst[c * HW] = fmaf(__ldg(M + 4 * c + 2), v3[2], fmaf(__ldg(M + 4 * c + 1), v3[1], fmaf(__ldg(M + 4 * c), v3[0], __ldg(M + 4 * c + 3))));
    }
  }
}

// The extended indices m of source pixels [i0, i1] in mirrored copy k (0: m = i; 1: m = -i, i >= 1; 2: m = 2(N-1) - i, i <= N-2),
// as a box [m0, m1]; false when empty.  m of pixel i in copy k: res_copy_index.
__device__ __forceinline__ bool res_copy_box(int k, int i0, int i1, int N, int& m0, int& m1) {
  if (k == 0) { m0 = i0; m1 = i1; }
  else if (k == 1) { m0 = -i1; m1 = -max(i0, 1); }
  else { m0 = 2 * (N - 1) - min(i1, N - 2); m1 = 2 * (N - 1) - i0; }
  return m0 <= m1;
}
__device__ __forceinline__ int res_copy_index(int k, int i, int N) { return k == 0 ? i : (k == 1 ? -i : 2 * (N - 1) - i); }

// Transposed bilinear at the integer 2x-source point (nux, nuy): the sum over the 2x output points q of the box [qx0, qx1] x
// [qy0, qy1] whose nu(q) has it as a tap, of that tap's weight times gv(q), walked row by row over the preimage's bounding box.
template <class GV>
__device__ __forceinline__ float res_gather_bilinear(const ResMap& m, float i00, float i01, float i10, float i11, float hx, float hy,
                                                     int nux, int nuy, int qx0, int qx1, int qy0, int qy1, GV gv) {
  const float dx = (float)nux - m.e0, dy = (float)nuy - m.e1;
  const float cx = fmaf(i00, dx, i01 * dy), cy = fmaf(i10, dx, i11 * dy);
  const int ax0 = max((int)floorf(cx - hx), qx0), ax1 = min((int)ceilf(cx + hx), qx1);
  const int ay0 = max((int)floorf(cy - hy), qy0), ay1 = min((int)ceilf(cy + hy), qy1);
  float acc = 0.f;
  for (int qy = ay0; qy <= ay1; ++qy)
    for (int qx = ax0; qx <= ax1; ++qx) {
      const float2 nu = res_nu(m, (float)qx, (float)qy);
      const float fx = floorf(nu.x), fy = floorf(nu.y);
      const int jx = (int)fx, jy = (int)fy;
      const float wx = jx == nux ? 1.f - (nu.x - fx) : (jx + 1 == nux ? nu.x - fx : 0.f);
      const float wy = jy == nuy ? 1.f - (nu.y - fy) : (jy + 1 == nuy ? nu.y - fy : 0.f);
      if (wx != 0.f && wy != 0.f) acc = fmaf(wy * wx, gv(qx, qy), acc);
    }
  return acc;
}

// Adjoint, gather only.  Per 16 x 16 source tile and channel, for each mirrored copy (3 x 3, fixed order) that meets the extended
// region the output can reach: the colour-transposed gy box -> transposed down-filter (x, then y) -> transposed bilinear -> transposed
// up-filter (x, then y), all in shared memory: the copy's 2x output points are staged in 64 x 64 chunks whose transposed-bilinear
// shares add into one gU accumulator in a fixed order, so any zoom-in fits the plan; each pixel sums its copies.
__global__ void __launch_bounds__(RS_T * RS_T) augment_resample_adjoint_kernel(const float* __restrict__ gy, float* __restrict__ gx,
                                                                                 const int* __restrict__ geom, const float* __restrict__ frac,
                                                                                 const float* __restrict__ color, int C, int H, int W,
                                                                                 long long tiles, int tiles_x, int tiles_y) {
  extern __shared__ float rs_smem[];
  float* sA = rs_smem;
  float* sB = rs_smem + RS_CAP;
  const size_t HW = (size_t)H * W;
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * RS_T + tx;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int b = (int)(tile / ((long long)tiles_x * tiles_y));
    const int rem = (int)(tile % ((long long)tiles_x * tiles_y));
    const int sx0 = (rem % tiles_x) * RS_T, sy0 = (rem / tiles_x) * RS_T;
    const int nsx = min(RS_T, W - sx0), nsy = min(RS_T, H - sy0);
    const bool mine = tx < nsx && ty < nsy;
    const int qx = sx0 + tx, qy = sy0 + ty;                           // this thread's source pixel
    const ResMap m = res_map(geom, frac, b, H, W);
    float* dst = gx + (size_t)b * C * HW + (size_t)qy * W + qx;
    const float* gb = gy + (size_t)b * C * HW;
    if (m.ident) {                                                    // the blit's adjoint, as augment_adjoint_kernel computes it
      if (!mine) continue;
      const AugGeom g = aug_geom(geom, b, H, W);
      int sxs[2], sys[2];
      const int nx = aug_preimages(qx, g.tx, W, sxs), ny = aug_preimages(qy, g.ty, H, sys);
      if (color) {
        const float* M = color + 12 * b;
        float mm[3][3];
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int j = 0; j < 3; ++j) mm[c][j] = __ldg(M + 4 * c + j);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int iy = 0; iy < ny; ++iy)
          for (int ix = 0; ix < nx; ++ix) {
            int px, py;
            aug_dihedral_inv(g.code, sxs[ix] + g.tx, sys[iy] + g.ty, H, W, px, py);
            const float* s = gb + (size_t)py * W + px;
            const float g0 = __ldg(s), g1 = __ldg(s + HW), g2 = __ldg(s + 2 * HW);
            a0 += fmaf(mm[2][0], g2, fmaf(mm[1][0], g1, mm[0][0] * g0));
            a1 += fmaf(mm[2][1], g2, fmaf(mm[1][1], g1, mm[0][1] * g0));
            a2 += fmaf(mm[2][2], g2, fmaf(mm[1][2], g1, mm[0][2] * g0));
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
          for (int i = 0; i < n; ++i) a += __ldg(gb + c * HW + off[i]);
          dst[c * HW] = a;
        }
      }
      continue;
    }
    if (!m.ok) {
      if (mine) res_write_nan(dst, HW, C);
      continue;
    }
    // the inverse of L: preimages of 2x-source boxes; (hx, hy) the half-extents of the preimage of a 2 x 2 square
    const float det = m.l00 * m.l11 - m.l01 * m.l10;
    const float i00 = m.l11 / det, i01 = -m.l01 / det, i10 = -m.l10 / det, i11 = m.l00 / det;
    const float hx = fabsf(i00) + fabsf(i01), hy = fabsf(i10) + fabsf(i11);
    const int QX = 2 * W + 10, QY = 2 * H + 10;                       // the 2x output grid the down filter reads: q in [1, 2N + 10]
    int rx0, rx1, ry0, ry1;                                           // the extended region the whole output can reach
    res_nu_box(m, 1, QX, 1, QY, H, W, rx0, rx1, ry0, ry1);
    const int rmx0 = max(cdiv2(rx0 - 6), -(W - 1)), rmx1 = min(fdiv2(rx1 + 5), 2 * (W - 1));
    const int rmy0 = max(cdiv2(ry0 - 6), -(H - 1)), rmy1 = min(fdiv2(ry1 + 5), 2 * (H - 1));
    const float* M = color ? color + 12 * b : nullptr;
    for (int c = 0; c < C; ++c) {
      float total = 0.f;
      for (int k = 0; k < 9; ++k) {
        const int kx = k % 3, ky = k / 3;
        int mx0, mx1, my0, my1;
        if (!res_copy_box(kx, sx0, sx0 + nsx - 1, W, mx0, mx1) || !res_copy_box(ky, sy0, sy0 + nsy - 1, H, my0, my1)) continue;
        mx0 = max(mx0, rmx0); mx1 = min(mx1, rmx1); my0 = max(my0, rmy0); my1 = min(my1, rmy1);
        if (mx0 > mx1 || my0 > my1 || rx0 > rx1 || ry0 > ry1) continue;   // block-uniform: no pixel of this copy is reachable
        const int mx = res_copy_index(kx, qx, W), my = res_copy_index(ky, qy, H);
        const bool here = mine && (kx != 1 || qx >= 1) && (kx != 2 || qx <= W - 2) && (ky != 1 || qy >= 1) && (ky != 2 || qy <= H - 2) &&
                          mx >= mx0 && mx <= mx1 && my >= my0 && my <= my1;
        const int ux0 = max(2 * mx0 - 5, -2 * (W - 1)), ux1 = min(2 * mx1 + 6, 4 * W - 3);
        const int uy0 = max(2 * my0 - 5, -2 * (H - 1)), uy1 = min(2 * my1 + 6, 4 * H - 3);
        const int nux = ux1 - ux0 + 1, nuy = uy1 - uy0 + 1;
        if (nux <= 0 || nuy <= 0) continue;
        float cq[4][2];                                               // preimage of [u0 - 1, u1 + 1]^2 -> the q box
        const float bx[2] = {(float)(ux0 - 1), (float)(ux1 + 1)}, by[2] = {(float)(uy0 - 1), (float)(uy1 + 1)};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float dx = bx[j & 1] - m.e0, dy = by[j >> 1] - m.e1;
          cq[j][0] = fmaf(i00, dx, i01 * dy); cq[j][1] = fmaf(i10, dx, i11 * dy);
        }
        const float cxmin = fminf(fminf(cq[0][0], cq[1][0]), fminf(cq[2][0], cq[3][0])), cxmax = fmaxf(fmaxf(cq[0][0], cq[1][0]), fmaxf(cq[2][0], cq[3][0]));
        const float cymin = fminf(fminf(cq[0][1], cq[1][1]), fminf(cq[2][1], cq[3][1])), cymax = fmaxf(fmaxf(cq[0][1], cq[1][1]), fmaxf(cq[2][1], cq[3][1]));
        const int qx0 = max((int)floorf(fmaxf(cxmin, -1e8f)) - 1, 1), qx1 = min((int)ceilf(fminf(cxmax, 1e8f)) + 1, QX);
        const int qy0 = max((int)floorf(fmaxf(cymin, -1e8f)) - 1, 1), qy1 = min((int)ceilf(fminf(cymax, 1e8f)) + 1, QY);
        if (qx0 > qx1 || qy0 > qy1) continue;
        const int nmx = mx1 - mx0 + 1;
        auto gcol = [&](int oy, int ox) {                               // colour-transposed gy at an output pixel
          const float* s = gb + (size_t)oy * W + ox;
          if (!M) return __ldg(s + c * HW);
          return fmaf(__ldg(M + 8 + c), __ldg(s + 2 * HW), fmaf(__ldg(M + 4 + c), __ldg(s + HW), __ldg(M + c) * __ldg(s)));
        };
        float* gU = sB + RS_GU;
        for (int i = tid; i < nuy * nux; i += RS_T * RS_T) gU[i] = 0.f;
        // the q box in RS_QC x RS_QC chunks, in a fixed order: gy box -> transposed down-filter (x, y) -> gU += transposed bilinear
        for (int cy0 = qy0; cy0 <= qy1; cy0 += RS_QC)
          for (int cx0 = qx0; cx0 <= qx1; cx0 += RS_QC) {
            const int cx1 = min(cx0 + RS_QC - 1, qx1), cy1 = min(cy0 + RS_QC - 1, qy1);
            const int ox0 = max(cdiv2(cx0 - 12), 0), ox1 = min(fdiv2(cx1 - 1), W - 1);
            const int oy0 = max(cdiv2(cy0 - 12), 0), oy1 = min(fdiv2(cy1 - 1), H - 1);
            const int nqx = cx1 - cx0 + 1, nqy = cy1 - cy0 + 1, nox = ox1 - ox0 + 1, noy = oy1 - oy0 + 1;
            for (int i = tid; i < noy * nox; i += RS_T * RS_T) { const int iy = i / nox; sA[i] = gcol(oy0 + iy, ox0 + i - iy * nox); }
            __syncthreads();
            for (int i = tid; i < noy * nqx; i += RS_T * RS_T) {      // transposed down-filter along x
              const int iy = i / nqx, jx = i - iy * nqx, q = cx0 + jx;
              float acc = 0.f;
#pragma unroll
              for (int t = 0; t < 6; ++t) {                               // o = cdiv2(q - 12) + t: taps 11 - 2t or 10 - 2t
                const int o = cdiv2(q - 12) + t;
                if (o >= ox0 && o <= ox1) acc = fmaf(rs_f[q - 1 - 2 * o], sA[iy * nox + o - ox0], acc);
              }
              sB[i] = acc;
            }
            __syncthreads();
            for (int i = tid; i < nqy * nqx; i += RS_T * RS_T) {      // ... along y: gV
              const int jy = i / nqx, jx = i - jy * nqx, q = cy0 + jy;
              float acc = 0.f;
#pragma unroll
              for (int t = 0; t < 6; ++t) {
                const int o = cdiv2(q - 12) + t;
                if (o >= oy0 && o <= oy1) acc = fmaf(rs_f[q - 1 - 2 * o], sB[(o - oy0) * nqx + jx], acc);
              }
              sA[i] = acc;
            }
            __syncthreads();
            for (int i = tid; i < nuy * nux; i += RS_T * RS_T) {      // transposed bilinear, this chunk's share of gU
              const int jy = i / nux, jx = i - jy * nux;
              gU[i] += res_gather_bilinear(m, i00, i01, i10, i11, hx, hy, ux0 + jx, uy0 + jy, cx0, cx1, cy0, cy1,
                                           [&](int a, int bb) { return sA[(bb - cy0) * nqx + a - cx0]; });
            }
            __syncthreads();
          }
        for (int i = tid; i < nuy * nmx; i += RS_T * RS_T) {          // transposed up-filter along x
          const int jy = i / nmx, ix = i - jy * nmx, mm = mx0 + ix;
          float acc = 0.f;
          for (int nu = max(2 * mm - 5, ux0); nu <= min(2 * mm + 6, ux1); ++nu) acc = fmaf(rs_f[nu + 5 - 2 * mm], gU[jy * nux + nu - ux0], acc);
          sA[i] = 2.f * acc;
        }
        __syncthreads();
        if (here) {                                                   // ... along y, at this pixel's copy
          float acc = 0.f;
          for (int nu = max(2 * my - 5, uy0); nu <= min(2 * my + 6, uy1); ++nu) acc = fmaf(rs_f[nu + 5 - 2 * my], sA[(nu - uy0) * nmx + mx - mx0], acc);
          total += 2.f * acc;
        }
        __syncthreads();
      }
      if (mine) dst[c * HW] = total;
    }
  }
}

// ================================================================================================ image-space filter (item 17)
// ADA's imgfilter: per image, 43 taps h_b = sum_i gains[b][i] bank[i] applied separably with the mirror R_N (21-pixel halo), then
// the additive noise y += sigma_b n.  Both kernels walk 64 x 32 output tiles of one (b, c) plane with a tile-stride loop: the tile's
// 74 x 106 input box goes to shared memory (mirrored forward, zero-padded in the adjoint), a vertical pass writes 32 x 106 partial
// sums, a horizontal pass the 64 x 32 outputs.  Each thread of a pass keeps a window of its column (row) in registers and
// accumulates 16 (8) outputs, so each shared-memory value it loads feeds 16 (8) FMAs.
constexpr int FL_TAPS = 43, FL_R = 21;                               // taps, halo
constexpr int FL_TW = 64, FL_TH = 32;                                // output tile
constexpr int FL_IW = FL_TW + 2 * FL_R, FL_IH = FL_TH + 2 * FL_R;    // input box: 106 x 74
constexpr int FL_PITCH = FL_IW + 1;                                  // odd pitch: a warp reading down 32 rows hits 32 banks
constexpr int FL_RV = 16, FL_RH = 8;                                 // outputs per thread: vertical pass, horizontal pass
constexpr int FL_THREADS = 256;
static_assert(FL_TH % FL_RV == 0 && FL_TW % FL_RH == 0 && FL_TH * (FL_TW / FL_RH) == FL_THREADS, "filter tile shape");
static_assert(FL_TH > FL_R && FL_TW > FL_R, "a tile holding a pixel within the halo of an edge must start at that edge");

// The bank [4, 43] as integer numerators over 2^15 (SURVEY A.4 item 17): every entry and every sum of entries of the four rows is
// exact in fp32.  Row i (i >= 1) is band i's high-pass.
__constant__ short fl_bank[4][FL_TAPS] = {
    {-1, 0, 9, 16, 18, 0, -66, -144, -207, -256, -297, -288, -212, 0, 468, 1056, 1674, 2304, 2918, 3456, 3888, 4096, 3888, 3456, 2918,
     2304, 1674, 1056, 468, 0, -212, -288, -297, -256, -207, -144, -66, 0, 18, 16, 9, 0, -1},
    {1, 0, -9, -16, -18, 0, 66, 144, 207, 256, 297, 288, 244, 0, -756, -1568, -2250, -2304, -806, 1152, 3024, 4096, 3024, 1152, -806,
     -2304, -2250, -1568, -756, 0, 244, 288, 297, 256, 207, 144, 66, 0, -18, -16, -9, 0, 1},
    {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, -32, 0, 288, 512, 576, 0, -3136, -4608, 2304, 8192, 2304, -4608, -3136, 0, 576, 512, 288, 0,
     -32, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0},
    {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1024, 0, -9216, 16384, -9216, 0, 1024, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
     0, 0, 0, 0, 0}};

// Gains exactly (1, 1, 1, 1): the taps are exactly the unit impulse, and the kernels copy the plane (bit for bit, -0 and non-finite
// neighbours included) instead of filtering it.
__device__ __forceinline__ bool fl_identity(const float* __restrict__ gains, int b) {
  return __ldg(gains + 4 * b) == 1.f && __ldg(gains + 4 * b + 1) == 1.f && __ldg(gains + 4 * b + 2) == 1.f && __ldg(gains + 4 * b + 3) == 1.f;
}

// The reflected preimages' contributions to the adjoint along one axis at source index m (N the axis length), read from a line
// `s` of the tile's zero-padded buffer whose element 0 is index o - 21: e[-m] for 1 <= m <= 21, e[2(N-1) - m] for N-22 <= m <= N-2,
// with e[k] = sum_t h[t] g[k - t + 21] (only the terms with g inside [0, N) are summed).  Returned separately, to be added in order.
__device__ __forceinline__ float2 fl_reflected(const float* s, int stride, const float* h, int m, int N, int o) {
  float lo = 0.f, hi = 0.f;
  if (m >= 1 && m <= FL_R)
    for (int t = 0; t <= FL_R - m; ++t) lo = fmaf(h[t], s[(FL_R - m - t - o + FL_R) * stride], lo);
  if (m >= N - 1 - FL_R && m <= N - 2)
    for (int t = N + FL_R - 1 - m; t < FL_TAPS; ++t) hi = fmaf(h[t], s[(2 * N + FL_R - 2 - m - t - o + FL_R) * stride], hi);
  return make_float2(lo, hi);
}

// ADJ = false: y = V H x (+ sigma n).  ADJ = true: gx = H^T V^T gy, each source pixel summing its at most 3 preimages per axis
// (itself, -m, 2(N-1) - m) in that order; with symmetric taps the transposed pass is the same correlation with h[42 - t].
template <bool ADJ>
__global__ void __launch_bounds__(FL_THREADS, 2) augment_filter_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                    const float* __restrict__ gains, const float* __restrict__ sigma,
                                                                    const float* __restrict__ noise, int C, int H, int W,
                                                                    long long tiles, int tiles_x, int tiles_y) {
  __shared__ float s_in[FL_IH * FL_PITCH];
  __shared__ float s_v[FL_TH * FL_PITCH];
  __shared__ float s_h[FL_TAPS + 1];
  const size_t HW = (size_t)H * W;
  const int tid = threadIdx.x;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long plane = tile / ((long long)tiles_x * tiles_y);
    const int rem = (int)(tile % ((long long)tiles_x * tiles_y));
    const int b = (int)(plane / C);
    const int x0 = (rem % tiles_x) * FL_TW, y0 = (rem / tiles_x) * FL_TH;
    const float* src = x + (size_t)plane * HW;
    float* dst = y + (size_t)plane * HW;
    const float* nz = noise ? noise + (size_t)plane * HW : nullptr;
    const float sig = (!ADJ && sigma) ? __ldg(sigma + b) : 0.f;
    if (fl_identity(gains, b)) {
      for (int i = tid; i < FL_TH * FL_TW; i += FL_THREADS) {
        const int gy = y0 + i / FL_TW, gx = x0 + i % FL_TW;
        if (gy >= H || gx >= W) continue;
        const size_t o = (size_t)gy * W + gx;
        float v = __ldg(src + o);
        if (sig != 0.f) v = fmaf(sig, __ldg(nz + o), v);
        dst[o] = v;
      }
      continue;
    }
    if (tid < FL_TAPS) {                                              // h_b[t], summed over the bands in a fixed order
      const float* g = gains + 4 * b;
      float h = __ldg(g) * ((float)fl_bank[0][tid] * (1.f / 32768.f));
#pragma unroll
      for (int i = 1; i < 4; ++i) h = fmaf(__ldg(g + i), (float)fl_bank[i][tid] * (1.f / 32768.f), h);
      s_h[tid] = h;
    }
    for (int i = tid; i < FL_IH * FL_IW; i += FL_THREADS) {           // the input box: mirrored (forward) or zero-padded (adjoint)
      const int r = i / FL_IW, c = i - r * FL_IW;
      int gy = y0 - FL_R + r, gx = x0 - FL_R + c;
      float v;
      if (ADJ) {
        v = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(src + (size_t)gy * W + gx) : 0.f;
      } else {                                                        // beyond N + 20 only feeds outputs past the edge
        gy = aug_mirror(min(gy, H - 1 + FL_R), H);
        gx = aug_mirror(min(gx, W - 1 + FL_R), W);
        v = __ldg(src + (size_t)gy * W + gx);
      }
      s_in[r * FL_PITCH + c] = v;
    }
    __syncthreads();
    for (int it = tid; it < FL_IW * (FL_TH / FL_RV); it += FL_THREADS) {   // vertical pass: FL_RV rows of one column
      const int c = it % FL_IW, r0 = (it / FL_IW) * FL_RV;
      float w[FL_RV + FL_TAPS - 1], acc[FL_RV];
#pragma unroll
      for (int k = 0; k < FL_RV + FL_TAPS - 1; ++k) w[k] = s_in[(r0 + k) * FL_PITCH + c];
#pragma unroll
      for (int k = 0; k < FL_RV; ++k) acc[k] = 0.f;
#pragma unroll
      for (int t = 0; t < FL_TAPS; ++t) {
        const float h = s_h[ADJ ? FL_TAPS - 1 - t : t];
#pragma unroll
        for (int k = 0; k < FL_RV; ++k) acc[k] = fmaf(h, w[k + t], acc[k]);
      }
#pragma unroll
      for (int k = 0; k < FL_RV; ++k) s_v[(r0 + k) * FL_PITCH + c] = acc[k];
      if (ADJ && (y0 <= FL_R || y0 + FL_TH >= H - 1 - FL_R)) {        // tiles that hold a row within the halo of an edge
#pragma unroll 1
        for (int k = 0; k < FL_RV; ++k) {                             // this thread's own sums: no barrier needed
          const float2 e = fl_reflected(s_in + c, FL_PITCH, s_h, y0 + r0 + k, H, y0);
          float v = s_v[(r0 + k) * FL_PITCH + c];
          v += e.x;
          v += e.y;
          s_v[(r0 + k) * FL_PITCH + c] = v;
        }
      }
    }
    __syncthreads();
    {                                                                 // horizontal pass: FL_RH columns of one row per thread
      const int r = tid % FL_TH, c0 = (tid / FL_TH) * FL_RH;
      const float* row = s_v + r * FL_PITCH;
      float w[FL_RH + FL_TAPS - 1], acc[FL_RH];
#pragma unroll
      for (int k = 0; k < FL_RH + FL_TAPS - 1; ++k) w[k] = row[c0 + k];
#pragma unroll
      for (int k = 0; k < FL_RH; ++k) acc[k] = 0.f;
#pragma unroll
      for (int t = 0; t < FL_TAPS; ++t) {
        const float h = s_h[ADJ ? FL_TAPS - 1 - t : t];
#pragma unroll
        for (int k = 0; k < FL_RH; ++k) acc[k] = fmaf(h, w[k + t], acc[k]);
      }
      const int gy = y0 + r;
      if (gy < H) {
#pragma unroll
        for (int k = 0; k < FL_RH; ++k) {
          const int gx = x0 + c0 + k;
          if (gx >= W) continue;
          float v = acc[k];
          if (ADJ) {
            const float2 e = fl_reflected(row, 1, s_h, gx, W, x0);
            v += e.x;
            v += e.y;
          }
          const size_t o = (size_t)gy * W + gx;
          if (sig != 0.f) v = fmaf(sig, __ldg(nz + o), v);
          dst[o] = v;
        }
      }
    }
    __syncthreads();
  }
}

// No filter: y = x, plus sigma_b n where sigma_b != 0 (an image with sigma_b == 0 does not read n).
__global__ void augment_noise_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ sigma,
                                     const float* __restrict__ noise, size_t n, size_t per_image) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = __ldg(x + i);
    if (sigma) {
      const float s = __ldg(sigma + i / per_image);
      if (s != 0.f) v = fmaf(s, __ldg(noise + i), v);
    }
    y[i] = v;
  }
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

// Both resampler entry points: the blit's checks plus a NULL frac; 16 x 16 tiles, 2 CTAs per SM (80 KB of shared memory each).
static int augment_resample_launch(const char* name, bool adjoint, const float* in, float* out, const int* geom, const float* frac,
                                   const float* color, int B, int C, int H, int W, void* stream) {
  long long tiles; int tx, ty;
  const int rc = augment_check(name, in, out, geom, color, B, C, H, W, &tiles, &tx, &ty);
  if (rc != GF_OK) return rc;
  if (!frac) { set_error("%s: null pointer (frac)", name); return GF_ERR_INVALID; }
  tx = (W + RS_T - 1) / RS_T;
  ty = (H + RS_T - 1) / RS_T;
  tiles = (long long)B * tx * ty;
  const long long cap = (long long)num_sms() * 2;
  const int grid = (int)(tiles < cap ? tiles : cap);
  const int smem = 2 * RS_CAP * (int)sizeof(float);
  if (adjoint) {
    GF_CUDA_OK(cudaFuncSetAttribute(augment_resample_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    augment_resample_adjoint_kernel<<<grid, dim3(RS_T, RS_T), smem, (cudaStream_t)stream>>>(in, out, geom, frac, color, C, H, W, tiles, tx, ty);
  } else {
    GF_CUDA_OK(cudaFuncSetAttribute(augment_resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    augment_resample_kernel<<<grid, dim3(RS_T, RS_T), smem, (cudaStream_t)stream>>>(in, out, geom, frac, color, C, H, W, tiles, tx, ty);
  }
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_augment_resample_nchw(const float* x, float* y, const int* geom, const float* frac, const float* color, int B, int C, int H, int W,
                             void* stream) {
  return augment_resample_launch("gf_augment_resample_nchw", false, x, y, geom, frac, color, B, C, H, W, stream);
}

int gf_augment_resample_adjoint_nchw(const float* gy, float* gx, const int* geom, const float* frac, const float* color, int B, int C, int H,
                                     int W, void* stream) {
  return augment_resample_launch("gf_augment_resample_adjoint_nchw", true, gy, gx, geom, frac, color, B, C, H, W, stream);
}

// Both filter entry points: the checks, then one launch (the tiled filter, or the elementwise noise pass without gains).
static int augment_filter_launch(const char* name, bool adjoint, const float* in, float* out, const float* gains, const float* sigma,
                                 const float* noise, int B, int C, int H, int W, void* stream) {
  if (!in || !out || (adjoint && !gains)) { set_error("%s: null pointer", name); return GF_ERR_INVALID; }
  if ((sigma == nullptr) != (noise == nullptr)) {
    set_error("%s: sigma and noise must both be given or both be NULL", name); return GF_ERR_INVALID;
  }
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("%s: bad sizes B=%d C=%d H=%d W=%d", name, B, C, H, W); return GF_ERR_INVALID; }
  if (gains && (H < FL_R + 1 || W < FL_R + 1)) {
    set_error("%s: the 43-tap filter's mirror needs H and W of at least 22 (H=%d W=%d)", name, H, W); return GF_ERR_UNSUPPORTED;
  }
  if (H > 32768 || W > 32768 || (long long)C * H * W > 0x7fffffffLL) {
    set_error("%s: image too large (C=%d H=%d W=%d): H, W <= 32768 and C*H*W < 2^31", name, C, H, W); return GF_ERR_UNSUPPORTED;
  }
  const size_t n = (size_t)B * C * H * W;
  if (in < out + n && out < in + n) { set_error("%s: the output must not alias the input", name); return GF_ERR_INVALID; }
  const cudaStream_t st = (cudaStream_t)stream;
  if (!gains) {
    const size_t blocks = (n + 255) / 256, cap = (size_t)num_sms() * 8;
    augment_noise_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(in, out, sigma, noise, n, (size_t)C * H * W);
  } else {
    const int tx = (W + FL_TW - 1) / FL_TW, ty = (H + FL_TH - 1) / FL_TH;
    const long long tiles = (long long)B * C * tx * ty, cap = (long long)num_sms() * 2;   // 2 CTAs per SM (registers)
    const int grid = (int)(tiles < cap ? tiles : cap);
    if (adjoint)
      augment_filter_kernel<true><<<grid, FL_THREADS, 0, st>>>(in, out, gains, nullptr, nullptr, C, H, W, tiles, tx, ty);
    else
      augment_filter_kernel<false><<<grid, FL_THREADS, 0, st>>>(in, out, gains, sigma, noise, C, H, W, tiles, tx, ty);
  }
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_augment_filter_nchw(const float* x, float* y, const float* gains, const float* sigma, const float* noise, int B, int C, int H, int W,
                           void* stream) {
  return augment_filter_launch("gf_augment_filter_nchw", false, x, y, gains, sigma, noise, B, C, H, W, stream);
}

int gf_augment_filter_adjoint_nchw(const float* gy, float* gx, const float* gains, int B, int C, int H, int W, void* stream) {
  return augment_filter_launch("gf_augment_filter_adjoint_nchw", true, gy, gx, gains, nullptr, nullptr, B, C, H, W, stream);
}

}  // extern "C"
