// gf_ops.cu -- memory-bound companions of the attention hot path (include/gf_ops.h): channel scaling
// (style modulation / demodulation), the two upfirdn_2d uses of the generator, and fused bias + noise + activation.
//
// sm_90a equivalents of the reference's native ops dnnlib/tflib/ops/{fused_bias_act,upfirdn_2d}.cu (expected
// upstream; not in the checkout).  All are pure streaming kernels: float4 accesses on channels-last rows, grids
// sized to a few waves of the device's SMs, no shared memory (the FIR reuse is served by L1/L2).
#include "gf_common.cuh"
#include "../../include/gf_ops.h"

namespace gf {

static inline int grid_for(size_t work_items, int threads) {
  size_t b = (work_items + threads - 1) / threads;
  const size_t cap = (size_t)num_sms() * 16;
  return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}

// the streaming kernels move float4s: every operand they access that way must start on a 16-byte boundary (NULL passes:
// the optional operands are checked for presence elsewhere)
static inline bool misaligned16(const void* p) { return ((uintptr_t)p & 15) != 0; }

__global__ void __launch_bounds__(256) chan_scale_kernel(const float4* __restrict__ x, const float4* __restrict__ s,
                                                         float4* __restrict__ y, size_t total4, int hw_c4, int c4n, int s_ld4) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / hw_c4), c4 = (int)(i % c4n);
    const float4 v = x[i], sc = __ldg(s + (size_t)b * s_ld4 + c4);
    y[i] = make_float4(v.x * sc.x, v.y * sc.y, v.z * sc.z, v.w * sc.w);
  }
}

// One thread: a column (w, 4 channels) of ROWS consecutive output rows; horizontal 4-tap pass per input row on the
// fly, vertical pass over a sliding window of 4 horizontally filtered rows.
template <int ROWS>
__global__ void __launch_bounds__(256) blur_up_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                      const float* __restrict__ scale, int Hout, int Wout, int C, float gain, int pad) {
  const int c4n = C >> 2;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Wout * c4n) return;
  const int w = t / c4n, c = (t % c4n) * 4;
  const int h0 = blockIdx.y * ROWS, b = blockIdx.z;
  const int Hin = Hout + 3 - 2 * pad, Win = Wout + 3 - 2 * pad;   // pad 1: the blur after an upsampling conv; pad 2: its adjoint
  const float f0 = 0.125f, f1 = 0.375f;
  const float* xb = x + (size_t)b * Hin * Win * C;
  float4 win[4];
  auto hrow = [&](int u) -> float4 {            // u: row of the padded input, x_pad[u][v] = x[u-pad][v-pad]
    const int r = u - pad;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < 0 || r >= Hin) return a;
    const float* row = xb + (size_t)r * Win * C + c;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int v = w + j - pad;
      if (v >= 0 && v < Win) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(row + (size_t)v * C));
        const float f = (j == 0 || j == 3) ? f0 : f1;
        a.x = fmaf(f, q.x, a.x); a.y = fmaf(f, q.y, a.y); a.z = fmaf(f, q.z, a.z); a.w = fmaf(f, q.w, a.w);
      }
    }
    return a;
  };
  win[0] = hrow(h0); win[1] = hrow(h0 + 1); win[2] = hrow(h0 + 2);
  float4 sc = make_float4(gain, gain, gain, gain);
  if (scale) {
    const float4 s = __ldg(reinterpret_cast<const float4*>(scale + (size_t)b * C + c));
    sc = make_float4(gain * s.x, gain * s.y, gain * s.z, gain * s.w);
  }
#pragma unroll
  for (int i = 0; i < ROWS; ++i) {
    const int h = h0 + i;
    if (h >= Hout) break;
    win[3] = hrow(h + 3);
    float4 o;
    o.x = (f0 * (win[0].x + win[3].x) + f1 * (win[1].x + win[2].x)) * sc.x;
    o.y = (f0 * (win[0].y + win[3].y) + f1 * (win[1].y + win[2].y)) * sc.y;
    o.z = (f0 * (win[0].z + win[3].z) + f1 * (win[1].z + win[2].z)) * sc.z;
    o.w = (f0 * (win[0].w + win[3].w) + f1 * (win[1].w + win[2].w)) * sc.w;
    *reinterpret_cast<float4*>(y + (((size_t)b * Hout + h) * Wout + w) * C + c) = o;
    win[0] = win[1]; win[1] = win[2]; win[2] = win[3];
  }
}

// The same blur, reading the stride-2 transposed convolution's output T [2H+1, 2W+1] as its four polyphase components
// P[a][b][i, j] = T[2i + a, 2j + b] (sizes (H+1-a) x (W+1-b)): the host computes them as four stride-1 convolutions of
// the low-resolution input (cuDNN fprop kernels: 1.3-1.7x faster than its strided dgrad) and never interleaves them.
struct PhasePtrs { const float* p[2][2]; };
template <int ROWS>
__global__ void __launch_bounds__(256) blur_up_phases_kernel(const PhasePtrs P, float* __restrict__ y, const float* __restrict__ scale,
                                                             int Hout, int Wout, int C, float gain) {
  // One thread: 4 channels of the output column PAIR (2q, 2q+1) for ROWS consecutive rows.  The pair needs T columns
  // 2q-1 .. 2q+3: three from the odd-column phase (q-1, q, q+1) and two from the even one (q, q+1) -- 5 loads per T row for
  // two outputs instead of 8; the kernel is load-issue bound, not DRAM bound.
  const int c4n = C >> 2;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int H = Hout >> 1, W = Wout >> 1;          // low-resolution grid; T is (2H+1) x (2W+1)
  if (t >= W * c4n) return;
  const int q = t / c4n, c = (t % c4n) * 4;
  const int h0 = blockIdx.y * ROWS, b = blockIdx.z;
  const float f0 = 0.125f, f1 = 0.375f;
  const bool has_m1 = q >= 1;                      // odd column 2q-1 exists (otherwise it is the zero padding)
  // T has columns 0..2W: odd phase column q+1 (= T column 2q+3) exists iff q+1 <= W-1; even phase column q+1 (T column 2q+2) always (<= 2W)
  const bool has_p3 = q + 1 < W;
  float4 wa[4], wb[4];                             // horizontally filtered rows of the two outputs (sliding window over 4 T rows)
  auto hrow = [&](int u, float4& oa, float4& ob) { // u: row of the padded T, T_pad[u] = T[u-1]
    const int r = u - 1;
    oa = ob = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < 0 || r > 2 * H) return;
    const int pa = r & 1, ri = r >> 1, Hp = H + 1 - pa;
    const size_t rowi = (size_t)b * Hp + ri;
    const float* rb0 = (pa ? P.p[1][0] : P.p[0][0]) + (rowi * (size_t)(W + 1) + q) * C + c;   // even columns 2q, 2q+2
    const float* rb1 = (pa ? P.p[1][1] : P.p[0][1]) + (rowi * (size_t)W + q) * C + c;         // odd columns 2q-1, 2q+1, 2q+3
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 e0 = __ldg(reinterpret_cast<const float4*>(rb0));
    const float4 e1 = __ldg(reinterpret_cast<const float4*>(rb0 + C));
    const float4 o0 = has_m1 ? __ldg(reinterpret_cast<const float4*>(rb1 - C)) : z;
    const float4 o1 = __ldg(reinterpret_cast<const float4*>(rb1));
    const float4 o2 = has_p3 ? __ldg(reinterpret_cast<const float4*>(rb1 + C)) : z;
    // output 2q  : T columns 2q-1, 2q, 2q+1, 2q+2  = o0, e0, o1, e1 ;  output 2q+1: 2q, 2q+1, 2q+2, 2q+3 = e0, o1, e1, o2
    oa.x = f0 * (o0.x + e1.x) + f1 * (e0.x + o1.x); oa.y = f0 * (o0.y + e1.y) + f1 * (e0.y + o1.y);
    oa.z = f0 * (o0.z + e1.z) + f1 * (e0.z + o1.z); oa.w = f0 * (o0.w + e1.w) + f1 * (e0.w + o1.w);
    ob.x = f0 * (e0.x + o2.x) + f1 * (o1.x + e1.x); ob.y = f0 * (e0.y + o2.y) + f1 * (o1.y + e1.y);
    ob.z = f0 * (e0.z + o2.z) + f1 * (o1.z + e1.z); ob.w = f0 * (e0.w + o2.w) + f1 * (o1.w + e1.w);
  };
  hrow(h0, wa[0], wb[0]); hrow(h0 + 1, wa[1], wb[1]); hrow(h0 + 2, wa[2], wb[2]);
  float4 sc = make_float4(gain, gain, gain, gain);
  if (scale) {
    const float4 s = __ldg(reinterpret_cast<const float4*>(scale + (size_t)b * C + c));
    sc = make_float4(gain * s.x, gain * s.y, gain * s.z, gain * s.w);
  }
#pragma unroll
  for (int i = 0; i < ROWS; ++i) {
    const int h = h0 + i;
    if (h >= Hout) break;
    hrow(h + 3, wa[3], wb[3]);
    float4 o;
    float* dst = y + (((size_t)b * Hout + h) * Wout + 2 * q) * C + c;
    o.x = (f0 * (wa[0].x + wa[3].x) + f1 * (wa[1].x + wa[2].x)) * sc.x; o.y = (f0 * (wa[0].y + wa[3].y) + f1 * (wa[1].y + wa[2].y)) * sc.y;
    o.z = (f0 * (wa[0].z + wa[3].z) + f1 * (wa[1].z + wa[2].z)) * sc.z; o.w = (f0 * (wa[0].w + wa[3].w) + f1 * (wa[1].w + wa[2].w)) * sc.w;
    *reinterpret_cast<float4*>(dst) = o;
    o.x = (f0 * (wb[0].x + wb[3].x) + f1 * (wb[1].x + wb[2].x)) * sc.x; o.y = (f0 * (wb[0].y + wb[3].y) + f1 * (wb[1].y + wb[2].y)) * sc.y;
    o.z = (f0 * (wb[0].z + wb[3].z) + f1 * (wb[1].z + wb[2].z)) * sc.z; o.w = (f0 * (wb[0].w + wb[3].w) + f1 * (wb[1].w + wb[2].w)) * sc.w;
    *reinterpret_cast<float4*>(dst + C) = o;
    wa[0] = wa[1]; wa[1] = wa[2]; wa[2] = wa[3];
    wb[0] = wb[1]; wb[1] = wb[2]; wb[2] = wb[3];
  }
}

// Polyphase form of upfirdn2d(x, [1,3,3,1]/8, up=2, pad=(2,1), gain=4): per dimension out[2i] = 0.25 x[i-1] + 0.75 x[i],
// out[2i+1] = 0.75 x[i] + 0.25 x[i+1] (zero outside).  One thread per INPUT pixel: its 3x3 neighbourhood gives the 2x2 output quad,
// stored as two float2 (a warp writes 256 contiguous bytes per output row).
__global__ void __launch_bounds__(256) upsample2x_nchw_kernel(const float* __restrict__ x, const float* __restrict__ add,
                                                              float* __restrict__ y, int planes, int H, int W) {
  const long long total = (long long)planes * H * W;
  const int OW = 2 * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % W);
    const long long r = i / W;
    const int h = (int)(r % H);
    const long long pl = r / H;
    const float* xp = x + pl * H * W;
    float v[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int hh = h + a - 1, jj = j + b - 1;
        v[a][b] = (hh >= 0 && hh < H && jj >= 0 && jj < W) ? __ldg(xp + (size_t)hh * W + jj) : 0.f;
      }
    float lo[3], hi[3];                               // vertical pass: output rows 2h and 2h+1, per input column
#pragma unroll
    for (int b = 0; b < 3; ++b) { lo[b] = 0.25f * v[0][b] + 0.75f * v[1][b]; hi[b] = 0.75f * v[1][b] + 0.25f * v[2][b]; }
    float2 o0 = make_float2(0.25f * lo[0] + 0.75f * lo[1], 0.75f * lo[1] + 0.25f * lo[2]);
    float2 o1 = make_float2(0.25f * hi[0] + 0.75f * hi[1], 0.75f * hi[1] + 0.25f * hi[2]);
    const size_t o = ((size_t)pl * 2 * H + 2 * h) * OW + 2 * j;
    if (add) {
      const float2 a0 = __ldg(reinterpret_cast<const float2*>(add + o)), a1 = __ldg(reinterpret_cast<const float2*>(add + o + OW));
      o0.x += a0.x; o0.y += a0.y; o1.x += a1.x; o1.y += a1.y;
    }
    *reinterpret_cast<float2*>(y + o) = o0;
    *reinterpret_cast<float2*>(y + o + OW) = o1;
  }
}

__global__ void __launch_bounds__(256) bias_act_kernel(const float4* __restrict__ x, float4* __restrict__ y,
                                                       const float* __restrict__ bias, const float* __restrict__ noise,
                                                       const float* __restrict__ strength, long long noise_bstride,
                                                       size_t total4, int HW, int c4n, int act, float gain) {
  const float st = (noise && strength) ? __ldg(strength) : (noise ? 1.f : 0.f);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % c4n);
    const size_t tok = i / c4n;
    const int t = (int)(tok % HW);
    const size_t b = tok / HW;
    float4 v = x[i];
    float nz = 0.f;
    if (noise) nz = __ldg(noise + b * noise_bstride + t) * st;
    float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) bb = __ldg(reinterpret_cast<const float4*>(bias) + c4);
    v.x += nz + bb.x; v.y += nz + bb.y; v.z += nz + bb.z; v.w += nz + bb.w;
    if (act == 1) {
      v.x = fmaxf(v.x, 0.2f * v.x); v.y = fmaxf(v.y, 0.2f * v.y); v.z = fmaxf(v.z, 0.2f * v.z); v.w = fmaxf(v.w, 0.2f * v.w);
    }
    y[i] = make_float4(v.x * gain, v.y * gain, v.z * gain, v.w * gain);
  }
}

// d[b,o] = rsqrt(sum_i s[b,i]^2 * wsq[o,i] + eps): one warp per output, lanes stride over i
__global__ void __launch_bounds__(256) demod_coef_kernel(const float* __restrict__ s, const float* __restrict__ wsq,
                                                         float* __restrict__ d, int B, int O, int I, float eps, int s_ld) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * O) return;
  const int b = warp / O, o = warp % O;
  const float* sb = s + (size_t)b * s_ld;
  const float* wo = wsq + (size_t)o * I;
  float acc = 0.f;
  for (int i = lane; i < I; i += 32) { const float v = sb[i]; acc = fmaf(v * v, wo[i], acc); }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) d[warp] = rsqrtf(acc + eps);
}

// every convolution layer of a network in one launch: blockIdx.y = layer.  One warp per output channel o: its wsq row stays in
// registers (first 512 input channels; the rest is re-read) while the warp walks the batch, two samples in flight
// (one warp per (b, o) was latency-bound: 213 k short-lived warps for config 2, 65 us)
struct DemodBatch { gf_demod_job job[GF_DEMOD_MAX_JOBS]; };
__global__ void __launch_bounds__(256) demod_coef_batch_kernel(const __grid_constant__ DemodBatch Jb, int B, float eps) {
  const gf_demod_job& J = Jb.job[blockIdx.y];
  const int o = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (o >= J.O) return;
  const float* wo = J.wsq + (size_t)o * J.I;
  float wr[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) { const int i = lane + 32 * q; wr[q] = i < J.I ? __ldg(wo + i) : 0.f; }
  for (int b = 0; b < B; b += 2) {
    const float* s0 = J.styles + (size_t)b * J.s_ld;
    const bool two = b + 1 < B;
    const float* s1 = two ? s0 + J.s_ld : s0;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int i = lane + 32 * q;
      if (i < J.I) { const float v0 = __ldg(s0 + i), v1 = __ldg(s1 + i); a0 = fmaf(v0 * v0, wr[q], a0); a1 = fmaf(v1 * v1, wr[q], a1); }
    }
    for (int i = 512 + lane; i < J.I; i += 32) { const float w = __ldg(wo + i), v0 = s0[i], v1 = s1[i]; a0 = fmaf(v0 * v0, w, a0); a1 = fmaf(v1 * v1, w, a1); }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { a0 += __shfl_xor_sync(0xffffffffu, a0, off); a1 += __shfl_xor_sync(0xffffffffu, a1, off); }
    if (lane == 0) {
      J.d[(size_t)b * J.O + o] = rsqrtf(a0 + eps);
      if (two) J.d[(size_t)(b + 1) * J.O + o] = rsqrtf(a1 + eps);
    }
  }
}

}  // namespace gf

using namespace gf;


// ------------------------------------------------------------------------------------------------------
// tRGB: 1x1 modulated convolution without demodulation, channels-last input -> planar image
//   y[b,o,t] = sum_c x[b,t,c] * w[o,c] * styles[b,c] * wscale + bias[o]
// One warp per 32 tokens: lane l owns the float4 channel chunks l, l+32, ... (its slice of the per-sample weights lives
// in registers), 4 tokens in flight per step, butterfly reduction, lane i keeps token i -> coalesced planar stores.
// ------------------------------------------------------------------------------------------------------
template <int O, int NQ>
__global__ void __launch_bounds__(256) torgb_kernel(const float4* __restrict__ x, const float* __restrict__ w, const float* __restrict__ styles,
                                                    int s_ld, const float* __restrict__ bias, float wscale, float* __restrict__ y,
                                                    int HW, int C4, int tok_per_cta, const float* __restrict__ s2, int s2_ld,
                                                    float4* __restrict__ xs_out) {
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 wr[O][NQ];
  float4 s2r[NQ];                                  // optional second output: x * s2 (the next convolution's style modulation)
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const int c4 = lane + q * 32;
    s2r[q] = (xs_out && c4 < C4) ? *reinterpret_cast<const float4*>(s2 + (size_t)b * s2_ld + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < C4) s4 = *reinterpret_cast<const float4*>(styles + (size_t)b * s_ld + c4 * 4);
#pragma unroll
    for (int o = 0; o < O; ++o) {
      float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c4 < C4) w4 = *reinterpret_cast<const float4*>(w + (size_t)o * C4 * 4 + c4 * 4);
      wr[o][q] = make_float4(w4.x * s4.x * wscale, w4.y * s4.y * wscale, w4.z * s4.z * wscale, w4.w * s4.w * wscale);
    }
  }
  const int t_beg = blockIdx.x * tok_per_cta, t_end = min(HW, t_beg + tok_per_cta);
  const float4* xb = x + (size_t)b * HW * C4;
  for (int t0 = t_beg + warp * 32; t0 < t_end; t0 += 8 * 32) {
    float keep[O];
#pragma unroll
    for (int o = 0; o < O; ++o) keep[o] = 0.f;
#pragma unroll 1
    for (int i0 = 0; i0 < 32; i0 += 4) {
      float acc[4][O];
      float4 xv[4][NQ];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int t = t0 + i0 + u;
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
          const int c4 = lane + q * 32;
          xv[u][q] = (t < t_end && c4 < C4) ? __ldg(xb + (size_t)t * C4 + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
          if (xs_out && t < t_end && c4 < C4)
            xs_out[((size_t)b * HW + t) * C4 + c4] = make_float4(xv[u][q].x * s2r[q].x, xv[u][q].y * s2r[q].y, xv[u][q].z * s2r[q].z, xv[u][q].w * s2r[q].w);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
#pragma unroll
        for (int o = 0; o < O; ++o) {
          float a = 0.f;
#pragma unroll
          for (int q = 0; q < NQ; ++q)
            a = fmaf(xv[u][q].x, wr[o][q].x, fmaf(xv[u][q].y, wr[o][q].y, fmaf(xv[u][q].z, wr[o][q].z, fmaf(xv[u][q].w, wr[o][q].w, a))));
          acc[u][o] = a;
        }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
          for (int o = 0; o < O; ++o) acc[u][o] += __shfl_xor_sync(0xffffffffu, acc[u][o], off);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (lane == i0 + u) {
#pragma unroll
          for (int o = 0; o < O; ++o) keep[o] = acc[u][o];
        }
      }
    }
    const int t = t0 + lane;
    if (t < t_end) {
#pragma unroll
      for (int o = 0; o < O; ++o) y[((size_t)b * O + o) * HW + t] = keep[o] + (bias ? bias[o] : 0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// G_mapping as ONE kernel (SURVEY row f4): pixel-norm of every latent, then L fully connected layers (+ leaky-ReLU) --
// one MLP shared by the k local components, one for the global latent -- and the truncation lerp.  All 2 L weight
// matrices (D x D, equalised-LR and activation gains pre-folded, [in][out]) are staged in shared memory once per CTA;
// one warp owns one latent row at a time (lane = output feature, the input vector is broadcast from shared memory).
// Replaces 16 small GEMMs + 16 activation kernels + 6 elementwise kernels per step of the eager form.
// ------------------------------------------------------------------------------------------------------
constexpr int MAP_WARPS = 8, MAP_MAXM = 4;          // D <= 128
__global__ void __launch_bounds__(MAP_WARPS * 32) mapping_kernel(const float* __restrict__ z, const float* __restrict__ Wt,
                                                                 const float* __restrict__ bias, const float* __restrict__ w_avg, float psi,
                                                                 float* __restrict__ out, int rows, int k, int D, int L) {
  extern __shared__ float msm[];
  float* Ws = msm;                                   // [2][L][D][D]
  float* bs = Ws + (size_t)2 * L * D * D;            // [2][L][D]
  float* xs = bs + (size_t)2 * L * D;                // [MAP_WARPS][D]
  for (int i = threadIdx.x; i < 2 * L * D * D; i += blockDim.x) Ws[i] = Wt[i];
  for (int i = threadIdx.x; i < 2 * L * D; i += blockDim.x) bs[i] = bias[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* x = xs + warp * D;
  const int nm = (D + 31) >> 5;
  for (int row = blockIdx.x * MAP_WARPS + warp; row < rows; row += gridDim.x * MAP_WARPS) {
    const int comp = row % (k + 1);
    const int path = comp == k ? 1 : 0;              // the last latent of every sample is the global one
    // pixel norm: x * rsqrt(mean(x^2) + 1e-8)
    float v[MAP_MAXM], ss = 0.f;
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) {
      const int o = lane + 32 * m;
      v[m] = (m < nm && o < D) ? z[(size_t)row * D + o] : 0.f;
      ss = fmaf(v[m], v[m], ss);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rn = rsqrtf(ss / (float)D + 1e-8f);
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) x[lane + 32 * m] = v[m] * rn;
    __syncwarp();
    for (int l = 0; l < L; ++l) {
      const float* W = Ws + ((size_t)path * L + l) * D * D;
      const float* bb = bs + ((size_t)path * L + l) * D;
      float acc[MAP_MAXM];
#pragma unroll
      for (int m = 0; m < MAP_MAXM; ++m) acc[m] = (m < nm && lane + 32 * m < D) ? bb[lane + 32 * m] : 0.f;
      for (int i = 0; i < D; ++i) {
        const float xi = x[i];                       // broadcast
#pragma unroll
        for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) acc[m] = fmaf(xi, W[(size_t)i * D + lane + 32 * m], acc[m]);
      }
      __syncwarp();
#pragma unroll
      for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) x[lane + 32 * m] = fmaxf(acc[m], 0.2f * acc[m]);   // gain sqrt(2) is in W, b
      __syncwarp();
    }
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) {
      const int o = lane + 32 * m;
      if (m < nm && o < D) {
        float r = x[o];
        if (w_avg) { const float a = w_avg[path * D + o]; r = a + psi * (r - a); }      // truncation trick: lerp(w_avg, w, psi)
        out[(size_t)row * D + o] = r;
      }
    }
    __syncwarp();
  }
}

// Class-conditional G_mapping (SURVEY A.4 item 14): mapping_kernel with the label embedding e_b = c_b E concatenated to every
// latent of image b = row / (k+1) before the pixel norm, so layer 0 has fan-in 2D.  A warp computes e_b itself: its lanes load 32
// labels at a time, and the nonzero ones (a warp-uniform ballot) add their row of E in ascending order, read through L2.  Layer 0
// reads its latent half [D][D] from shared memory and its label half from L2; layers 1..L-1 are staged as in mapping_kernel.
__global__ void __launch_bounds__(MAP_WARPS * 32) mapping_cond_kernel(const float* __restrict__ z, const float* __restrict__ c, int c_dim,
                                                                      const float* __restrict__ E, const float* __restrict__ W0,
                                                                      const float* __restrict__ Wt, const float* __restrict__ bias,
                                                                      const float* __restrict__ w_avg, float psi, float* __restrict__ out,
                                                                      int rows, int k, int D, int L) {
  extern __shared__ float msm[];
  const int DD = D * D;
  float* W0s = msm;                                  // [2][D][D]: rows 0..D-1 (the latent half) of each path's [2D][D]
  float* Ws = W0s + (size_t)2 * DD;                  // [2][L-1][D][D]
  float* bs = Ws + (size_t)2 * (L - 1) * DD;         // [2][L][D]
  float* xs = bs + (size_t)2 * L * D;                // [MAP_WARPS][2D]
  for (int i = threadIdx.x; i < 2 * DD; i += blockDim.x) W0s[i] = W0[(size_t)(i / DD) * 2 * DD + i % DD];
  for (int i = threadIdx.x; i < 2 * (L - 1) * DD; i += blockDim.x) Ws[i] = Wt[i];
  for (int i = threadIdx.x; i < 2 * L * D; i += blockDim.x) bs[i] = bias[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* x = xs + warp * 2 * D;
  const int nm = (D + 31) >> 5;
  for (int row = blockIdx.x * MAP_WARPS + warp; row < rows; row += gridDim.x * MAP_WARPS) {
    const int b = row / (k + 1), comp = row % (k + 1);
    const int path = comp == k ? 1 : 0;              // the last latent of every sample is the global one
    // e_b = c_b . E
    float e[MAP_MAXM];
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) e[m] = 0.f;
    const float* cb = c + (size_t)b * c_dim;
    for (int j0 = 0; j0 < c_dim; j0 += 32) {
      const float cv = j0 + lane < c_dim ? cb[j0 + lane] : 0.f;
      unsigned nz = __ballot_sync(0xffffffffu, cv != 0.f);
      while (nz) {
        const int s = __ffs(nz) - 1;
        nz &= nz - 1;
        const float cj = __shfl_sync(0xffffffffu, cv, s);
        const float* Er = E + (size_t)(j0 + s) * D;
#pragma unroll
        for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) e[m] = fmaf(cj, __ldg(Er + lane + 32 * m), e[m]);
      }
    }
    // pixel norm of [z || e]: x * rsqrt(mean over the 2D entries of x^2 + 1e-8)
    float v[MAP_MAXM], ss = 0.f;
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) {
      const int o = lane + 32 * m;
      v[m] = (m < nm && o < D) ? z[(size_t)row * D + o] : 0.f;
      ss = fmaf(v[m], v[m], ss);
      ss = fmaf(e[m], e[m], ss);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rn = rsqrtf(ss / (float)(2 * D) + 1e-8f);
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) { x[lane + 32 * m] = v[m] * rn; x[D + lane + 32 * m] = e[m] * rn; }
    __syncwarp();
    for (int l = 0; l < L; ++l) {
      const float* bb = bs + ((size_t)path * L + l) * D;
      float acc[MAP_MAXM];
#pragma unroll
      for (int m = 0; m < MAP_MAXM; ++m) acc[m] = (m < nm && lane + 32 * m < D) ? bb[lane + 32 * m] : 0.f;
      if (l == 0) {
        const float* W = W0s + (size_t)path * DD;
        const float* We = W0 + ((size_t)path * 2 + 1) * DD;     // the label half of layer 0
        for (int i = 0; i < D; ++i) {
          const float xi = x[i];
#pragma unroll
          for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) acc[m] = fmaf(xi, W[(size_t)i * D + lane + 32 * m], acc[m]);
        }
        for (int i = 0; i < D; ++i) {
          const float xi = x[D + i];
#pragma unroll
          for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) acc[m] = fmaf(xi, __ldg(We + (size_t)i * D + lane + 32 * m), acc[m]);
        }
      } else {
        const float* W = Ws + ((size_t)path * (L - 1) + (l - 1)) * DD;
        for (int i = 0; i < D; ++i) {
          const float xi = x[i];
#pragma unroll
          for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) acc[m] = fmaf(xi, W[(size_t)i * D + lane + 32 * m], acc[m]);
        }
      }
      __syncwarp();
#pragma unroll
      for (int m = 0; m < MAP_MAXM; ++m) if (m < nm && lane + 32 * m < D) x[lane + 32 * m] = fmaxf(acc[m], 0.2f * acc[m]);
      __syncwarp();
    }
#pragma unroll
    for (int m = 0; m < MAP_MAXM; ++m) {
      const int o = lane + 32 * m;
      if (m < nm && o < D) {
        float r = x[o];
        if (w_avg) { const float a = w_avg[path * D + o]; r = a + psi * (r - a); }      // one label-agnostic w_avg
        out[(size_t)row * D + o] = r;
      }
    }
    __syncwarp();
  }
}

extern "C" {

int gf_chan_scale_nhwc(const float* x, const float* s, int s_ld, float* y, int B, int HW, int C, void* stream) {
  if (!x || !s || !y) { set_error("gf_chan_scale_nhwc: null pointer"); return GF_ERR_INVALID; }
  if (misaligned16(x) || misaligned16(s) || misaligned16(y)) { set_error("gf_chan_scale_nhwc: x, s and y must be 16-byte aligned"); return GF_ERR_INVALID; }
  if (B <= 0 || HW <= 0 || C <= 0 || (C & 3) || s_ld < C || (s_ld & 3)) {
    set_error("gf_chan_scale_nhwc: need B,HW,C > 0, C %% 4 == 0, s_ld >= C, s_ld %% 4 == 0 (C=%d s_ld=%d)", C, s_ld);
    return GF_ERR_UNSUPPORTED;
  }
  const size_t total4 = (size_t)B * HW * (C >> 2);
  chan_scale_kernel<<<grid_for(total4, 256 * 4), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(s), reinterpret_cast<float4*>(y), total4, HW * (C >> 2), C >> 2, s_ld >> 2);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_blur_up_nhwc(const float* x, float* y, const float* scale, int B, int Hout, int Wout, int C, float gain, void* stream) {
  if (!x || !y) { set_error("gf_blur_up_nhwc: null pointer"); return GF_ERR_INVALID; }
  if (misaligned16(x) || misaligned16(y) || misaligned16(scale)) { set_error("gf_blur_up_nhwc: x, y and scale must be 16-byte aligned"); return GF_ERR_INVALID; }
  if (B <= 0 || Hout <= 0 || Wout <= 0 || C <= 0 || (C & 3) || B > 65535) { set_error("gf_blur_up_nhwc: bad shape (B=%d Hout=%d Wout=%d C=%d)", B, Hout, Wout, C); return GF_ERR_UNSUPPORTED; }
  constexpr int ROWS = 8;
  dim3 grid((Wout * (C >> 2) + 255) / 256, (Hout + ROWS - 1) / ROWS, B);
  blur_up_kernel<ROWS><<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, scale, Hout, Wout, C, gain, 1);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_blur_up_phases_nhwc(const float* p00, const float* p01, const float* p10, const float* p11, float* y, const float* scale,
                           int B, int Hout, int Wout, int C, float gain, void* stream) {
  if (!p00 || !p01 || !p10 || !p11 || !y) { set_error("gf_blur_up_phases_nhwc: null pointer"); return GF_ERR_INVALID; }
  if (misaligned16(p00) || misaligned16(p01) || misaligned16(p10) || misaligned16(p11) || misaligned16(y) || misaligned16(scale)) {
    set_error("gf_blur_up_phases_nhwc: the four phases, y and scale must be 16-byte aligned"); return GF_ERR_INVALID;
  }
  if (B <= 0 || Hout <= 0 || Wout <= 0 || (Hout & 1) || (Wout & 1) || C <= 0 || (C & 3) || B > 65535) {
    set_error("gf_blur_up_phases_nhwc: bad shape (B=%d Hout=%d Wout=%d C=%d)", B, Hout, Wout, C); return GF_ERR_UNSUPPORTED;
  }
  constexpr int ROWS = 8;
  PhasePtrs P;
  P.p[0][0] = p00; P.p[0][1] = p01; P.p[1][0] = p10; P.p[1][1] = p11;
  dim3 grid(((Wout >> 1) * (C >> 2) + 255) / 256, (Hout + ROWS - 1) / ROWS, B);
  blur_up_phases_kernel<ROWS><<<grid, 256, 0, (cudaStream_t)stream>>>(P, y, scale, Hout, Wout, C, gain);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_fir4_nhwc(const float* x, float* y, int B, int Hin, int Win, int C, int pad, float gain, void* stream) {
  if (!x || !y) { set_error("gf_fir4_nhwc: null pointer"); return GF_ERR_INVALID; }
  if (misaligned16(x) || misaligned16(y)) { set_error("gf_fir4_nhwc: x and y must be 16-byte aligned"); return GF_ERR_INVALID; }
  const int Hout = Hin + 2 * pad - 3, Wout = Win + 2 * pad - 3;
  if (B <= 0 || Hout <= 0 || Wout <= 0 || C <= 0 || (C & 3) || B > 65535 || pad < 0 || pad > 3) {
    set_error("gf_fir4_nhwc: bad arguments (B=%d Hin=%d Win=%d C=%d pad=%d)", B, Hin, Win, C, pad); return GF_ERR_UNSUPPORTED;
  }
  constexpr int ROWS = 8;
  dim3 grid((Wout * (C >> 2) + 255) / 256, (Hout + ROWS - 1) / ROWS, B);
  blur_up_kernel<ROWS><<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, nullptr, Hout, Wout, C, gain, pad);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_upsample2x_nchw(const float* x, const float* add, float* y, int B, int C, int H, int W, void* stream) {
  if (!x || !y) { set_error("gf_upsample2x_nchw: null pointer"); return GF_ERR_INVALID; }
  if (B <= 0 || C <= 0 || H <= 0 || W <= 0) { set_error("gf_upsample2x_nchw: bad shape"); return GF_ERR_INVALID; }
  if (((uintptr_t)y & 7) || (add && ((uintptr_t)add & 7))) { set_error("gf_upsample2x_nchw: y / add must be 8-byte aligned"); return GF_ERR_INVALID; }
  const size_t total = (size_t)B * C * H * W;                    // one thread per input pixel
  upsample2x_nchw_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, add, y, B * C, H, W);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_bias_act_nhwc(const float* x, float* y, const float* bias, const float* noise, const float* strength,
                     long long noise_bstride, int B, int HW, int C, int act, float gain, void* stream) {
  if (!x || !y) { set_error("gf_bias_act_nhwc: null pointer"); return GF_ERR_INVALID; }
  if (misaligned16(x) || misaligned16(y) || misaligned16(bias)) { set_error("gf_bias_act_nhwc: x, y and bias must be 16-byte aligned"); return GF_ERR_INVALID; }
  if (B <= 0 || HW <= 0 || C <= 0 || (C & 3) || act < 0 || act > 1) { set_error("gf_bias_act_nhwc: bad arguments (C=%d act=%d)", C, act); return GF_ERR_UNSUPPORTED; }
  const size_t total4 = (size_t)B * HW * (C >> 2);
  bias_act_kernel<<<grid_for(total4, 256 * 4), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), bias, noise, strength, noise_bstride, total4, HW, C >> 2, act, gain);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_demod_coef(const float* styles, int s_ld, const float* wsq, float* d, int B, int O, int I, float eps, void* stream) {
  if (!styles || !wsq || !d) { set_error("gf_demod_coef: null pointer"); return GF_ERR_INVALID; }
  if (B <= 0 || O <= 0 || I <= 0 || s_ld < I) { set_error("gf_demod_coef: bad shape"); return GF_ERR_INVALID; }
  const long long warps = (long long)B * O;
  demod_coef_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(styles, wsq, d, B, O, I, eps, s_ld);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_demod_coef_batch(const gf_demod_job* jobs, int n, int B, float eps, void* stream) {
  if (!jobs || n <= 0 || n > GF_DEMOD_MAX_JOBS || B <= 0) { set_error("gf_demod_coef_batch: needs 1 <= n <= %d jobs and B > 0 (got n=%d B=%d)", GF_DEMOD_MAX_JOBS, n, B); return GF_ERR_INVALID; }
  DemodBatch Jb;
  int max_o = 0;
  for (int i = 0; i < n; ++i) {
    const gf_demod_job& J = jobs[i];
    if (!J.styles || !J.wsq || !J.d || J.O <= 0 || J.I <= 0 || J.s_ld < J.I) { set_error("gf_demod_coef_batch: job %d: null pointer or bad shape", i); return GF_ERR_INVALID; }
    Jb.job[i] = J;
    if (J.O > max_o) max_o = J.O;
  }
  dim3 grid((unsigned)(((long long)max_o * 32 + 255) / 256), (unsigned)n);
  demod_coef_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(Jb, B, eps);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_torgb_nhwc(const float* x, const float* w, const float* styles, int s_ld, const float* bias, float wscale, float* y,
                  int B, int HW, int C, void* stream) {
  return gf_torgb_scale_nhwc(x, w, styles, s_ld, bias, wscale, y, nullptr, 0, nullptr, B, HW, C, stream);
}

int gf_torgb_scale_nhwc(const float* x, const float* w, const float* styles, int s_ld, const float* bias, float wscale, float* y,
                        const float* s2, int s2_ld, float* xs_out, int B, int HW, int C, void* stream) {
  if (!x || !w || !styles || !y) { set_error("gf_torgb_nhwc: null pointer"); return GF_ERR_INVALID; }
  if (misaligned16(x) || misaligned16(w) || misaligned16(styles)) { set_error("gf_torgb_nhwc: x, w and styles must be 16-byte aligned"); return GF_ERR_INVALID; }
  if ((xs_out != nullptr) != (s2 != nullptr) || (xs_out && (s2_ld < C || (s2_ld & 3) || ((uintptr_t)s2 & 15) || ((uintptr_t)xs_out & 15)))) {
    set_error("gf_torgb_scale_nhwc: s2 / xs_out must both be given, 16-byte aligned, s2_ld >= C and %% 4 == 0"); return GF_ERR_INVALID;
  }
  if (B <= 0 || HW <= 0 || C <= 0 || (C & 3) || C > 512 || s_ld < C || (s_ld & 3) || B > 65535) {
    set_error("gf_torgb_nhwc: unsupported arguments (C=%d s_ld=%d B=%d)", C, s_ld, B); return GF_ERR_UNSUPPORTED;
  }
  const int C4 = C >> 2, nq = (C4 + 31) / 32;
  // 1024 tokens per CTA amortise the per-sample weight load; small images take fewer so that the grid still covers the SMs
  // (res 32 / 64 at B = 32 ran on 32 / 128 CTAs: 144 / 171 us for 67 / 268 MB)
  int tok_per_cta = 1024;
  while (tok_per_cta > 256 && (long long)((HW + tok_per_cta - 1) / tok_per_cta) * B < 4LL * num_sms()) tok_per_cta >>= 1;
  dim3 grid((HW + tok_per_cta - 1) / tok_per_cta, B);
  const float4* x4 = reinterpret_cast<const float4*>(x);
  cudaStream_t st = (cudaStream_t)stream;
  switch (nq) {
    case 1: torgb_kernel<3, 1><<<grid, 256, 0, st>>>(x4, w, styles, s_ld, bias, wscale, y, HW, C4, tok_per_cta, s2, s2_ld, reinterpret_cast<float4*>(xs_out)); break;
    case 2: torgb_kernel<3, 2><<<grid, 256, 0, st>>>(x4, w, styles, s_ld, bias, wscale, y, HW, C4, tok_per_cta, s2, s2_ld, reinterpret_cast<float4*>(xs_out)); break;
    case 3: torgb_kernel<3, 3><<<grid, 256, 0, st>>>(x4, w, styles, s_ld, bias, wscale, y, HW, C4, tok_per_cta, s2, s2_ld, reinterpret_cast<float4*>(xs_out)); break;
    default: torgb_kernel<3, 4><<<grid, 256, 0, st>>>(x4, w, styles, s_ld, bias, wscale, y, HW, C4, tok_per_cta, s2, s2_ld, reinterpret_cast<float4*>(xs_out)); break;
  }
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_mapping_fwd(const float* z, const float* w, const float* b, const float* w_avg, float psi, float* out,
                   int B, int k, int D, int L, void* stream) {
  if (!z || !w || !b || !out) { set_error("gf_mapping_fwd: null pointer"); return GF_ERR_INVALID; }
  if (B <= 0 || k < 0 || D <= 0 || L <= 0) { set_error("gf_mapping_fwd: bad sizes B=%d k=%d D=%d L=%d", B, k, D, L); return GF_ERR_INVALID; }
  if (D > 32 * MAP_MAXM) { set_error("gf_mapping_fwd: latent width D=%d > %d is not served by the fused kernel", D, 32 * MAP_MAXM); return GF_ERR_UNSUPPORTED; }
  const size_t smem = ((size_t)2 * L * D * D + (size_t)2 * L * D + (size_t)MAP_WARPS * D) * sizeof(float);
  int dev = 0, optin = 0;
  GF_CUDA_OK(cudaGetDevice(&dev));
  GF_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  if (smem > (size_t)optin) { set_error("gf_mapping_fwd: 2*L*D*D weights (%zu bytes) do not fit shared memory", smem); return GF_ERR_UNSUPPORTED; }
  GF_CUDA_OK(cudaFuncSetAttribute(mapping_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int rows = B * (k + 1);
  int grid = (rows + MAP_WARPS - 1) / MAP_WARPS;
  if (grid > num_sms()) grid = num_sms();
  mapping_kernel<<<grid, MAP_WARPS * 32, smem, (cudaStream_t)stream>>>(z, w, b, w_avg, psi, out, rows, k, D, L);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_mapping_fwd_cond(const float* z, const float* c, int c_dim, const float* E, const float* w0, const float* w, const float* b,
                        const float* w_avg, float psi, float* out, int B, int k, int D, int L, void* stream) {
  if (!z || !c || !E || !w0 || !b || !out || (L > 1 && !w)) { set_error("gf_mapping_fwd_cond: null pointer"); return GF_ERR_INVALID; }
  if (B <= 0 || k < 0 || D <= 0 || L <= 0 || c_dim < 1) {
    set_error("gf_mapping_fwd_cond: bad sizes B=%d k=%d D=%d L=%d c_dim=%d", B, k, D, L, c_dim); return GF_ERR_INVALID;
  }
  if (D > 32 * MAP_MAXM) { set_error("gf_mapping_fwd_cond: latent width D=%d > %d is not served by the fused kernel", D, 32 * MAP_MAXM); return GF_ERR_UNSUPPORTED; }
  const size_t smem = ((size_t)2 * L * D * D + (size_t)2 * L * D + (size_t)MAP_WARPS * 2 * D) * sizeof(float);
  int dev = 0, optin = 0;
  GF_CUDA_OK(cudaGetDevice(&dev));
  GF_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  if (smem > (size_t)optin) { set_error("gf_mapping_fwd_cond: 2*L*D*D weights (%zu bytes) do not fit shared memory", smem); return GF_ERR_UNSUPPORTED; }
  GF_CUDA_OK(cudaFuncSetAttribute(mapping_cond_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int rows = B * (k + 1);
  int grid = (rows + MAP_WARPS - 1) / MAP_WARPS;
  if (grid > num_sms()) grid = num_sms();
  mapping_cond_kernel<<<grid, MAP_WARPS * 32, smem, (cudaStream_t)stream>>>(z, c, c_dim, E, w0, w, b, w_avg, psi, out, rows, k, D, L);
  GF_LAUNCH_OK();
  return GF_OK;
}

}  // extern "C"
