// gf_bwd.cu -- backward of stage T (SURVEY row f2): the per-token part of d(loss)/d(x, K', V^T, Rt, Ct).
//
// Forward (oracle/folded.py per_token):  s = x.K'^T + Rt[h] + Ct[w];  p = softmax(s);  ctl = p.V^T (gain | bias);
//     xn = LayerNorm(x) (or x);   out = xn*g  |  xn + g  |  xn*g + b.
// Given dOut this kernel recomputes s, p and the statistics and writes, in three sweeps over the 32-channel chunks of a
// 128-token tile (thread = token, fp32 FMA):
//     dX   [B,n,C]     = LN^T(dxn) + ds.K'                      (the activation gradient)
//     dS   [B,n,KP]    = p * (dp - <p, dp>),  dp = dCtl.V^T     (gradient w.r.t. the logits)
//     P    [B,n,KP]    the probabilities
//     dCtl [B,n,Cout]  = dOut*xn (gain half) | dOut (bias half) (gradient w.r.t. the control signal)
// The remaining reductions over tokens are plain batched GEMMs / sums done by the caller (autograd.py):
//     dK'[b] = dS[b]^T X[b],   dV^T[b] = dCtl[b]^T P[b],   dRt = sum_w dS,   dCt = sum_h dS,
// and the chain rule through stages I and W is torch autograd over tiny [B,k,*] tensors.
// Replaces ~45 full passes over [B,n,C]-sized tensors of the direct-form autograd composite by 8.
//
// Also here: the backward of duplex pass A (centroid_bwd_kernel, gf_attn_centroid_stats / gf_attn_centroid_bwd).  Stage T of a
// duplex layer is the computation above with keys from the centroids, so a duplex layer's backward is token_bwd_kernel, then
// centroid_bwd_kernel adding the pass-A part of dX.
#include <string.h>
#include "gf_common.cuh"

namespace gf {

static constexpr int BTM = 128;     // tokens per CTA (one thread per token)
static constexpr int BCH = 32;      // channels per chunk
static constexpr int BXS = BCH + 4; // padded smem row

struct BwdParams {
  const float* X; const float* dOut; const float* Kp; const float* Vt; const float* Rt; const float* Ct;
  float* dX; float* dS; float* P; float* dCtl;
  int n, H, W, C, k, Cout, norm, integration;
  DropoutArgs dp;            // attention dropout of the forward call (thr = 0: off)
  const float* cb;           // [Cout] bo (+1): ctl = sum_j q_j (Vt_j - cb) + cb when dropout is on
};

__device__ __forceinline__ void bwd_load_chunk(float (*dst)[BXS], const float* __restrict__ src, int t0, int n, int ld, int c0) {
#pragma unroll
  for (int it = 0; it < BTM / 16; ++it) {
    const int row = it * 16 + (threadIdx.x >> 3), c4 = (threadIdx.x & 7) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + row < n) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)(t0 + row) * ld + c0 + c4));
    *reinterpret_cast<float4*>(&dst[row][c4]) = v;
  }
}
__device__ __forceinline__ void bwd_store_chunk(float* __restrict__ dst, float (*src)[BXS], int t0, int n, int ld, int c0) {
#pragma unroll
  for (int it = 0; it < BTM / 16; ++it) {
    const int row = it * 16 + (threadIdx.x >> 3), c4 = (threadIdx.x & 7) * 4;
    if (t0 + row < n) *reinterpret_cast<float4*>(dst + (size_t)(t0 + row) * ld + c0 + c4) = *reinterpret_cast<const float4*>(&src[row][c4]);
  }
}

template <int KP>
__global__ void __launch_bounds__(BTM) token_bwd_kernel(const BwdParams P) {
  extern __shared__ __align__(16) uint8_t bsm_raw[];
  float (*xs)[BXS] = reinterpret_cast<float (*)[BXS]>(bsm_raw);                               // x chunk / result staging
  float (*gs)[BXS] = reinterpret_cast<float (*)[BXS]>(bsm_raw + sizeof(float) * BTM * BXS);   // dOut chunk / dCtl staging
  float (*ks)[BCH] = reinterpret_cast<float (*)[BCH]>(bsm_raw + 2 * sizeof(float) * BTM * BXS);         // K' chunk [KP][32]
  float (*vs)[KP] = reinterpret_cast<float (*)[KP]>(reinterpret_cast<uint8_t*>(ks) + sizeof(float) * KP * BCH);   // V^T gain chunk [32][KP]
  float (*vs2)[KP] = reinterpret_cast<float (*)[KP]>(reinterpret_cast<uint8_t*>(vs) + sizeof(float) * KP * BCH);   // V^T bias chunk

  const int b = blockIdx.y, t0 = blockIdx.x * BTM, tid = threadIdx.x, t = t0 + tid;
  const int n = P.n, C = P.C, Cout = P.Cout, integ = P.integration;
  const bool valid = t < n;
  const float* Xb = P.X + (size_t)b * n * C;
  const float* Gb = P.dOut + (size_t)b * n * C;
  const float* Kpb = P.Kp + (size_t)b * KP * C;
  const float* Vtb = P.Vt + (size_t)b * Cout * KP;
  float* dXb = P.dX + (size_t)b * n * C;
  float* dCb = P.dCtl + (size_t)b * n * Cout;

  float s[KP];
  {
    const int h = valid ? t / P.W : 0, w = valid ? t % P.W : 0;
    const float* rt = P.Rt + ((size_t)b * P.H + h) * KP;
    const float* ct = P.Ct + ((size_t)b * P.W + w) * KP;
#pragma unroll
    for (int j = 0; j < KP; ++j) s[j] = rt[j] + ct[j];
  }
  // ---- sweep 1: logits + layer-norm statistics (as the forward)
  float sum = 0.f, sumsq = 0.f, shift = 0.f;
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    for (int i = tid; i < KP * BCH / 4; i += BTM) {
      const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
      *reinterpret_cast<float4*>(&ks[j][c4]) = __ldg(reinterpret_cast<const float4*>(Kpb + (size_t)j * C + c0 + c4));
    }
    __syncthreads();
    if (c0 == 0) shift = xs[tid][0];
#pragma unroll
    for (int c4 = 0; c4 < BCH; c4 += 4) {
      const float4 x = *reinterpret_cast<const float4*>(&xs[tid][c4]);
      const float d0 = x.x - shift, d1 = x.y - shift, d2 = x.z - shift, d3 = x.w - shift;
      sum += (d0 + d1) + (d2 + d3);
      sumsq = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, sumsq))));
#pragma unroll
      for (int j = 0; j < KP; ++j) {
        const float4 kv = *reinterpret_cast<const float4*>(&ks[j][c4]);
        s[j] = fmaf(x.x, kv.x, fmaf(x.y, kv.y, fmaf(x.z, kv.z, fmaf(x.w, kv.w, s[j]))));
      }
    }
  }
  float mx = s[0];
#pragma unroll
  for (int j = 1; j < KP; ++j) mx = fmaxf(mx, s[j]);
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < KP; ++j) { s[j] = expf(s[j] - mx); den += s[j]; }
  const float inv = 1.f / den;
#pragma unroll
  for (int j = 0; j < KP; ++j) s[j] *= inv;                       // s = p from here on
  // attention dropout: q = p * mk feeds the control signal (and the dV^T reduction); the softmax backward uses p itself
  float pk[KP];                                                  // p before dropout (only read when dropout is on)
  float mk[KP];
#pragma unroll
  for (int j = 0; j < KP; ++j) { pk[j] = s[j]; mk[j] = 1.f; }
  if (P.dp.thr) {
    const unsigned long long seed = P.dp.state[0], step = P.dp.state[1];
#pragma unroll
    for (int q = 0; q < KP / 4; ++q) {
      dropout_mult4(P.dp, seed, step, (uint32_t)((size_t)b * n + (valid ? t : 0)), q, mk + q * 4);
      s[q * 4] *= mk[q * 4]; s[q * 4 + 1] *= mk[q * 4 + 1]; s[q * 4 + 2] *= mk[q * 4 + 2]; s[q * 4 + 3] *= mk[q * 4 + 3];
    }
  }                                                              // s = q (= p without dropout) from here on
  float qdef = 0.f;                                              // 1 - sum q (0 without dropout)
  if (P.dp.thr) {
    float qs = 0.f;
#pragma unroll
    for (int j = 0; j < KP; ++j) qs += s[j];
    qdef = 1.f - qs;
  }
  float dcb = 0.f;                                               // sum_c dctl[c] * cb[c]: d/dq_j of the (1 - sum q) cb term is -cb
  float mean = 0.f, rstd = 1.f;
  const bool ln = P.norm == GF_NORM_LAYER;
  if (ln) {
    const float invC = 1.f / (float)C;
    const float md = sum * invC;
    const float var = fmaxf(sumsq * invC - md * md, 0.f);
    mean = md + shift;
    rstd = rsqrtf(var + 1e-8f);
  }

  // ---- sweep 2: dCtl (stored), dp, and the two LayerNorm-backward sums
  float dp[KP];
#pragma unroll
  for (int j = 0; j < KP; ++j) dp[j] = 0.f;
  float a1 = 0.f, a2 = 0.f;                                      // sum_c dxn, sum_c dxn * xn
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    bwd_load_chunk(gs, Gb, t0, n, C, c0);
    for (int i = tid; i < BCH * KP / 4; i += BTM)
      reinterpret_cast<float4*>(&vs[0][0])[i] = __ldg(reinterpret_cast<const float4*>(Vtb + (size_t)c0 * KP) + i);
    if (integ == GF_INT_BOTH)
      for (int i = tid; i < BCH * KP / 4; i += BTM)
        reinterpret_cast<float4*>(&vs2[0][0])[i] = __ldg(reinterpret_cast<const float4*>(Vtb + (size_t)(C + c0) * KP) + i);
    __syncthreads();
    if (integ == GF_INT_BOTH) bwd_store_chunk(dCb, gs, t0, n, Cout, C + c0);      // bias half of dCtl = dOut (before gs is reused)
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      const float go = gs[tid][cc];
      const float xn = (xs[tid][cc] - mean) * rstd;
      float dxn, dc;
      if (integ == GF_INT_ADD) { dxn = go; dc = go; }
      else {
        float g = 0.f;
#pragma unroll
        for (int j4 = 0; j4 < KP; j4 += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&vs[cc][j4]);
          g = fmaf(s[j4], v.x, fmaf(s[j4 + 1], v.y, fmaf(s[j4 + 2], v.z, fmaf(s[j4 + 3], v.w, g))));
        }
        if (P.dp.thr) g = fmaf(qdef, __ldg(P.cb + c0 + cc), g);
        dxn = go * g; dc = go * xn;
      }
      if (P.dp.thr) {
        dcb = fmaf(dc, __ldg(P.cb + c0 + cc), dcb);
        if (integ == GF_INT_BOTH) dcb = fmaf(go, __ldg(P.cb + C + c0 + cc), dcb);
      }
      a1 += dxn; a2 = fmaf(dxn, xn, a2);
#pragma unroll
      for (int j4 = 0; j4 < KP; j4 += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&vs[cc][j4]);
        dp[j4] = fmaf(dc, v.x, dp[j4]); dp[j4 + 1] = fmaf(dc, v.y, dp[j4 + 1]);
        dp[j4 + 2] = fmaf(dc, v.z, dp[j4 + 2]); dp[j4 + 3] = fmaf(dc, v.w, dp[j4 + 3]);
      }
      if (integ == GF_INT_BOTH) {
#pragma unroll
        for (int j4 = 0; j4 < KP; j4 += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&vs2[cc][j4]);
          dp[j4] = fmaf(go, v.x, dp[j4]); dp[j4 + 1] = fmaf(go, v.y, dp[j4 + 1]);
          dp[j4 + 2] = fmaf(go, v.z, dp[j4 + 2]); dp[j4 + 3] = fmaf(go, v.w, dp[j4 + 3]);
        }
      }
      gs[tid][cc] = dc;                                          // own row only: no hazard with other threads
    }
    __syncthreads();
    bwd_store_chunk(dCb, gs, t0, n, Cout, c0);                    // gain half (or the only half) of dCtl
  }
  // ---- softmax backward; dS and P rows
  float pd = 0.f;
#pragma unroll
  for (int j = 0; j < KP; ++j) { dp[j] = (dp[j] - dcb) * mk[j]; pd = fmaf(pk[j], dp[j], pd); }   // d/dq (minus the cb term) -> d/dp through the mask
#pragma unroll
  for (int j = 0; j < KP; ++j) dp[j] = pk[j] * (dp[j] - pd);     // dp = ds from here on
  if (valid) {
    float4* ds4 = reinterpret_cast<float4*>(P.dS + ((size_t)b * n + t) * KP);
    float4* p4 = reinterpret_cast<float4*>(P.P + ((size_t)b * n + t) * KP);
#pragma unroll
    for (int j4 = 0; j4 < KP / 4; ++j4) {
      ds4[j4] = make_float4(dp[j4 * 4], dp[j4 * 4 + 1], dp[j4 * 4 + 2], dp[j4 * 4 + 3]);
      p4[j4] = make_float4(s[j4 * 4], s[j4 * 4 + 1], s[j4 * 4 + 2], s[j4 * 4 + 3]);
    }
  }
  const float m1 = a1 / (float)C, m2 = a2 / (float)C;

  // ---- sweep 3: dX = LayerNorm^T(dxn) + ds.K'
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    bwd_load_chunk(gs, Gb, t0, n, C, c0);
    for (int i = tid; i < KP * BCH / 4; i += BTM) {
      const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
      *reinterpret_cast<float4*>(&ks[j][c4]) = __ldg(reinterpret_cast<const float4*>(Kpb + (size_t)j * C + c0 + c4));
    }
    if (integ != GF_INT_ADD)
      for (int i = tid; i < BCH * KP / 4; i += BTM)
        reinterpret_cast<float4*>(&vs[0][0])[i] = __ldg(reinterpret_cast<const float4*>(Vtb + (size_t)c0 * KP) + i);
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      const float go = gs[tid][cc];
      float dxn = go;
      if (integ != GF_INT_ADD) {
        float g = 0.f;
#pragma unroll
        for (int j4 = 0; j4 < KP; j4 += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&vs[cc][j4]);
          g = fmaf(s[j4], v.x, fmaf(s[j4 + 1], v.y, fmaf(s[j4 + 2], v.z, fmaf(s[j4 + 3], v.w, g))));
        }
        if (P.dp.thr) g = fmaf(qdef, __ldg(P.cb + c0 + cc), g);
        dxn = go * g;
      }
      float dx = dxn;
      if (ln) {
        const float xn = (xs[tid][cc] - mean) * rstd;
        dx = rstd * (dxn - m1 - xn * m2);
      }
#pragma unroll
      for (int j = 0; j < KP; ++j) dx = fmaf(dp[j], ks[j][cc], dx);
      xs[tid][cc] = dx;
    }
    __syncthreads();
    bwd_store_chunk(dXb, xs, t0, n, C, c0);
  }
}

// ---- backward of duplex pass A (the centroid pass: the latents attend to the grid, softmax over the n tokens) ------------------
// Forward (oracle/folded.py centroid_pass):  s[t,j] = x_t.M_j + Rt2[h,j] + Ct2[w,j];  A[t,j] = exp(s[t,j] - lse_j);
//     Xbar_j = sum_t A[t,j] x_t.
// Given dXbar and r_j = dXbar_j.Xbar_j, two sweeps over the 32-channel chunks of a 128-token tile (thread = token, fp32 FMA):
//     sweep 1:  s_j, g_j = x_t.dXbar_j;   then a_j = A[t,j], ds_j = a_j (g_j - r_j)       -> dS [B,n,KP]
//     sweep 2:  dX_t += sum_j a_j dXbar_j + sum_j ds_j M_j                                (in place, on top of stage T's dX)
// The reductions over tokens are the caller's: dM = dS^T X, dRt2 = sum_w dS, dCt2 = sum_h dS.  Reads X once and dX once, writes dX
// and dS: with stage T's backward and the recompute of the statistics, about 16 [B,n,C]-sized passes for a duplex layer.
struct CenBwdParams {
  const float* X; const float* M; const float* Rt; const float* Ct; const float* lse; const float* dXbar; const float* r;
  float* dX; float* dS;
  int n, H, W, C, k;
};

template <int KP>
__global__ void __launch_bounds__(BTM) centroid_bwd_kernel(const CenBwdParams P) {
  __shared__ __align__(16) float xs[BTM][BXS];       // x chunk (sweep 1), dX chunk (sweep 2)
  __shared__ __align__(16) float ms[KP * BCH];       // M chunk: [KP][32] in sweep 1, [32][KP] in sweep 2
  __shared__ __align__(16) float gs[KP * BCH];       // dXbar chunk, same two layouts; zero rows for the padded latents

  const int b = blockIdx.y, t0 = blockIdx.x * BTM, tid = threadIdx.x, t = t0 + tid;
  const int n = P.n, C = P.C, k = P.k;
  const bool valid = t < n;
  const float* Xb = P.X + (size_t)b * n * C;
  const float* Mb = P.M + (size_t)b * KP * C;
  const float* Gb = P.dXbar + (size_t)b * k * C;
  float* dXb = P.dX + (size_t)b * n * C;

  float s[KP], g[KP];
  {
    const int h = valid ? t / P.W : 0, w = valid ? t % P.W : 0;
    const float* rt = P.Rt + ((size_t)b * P.H + h) * KP;
    const float* ct = P.Ct + ((size_t)b * P.W + w) * KP;
#pragma unroll
    for (int j = 0; j < KP; ++j) { s[j] = rt[j] + ct[j]; g[j] = 0.f; }
  }
  // ---- sweep 1: logits of pass A and g = x.dXbar
  {
    float (*mk)[BCH] = reinterpret_cast<float (*)[BCH]>(ms);
    float (*gk)[BCH] = reinterpret_cast<float (*)[BCH]>(gs);
    for (int c0 = 0; c0 < C; c0 += BCH) {
      __syncthreads();
      bwd_load_chunk(xs, Xb, t0, n, C, c0);
      for (int i = tid; i < KP * BCH / 4; i += BTM) {
        const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
        *reinterpret_cast<float4*>(&mk[j][c4]) = __ldg(reinterpret_cast<const float4*>(Mb + (size_t)j * C + c0 + c4));
        *reinterpret_cast<float4*>(&gk[j][c4]) = j < k ? __ldg(reinterpret_cast<const float4*>(Gb + (size_t)j * C + c0 + c4))
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncthreads();
#pragma unroll
      for (int c4 = 0; c4 < BCH; c4 += 4) {
        const float4 x = *reinterpret_cast<const float4*>(&xs[tid][c4]);
#pragma unroll
        for (int j = 0; j < KP; ++j) {
          const float4 mv = *reinterpret_cast<const float4*>(&mk[j][c4]);
          const float4 gv = *reinterpret_cast<const float4*>(&gk[j][c4]);
          s[j] = fmaf(x.x, mv.x, fmaf(x.y, mv.y, fmaf(x.z, mv.z, fmaf(x.w, mv.w, s[j]))));
          g[j] = fmaf(x.x, gv.x, fmaf(x.y, gv.y, fmaf(x.z, gv.z, fmaf(x.w, gv.w, g[j]))));
        }
      }
    }
  }
  // ---- probabilities of pass A (softmax over the tokens, from the merged log-denominators) and the gradient of their logits
#pragma unroll
  for (int j = 0; j < KP; ++j) {
    const float l = __ldg(P.lse + (size_t)b * KP + j);
    const float a = (l == -INFINITY) ? 0.f : expf(s[j] - l);     // padded latents (Rt2 = lse = -inf) stay inert
    const float rj = j < k ? __ldg(P.r + (size_t)b * k + j) : 0.f;
    s[j] = a;                                                    // s = a from here on
    g[j] = a * (g[j] - rj);                                      // g = ds from here on
  }
  if (valid) {
    float4* ds4 = reinterpret_cast<float4*>(P.dS + ((size_t)b * n + t) * KP);
#pragma unroll
    for (int j4 = 0; j4 < KP / 4; ++j4) ds4[j4] = make_float4(g[j4 * 4], g[j4 * 4 + 1], g[j4 * 4 + 2], g[j4 * 4 + 3]);
  }
  // ---- sweep 2: dX += a.dXbar + ds.M
  float (*mt)[KP] = reinterpret_cast<float (*)[KP]>(ms);
  float (*gt)[KP] = reinterpret_cast<float (*)[KP]>(gs);
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
#pragma unroll
    for (int it = 0; it < BTM / 16; ++it) {            // plain loads: this kernel writes dX
      const int row = it * 16 + (tid >> 3), c4 = (tid & 7) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t0 + row < n) v = *reinterpret_cast<const float4*>(dXb + (size_t)(t0 + row) * C + c0 + c4);
      *reinterpret_cast<float4*>(&xs[row][c4]) = v;
    }
    for (int i = tid; i < KP * BCH / 4; i += BTM) {    // transposed: [channel][latent]
      const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
      const float4 mv = __ldg(reinterpret_cast<const float4*>(Mb + (size_t)j * C + c0 + c4));
      const float4 gv = j < k ? __ldg(reinterpret_cast<const float4*>(Gb + (size_t)j * C + c0 + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      mt[c4][j] = mv.x; mt[c4 + 1][j] = mv.y; mt[c4 + 2][j] = mv.z; mt[c4 + 3][j] = mv.w;
      gt[c4][j] = gv.x; gt[c4 + 1][j] = gv.y; gt[c4 + 2][j] = gv.z; gt[c4 + 3][j] = gv.w;
    }
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      float dx = xs[tid][cc];
#pragma unroll
      for (int j4 = 0; j4 < KP; j4 += 4) {
        const float4 mv = *reinterpret_cast<const float4*>(&mt[cc][j4]);
        const float4 gv = *reinterpret_cast<const float4*>(&gt[cc][j4]);
        dx = fmaf(s[j4], gv.x, fmaf(g[j4], mv.x, dx));
        dx = fmaf(s[j4 + 1], gv.y, fmaf(g[j4 + 1], mv.y, dx));
        dx = fmaf(s[j4 + 2], gv.z, fmaf(g[j4 + 2], mv.z, dx));
        dx = fmaf(s[j4 + 3], gv.w, fmaf(g[j4 + 3], mv.w, dx));
      }
      xs[tid][cc] = dx;                                // own row only
    }
    __syncthreads();
    bwd_store_chunk(dXb, xs, t0, n, C, c0);
  }
}

// ---- double backward: the VJP of the stage-T backward (gf_attn_simplex_bwd_vjp) --------------------------------------------------
// The first-order backward above (without dropout) plus its token reductions is one function
//     (X, dOut, Kp, Vt, Rt, Ct) -> (dX, dKp = dS^T X, dVt = dCtl^T P, dRt = sum_w dS, dCt = sum_h dS).
// Given the cotangents U [B,n,C] of dX and Kg [B,KP,C], Vg [B,Cout,KP], Rg [B,H,KP], Cg [B,W,KP] of the tables, each token forms
//     e = cotangent of dS = Kg x + Rg[h] + Cg[w] + K U,   cotangent of P += Vg^T dCtl,   cotangent of dCtl = Vg p (+ Vt f below),
// and the kernel reverses the first-order arithmetic (recomputing s, p, the statistics, ctl, dCtl and dp as token_bwd_kernel does):
//     softmax backward  dS = p (dp - <p,dp>):  f = cotangent of dp = p (e - <p,e>),  cotangent of p += e (dp - <p,dp>) - <p,e> dp
//     dp = Vt^T dCtl:   cotangent of dCtl += Vt f
//     dxn = dOut * g (g = gain of ctl),  dCtl = dOut * xn | dOut:  the product terms in which x and dOut meet
//     dX = LN^T(dxn) + K^T dS:  cotangent of dxn = J U (J = dxn/dx, symmetric), and the LayerNorm Hessian term: with
//         d = dxn, m1 = mean d, m2 = mean d*xn,  U.J d = rstd (U.d - sum U m1 - (U.xn) m2), whose derivative in xn is
//         -rstd (U m2 + (U.xn) d / C) and in rstd is (U.d - sum U m1 - (U.xn) m2); drstd/dx = -rstd^2 xn / C
//     p = softmax(s):   Sg = cotangent of s = p (pbar - <p,pbar>);   x gets K^T Sg + Kg^T dS.
// Outputs per token: Xg [B,n,C] and dOutg [B,n,C] (the cotangents of X and dOut), Sg [B,n,KP], dPg = f [B,n,KP], Ctlg [B,n,Cout]
// (the cotangent of ctl: dOut * (J U) on the gain half, 0 on the bias half and for "add", where ctl does not enter the backward),
// and the first-order dS, P, dCtl again.  The caller reduces Kpg = Sg^T X + dS^T U, Vtg = Ctlg^T P + dCtl^T dPg, Rtg / Ctg = sums of Sg.
// Four sweeps over the 32-channel chunks; Xg doubles as the staging buffer of the cotangent of xn between sweeps 3 and 4 (each
// element is stored and reloaded by the same thread).
//
// With attention dropout (gf_attn_simplex_bwd_vjp_ex, the generator's path-length penalty) the first-order backward is the one of
// token_bwd_kernel: mask mk (0 or 1/(1-p)) from the same Philox draw, q = p mk, qdef = 1 - sum q, the gain of ctl
// g = sum_j q_j Vt_j + qdef cb, dp = Vt^T dCtl, dcbt = dCtl.cb, dS = p (dpp - <p,dpp>) with dpp = mk (dp - dcbt), and P = q; the
// function gains one reduction, dcb = sum_tokens qdef dCtl, whose cotangent cbg [Cout] comes in.  Reversed:
//     f = p (e - <p,e>) as above, fq = mk f = cotangent of dp (dPg),  F = sum_j fq_j = -(cotangent of dcbt)
//     cotangent of dCtl = Vt fq + Vg q - F cb + qdef cbg                (each half with its own rows of Vt, Vg, cb, cbg)
//     cotangent of q    = Vg^T dCtl - dCtl.cbg + Vt_gain^T gbar - gbar.cb   (gbar = cotangent of the gain, as above)
//     cotangent of p    = mk (cotangent of q) + e (dpp - <p,dpp>) - <p,e> dpp,   then Sg = p (pbar - <p,pbar>) as above
//     cotangent of cb   = sum_tokens qdef gbar - F dCtl: the caller forms it from the outputs, (1 - sum P) Ctlg - (sum dPg) dCtl.
// The LayerNorm terms are unchanged.  dS, the direct softmax term of pbar (staged in Sg) and q (in P) leave the registers after
// sweep 2 and dS is reloaded for sweep 4, so the dropout variant holds as many [KP] arrays as the plain one; the mask is one word.
// Without dropout the cotangent cbg is ignored: dcb is 0 for every input (sum p = 1).
struct VjpParams {
  const float* X; const float* dOut; const float* Kp; const float* Vt; const float* Rt; const float* Ct;
  const float* U; const float* Kg; const float* Vg; const float* Rg; const float* Cg;
  float* Xg; float* dOutg; float* Sg; float* dPg; float* Ctlg; float* dS; float* P; float* dCtl;
  int n, H, W, C, Cout, norm, integration;
  DropoutArgs dp;            // attention dropout of the forward call (thr = 0: off)
  const float* cb;           // [Cout] bo (+1 on the gain half), read when dropout is on
  const float* cbg;          // [Cout] cotangent of dcb, read when dropout is on
};

__device__ __forceinline__ void bwd_zero_chunk(float* __restrict__ dst, int t0, int n, int ld, int c0) {
#pragma unroll
  for (int it = 0; it < BTM / 16; ++it) {
    const int row = it * 16 + (threadIdx.x >> 3), c4 = (threadIdx.x & 7) * 4;
    if (t0 + row < n) *reinterpret_cast<float4*>(dst + (size_t)(t0 + row) * ld + c0 + c4) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
__device__ __forceinline__ void bwd_load_own_chunk(float (*dst)[BXS], const float* src, int t0, int n, int ld, int c0) {
#pragma unroll
  for (int it = 0; it < BTM / 16; ++it) {            // plain loads of what the same thread stored with bwd_store_chunk
    const int row = it * 16 + (threadIdx.x >> 3), c4 = (threadIdx.x & 7) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + row < n) v = *reinterpret_cast<const float4*>(src + (size_t)(t0 + row) * ld + c0 + c4);
    *reinterpret_cast<float4*>(&dst[row][c4]) = v;
  }
}
template <int KP>
__device__ __forceinline__ void vjp_load_rows(float (*dst)[BCH], const float* __restrict__ src, int ld, int c0) {   // [KP][32]
  for (int i = threadIdx.x; i < KP * BCH / 4; i += BTM) {
    const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
    *reinterpret_cast<float4*>(&dst[j][c4]) = __ldg(reinterpret_cast<const float4*>(src + (size_t)j * ld + c0 + c4));
  }
}
template <int KP>
__device__ __forceinline__ void vjp_load_cols(float (*dst)[KP], const float* __restrict__ src, int c0) {          // [32][KP]
  for (int i = threadIdx.x; i < BCH * KP / 4; i += BTM)
    reinterpret_cast<float4*>(&dst[0][0])[i] = __ldg(reinterpret_cast<const float4*>(src + (size_t)c0 * KP) + i);
}

template <int KP, bool DROP>
__global__ void __launch_bounds__(BTM) token_bwd_vjp_kernel(const VjpParams P) {
  extern __shared__ __align__(16) uint8_t vsm_raw[];
  float (*xs)[BXS] = reinterpret_cast<float (*)[BXS]>(vsm_raw);
  float (*gs)[BXS] = reinterpret_cast<float (*)[BXS]>(vsm_raw + sizeof(float) * BTM * BXS);
  float (*us)[BXS] = reinterpret_cast<float (*)[BXS]>(vsm_raw + 2 * sizeof(float) * BTM * BXS);
  float* tab = reinterpret_cast<float*>(vsm_raw + 3 * sizeof(float) * BTM * BXS);       // 4 [KP x 32] table chunks
  float (*ka)[BCH] = reinterpret_cast<float (*)[BCH]>(tab);                           // K' chunk [KP][32]
  float (*kb)[BCH] = reinterpret_cast<float (*)[BCH]>(tab + KP * BCH);                // Kg chunk [KP][32]
  float (*va)[KP] = reinterpret_cast<float (*)[KP]>(tab);                             // V^T gain chunk [32][KP]
  float (*vb)[KP] = reinterpret_cast<float (*)[KP]>(tab + KP * BCH);                  // V^T bias chunk
  float (*wa)[KP] = reinterpret_cast<float (*)[KP]>(tab + 2 * KP * BCH);              // Vg gain chunk
  float (*wb)[KP] = reinterpret_cast<float (*)[KP]>(tab + 3 * KP * BCH);              // Vg bias chunk
  float (*cbs)[BCH] = reinterpret_cast<float (*)[BCH]>(tab + 4 * KP * BCH);           // with dropout: cb, cbg chunks (gain, bias)

  const int b = blockIdx.y, t0 = blockIdx.x * BTM, tid = threadIdx.x, t = t0 + tid;
  const int n = P.n, C = P.C, Cout = P.Cout, integ = P.integration;
  const bool valid = t < n, ln = P.norm == GF_NORM_LAYER, add = integ == GF_INT_ADD, both = integ == GF_INT_BOTH;
  const float invC = 1.f / (float)C;
  const float* Xb = P.X + (size_t)b * n * C;
  const float* Gb = P.dOut + (size_t)b * n * C;
  const float* Ub = P.U + (size_t)b * n * C;
  const float* Kpb = P.Kp + (size_t)b * KP * C;
  const float* Kgb = P.Kg + (size_t)b * KP * C;
  const float* Vtb = P.Vt + (size_t)b * Cout * KP;
  const float* Vgb = P.Vg + (size_t)b * Cout * KP;
  float* Xgb = P.Xg + (size_t)b * n * C;
  float* dOgb = P.dOutg + (size_t)b * n * C;
  float* dCb = P.dCtl + (size_t)b * n * Cout;
  float* Cgb = P.Ctlg + (size_t)b * n * Cout;
  const size_t orow = ((size_t)b * n + t) * KP;                   // this token's row of the [B,n,KP] outputs

  float s[KP], e[KP];
  {
    const int h = valid ? t / P.W : 0, w = valid ? t % P.W : 0;
    const float* rt = P.Rt + ((size_t)b * P.H + h) * KP;
    const float* ct = P.Ct + ((size_t)b * P.W + w) * KP;
    const float* rg = P.Rg + ((size_t)b * P.H + h) * KP;
    const float* cg = P.Cg + ((size_t)b * P.W + w) * KP;
#pragma unroll
    for (int j = 0; j < KP; ++j) { s[j] = rt[j] + ct[j]; e[j] = rg[j] + cg[j]; }
  }
  // ---- sweep 1: logits, layer-norm statistics, e = cotangent of dS (Kg x + Rg + Cg + K U)
  float sum = 0.f, sumsq = 0.f, shift = 0.f;
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    bwd_load_chunk(us, Ub, t0, n, C, c0);
    vjp_load_rows<KP>(ka, Kpb, C, c0);
    vjp_load_rows<KP>(kb, Kgb, C, c0);
    __syncthreads();
    if (c0 == 0) shift = xs[tid][0];
#pragma unroll
    for (int c4 = 0; c4 < BCH; c4 += 4) {
      const float4 x = *reinterpret_cast<const float4*>(&xs[tid][c4]);
      const float4 u = *reinterpret_cast<const float4*>(&us[tid][c4]);
      const float d0 = x.x - shift, d1 = x.y - shift, d2 = x.z - shift, d3 = x.w - shift;
      sum += (d0 + d1) + (d2 + d3);
      sumsq = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, sumsq))));
#pragma unroll
      for (int j = 0; j < KP; ++j) {
        const float4 kv = *reinterpret_cast<const float4*>(&ka[j][c4]);
        const float4 gv = *reinterpret_cast<const float4*>(&kb[j][c4]);
        s[j] = fmaf(x.x, kv.x, fmaf(x.y, kv.y, fmaf(x.z, kv.z, fmaf(x.w, kv.w, s[j]))));
        e[j] = fmaf(x.x, gv.x, fmaf(x.y, gv.y, fmaf(x.z, gv.z, fmaf(x.w, gv.w, e[j]))));
        e[j] = fmaf(u.x, kv.x, fmaf(u.y, kv.y, fmaf(u.z, kv.z, fmaf(u.w, kv.w, e[j]))));
      }
    }
  }
  float mx = s[0];
#pragma unroll
  for (int j = 1; j < KP; ++j) mx = fmaxf(mx, s[j]);
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < KP; ++j) { s[j] = expf(s[j] - mx); den += s[j]; }
  const float inv = 1.f / den;
#pragma unroll
  for (int j = 0; j < KP; ++j) s[j] *= inv;                       // s = p from here on
  // attention dropout: the mask of token_bwd_kernel as one bit per latent (multiplier 1/(1-p) where set), q = p mk
  uint32_t keep = 0;
  float q[KP], qdef = 0.f;                                       // q (without dropout: p itself, s is read instead)
  if constexpr (DROP) {
    const unsigned long long seed = P.dp.state[0], step = P.dp.state[1];
#pragma unroll 1                                                 // unrolled, the Philox rounds push s and e out of the registers
    for (int g4 = 0; g4 < KP / 4; ++g4) {
      float m4[4];
      dropout_mult4(P.dp, seed, step, (uint32_t)((size_t)b * n + (valid ? t : 0)), g4, m4);
#pragma unroll
      for (int i = 0; i < 4; ++i) keep |= (m4[i] != 0.f ? 1u : 0u) << (g4 * 4 + i);
    }
    float qs = 0.f;
#pragma unroll
    for (int j = 0; j < KP; ++j) { q[j] = s[j] * (((keep >> j) & 1u) ? P.dp.scale : 0.f); qs += q[j]; }
    qdef = 1.f - qs;
  }
  if constexpr (DROP) {                                          // e is not read in sweep 2: parked in Sg (same thread) meanwhile
    if (valid) {
#pragma unroll
      for (int j4 = 0; j4 < KP; j4 += 4)
        *reinterpret_cast<float4*>(P.Sg + orow + j4) = make_float4(e[j4], e[j4 + 1], e[j4 + 2], e[j4 + 3]);
    }
  }
  float mean = 0.f, rstd = 1.f;
  if (ln) {
    const float md = sum * invC;
    const float var = fmaxf(sumsq * invC - md * md, 0.f);
    mean = md + shift;
    rstd = rsqrtf(var + 1e-8f);
  }

  // ---- sweep 2: dCtl (stored), dp, the LayerNorm-backward sums, pbar = Vg^T dCtl (with dropout: the cotangent of q, from the
  //      reduction dVt = dCtl^T q), the sums of U against 1, xn and dxn; with dropout also dCtl.cb and dCtl.cbg
  float dp[KP], pb[KP];
#pragma unroll
  for (int j = 0; j < KP; ++j) { dp[j] = 0.f; pb[j] = 0.f; }
  float a1 = 0.f, a2 = 0.f, su = 0.f, sux = 0.f, sud = 0.f, dcbt = 0.f, dcg = 0.f;
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    bwd_load_chunk(gs, Gb, t0, n, C, c0);
    bwd_load_chunk(us, Ub, t0, n, C, c0);
    vjp_load_cols<KP>(va, Vtb, c0);
    vjp_load_cols<KP>(wa, Vgb, c0);
    if (both) { vjp_load_cols<KP>(vb, Vtb, C + c0); vjp_load_cols<KP>(wb, Vgb, C + c0); }
    if constexpr (DROP) {
      if (tid < 4 * BCH) {                                       // rows: cb gain, cb bias, cbg gain, cbg bias
        const int r = tid / BCH, c = tid % BCH;
        cbs[r][c] = (r & 1) && !both ? 0.f : __ldg((r < 2 ? P.cb : P.cbg) + ((r & 1) ? C : 0) + c0 + c);
      }
    }
    __syncthreads();
    if (both) bwd_store_chunk(dCb, gs, t0, n, Cout, C + c0);      // bias half of dCtl = dOut (before gs is reused)
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      const float go = gs[tid][cc], u = us[tid][cc];
      const float xn = (xs[tid][cc] - mean) * rstd;
      float dxn, dc;
      if (add) { dxn = go; dc = go; }
      else {
        float g = 0.f;
#pragma unroll
        for (int j = 0; j < KP; ++j) g = fmaf(DROP ? q[j] : s[j], va[cc][j], g);
        if constexpr (DROP) g = fmaf(qdef, cbs[0][cc], g);
        dxn = go * g; dc = go * xn;
      }
      if constexpr (DROP) {
        dcbt = fmaf(dc, cbs[0][cc], dcbt); dcg = fmaf(dc, cbs[2][cc], dcg);
        if (both) { dcbt = fmaf(go, cbs[1][cc], dcbt); dcg = fmaf(go, cbs[3][cc], dcg); }
      }
      a1 += dxn; a2 = fmaf(dxn, xn, a2);
      su += u; sux = fmaf(u, xn, sux); sud = fmaf(u, dxn, sud);
#pragma unroll
      for (int j = 0; j < KP; ++j) { dp[j] = fmaf(dc, va[cc][j], dp[j]); pb[j] = fmaf(dc, wa[cc][j], pb[j]); }
      if (both) {
#pragma unroll
        for (int j = 0; j < KP; ++j) { dp[j] = fmaf(go, vb[cc][j], dp[j]); pb[j] = fmaf(go, wb[cc][j], pb[j]); }
      }
      gs[tid][cc] = dc;                                          // own row only
    }
    __syncthreads();
    bwd_store_chunk(dCb, gs, t0, n, Cout, c0);                    // gain half (or the only half) of dCtl
  }
  // ---- the softmax backward and its reverse: dS (kept in dp), f = cotangent of dp (kept in e), pbar += e (dp - pd) - pe dp
  float fsum = 0.f;                                              // with dropout: F = sum_j fq_j
  if constexpr (!DROP) {
    float pd = 0.f, pe = 0.f;
#pragma unroll
    for (int j = 0; j < KP; ++j) { pd = fmaf(s[j], dp[j], pd); pe = fmaf(s[j], e[j], pe); }
#pragma unroll
    for (int j = 0; j < KP; ++j) {
      const float d = dp[j] - pd;
      pb[j] = fmaf(e[j], d, fmaf(-pe, dp[j], pb[j]));
      dp[j] = s[j] * d;                                          // dp = dS from here on
      e[j] = s[j] * (e[j] - pe);                                 // e = f from here on
    }
    if (valid) {
#pragma unroll
      for (int j4 = 0; j4 < KP / 4; ++j4) {
        reinterpret_cast<float4*>(P.dS + orow)[j4] = make_float4(dp[j4 * 4], dp[j4 * 4 + 1], dp[j4 * 4 + 2], dp[j4 * 4 + 3]);
        reinterpret_cast<float4*>(P.P + orow)[j4] = make_float4(s[j4 * 4], s[j4 * 4 + 1], s[j4 * 4 + 2], s[j4 * 4 + 3]);
        reinterpret_cast<float4*>(P.dPg + orow)[j4] = make_float4(e[j4 * 4], e[j4 * 4 + 1], e[j4 * 4 + 2], e[j4 * 4 + 3]);
      }
    }
  } else {
    // dpp = mk (dp - dcbt) is what the softmax backward saw; its direct term of pbar is staged in Sg (same thread, reloaded after
    // sweep 3), dS goes out and is reloaded for sweep 4, e becomes fq = mk f; pb keeps the cotangent of q
    float pd = 0.f, pe = 0.f;
#pragma unroll
    for (int j4 = 0; j4 < KP; j4 += 4) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (valid) v = *reinterpret_cast<const float4*>(P.Sg + orow + j4);
      e[j4] = v.x; e[j4 + 1] = v.y; e[j4 + 2] = v.z; e[j4 + 3] = v.w;
    }
#pragma unroll
    for (int j = 0; j < KP; ++j) {
      dp[j] = (dp[j] - dcbt) * (((keep >> j) & 1u) ? P.dp.scale : 0.f);
      pd = fmaf(s[j], dp[j], pd); pe = fmaf(s[j], e[j], pe);
    }
#pragma unroll
    for (int j4 = 0; j4 < KP; j4 += 4) {
      float dr[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = j4 + i;
        const float d = dp[j] - pd;
        dr[i] = fmaf(e[j], d, -pe * dp[j]);
        dp[j] = s[j] * d;
        e[j] = (((keep >> j) & 1u) ? P.dp.scale : 0.f) * (s[j] * (e[j] - pe));
        fsum += e[j];
      }
      if (valid) {
        *reinterpret_cast<float4*>(P.Sg + orow + j4) = make_float4(dr[0], dr[1], dr[2], dr[3]);
        *reinterpret_cast<float4*>(P.dS + orow + j4) = make_float4(dp[j4], dp[j4 + 1], dp[j4 + 2], dp[j4 + 3]);
        *reinterpret_cast<float4*>(P.P + orow + j4) = make_float4(q[j4], q[j4 + 1], q[j4 + 2], q[j4 + 3]);
        *reinterpret_cast<float4*>(P.dPg + orow + j4) = make_float4(e[j4], e[j4 + 1], e[j4 + 2], e[j4 + 3]);
      }
    }
  }
  const float m2 = a2 * invC;
  const float hb = ln ? sud - su * (a1 * invC) - sux * m2 : 0.f;     // derivative of U.J dxn in rstd
  const float su_c = su * invC, sux_c = sux * invC;

  // ---- sweep 3: cotangents of dCtl, dxn, ctl, dOut and xn; pbar += Vt_gain ctlbar (with dropout: the cotangent of q, and gcb)
  float t1 = 0.f, t2 = 0.f;                                      // sum_c xnbar, sum_c xnbar * xn
  float gcb = 0.f;                                               // with dropout: gbar.cb
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    bwd_load_chunk(gs, Gb, t0, n, C, c0);
    bwd_load_chunk(us, Ub, t0, n, C, c0);
    vjp_load_cols<KP>(va, Vtb, c0);
    vjp_load_cols<KP>(wa, Vgb, c0);
    if (both) { vjp_load_cols<KP>(vb, Vtb, C + c0); vjp_load_cols<KP>(wb, Vgb, C + c0); }
    if constexpr (DROP) {
      if (tid < 4 * BCH) {                                       // rows: cb gain, cb bias, cbg gain, cbg bias
        const int r = tid / BCH, c = tid % BCH;
        cbs[r][c] = (r & 1) && !both ? 0.f : __ldg((r < 2 ? P.cb : P.cbg) + ((r & 1) ? C : 0) + c0 + c);
      }
    }
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      const float go = gs[tid][cc], u = us[tid][cc];
      const float xn = (xs[tid][cc] - mean) * rstd;
      const float dxnb = ln ? rstd * (u - su_c - xn * sux_c) : u;   // cotangent of dxn = J U
      float g = 0.f, cg = 0.f, cbias = 0.f;
#pragma unroll
      for (int j = 0; j < KP; ++j) {
        const float qj = DROP ? q[j] : s[j];
        if (!add) g = fmaf(qj, va[cc][j], g);
        cg = fmaf(wa[cc][j], qj, fmaf(va[cc][j], e[j], cg));         // cotangent of dCtl (gain half, or the only half)
      }
      if (both) {
#pragma unroll
        for (int j = 0; j < KP; ++j) cbias = fmaf(wb[cc][j], DROP ? q[j] : s[j], fmaf(vb[cc][j], e[j], cbias));
      }
      float cbc = 0.f;
      if constexpr (DROP) {
        cbc = cbs[0][cc];
        if (!add) g = fmaf(qdef, cbc, g);
        cg = fmaf(qdef, cbs[2][cc], fmaf(-fsum, cbc, cg));
        if (both) cbias = fmaf(qdef, cbs[3][cc], fmaf(-fsum, cbs[1][cc], cbias));
      }
      const float dxn = add ? go : go * g;
      float gbar = 0.f, dog, xnb;
      if (add) { dog = dxnb + cg; xnb = 0.f; }
      else {
        gbar = dxnb * go;                                        // cotangent of ctl (gain half)
#pragma unroll
        for (int j = 0; j < KP; ++j) pb[j] = fmaf(gbar, va[cc][j], pb[j]);
        if constexpr (DROP) gcb = fmaf(gbar, cbc, gcb);
        dog = fmaf(dxnb, g, cg * xn) + cbias;
        xnb = cg * go;
      }
      if (ln) {
        xnb = fmaf(-rstd, fmaf(u, m2, sux_c * dxn), xnb);         // the LayerNorm Hessian term
        t1 += xnb; t2 = fmaf(xnb, xn, t2);
      }
      xs[tid][cc] = xnb; gs[tid][cc] = dog; us[tid][cc] = gbar;  // own row only
    }
    __syncthreads();
    bwd_store_chunk(Xgb, xs, t0, n, C, c0);                       // staging: the cotangent of xn
    bwd_store_chunk(dOgb, gs, t0, n, C, c0);
    bwd_store_chunk(Cgb, us, t0, n, Cout, c0);
    if (both) bwd_zero_chunk(Cgb, t0, n, Cout, C + c0);
  }
  if constexpr (DROP) {
    // pbar = mk (cotangent of q) + the staged direct term; dS back for sweep 4
    const float sh = dcg + gcb;
#pragma unroll
    for (int j4 = 0; j4 < KP; j4 += 4) {
      float4 dr = make_float4(0.f, 0.f, 0.f, 0.f), ds = dr;
      if (valid) { dr = *reinterpret_cast<const float4*>(P.Sg + orow + j4); ds = *reinterpret_cast<const float4*>(P.dS + orow + j4); }
      const float drv[4] = {dr.x, dr.y, dr.z, dr.w}, dsv[4] = {ds.x, ds.y, ds.z, ds.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = j4 + i;
        pb[j] = fmaf(((keep >> j) & 1u) ? P.dp.scale : 0.f, pb[j] - sh, drv[i]);
        dp[j] = dsv[i];
      }
    }
  }
  // ---- Sg = p (pbar - <p, pbar>)
  float pp = 0.f;
#pragma unroll
  for (int j = 0; j < KP; ++j) pp = fmaf(s[j], pb[j], pp);
#pragma unroll
  for (int j = 0; j < KP; ++j) pb[j] = s[j] * (pb[j] - pp);      // pb = Sg from here on
  if (valid) {
    float4* sg4 = reinterpret_cast<float4*>(P.Sg + orow);
#pragma unroll
    for (int j4 = 0; j4 < KP / 4; ++j4) sg4[j4] = make_float4(pb[j4 * 4], pb[j4 * 4 + 1], pb[j4 * 4 + 2], pb[j4 * 4 + 3]);
  }
  const float q1 = t1 * invC, q2 = (t2 + rstd * hb) * invC;

  // ---- sweep 4: Xg = J xnbar + (U.J dxn)_rstd drstd/dx + K^T Sg + Kg^T dS
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    bwd_load_chunk(xs, Xb, t0, n, C, c0);
    bwd_load_own_chunk(gs, Xgb, t0, n, C, c0);
    vjp_load_rows<KP>(ka, Kpb, C, c0);
    vjp_load_rows<KP>(kb, Kgb, C, c0);
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      float dx = gs[tid][cc];
      if (ln) {
        const float xn = (xs[tid][cc] - mean) * rstd;
        dx = rstd * (dx - q1 - xn * q2);
      }
#pragma unroll
      for (int j = 0; j < KP; ++j) dx = fmaf(pb[j], ka[j][cc], fmaf(dp[j], kb[j][cc], dx));
      gs[tid][cc] = dx;
    }
    __syncthreads();
    bwd_store_chunk(Xgb, gs, t0, n, C, c0);
  }
}

// ---- double backward: the VJP of the pass-A backward (gf_attn_centroid_bwd_vjp) -------------------------------------------------
// gf_attn_centroid_bwd plus its reductions is the function (X, M, Rt2, Ct2, lse, dXbar, r, dX_in) -> (dX_out, dM = dS^T X, dRt2, dCt2)
// with a = exp(s - lse), g = x.dXbar, dS = a (g - r), dX_out = dX_in + sum_j a_j dXbar_j + sum_j dS_j M_j.  Given the cotangents
// U [B,n,C] of dX_out and Mg [B,KP,C], Rg [B,H,KP], Cg [B,W,KP] of the tables, per token (thread = token, fp32 FMA):
//     e = cotangent of dS = Mg x + Rg[h] + Cg[w] + M U;   abar = U.dXbar + e (g - r);   Gg = cotangent of g = a e;   Sg = a abar
//     Xg = sum_j Sg_j M_j + Gg_j dXbar_j + dS_j Mg_j                                    (a new tensor: nothing is accumulated)
// The kernel writes Xg, Sg, Gg, A and dS [B,n,KP]; the caller reduces dXbarg = A^T U + Gg^T X, Mg' = Sg^T X + dS^T U,
// rg = -sum_t Gg, lseg = -sum_t Sg, Rt2g / Ct2g = sums of Sg; the cotangent of dX_in is U itself.
struct CenVjpParams {
  const float* X; const float* M; const float* Rt; const float* Ct; const float* lse; const float* dXbar; const float* r;
  const float* U; const float* Mg; const float* Rg; const float* Cg;
  float* Xg; float* Sg; float* Gg; float* A; float* dS;
  int n, H, W, C, k;
};

template <int KP>
__global__ void __launch_bounds__(BTM) centroid_bwd_vjp_kernel(const CenVjpParams P) {
  extern __shared__ __align__(16) uint8_t csm_raw[];
  float (*xs)[BXS] = reinterpret_cast<float (*)[BXS]>(csm_raw);
  float (*us)[BXS] = reinterpret_cast<float (*)[BXS]>(csm_raw + sizeof(float) * BTM * BXS);
  float* ms = reinterpret_cast<float*>(csm_raw + 2 * sizeof(float) * BTM * BXS);   // M chunk: [KP][32] in sweep 1, [32][KP] in sweep 2
  float* gs = ms + KP * BCH;                                                         // dXbar chunk (zero rows in the padded latents)
  float* hs = gs + KP * BCH;                                                         // Mg chunk

  const int b = blockIdx.y, t0 = blockIdx.x * BTM, tid = threadIdx.x, t = t0 + tid;
  const int n = P.n, C = P.C, k = P.k;
  const bool valid = t < n;
  const float* Xb = P.X + (size_t)b * n * C;
  const float* Ub = P.U + (size_t)b * n * C;
  const float* Mb = P.M + (size_t)b * KP * C;
  const float* Mgb = P.Mg + (size_t)b * KP * C;
  const float* Gb = P.dXbar + (size_t)b * k * C;
  float* Xgb = P.Xg + (size_t)b * n * C;

  float s[KP], g[KP], e[KP], ug[KP];
  {
    const int h = valid ? t / P.W : 0, w = valid ? t % P.W : 0;
    const float* rt = P.Rt + ((size_t)b * P.H + h) * KP;
    const float* ct = P.Ct + ((size_t)b * P.W + w) * KP;
    const float* rg = P.Rg + ((size_t)b * P.H + h) * KP;
    const float* cg = P.Cg + ((size_t)b * P.W + w) * KP;
#pragma unroll
    for (int j = 0; j < KP; ++j) { s[j] = rt[j] + ct[j]; e[j] = rg[j] + cg[j]; g[j] = 0.f; ug[j] = 0.f; }
  }
  // ---- sweep 1: logits, g = x.dXbar, e (without a), U.dXbar
  {
    float (*mk)[BCH] = reinterpret_cast<float (*)[BCH]>(ms);
    float (*gk)[BCH] = reinterpret_cast<float (*)[BCH]>(gs);
    float (*hk)[BCH] = reinterpret_cast<float (*)[BCH]>(hs);
    for (int c0 = 0; c0 < C; c0 += BCH) {
      __syncthreads();
      bwd_load_chunk(xs, Xb, t0, n, C, c0);
      bwd_load_chunk(us, Ub, t0, n, C, c0);
      for (int i = tid; i < KP * BCH / 4; i += BTM) {
        const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
        *reinterpret_cast<float4*>(&mk[j][c4]) = __ldg(reinterpret_cast<const float4*>(Mb + (size_t)j * C + c0 + c4));
        *reinterpret_cast<float4*>(&hk[j][c4]) = __ldg(reinterpret_cast<const float4*>(Mgb + (size_t)j * C + c0 + c4));
        *reinterpret_cast<float4*>(&gk[j][c4]) = j < k ? __ldg(reinterpret_cast<const float4*>(Gb + (size_t)j * C + c0 + c4))
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncthreads();
#pragma unroll 1                                         // four [KP] accumulators: unrolled, KP = 32 spills
      for (int c4 = 0; c4 < BCH; c4 += 4) {
        const float4 x = *reinterpret_cast<const float4*>(&xs[tid][c4]);
        const float4 u = *reinterpret_cast<const float4*>(&us[tid][c4]);
#pragma unroll
        for (int j = 0; j < KP; ++j) {
          const float4 mv = *reinterpret_cast<const float4*>(&mk[j][c4]);
          const float4 gv = *reinterpret_cast<const float4*>(&gk[j][c4]);
          const float4 hv = *reinterpret_cast<const float4*>(&hk[j][c4]);
          s[j] = fmaf(x.x, mv.x, fmaf(x.y, mv.y, fmaf(x.z, mv.z, fmaf(x.w, mv.w, s[j]))));
          g[j] = fmaf(x.x, gv.x, fmaf(x.y, gv.y, fmaf(x.z, gv.z, fmaf(x.w, gv.w, g[j]))));
          e[j] = fmaf(x.x, hv.x, fmaf(x.y, hv.y, fmaf(x.z, hv.z, fmaf(x.w, hv.w, e[j]))));
          e[j] = fmaf(u.x, mv.x, fmaf(u.y, mv.y, fmaf(u.z, mv.z, fmaf(u.w, mv.w, e[j]))));
          ug[j] = fmaf(u.x, gv.x, fmaf(u.y, gv.y, fmaf(u.z, gv.z, fmaf(u.w, gv.w, ug[j]))));
        }
      }
    }
  }
  // ---- per latent: a, dS, and the cotangents Gg = a e, Sg = a (U.dXbar + e (g - r))
#pragma unroll
  for (int j = 0; j < KP; ++j) {
    const float l = __ldg(P.lse + (size_t)b * KP + j);
    const float a = (l == -INFINITY) ? 0.f : expf(s[j] - l);     // padded latents (Rt2 = lse = -inf) stay inert
    const float rj = j < k ? __ldg(P.r + (size_t)b * k + j) : 0.f;
    const float gr = g[j] - rj;
    s[j] = a;                                                    // s = a
    g[j] = a * gr;                                               // g = dS
    ug[j] = a * fmaf(e[j], gr, ug[j]);                           // ug = Sg
    e[j] = a * e[j];                                             // e = Gg
  }
  if (valid) {
    const size_t o = ((size_t)b * n + t) * KP;
#pragma unroll
    for (int j4 = 0; j4 < KP / 4; ++j4) {
      reinterpret_cast<float4*>(P.A + o)[j4] = make_float4(s[j4 * 4], s[j4 * 4 + 1], s[j4 * 4 + 2], s[j4 * 4 + 3]);
      reinterpret_cast<float4*>(P.dS + o)[j4] = make_float4(g[j4 * 4], g[j4 * 4 + 1], g[j4 * 4 + 2], g[j4 * 4 + 3]);
      reinterpret_cast<float4*>(P.Sg + o)[j4] = make_float4(ug[j4 * 4], ug[j4 * 4 + 1], ug[j4 * 4 + 2], ug[j4 * 4 + 3]);
      reinterpret_cast<float4*>(P.Gg + o)[j4] = make_float4(e[j4 * 4], e[j4 * 4 + 1], e[j4 * 4 + 2], e[j4 * 4 + 3]);
    }
  }
  // ---- sweep 2: Xg = Sg.M + Gg.dXbar + dS.Mg
  float (*mt)[KP] = reinterpret_cast<float (*)[KP]>(ms);
  float (*gt)[KP] = reinterpret_cast<float (*)[KP]>(gs);
  float (*ht)[KP] = reinterpret_cast<float (*)[KP]>(hs);
  for (int c0 = 0; c0 < C; c0 += BCH) {
    __syncthreads();
    for (int i = tid; i < KP * BCH / 4; i += BTM) {    // transposed: [channel][latent]
      const int j = i / (BCH / 4), c4 = (i % (BCH / 4)) * 4;
      const float4 mv = __ldg(reinterpret_cast<const float4*>(Mb + (size_t)j * C + c0 + c4));
      const float4 hv = __ldg(reinterpret_cast<const float4*>(Mgb + (size_t)j * C + c0 + c4));
      const float4 gv = j < k ? __ldg(reinterpret_cast<const float4*>(Gb + (size_t)j * C + c0 + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      mt[c4][j] = mv.x; mt[c4 + 1][j] = mv.y; mt[c4 + 2][j] = mv.z; mt[c4 + 3][j] = mv.w;
      gt[c4][j] = gv.x; gt[c4 + 1][j] = gv.y; gt[c4 + 2][j] = gv.z; gt[c4 + 3][j] = gv.w;
      ht[c4][j] = hv.x; ht[c4 + 1][j] = hv.y; ht[c4 + 2][j] = hv.z; ht[c4 + 3][j] = hv.w;
    }
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < BCH; ++cc) {
      float dx = 0.f;
#pragma unroll
      for (int j = 0; j < KP; ++j) dx = fmaf(ug[j], mt[cc][j], fmaf(e[j], gt[cc][j], fmaf(g[j], ht[cc][j], dx)));
      xs[tid][cc] = dx;                                // own row only
    }
    __syncthreads();
    bwd_store_chunk(Xgb, xs, t0, n, C, c0);
  }
}

// The configurations the pass-A backward serves: a duplex layer with one k-means iteration, norm layer / none, B <= 65535 (grid.y).
static int centroid_bwd_config(const char* who, const gf_attn_desc* desc, const Layout& L) {
  if (!L.duplex) { set_error("%s: desc.duplex is 0 (pass A belongs to duplex layers)", who); return GF_ERR_INVALID; }
  if (desc->duplex != 1) { set_error("%s: one k-means iteration (desc.duplex = 1) is supported, got %d", who, desc->duplex); return GF_ERR_UNSUPPORTED; }
  if (desc->norm != GF_NORM_LAYER && desc->norm != GF_NORM_NONE) { set_error("%s: norm must be layer or none", who); return GF_ERR_UNSUPPORTED; }
  if (L.B > 65535) { set_error("%s: B > 65535", who); return GF_ERR_UNSUPPORTED; }
  return GF_OK;
}

}  // namespace gf

using namespace gf;

extern "C" int gf_attn_simplex_bwd(const gf_attn_desc* desc, const float* X, const float* dOut, const float* Kp, const float* Vt,
                                   const float* Rt, const float* Ct, float* dX, float* dS, float* Pout, float* dCtl, void* stream) {
  return gf_attn_simplex_bwd_ex(desc, X, dOut, Kp, Vt, Rt, Ct, dX, dS, Pout, dCtl, 0.f, 0, nullptr, nullptr, stream);
}

extern "C" int gf_attn_simplex_bwd_ex(const gf_attn_desc* desc, const float* X, const float* dOut, const float* Kp, const float* Vt,
                                      const float* Rt, const float* Ct, float* dX, float* dS, float* Pout, float* dCtl,
                                      float att_dp, uint32_t dp_salt, const unsigned long long* dp_state, const float* cb, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !dOut || !Kp || !Vt || !Rt || !Ct || !dX || !dS || !Pout || !dCtl) { set_error("gf_attn_simplex_bwd: null pointer"); return GF_ERR_INVALID; }
  if (L.duplex) { set_error("gf_attn_simplex_bwd: duplex layers use the composite backward"); return GF_ERR_UNSUPPORTED; }
  if (desc->norm != GF_NORM_LAYER && desc->norm != GF_NORM_NONE) { set_error("gf_attn_simplex_bwd: norm must be layer or none"); return GF_ERR_UNSUPPORTED; }
  if (L.B > 65535) { set_error("gf_attn_simplex_bwd: B > 65535"); return GF_ERR_UNSUPPORTED; }
  if ((rc = check_device())) return rc;
  BwdParams P;
  P.X = X; P.dOut = dOut; P.Kp = Kp; P.Vt = Vt; P.Rt = Rt; P.Ct = Ct; P.dX = dX; P.dS = dS; P.P = Pout; P.dCtl = dCtl;
  P.n = L.n; P.H = L.H; P.W = L.W; P.C = L.C; P.k = L.k; P.Cout = L.Cout; P.norm = desc->norm; P.integration = desc->integration;
  {
    gf_attn_postop post;
    memset(&post, 0, sizeof(post));
    post.att_dp = att_dp; post.dp_salt = dp_salt; post.dp_state = dp_state;
    if ((rc = dropout_args(&post, &P.dp))) return rc;
    if (P.dp.thr && !cb) { set_error("gf_attn_simplex_bwd_ex: attention dropout needs cb (bo, +1 on the gain half)"); return GF_ERR_INVALID; }
    P.cb = cb;
  }
  if (L.heads != 1) { set_error("gf_attn_simplex_bwd: one head (multi-head layers use the composite backward)"); return GF_ERR_UNSUPPORTED; }
  dim3 grid((L.n + BTM - 1) / BTM, L.B);
  const int smem = (int)(2 * sizeof(float) * BTM * BXS + 3 * sizeof(float) * L.KP * BCH);
  cudaStream_t st = (cudaStream_t)stream;
  if (L.KP == 16) {
    GF_CUDA_OK(cudaFuncSetAttribute(token_bwd_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    token_bwd_kernel<16><<<grid, BTM, smem, st>>>(P);
  } else {
    GF_CUDA_OK(cudaFuncSetAttribute(token_bwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    token_bwd_kernel<32><<<grid, BTM, smem, st>>>(P);
  }
  GF_LAUNCH_OK();
  return GF_OK;
}

extern "C" int gf_attn_centroid_stats(const gf_attn_desc* desc, const float* X, const float* M, const float* Rt2, const float* Ct2,
                                      float* Xbar, float* lse, void* ws, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !M || !Rt2 || !Ct2 || !Xbar || !lse || !ws) { set_error("gf_attn_centroid_stats: null pointer"); return GF_ERR_INVALID; }
  if ((rc = centroid_bwd_config("gf_attn_centroid_stats", desc, L))) return rc;
  if ((rc = check_device())) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  float* part = (float*)ws;                            // split-n partials [B][nsplit][KP][C + 4]
  if ((rc = centroid_partials_simt(L, X, M, Rt2, Ct2, part, st))) return rc;
  return centroid_merge_into(L, part, Xbar, lse, st);
}

extern "C" int gf_attn_centroid_bwd(const gf_attn_desc* desc, const float* X, const float* M, const float* Rt2, const float* Ct2,
                                    const float* lse, const float* dXbar, const float* r, float* dX, float* dS, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !M || !Rt2 || !Ct2 || !lse || !dXbar || !r || !dX || !dS) { set_error("gf_attn_centroid_bwd: null pointer"); return GF_ERR_INVALID; }
  if ((rc = centroid_bwd_config("gf_attn_centroid_bwd", desc, L))) return rc;
  if ((rc = check_device())) return rc;
  CenBwdParams P;
  P.X = X; P.M = M; P.Rt = Rt2; P.Ct = Ct2; P.lse = lse; P.dXbar = dXbar; P.r = r; P.dX = dX; P.dS = dS;
  P.n = L.n; P.H = L.H; P.W = L.W; P.C = L.C; P.k = L.k;
  dim3 grid((L.n + BTM - 1) / BTM, L.B);
  cudaStream_t st = (cudaStream_t)stream;
  if (L.KP == 16) centroid_bwd_kernel<16><<<grid, BTM, 0, st>>>(P);
  else centroid_bwd_kernel<32><<<grid, BTM, 0, st>>>(P);
  GF_LAUNCH_OK();
  return GF_OK;
}

extern "C" int gf_attn_simplex_bwd_vjp(const gf_attn_desc* desc, const float* X, const float* dOut, const float* Kp, const float* Vt,
                                       const float* Rt, const float* Ct, const float* U, const float* Kpg, const float* Vtg,
                                       const float* Rtg, const float* Ctg, float* Xg, float* dOutg, float* Sg, float* dPg, float* Ctlg,
                                       float* dS, float* Pout, float* dCtl, void* stream) {
  return gf_attn_simplex_bwd_vjp_ex(desc, X, dOut, Kp, Vt, Rt, Ct, U, Kpg, Vtg, Rtg, Ctg, Xg, dOutg, Sg, dPg, Ctlg, dS, Pout, dCtl,
                                    0.f, 0, nullptr, nullptr, nullptr, stream);
}

template <int KP, bool DROP>
static int launch_token_bwd_vjp(const VjpParams& P, dim3 grid, int smem, cudaStream_t st) {
  GF_CUDA_OK(cudaFuncSetAttribute(token_bwd_vjp_kernel<KP, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  token_bwd_vjp_kernel<KP, DROP><<<grid, BTM, smem, st>>>(P);
  return GF_OK;
}

extern "C" int gf_attn_simplex_bwd_vjp_ex(const gf_attn_desc* desc, const float* X, const float* dOut, const float* Kp, const float* Vt,
                                          const float* Rt, const float* Ct, const float* U, const float* Kpg, const float* Vtg,
                                          const float* Rtg, const float* Ctg, float* Xg, float* dOutg, float* Sg, float* dPg, float* Ctlg,
                                          float* dS, float* Pout, float* dCtl, float att_dp, uint32_t dp_salt,
                                          const unsigned long long* dp_state, const float* cb, const float* cbg, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !dOut || !Kp || !Vt || !Rt || !Ct || !U || !Kpg || !Vtg || !Rtg || !Ctg || !Xg || !dOutg || !Sg || !dPg || !Ctlg || !dS ||
      !Pout || !dCtl) { set_error("gf_attn_simplex_bwd_vjp: null pointer"); return GF_ERR_INVALID; }
  if (L.duplex) { set_error("gf_attn_simplex_bwd_vjp: stage T runs on a simplex descriptor (desc.duplex = 0)"); return GF_ERR_UNSUPPORTED; }
  if (desc->norm != GF_NORM_LAYER && desc->norm != GF_NORM_NONE) { set_error("gf_attn_simplex_bwd_vjp: norm must be layer or none"); return GF_ERR_UNSUPPORTED; }
  if (L.heads != 1) { set_error("gf_attn_simplex_bwd_vjp: one head"); return GF_ERR_UNSUPPORTED; }
  if (L.B > 65535) { set_error("gf_attn_simplex_bwd_vjp: B > 65535"); return GF_ERR_UNSUPPORTED; }
  VjpParams P;
  {
    gf_attn_postop post;
    memset(&post, 0, sizeof(post));
    post.att_dp = att_dp; post.dp_salt = dp_salt; post.dp_state = dp_state;
    if ((rc = dropout_args(&post, &P.dp))) return rc;
    if (P.dp.thr && (!cb || !cbg)) {
      set_error("gf_attn_simplex_bwd_vjp_ex: attention dropout needs cb (bo, +1 on the gain half) and its cotangent cbg"); return GF_ERR_INVALID;
    }
    P.cb = cb; P.cbg = cbg;
  }
  if ((rc = check_device())) return rc;
  P.X = X; P.dOut = dOut; P.Kp = Kp; P.Vt = Vt; P.Rt = Rt; P.Ct = Ct; P.U = U; P.Kg = Kpg; P.Vg = Vtg; P.Rg = Rtg; P.Cg = Ctg;
  P.Xg = Xg; P.dOutg = dOutg; P.Sg = Sg; P.dPg = dPg; P.Ctlg = Ctlg; P.dS = dS; P.P = Pout; P.dCtl = dCtl;
  P.n = L.n; P.H = L.H; P.W = L.W; P.C = L.C; P.Cout = L.Cout; P.norm = desc->norm; P.integration = desc->integration;
  dim3 grid((L.n + BTM - 1) / BTM, L.B);
  const int smem = (int)(3 * sizeof(float) * BTM * BXS + 4 * sizeof(float) * L.KP * BCH + (P.dp.thr ? 4 * sizeof(float) * BCH : 0));
  cudaStream_t st = (cudaStream_t)stream;
  if (L.KP == 16) rc = P.dp.thr ? launch_token_bwd_vjp<16, true>(P, grid, smem, st) : launch_token_bwd_vjp<16, false>(P, grid, smem, st);
  else rc = P.dp.thr ? launch_token_bwd_vjp<32, true>(P, grid, smem, st) : launch_token_bwd_vjp<32, false>(P, grid, smem, st);
  if (rc) return rc;
  GF_LAUNCH_OK();
  return GF_OK;
}

extern "C" int gf_attn_centroid_bwd_vjp(const gf_attn_desc* desc, const float* X, const float* M, const float* Rt2, const float* Ct2,
                                        const float* lse, const float* dXbar, const float* r, const float* U, const float* Mg,
                                        const float* Rt2g, const float* Ct2g, float* Xg, float* Sg, float* Gg, float* A, float* dS,
                                        void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !M || !Rt2 || !Ct2 || !lse || !dXbar || !r || !U || !Mg || !Rt2g || !Ct2g || !Xg || !Sg || !Gg || !A || !dS) {
    set_error("gf_attn_centroid_bwd_vjp: null pointer"); return GF_ERR_INVALID;
  }
  if ((rc = centroid_bwd_config("gf_attn_centroid_bwd_vjp", desc, L))) return rc;
  if ((rc = check_device())) return rc;
  CenVjpParams P;
  P.X = X; P.M = M; P.Rt = Rt2; P.Ct = Ct2; P.lse = lse; P.dXbar = dXbar; P.r = r; P.U = U; P.Mg = Mg; P.Rg = Rt2g; P.Cg = Ct2g;
  P.Xg = Xg; P.Sg = Sg; P.Gg = Gg; P.A = A; P.dS = dS;
  P.n = L.n; P.H = L.H; P.W = L.W; P.C = L.C; P.k = L.k;
  dim3 grid((L.n + BTM - 1) / BTM, L.B);
  const int smem = (int)(2 * sizeof(float) * BTM * BXS + 3 * sizeof(float) * L.KP * BCH);
  cudaStream_t st = (cudaStream_t)stream;
  if (L.KP == 16) {
    GF_CUDA_OK(cudaFuncSetAttribute(centroid_bwd_vjp_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    centroid_bwd_vjp_kernel<16><<<grid, BTM, smem, st>>>(P);
  } else {
    GF_CUDA_OK(cudaFuncSetAttribute(centroid_bwd_vjp_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    centroid_bwd_vjp_kernel<32><<<grid, BTM, smem, st>>>(P);
  }
  GF_LAUNCH_OK();
  return GF_OK;
}
