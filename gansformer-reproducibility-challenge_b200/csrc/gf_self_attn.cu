// gf_self_attn.cu -- dense self-attention over the image grid (img2img, SURVEY A.4 item 18) on the Hopper tensor path.
//
// Per image b and head j (columns [j d, (j+1) d) of the channels-last [B, n, C] tensors):
//     P = softmax_keys(Q_j K_j^T * scale),   O_j = P V_j,   lse = log2 sum_keys 2^(Q_j K_j^T * scale * log2 e)
// streamed over 64-key tiles with an online softmax (FlashAttention-2), so no n x n tensor is ever stored.
//
// wgmma takes 32-bit operands K-major only (gf_tc_cen.cu).  Every product below is therefore arranged so that each operand is read
// along its contraction index: S = Q K^T and dP = dO V^T contract over the head's d channels (natural layout), while O = P V,
// dV = P^T dO, dK = dS^T Q and dQ = dS K contract over tokens and read per-head transposed copies V^T, dO^T, Q^T, K^T ([B, C, n]
// = [B, h, d, n]).  The caller provides those copies.  P, P^T and dS never leave shared memory: they are written from the
// accumulators, rounded to TF32, as the A operand of the next product.
//
//   forward   grid (ceil(n / 128), h, B), 9 warps: warp 8 is the TMA producer (the two query tiles once, then K / V^T tiles of
//             64 keys through a 3-slot mbarrier ring); warpgroups 0 and 1 each own a 64-query tile.
//   backward  delta kernel: Delta = rowsum(dO o O) per head.  dK/dV kernel, grid (n / 64, h, B): one warpgroup per 64-key tile
//             streams the query tiles (Q, dO, Q^T, dO^T, lse, Delta); dQ kernel, grid (n / 64, h, B): one warpgroup per 64-query
//             tile streams the key tiles (K, V, K^T).  Each output is accumulated by one CTA in a fixed order: no atomics, the same
//             bits on every call.
//   double backward (gf_self_attn_bwd_vjp)  a row pass, a query-tile and a key-tile kernel, laid out as the backward (see below).
// Operands are truncated to TF32 by the tensor core (P and dS are rounded to nearest first); accumulation is fp32.
#include <limits.h>
#include <math.h>
#include "gf_common.cuh"
#include "gf_tc_common.cuh"
#include "../../include/gf_ops.h"

namespace gf {
namespace sa {

using namespace tc;

constexpr int T = 64;                         // tokens per tile (queries or keys)
constexpr int CHUNK = T * 128;                // [64 rows x 32 fp32], one SWIZZLE_128B K-major chunk
constexpr int PT_BYTES = 2 * CHUNK;           // a [64 x 64] staged operand (P, P^T, dS^T, dS): two 32-column chunks
constexpr float LOG2E = 1.4426950408889634f;

// byte offset of element (row, k) in a K-major SWIZZLE_128B chunk of 32 columns (the layout TMA writes with that swizzle)
__device__ __forceinline__ uint32_t sw_off(int row, int k) {
  return (uint32_t)(row * 128 + ((((k >> 2) ^ (row & 7))) << 4) + (k & 3) * 4);
}

template <int N>
__device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  static_assert(N == 32 || N == 64, "mma: N must be 32 or 64");
  if constexpr (N == 32) wgmma_ss_n32(d, a, b, acc);
  else wgmma_ss_n64(d, a, b, acc);
}

// d[64 x N] (+)= A[64 x K] . B[N x K]^T, both operands K-major in chunks of 32 columns: A chunk c at a + c * 64 * 128,
// B chunk c at b + c * N * 128.  Issues the MMAs only (the caller fences, commits and waits).
template <int N, int K>
__device__ __forceinline__ void gemm(float* d, uint32_t a, uint32_t b, bool accumulate) {
#pragma unroll
  for (int c = 0; c < K / 32; ++c)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      mma<N>(d, gmma_desc(a + c * CHUNK + kk * 32, 1024, LAYOUT_SW128), gmma_desc(b + c * N * 128 + kk * 32, 1024, LAYOUT_SW128),
             (accumulate || c || kk) ? 1u : 0u);
}

// A [64 x 64] accumulator (row 16 w + g + 8 i, column 8 jb + 2 t + e) -> a K-major operand in shared memory, rounded to TF32
__device__ __forceinline__ void stage_tile(uint8_t* dst, const float* acc, int w, int g, int t) {
#pragma unroll
  for (int jb = 0; jb < 8; ++jb)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = 16 * w + g + 8 * i, col = 8 * jb + 2 * t;
      *reinterpret_cast<float2*>(dst + (col >> 5) * CHUNK + sw_off(row, col & 31)) =
          make_float2(round_tf32_rn(acc[4 * jb + 2 * i]), round_tf32_rn(acc[4 * jb + 2 * i + 1]));
    }
}

// A [64 x D] accumulator * mul -> rows row0 .. row0 + 63, columns col0 .. col0 + D - 1 of a [*, C] row-major tensor
template <int D>
__device__ __forceinline__ void store_tile(float* out, const float* acc, size_t row0, int col0, int C, int w, int g, int t, float mul0,
                                           float mul1) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float mul = i ? mul1 : mul0;
    float* row = out + (row0 + 16 * w + g + 8 * i) * (size_t)C + col0 + 2 * t;
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb)
      *reinterpret_cast<float2*>(row + 8 * jb) = make_float2(acc[4 * jb + 2 * i] * mul, acc[4 * jb + 2 * i + 1] * mul);
  }
}

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) { return p + ((1024u - (smem_u32(p) & 1023u)) & 1023u); }

// ------------------------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int FWD_ST = 3;
constexpr int FWD_THREADS = 288;

struct Bars {
  uint64_t full[4], empty[4], once;
};

template <int D>
struct FwdCfg {
  static constexpr int TILE = T * D * 4;                   // a [64 x D] (or [D x 64]) fp32 tile
  static constexpr int OFF_Q = 0;                          // two query tiles
  static constexpr int OFF_P = OFF_Q + 2 * TILE;           // two staged P tiles
  static constexpr int OFF_RING = OFF_P + 2 * PT_BYTES;    // FWD_ST x (K tile [64 keys x D], V^T tile [D x 64 keys])
  static constexpr int STAGE = 2 * TILE;
  static constexpr int OFF_BARS = OFF_RING + FWD_ST * STAGE;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(Bars) + 1024;
};

template <int D>
__global__ void __launch_bounds__(FWD_THREADS, 1)
self_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmVt, float* __restrict__ O, float* __restrict__ lse, int n, int C, float sl2) {
  using CF = FwdCfg<D>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const uint32_t s_base = smem_u32(smem);
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int j = blockIdx.y, b = blockIdx.z, h = C / D, ntiles = n / T;
  const int qt0 = 2 * blockIdx.x;
  const int nwg = min(2, ntiles - qt0);                    // warpgroups with a query tile (n / 64 may be odd)
  if (threadIdx.x == 256) {
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmVt);
    for (int i = 0; i < FWD_ST; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), nwg); }
    mbar_init(smem_u32(&bars->once), 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // =============================== TMA producer ===============================
    if (lane == 0) {
      const uint32_t qb = smem_u32(&bars->once);
      mbar_expect_tx(qb, (uint32_t)(nwg * CF::TILE));
      for (int wg = 0; wg < nwg; ++wg)
#pragma unroll
        for (int c = 0; c < D / 32; ++c)
          tma_load_2d(s_base + CF::OFF_Q + wg * CF::TILE + c * CHUNK, &tmQ, qb, j * D + c * 32, b * n + (qt0 + wg) * T);
      for (int kt = 0; kt < ntiles; ++kt) {
        const int st = kt % FWD_ST;
        mbar_wait(smem_u32(&bars->empty[st]), ((kt / FWD_ST) & 1) ^ 1);
        const uint32_t fb = smem_u32(&bars->full[st]), dst = s_base + CF::OFF_RING + st * CF::STAGE;
        mbar_expect_tx(fb, (uint32_t)CF::STAGE);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) tma_load_2d(dst + c * CHUNK, &tmK, fb, j * D + c * 32, b * n + kt * T);
#pragma unroll
        for (int c = 0; c < 2; ++c) tma_load_2d(dst + CF::TILE + c * D * 128, &tmVt, fb, kt * T + c * 32, b * C + j * D);
      }
    }
    return;
  }

  // =============================== consumer warpgroups ===============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  if (wg >= nwg) return;
  const uint32_t sQ = s_base + CF::OFF_Q + wg * CF::TILE, sP = s_base + CF::OFF_P + wg * PT_BYTES;
  uint8_t* pP = smem + CF::OFF_P + wg * PT_BYTES;
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // running maximum (log2 units) and this thread's share of the sum
  mbar_wait(smem_u32(&bars->once), 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt % FWD_ST;
    mbar_wait(smem_u32(&bars->full[st]), (kt / FWD_ST) & 1);
    const uint32_t sK = s_base + CF::OFF_RING + st * CF::STAGE, sVt = sK + CF::TILE;
    float s[32];
    wgmma_fence();
    gemm<64, D>(s, sQ, sK, false);                          // S = Q K^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(s);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = m[i];
#pragma unroll
      for (int jb = 0; jb < 8; ++jb) {
        s[4 * jb + 2 * i] = __fmul_rn(s[4 * jb + 2 * i], sl2);            // rounded here and in the backward alike (no FMA)
        s[4 * jb + 2 * i + 1] = __fmul_rn(s[4 * jb + 2 * i + 1], sl2);
        mx = fmaxf(mx, fmaxf(s[4 * jb + 2 * i], s[4 * jb + 2 * i + 1]));
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float alpha = exp2f(m[i] - mx);                 // 0 on the first tile (m = -inf)
      m[i] = mx;
      float sum = 0.f;
#pragma unroll
      for (int jb = 0; jb < 8; ++jb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = exp2f(s[4 * jb + 2 * i + e] - mx);
          s[4 * jb + 2 * i + e] = p;
          sum += p;
        }
      l[i] = l[i] * alpha + sum;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) { o[4 * jb + 2 * i] *= alpha; o[4 * jb + 2 * i + 1] *= alpha; }
    }
    stage_tile(pP, s, w, g, t);                             // the previous tile's P V finished in every warp (barrier below)
    fence_proxy_async();
    named_bar_sync(1 + wg, 128);
    wgmma_fence();
    gemm<D, 64>(o, sP, sVt, true);                          // O += P V
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(o);
    named_bar_sync(1 + wg, 128);
    if (w == 0 && lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
  }
  float inv[2];
  const int qt = qt0 + wg;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float L = l[i];
    L += __shfl_xor_sync(0xffffffffu, L, 1);
    L += __shfl_xor_sync(0xffffffffu, L, 2);
    inv[i] = 1.f / L;
    if (t == 0) lse[((size_t)b * h + j) * n + qt * T + 16 * w + g + 8 * i] = m[i] + log2f(L);
  }
  store_tile<D>(O, o, (size_t)b * n + qt * T, j * D, C, w, g, t, inv[0], inv[1]);
}

// ------------------------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int BWD_THREADS = 160;                            // one consumer warpgroup + the producer warp

// delta[b, j, q] = sum over the head's channels of dO . O, in channel order
__global__ void self_attn_delta_kernel(const float* __restrict__ O, const float* __restrict__ dO, float* __restrict__ delta, int B, int n,
                                       int C, int D) {
  const int h = C / D;
  const long long total = (long long)B * h * n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(idx % n);
    const long long bj = idx / n;
    const int j = (int)(bj % h), b = (int)(bj / h);
    const float4* o = reinterpret_cast<const float4*>(O + ((size_t)b * n + q) * C + j * D);
    const float4* g = reinterpret_cast<const float4*>(dO + ((size_t)b * n + q) * C + j * D);
    float s = 0.f;
    for (int c = 0; c < D / 4; ++c) {
      const float4 a = __ldg(o + c), e = __ldg(g + c);
      s = fmaf(a.x, e.x, s); s = fmaf(a.y, e.y, s); s = fmaf(a.z, e.z, s); s = fmaf(a.w, e.w, s);
    }
    delta[idx] = s;
  }
}

constexpr int KV_ST = 2;

template <int D>
struct KvCfg {
  static constexpr int TILE = T * D * 4;
  static constexpr int OFF_K = 0, OFF_V = TILE;            // this CTA's key tile of K and of V
  static constexpr int OFF_PT = 2 * TILE;                  // staged P^T
  static constexpr int OFF_DST = OFF_PT + PT_BYTES;        // staged dS^T
  static constexpr int OFF_RING = OFF_DST + PT_BYTES;      // KV_ST x (Q, dO [64 q x D], Q^T, dO^T [D x 64 q], lse, Delta [64])
  static constexpr int STAGE_TX = 4 * TILE + 2 * T * 4;
  static constexpr int STAGE = 4 * TILE + 1024;
  static constexpr int OFF_BARS = OFF_RING + KV_ST * STAGE;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(Bars) + 1024;
};

template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
self_attn_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                     const __grid_constant__ CUtensorMap tmdO, const __grid_constant__ CUtensorMap tmQt,
                     const __grid_constant__ CUtensorMap tmdOt, const float* __restrict__ lse, const float* __restrict__ delta,
                     float* __restrict__ dK, float* __restrict__ dV, int n, int C, float sl2, float scale) {
  using CF = KvCfg<D>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const uint32_t s_base = smem_u32(smem);
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int kt = blockIdx.x, j = blockIdx.y, b = blockIdx.z, h = C / D, ntiles = n / T;
  if (threadIdx.x == 128) {
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV); prefetch_tmap(&tmdO); prefetch_tmap(&tmQt); prefetch_tmap(&tmdOt);
    for (int i = 0; i < KV_ST; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 1); }
    mbar_init(smem_u32(&bars->once), 1);
    fence_barrier_init();
  }
  __syncthreads();
  const float* lse_bj = lse + ((size_t)b * h + j) * n;
  const float* delta_bj = delta + ((size_t)b * h + j) * n;

  if (warp == 4) {
    if (lane == 0) {
      const uint32_t kb = smem_u32(&bars->once);
      mbar_expect_tx(kb, (uint32_t)(2 * CF::TILE));
#pragma unroll
      for (int c = 0; c < D / 32; ++c) {
        tma_load_2d(s_base + CF::OFF_K + c * CHUNK, &tmK, kb, j * D + c * 32, b * n + kt * T);
        tma_load_2d(s_base + CF::OFF_V + c * CHUNK, &tmV, kb, j * D + c * 32, b * n + kt * T);
      }
      for (int qt = 0; qt < ntiles; ++qt) {
        const int st = qt % KV_ST;
        mbar_wait(smem_u32(&bars->empty[st]), ((qt / KV_ST) & 1) ^ 1);
        const uint32_t fb = smem_u32(&bars->full[st]), dst = s_base + CF::OFF_RING + st * CF::STAGE;
        mbar_expect_tx(fb, (uint32_t)CF::STAGE_TX);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) {
          tma_load_2d(dst + c * CHUNK, &tmQ, fb, j * D + c * 32, b * n + qt * T);
          tma_load_2d(dst + CF::TILE + c * CHUNK, &tmdO, fb, j * D + c * 32, b * n + qt * T);
        }
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          tma_load_2d(dst + 2 * CF::TILE + c * D * 128, &tmQt, fb, qt * T + c * 32, b * C + j * D);
          tma_load_2d(dst + 3 * CF::TILE + c * D * 128, &tmdOt, fb, qt * T + c * 32, b * C + j * D);
        }
        bulk_load_1d(dst + 4 * CF::TILE, lse_bj + qt * T, T * 4, fb);
        bulk_load_1d(dst + 4 * CF::TILE + T * 4, delta_bj + qt * T, T * 4, fb);
      }
    }
    return;
  }

  const int w = warp, g = lane >> 2, t = lane & 3;
  const uint32_t sK = s_base + CF::OFF_K, sV = s_base + CF::OFF_V, sPt = s_base + CF::OFF_PT, sdSt = s_base + CF::OFF_DST;
  float dk[D / 2], dv[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) { dk[i] = 0.f; dv[i] = 0.f; }
  mbar_wait(smem_u32(&bars->once), 0);
  for (int qt = 0; qt < ntiles; ++qt) {
    const int st = qt % KV_ST;
    mbar_wait(smem_u32(&bars->full[st]), (qt / KV_ST) & 1);
    const uint32_t sQ = s_base + CF::OFF_RING + st * CF::STAGE, sdO = sQ + CF::TILE, sQt = sQ + 2 * CF::TILE, sdOt = sQ + 3 * CF::TILE;
    const float* lse_s = reinterpret_cast<const float*>(smem + CF::OFF_RING + st * CF::STAGE + 4 * CF::TILE);
    const float* delta_s = lse_s + T;
    float s[32], dp[32];
    wgmma_fence();
    gemm<64, D>(s, sK, sQ, false);                          // S^T [key, query] = K Q^T
    gemm<64, D>(dp, sV, sdO, false);                        // dP^T [key, query] = V dO^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(s); fence_regs<32>(dp);
#pragma unroll
    for (int jb = 0; jb < 8; ++jb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int q = 8 * jb + 2 * t + e;
        const float L = lse_s[q], Dl = delta_s[q];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float p = exp2f(__fmul_rn(s[4 * jb + 2 * i + e], sl2) - L);
          dp[4 * jb + 2 * i + e] = p * (dp[4 * jb + 2 * i + e] - Dl);   // dS^T
          s[4 * jb + 2 * i + e] = p;                                       // P^T
        }
      }
    stage_tile(smem + CF::OFF_PT, s, w, g, t);
    stage_tile(smem + CF::OFF_DST, dp, w, g, t);
    fence_proxy_async();
    named_bar_sync(1, 128);
    wgmma_fence();
    gemm<D, 64>(dv, sPt, sdOt, true);                       // dV += P^T dO
    gemm<D, 64>(dk, sdSt, sQt, true);                       // dK += dS^T Q
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(dv); fence_regs<D / 2>(dk);
    named_bar_sync(1, 128);
    if (w == 0 && lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
  }
  store_tile<D>(dK, dk, (size_t)b * n + kt * T, j * D, C, w, g, t, scale, scale);
  store_tile<D>(dV, dv, (size_t)b * n + kt * T, j * D, C, w, g, t, 1.f, 1.f);
}

constexpr int Q_ST = 3;

template <int D>
struct QCfg {
  static constexpr int TILE = T * D * 4;
  static constexpr int OFF_Q = 0, OFF_DO = TILE;           // this CTA's query tile of Q and of dO
  static constexpr int OFF_DS = 2 * TILE;                  // staged dS
  static constexpr int OFF_RING = OFF_DS + PT_BYTES;       // Q_ST x (K, V [64 keys x D], K^T [D x 64 keys])
  static constexpr int STAGE = 3 * TILE;
  static constexpr int OFF_BARS = OFF_RING + Q_ST * STAGE;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(Bars) + 1024;
};

template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
self_attn_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const __grid_constant__ CUtensorMap tmdO, const __grid_constant__ CUtensorMap tmKt, const float* __restrict__ lse,
                    const float* __restrict__ delta, float* __restrict__ dQ, int n, int C, float sl2, float scale) {
  using CF = QCfg<D>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const uint32_t s_base = smem_u32(smem);
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int qt = blockIdx.x, j = blockIdx.y, b = blockIdx.z, h = C / D, ntiles = n / T;
  if (threadIdx.x == 128) {
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV); prefetch_tmap(&tmdO); prefetch_tmap(&tmKt);
    for (int i = 0; i < Q_ST; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 1); }
    mbar_init(smem_u32(&bars->once), 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      const uint32_t qb = smem_u32(&bars->once);
      mbar_expect_tx(qb, (uint32_t)(2 * CF::TILE));
#pragma unroll
      for (int c = 0; c < D / 32; ++c) {
        tma_load_2d(s_base + CF::OFF_Q + c * CHUNK, &tmQ, qb, j * D + c * 32, b * n + qt * T);
        tma_load_2d(s_base + CF::OFF_DO + c * CHUNK, &tmdO, qb, j * D + c * 32, b * n + qt * T);
      }
      for (int kt = 0; kt < ntiles; ++kt) {
        const int st = kt % Q_ST;
        mbar_wait(smem_u32(&bars->empty[st]), ((kt / Q_ST) & 1) ^ 1);
        const uint32_t fb = smem_u32(&bars->full[st]), dst = s_base + CF::OFF_RING + st * CF::STAGE;
        mbar_expect_tx(fb, (uint32_t)CF::STAGE);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) {
          tma_load_2d(dst + c * CHUNK, &tmK, fb, j * D + c * 32, b * n + kt * T);
          tma_load_2d(dst + CF::TILE + c * CHUNK, &tmV, fb, j * D + c * 32, b * n + kt * T);
        }
#pragma unroll
        for (int c = 0; c < 2; ++c) tma_load_2d(dst + 2 * CF::TILE + c * D * 128, &tmKt, fb, kt * T + c * 32, b * C + j * D);
      }
    }
    return;
  }

  const int w = warp, g = lane >> 2, t = lane & 3;
  const uint32_t sQ = s_base + CF::OFF_Q, sdO = s_base + CF::OFF_DO, sdS = s_base + CF::OFF_DS;
  float L[2], Dl[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const size_t r = ((size_t)b * h + j) * n + qt * T + 16 * w + g + 8 * i;
    L[i] = __ldg(lse + r);
    Dl[i] = __ldg(delta + r);
  }
  float dq[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dq[i] = 0.f;
  mbar_wait(smem_u32(&bars->once), 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt % Q_ST;
    mbar_wait(smem_u32(&bars->full[st]), (kt / Q_ST) & 1);
    const uint32_t sK = s_base + CF::OFF_RING + st * CF::STAGE, sV = sK + CF::TILE, sKt = sK + 2 * CF::TILE;
    float s[32], dp[32];
    wgmma_fence();
    gemm<64, D>(s, sQ, sK, false);                          // S = Q K^T
    gemm<64, D>(dp, sdO, sV, false);                        // dP = dO V^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(s); fence_regs<32>(dp);
#pragma unroll
    for (int jb = 0; jb < 8; ++jb)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = exp2f(__fmul_rn(s[4 * jb + 2 * i + e], sl2) - L[i]);
          dp[4 * jb + 2 * i + e] = p * (dp[4 * jb + 2 * i + e] - Dl[i]);
        }
    stage_tile(smem + CF::OFF_DS, dp, w, g, t);
    fence_proxy_async();
    named_bar_sync(1, 128);
    wgmma_fence();
    gemm<D, 64>(dq, sdS, sKt, true);                        // dQ += dS K
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(dq);
    named_bar_sync(1, 128);
    if (w == 0 && lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
  }
  store_tile<D>(dQ, dq, (size_t)b * n + qt * T, j * D, C, w, g, t, scale, scale);
}

// ------------------------------------------------------------------------------------------------------------------------------
// double backward: the vector-Jacobian product of the backward (Q, K, V, dO) -> (dQ, dK, dV) with cotangents A of dQ, Bk of dK
// and Cv of dV.  P is recomputed from lse as above, Delta is the backward's; with s = scale:
//   dS = P o (dP - Delta),   GdS = s [A | Q] [K | Bk]^T,   r = rowsum(P o GdS),   u = rowsum(P o GdS o dP),   PC = P Cv
//   GdP = P o (GdS - r),   GP = GdS o (dP - Delta) - r o dP + dO Cv^T,   t = u - 2 Delta r + dO . PC (= rowsum(P o GP)),
//   GS = P o (GP - t);     gQ = s (dS Bk + GS K),   gK = s (dS^T A + GS^T Q),   gV = GdP^T dO,   gdO = GdP V + PC
//   rows kernel, grid (n / 64, h, B): one warpgroup per 64-query tile streams K, V, Bk, Cv^T over every key and writes r, t and
//               PC (into gdO);
//   q kernel,    grid (n / 64, h, B): one warpgroup per 64-query tile streams K, V, Bk, Cv, K^T, Bk^T, V^T: gQ, and gdO += GdP V;
//   kv kernel,   grid (n / 64, h, B): one warpgroup per 64-key tile streams Q, dO, A, Q^T, A^T, dO^T and lse, Delta, r, t of
//               each query tile: gK, gV.
// The q and kv kernels hold seven and six streamed tiles per stage: at d = 64 their ring has one slot (the shared memory of a
// second is not there), at d = 32 two.
// ------------------------------------------------------------------------------------------------------------------------------
// one pair of staged elements (row, col), (row, col + 1), col even, rounded to TF32
__device__ __forceinline__ void stage_pair(uint8_t* dst, int row, int col, float v0, float v1) {
  *reinterpret_cast<float2*>(dst + (col >> 5) * CHUNK + sw_off(row, col & 31)) = make_float2(round_tf32_rn(v0), round_tf32_rn(v1));
}

// out[row0 .., col0 ..] += a [64 x D] accumulator (the element's previous value added last)
template <int D>
__device__ __forceinline__ void add_tile(float* out, const float* acc, size_t row0, int col0, int C, int w, int g, int t) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float* row = out + (row0 + 16 * w + g + 8 * i) * (size_t)C + col0 + 2 * t;
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb) {
      float2* p = reinterpret_cast<float2*>(row + 8 * jb);
      const float2 o = *p;
      *p = make_float2(acc[4 * jb + 2 * i] + o.x, acc[4 * jb + 2 * i + 1] + o.y);
    }
  }
}

constexpr int VJP_ROW_ST = 2;

template <int D>
struct VjpRowCfg {
  static constexpr int TILE = T * D * 4;
  static constexpr int OFF_Q = 0, OFF_DO = TILE, OFF_A = 2 * TILE;   // this CTA's query tile of Q, dO and A
  static constexpr int OFF_P = 3 * TILE;                            // staged P
  static constexpr int OFF_RING = OFF_P + PT_BYTES;                 // VJP_ROW_ST x (K, V, Bk [64 keys x D], Cv^T [D x 64 keys])
  static constexpr int STAGE = 4 * TILE;
  static constexpr int OFF_BARS = OFF_RING + VJP_ROW_ST * STAGE;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(Bars) + 1024;
};

template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
self_attn_vjp_rows_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                          const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBk,
                          const __grid_constant__ CUtensorMap tmCvt, const float* __restrict__ lse, const float* __restrict__ delta,
                          float* __restrict__ rr, float* __restrict__ tt, float* __restrict__ gdO, int n, int C, float sl2, float scale) {
  using CF = VjpRowCfg<D>;
  constexpr int ST = VJP_ROW_ST;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const uint32_t s_base = smem_u32(smem);
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int qt = blockIdx.x, j = blockIdx.y, b = blockIdx.z, h = C / D, ntiles = n / T;
  if (threadIdx.x == 128) {
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV); prefetch_tmap(&tmdO); prefetch_tmap(&tmA); prefetch_tmap(&tmBk);
    prefetch_tmap(&tmCvt);
    for (int i = 0; i < ST; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 1); }
    mbar_init(smem_u32(&bars->once), 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      const uint32_t qb = smem_u32(&bars->once);
      mbar_expect_tx(qb, (uint32_t)(3 * CF::TILE));
#pragma unroll
      for (int c = 0; c < D / 32; ++c) {
        tma_load_2d(s_base + CF::OFF_Q + c * CHUNK, &tmQ, qb, j * D + c * 32, b * n + qt * T);
        tma_load_2d(s_base + CF::OFF_DO + c * CHUNK, &tmdO, qb, j * D + c * 32, b * n + qt * T);
        tma_load_2d(s_base + CF::OFF_A + c * CHUNK, &tmA, qb, j * D + c * 32, b * n + qt * T);
      }
      for (int kt = 0; kt < ntiles; ++kt) {
        const int st = kt % ST;
        mbar_wait(smem_u32(&bars->empty[st]), ((kt / ST) & 1) ^ 1);
        const uint32_t fb = smem_u32(&bars->full[st]), dst = s_base + CF::OFF_RING + st * CF::STAGE;
        mbar_expect_tx(fb, (uint32_t)CF::STAGE);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) {
          tma_load_2d(dst + c * CHUNK, &tmK, fb, j * D + c * 32, b * n + kt * T);
          tma_load_2d(dst + CF::TILE + c * CHUNK, &tmV, fb, j * D + c * 32, b * n + kt * T);
          tma_load_2d(dst + 2 * CF::TILE + c * CHUNK, &tmBk, fb, j * D + c * 32, b * n + kt * T);
        }
#pragma unroll
        for (int c = 0; c < 2; ++c) tma_load_2d(dst + 3 * CF::TILE + c * D * 128, &tmCvt, fb, kt * T + c * 32, b * C + j * D);
      }
    }
    return;
  }

  const int w = warp, g = lane >> 2, t = lane & 3;
  const uint32_t sQ = s_base + CF::OFF_Q, sdO = s_base + CF::OFF_DO, sA = s_base + CF::OFF_A, sP = s_base + CF::OFF_P;
  float L[2], Dl[2], rs[2] = {0.f, 0.f}, us[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const size_t r = ((size_t)b * h + j) * n + qt * T + 16 * w + g + 8 * i;
    L[i] = __ldg(lse + r);
    Dl[i] = __ldg(delta + r);
  }
  float pc[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) pc[i] = 0.f;
  mbar_wait(smem_u32(&bars->once), 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt % ST;
    mbar_wait(smem_u32(&bars->full[st]), (kt / ST) & 1);
    const uint32_t sK = s_base + CF::OFF_RING + st * CF::STAGE, sV = sK + CF::TILE, sBk = sK + 2 * CF::TILE, sCvt = sK + 3 * CF::TILE;
    float s[32], dp[32], gs[32];
    wgmma_fence();
    gemm<64, D>(s, sQ, sK, false);                          // S = Q K^T
    gemm<64, D>(dp, sdO, sV, false);                        // dP = dO V^T
    gemm<64, D>(gs, sA, sK, false);                         // GdS / s = A K^T + Q Bk^T
    gemm<64, D>(gs, sQ, sBk, true);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(s); fence_regs<32>(dp); fence_regs<32>(gs);
#pragma unroll
    for (int jb = 0; jb < 8; ++jb)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jb + 2 * i + e;
          const float p = exp2f(__fmul_rn(s[x], sl2) - L[i]);
          const float pg = p * (gs[x] * scale);
          rs[i] += pg;
          us[i] += pg * dp[x];
          s[x] = p;
        }
    stage_tile(smem + CF::OFF_P, s, w, g, t);
    fence_proxy_async();
    named_bar_sync(1, 128);
    wgmma_fence();
    gemm<D, 64>(pc, sP, sCvt, true);                        // PC += P Cv
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(pc);
    named_bar_sync(1, 128);
    if (w == 0 && lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
  }
  const uint8_t* pdO = smem + CF::OFF_DO;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = 16 * w + g + 8 * i;
    float dot = 0.f;                                        // dO . PC over this thread's columns, in column order
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * jb + 2 * t + e;
        dot = fmaf(*reinterpret_cast<const float*>(pdO + (col >> 5) * CHUNK + sw_off(row, col & 31)), pc[4 * jb + 2 * i + e], dot);
      }
    float R = rs[i], U = us[i];
    R += __shfl_xor_sync(0xffffffffu, R, 1); R += __shfl_xor_sync(0xffffffffu, R, 2);
    U += __shfl_xor_sync(0xffffffffu, U, 1); U += __shfl_xor_sync(0xffffffffu, U, 2);
    dot += __shfl_xor_sync(0xffffffffu, dot, 1); dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    if (t == 0) {
      const size_t r = ((size_t)b * h + j) * n + qt * T + row;
      rr[r] = R;
      tt[r] = (U - 2.f * Dl[i] * R) + dot;
    }
  }
  store_tile<D>(gdO, pc, (size_t)b * n + qt * T, j * D, C, w, g, t, 1.f, 1.f);
}

template <int D>
struct VjpQCfg {
  static constexpr int ST = D == 32 ? 2 : 1;
  static constexpr int TILE = T * D * 4;
  static constexpr int OFF_Q = 0, OFF_DO = TILE, OFF_A = 2 * TILE;   // this CTA's query tile of Q, dO and A
  static constexpr int OFF_DS = 3 * TILE, OFF_GS = OFF_DS + PT_BYTES, OFF_GDP = OFF_GS + PT_BYTES;   // staged dS, GS, GdP
  static constexpr int OFF_RING = OFF_GDP + PT_BYTES;     // ST x (K, V, Bk, Cv [64 keys x D], K^T, Bk^T, V^T [D x 64 keys])
  static constexpr int STAGE = 7 * TILE;
  static constexpr int OFF_BARS = OFF_RING + ST * STAGE;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(Bars) + 1024;
};

template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
self_attn_vjp_q_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                       const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBk,
                       const __grid_constant__ CUtensorMap tmCv, const __grid_constant__ CUtensorMap tmKt,
                       const __grid_constant__ CUtensorMap tmBkt, const __grid_constant__ CUtensorMap tmVt, const float* __restrict__ lse,
                       const float* __restrict__ delta, const float* __restrict__ rr, const float* __restrict__ tt, float* __restrict__ gQ,
                       float* __restrict__ gdO, int n, int C, float sl2, float scale) {
  using CF = VjpQCfg<D>;
  constexpr int ST = CF::ST;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const uint32_t s_base = smem_u32(smem);
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int qt = blockIdx.x, j = blockIdx.y, b = blockIdx.z, h = C / D, ntiles = n / T;
  if (threadIdx.x == 128) {
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV); prefetch_tmap(&tmdO); prefetch_tmap(&tmA); prefetch_tmap(&tmBk);
    prefetch_tmap(&tmCv); prefetch_tmap(&tmKt); prefetch_tmap(&tmBkt); prefetch_tmap(&tmVt);
    for (int i = 0; i < ST; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 1); }
    mbar_init(smem_u32(&bars->once), 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (lane == 0) {
      const uint32_t qb = smem_u32(&bars->once);
      mbar_expect_tx(qb, (uint32_t)(3 * CF::TILE));
#pragma unroll
      for (int c = 0; c < D / 32; ++c) {
        tma_load_2d(s_base + CF::OFF_Q + c * CHUNK, &tmQ, qb, j * D + c * 32, b * n + qt * T);
        tma_load_2d(s_base + CF::OFF_DO + c * CHUNK, &tmdO, qb, j * D + c * 32, b * n + qt * T);
        tma_load_2d(s_base + CF::OFF_A + c * CHUNK, &tmA, qb, j * D + c * 32, b * n + qt * T);
      }
      for (int kt = 0; kt < ntiles; ++kt) {
        const int st = kt % ST;
        mbar_wait(smem_u32(&bars->empty[st]), ((kt / ST) & 1) ^ 1);
        const uint32_t fb = smem_u32(&bars->full[st]), dst = s_base + CF::OFF_RING + st * CF::STAGE;
        mbar_expect_tx(fb, (uint32_t)CF::STAGE);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) {
          tma_load_2d(dst + c * CHUNK, &tmK, fb, j * D + c * 32, b * n + kt * T);
          tma_load_2d(dst + CF::TILE + c * CHUNK, &tmV, fb, j * D + c * 32, b * n + kt * T);
          tma_load_2d(dst + 2 * CF::TILE + c * CHUNK, &tmBk, fb, j * D + c * 32, b * n + kt * T);
          tma_load_2d(dst + 3 * CF::TILE + c * CHUNK, &tmCv, fb, j * D + c * 32, b * n + kt * T);
        }
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          tma_load_2d(dst + 4 * CF::TILE + c * D * 128, &tmKt, fb, kt * T + c * 32, b * C + j * D);
          tma_load_2d(dst + 5 * CF::TILE + c * D * 128, &tmBkt, fb, kt * T + c * 32, b * C + j * D);
          tma_load_2d(dst + 6 * CF::TILE + c * D * 128, &tmVt, fb, kt * T + c * 32, b * C + j * D);
        }
      }
    }
    return;
  }

  const int w = warp, g = lane >> 2, t = lane & 3;
  const uint32_t sQ = s_base + CF::OFF_Q, sdO = s_base + CF::OFF_DO, sA = s_base + CF::OFF_A;
  const uint32_t sdS = s_base + CF::OFF_DS, sGS = s_base + CF::OFF_GS, sGdP = s_base + CF::OFF_GDP;
  float L[2], Dl[2], R[2], Tr[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const size_t r = ((size_t)b * h + j) * n + qt * T + 16 * w + g + 8 * i;
    L[i] = __ldg(lse + r);
    Dl[i] = __ldg(delta + r);
    R[i] = __ldg(rr + r);
    Tr[i] = __ldg(tt + r);
  }
  float gq[D / 2], gdo[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) { gq[i] = 0.f; gdo[i] = 0.f; }
  mbar_wait(smem_u32(&bars->once), 0);
  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt % ST;
    mbar_wait(smem_u32(&bars->full[st]), (kt / ST) & 1);
    const uint32_t sK = s_base + CF::OFF_RING + st * CF::STAGE, sV = sK + CF::TILE, sBk = sK + 2 * CF::TILE, sCv = sK + 3 * CF::TILE;
    const uint32_t sKt = sK + 4 * CF::TILE, sBkt = sK + 5 * CF::TILE, sVt = sK + 6 * CF::TILE;
    float s[32], dp[32], gp[32];
    wgmma_fence();
    gemm<64, D>(s, sQ, sK, false);                          // S = Q K^T
    gemm<64, D>(dp, sdO, sV, false);                        // dP = dO V^T
    gemm<64, D>(gp, sA, sK, false);                         // GdS / s = A K^T + Q Bk^T
    gemm<64, D>(gp, sQ, sBk, true);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(s); fence_regs<32>(dp); fence_regs<32>(gp);
#pragma unroll
    for (int jb = 0; jb < 8; ++jb)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float gdp[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jb + 2 * i + e;
          const float p = exp2f(__fmul_rn(s[x], sl2) - L[i]);
          const float dpm = dp[x] - Dl[i], gds = gp[x] * scale;
          gdp[e] = p * (gds - R[i]);                                     // GdP
          gp[x] = gds * dpm - R[i] * dp[x];                              // GP, before dO Cv^T
          dp[x] = p * dpm;                                               // dS
          s[x] = p;
        }
        stage_pair(smem + CF::OFF_GDP, 16 * w + g + 8 * i, 8 * jb + 2 * t, gdp[0], gdp[1]);
      }
    stage_tile(smem + CF::OFF_DS, dp, w, g, t);
    wgmma_fence();
    gemm<64, D>(gp, sdO, sCv, true);                        // GP += dO Cv^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(gp);
#pragma unroll
    for (int x = 0; x < 32; ++x) gp[x] = s[x] * (gp[x] - Tr[(x >> 1) & 1]);   // GS
    stage_tile(smem + CF::OFF_GS, gp, w, g, t);
    fence_proxy_async();
    named_bar_sync(1, 128);
    wgmma_fence();
    gemm<D, 64>(gq, sdS, sBkt, true);                       // gQ / s += dS Bk + GS K
    gemm<D, 64>(gq, sGS, sKt, true);
    gemm<D, 64>(gdo, sGdP, sVt, true);                      // gdO += GdP V
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(gq); fence_regs<D / 2>(gdo);
    named_bar_sync(1, 128);
    if (w == 0 && lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
  }
  store_tile<D>(gQ, gq, (size_t)b * n + qt * T, j * D, C, w, g, t, scale, scale);
  add_tile<D>(gdO, gdo, (size_t)b * n + qt * T, j * D, C, w, g, t);
}

template <int D>
struct VjpKvCfg {
  static constexpr int ST = D == 32 ? 2 : 1;
  static constexpr int TILE = T * D * 4;
  static constexpr int OFF_K = 0, OFF_V = TILE, OFF_BK = 2 * TILE, OFF_CV = 3 * TILE;   // this CTA's key tile of K, V, Bk, Cv
  static constexpr int OFF_DST = 4 * TILE, OFF_GST = OFF_DST + PT_BYTES, OFF_GDPT = OFF_GST + PT_BYTES;   // staged dS^T, GS^T, GdP^T
  static constexpr int OFF_RING = OFF_GDPT + PT_BYTES;    // ST x (Q, dO, A [64 q x D], Q^T, A^T, dO^T [D x 64 q], lse, Delta, r, t [64])
  static constexpr int STAGE_TX = 6 * TILE + 4 * T * 4;
  static constexpr int STAGE = 6 * TILE + 1024;
  static constexpr int OFF_BARS = OFF_RING + ST * STAGE;
  static constexpr int SMEM = OFF_BARS + (int)sizeof(Bars) + 1024;
};

template <int D>
__global__ void __launch_bounds__(BWD_THREADS, 1)
self_attn_vjp_kv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                        const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBk,
                        const __grid_constant__ CUtensorMap tmCv, const __grid_constant__ CUtensorMap tmQt,
                        const __grid_constant__ CUtensorMap tmAt, const __grid_constant__ CUtensorMap tmdOt, const float* __restrict__ lse,
                        const float* __restrict__ delta, const float* __restrict__ rr, const float* __restrict__ tt, float* __restrict__ gK,
                        float* __restrict__ gV, int n, int C, float sl2, float scale) {
  using CF = VjpKvCfg<D>;
  constexpr int ST = CF::ST;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  const uint32_t s_base = smem_u32(smem);
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int kt = blockIdx.x, j = blockIdx.y, b = blockIdx.z, h = C / D, ntiles = n / T;
  if (threadIdx.x == 128) {
    prefetch_tmap(&tmQ); prefetch_tmap(&tmK); prefetch_tmap(&tmV); prefetch_tmap(&tmdO); prefetch_tmap(&tmA); prefetch_tmap(&tmBk);
    prefetch_tmap(&tmCv); prefetch_tmap(&tmQt); prefetch_tmap(&tmAt); prefetch_tmap(&tmdOt);
    for (int i = 0; i < ST; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 1); }
    mbar_init(smem_u32(&bars->once), 1);
    fence_barrier_init();
  }
  __syncthreads();
  const size_t bj = ((size_t)b * h + j) * n;

  if (warp == 4) {
    if (lane == 0) {
      const uint32_t kb = smem_u32(&bars->once);
      mbar_expect_tx(kb, (uint32_t)(4 * CF::TILE));
#pragma unroll
      for (int c = 0; c < D / 32; ++c) {
        tma_load_2d(s_base + CF::OFF_K + c * CHUNK, &tmK, kb, j * D + c * 32, b * n + kt * T);
        tma_load_2d(s_base + CF::OFF_V + c * CHUNK, &tmV, kb, j * D + c * 32, b * n + kt * T);
        tma_load_2d(s_base + CF::OFF_BK + c * CHUNK, &tmBk, kb, j * D + c * 32, b * n + kt * T);
        tma_load_2d(s_base + CF::OFF_CV + c * CHUNK, &tmCv, kb, j * D + c * 32, b * n + kt * T);
      }
      for (int qt = 0; qt < ntiles; ++qt) {
        const int st = qt % ST;
        mbar_wait(smem_u32(&bars->empty[st]), ((qt / ST) & 1) ^ 1);
        const uint32_t fb = smem_u32(&bars->full[st]), dst = s_base + CF::OFF_RING + st * CF::STAGE;
        mbar_expect_tx(fb, (uint32_t)CF::STAGE_TX);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) {
          tma_load_2d(dst + c * CHUNK, &tmQ, fb, j * D + c * 32, b * n + qt * T);
          tma_load_2d(dst + CF::TILE + c * CHUNK, &tmdO, fb, j * D + c * 32, b * n + qt * T);
          tma_load_2d(dst + 2 * CF::TILE + c * CHUNK, &tmA, fb, j * D + c * 32, b * n + qt * T);
        }
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          tma_load_2d(dst + 3 * CF::TILE + c * D * 128, &tmQt, fb, qt * T + c * 32, b * C + j * D);
          tma_load_2d(dst + 4 * CF::TILE + c * D * 128, &tmAt, fb, qt * T + c * 32, b * C + j * D);
          tma_load_2d(dst + 5 * CF::TILE + c * D * 128, &tmdOt, fb, qt * T + c * 32, b * C + j * D);
        }
        bulk_load_1d(dst + 6 * CF::TILE, lse + bj + qt * T, T * 4, fb);
        bulk_load_1d(dst + 6 * CF::TILE + T * 4, delta + bj + qt * T, T * 4, fb);
        bulk_load_1d(dst + 6 * CF::TILE + 2 * T * 4, rr + bj + qt * T, T * 4, fb);
        bulk_load_1d(dst + 6 * CF::TILE + 3 * T * 4, tt + bj + qt * T, T * 4, fb);
      }
    }
    return;
  }

  const int w = warp, g = lane >> 2, t = lane & 3;
  const uint32_t sK = s_base + CF::OFF_K, sV = s_base + CF::OFF_V, sBk = s_base + CF::OFF_BK, sCv = s_base + CF::OFF_CV;
  const uint32_t sdSt = s_base + CF::OFF_DST, sGSt = s_base + CF::OFF_GST, sGdPt = s_base + CF::OFF_GDPT;
  float gk[D / 2], gv[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) { gk[i] = 0.f; gv[i] = 0.f; }
  mbar_wait(smem_u32(&bars->once), 0);
  for (int qt = 0; qt < ntiles; ++qt) {
    const int st = qt % ST;
    mbar_wait(smem_u32(&bars->full[st]), (qt / ST) & 1);
    const uint32_t sQ = s_base + CF::OFF_RING + st * CF::STAGE, sdO = sQ + CF::TILE, sA = sQ + 2 * CF::TILE;
    const uint32_t sQt = sQ + 3 * CF::TILE, sAt = sQ + 4 * CF::TILE, sdOt = sQ + 5 * CF::TILE;
    const float* lse_s = reinterpret_cast<const float*>(smem + CF::OFF_RING + st * CF::STAGE + 6 * CF::TILE);
    const float *delta_s = lse_s + T, *r_s = lse_s + 2 * T, *t_s = lse_s + 3 * T;
    float s[32], dp[32], gp[32];
    wgmma_fence();
    gemm<64, D>(s, sK, sQ, false);                          // S^T [key, query] = K Q^T
    gemm<64, D>(dp, sV, sdO, false);                        // dP^T = V dO^T
    gemm<64, D>(gp, sK, sA, false);                         // GdS^T / s = K A^T + Bk Q^T
    gemm<64, D>(gp, sBk, sQ, true);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(s); fence_regs<32>(dp); fence_regs<32>(gp);
#pragma unroll
    for (int jb = 0; jb < 8; ++jb)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float gdp[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int x = 4 * jb + 2 * i + e, q = 8 * jb + 2 * t + e;
          const float Dl = delta_s[q], R = r_s[q];
          const float p = exp2f(__fmul_rn(s[x], sl2) - lse_s[q]);
          const float dpm = dp[x] - Dl, gds = gp[x] * scale;
          gdp[e] = p * (gds - R);                                        // GdP^T
          gp[x] = gds * dpm - R * dp[x];                                 // GP^T, before (dO Cv^T)^T
          dp[x] = p * dpm;                                               // dS^T
          s[x] = p;
        }
        stage_pair(smem + CF::OFF_GDPT, 16 * w + g + 8 * i, 8 * jb + 2 * t, gdp[0], gdp[1]);
      }
    stage_tile(smem + CF::OFF_DST, dp, w, g, t);
    wgmma_fence();
    gemm<64, D>(gp, sCv, sdO, true);                        // GP^T += Cv dO^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(gp);
#pragma unroll
    for (int jb = 0; jb < 8; ++jb)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float Tq = t_s[8 * jb + 2 * t + e];
#pragma unroll
        for (int i = 0; i < 2; ++i) gp[4 * jb + 2 * i + e] = s[4 * jb + 2 * i + e] * (gp[4 * jb + 2 * i + e] - Tq);   // GS^T
      }
    stage_tile(smem + CF::OFF_GST, gp, w, g, t);
    fence_proxy_async();
    named_bar_sync(1, 128);
    wgmma_fence();
    gemm<D, 64>(gk, sdSt, sAt, true);                       // gK / s += dS^T A + GS^T Q
    gemm<D, 64>(gk, sGSt, sQt, true);
    gemm<D, 64>(gv, sGdPt, sdOt, true);                     // gV += GdP^T dO
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<D / 2>(gk); fence_regs<D / 2>(gv);
    named_bar_sync(1, 128);
    if (w == 0 && lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
  }
  store_tile<D>(gK, gk, (size_t)b * n + kt * T, j * D, C, w, g, t, scale, scale);
  store_tile<D>(gV, gv, (size_t)b * n + kt * T, j * D, C, w, g, t, 1.f, 1.f);
}

// ------------------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------------------
static int check_args(const char* name, const void* const* ptrs, const char* const* names, int np, int B, int n, int C, int d, float scale) {
  for (int i = 0; i < np; ++i) {
    if (!ptrs[i]) { set_error("%s: null pointer (%s)", name, names[i]); return GF_ERR_INVALID; }
    if ((uintptr_t)ptrs[i] & 15) { set_error("%s: %s is not 16-byte aligned", name, names[i]); return GF_ERR_INVALID; }
  }
  if (B <= 0 || n <= 0 || C <= 0 || d <= 0) { set_error("%s: bad sizes B=%d n=%d C=%d d=%d", name, B, n, C, d); return GF_ERR_INVALID; }
  if (!(scale > 0.f) || !isfinite(scale)) { set_error("%s: scale must be positive and finite, got %g", name, (double)scale); return GF_ERR_INVALID; }
  if (C % d) { set_error("%s: C=%d is not a multiple of the head size d=%d", name, C, d); return GF_ERR_INVALID; }
  if (d != 32 && d != 64) { set_error("%s: head size d=%d (the kernels serve d = 32 and 64)", name, d); return GF_ERR_UNSUPPORTED; }
  if (n % T) { set_error("%s: n=%d tokens is not a multiple of 64", name, n); return GF_ERR_UNSUPPORTED; }
  if (B > 65535) { set_error("%s: batch B=%d exceeds 65535", name, B); return GF_ERR_UNSUPPORTED; }
  if ((long long)B * n * C > INT_MAX) { set_error("%s: B*n*C = %lld does not fit int32", name, (long long)B * n * C); return GF_ERR_UNSUPPORTED; }
  return GF_OK;
}

// natural [B*n, C] (box 64 tokens x 32 channels) and per-head transposed [B*C, n] (box d channels x 32 tokens) operand maps
static int map_nat(CUtensorMap* m, const float* p, int B, int n, int C) {
  return make_map(m, p, (uint64_t)B * n, (uint64_t)C, T, 32, CU_TENSOR_MAP_SWIZZLE_128B);
}
static int map_tr(CUtensorMap* m, const float* p, int B, int n, int C, int d) {
  return make_map(m, p, (uint64_t)B * C, (uint64_t)n, (uint32_t)d, 32, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <int D>
static int launch_fwd(const float* q, const float* k, const float* vt, float* o, float* lse, int B, int n, int C, float scale, cudaStream_t st) {
  CUtensorMap mq, mk, mvt;
  int rc;
  if ((rc = map_nat(&mq, q, B, n, C)) || (rc = map_nat(&mk, k, B, n, C)) || (rc = map_tr(&mvt, vt, B, n, C, D))) return rc;
  constexpr int smem = FwdCfg<D>::SMEM;
  GF_CUDA_OK(cudaFuncSetAttribute(self_attn_fwd_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const dim3 grid((n / T + 1) / 2, C / D, B);
  self_attn_fwd_kernel<D><<<grid, FWD_THREADS, smem, st>>>(mq, mk, mvt, o, lse, n, C, scale * LOG2E);
  GF_LAUNCH_OK();
  return GF_OK;
}

template <int D>
static int launch_bwd(const float* q, const float* qt, const float* k, const float* kt, const float* v, const float* o, const float* lse,
                      const float* dO, const float* dOt, float* delta, float* dq, float* dk, float* dv, int B, int n, int C, float scale,
                      cudaStream_t st) {
  CUtensorMap mq, mk, mv, mdo, mqt, mkt, mdot;
  int rc;
  if ((rc = map_nat(&mq, q, B, n, C)) || (rc = map_nat(&mk, k, B, n, C)) || (rc = map_nat(&mv, v, B, n, C)) ||
      (rc = map_nat(&mdo, dO, B, n, C)) || (rc = map_tr(&mqt, qt, B, n, C, D)) || (rc = map_tr(&mkt, kt, B, n, C, D)) ||
      (rc = map_tr(&mdot, dOt, B, n, C, D)))
    return rc;
  const long long rows = (long long)B * (C / D) * n;
  const long long blocks = (rows + 255) / 256, cap = (long long)num_sms() * 8;
  self_attn_delta_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, st>>>(o, dO, delta, B, n, C, D);
  GF_LAUNCH_OK();
  const dim3 grid(n / T, C / D, B);
  const float sl2 = scale * LOG2E;
  constexpr int smem_kv = KvCfg<D>::SMEM, smem_q = QCfg<D>::SMEM;
  GF_CUDA_OK(cudaFuncSetAttribute(self_attn_dkv_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_kv));
  self_attn_dkv_kernel<D><<<grid, BWD_THREADS, smem_kv, st>>>(mq, mk, mv, mdo, mqt, mdot, lse, delta, dk, dv, n, C, sl2, scale);
  GF_LAUNCH_OK();
  GF_CUDA_OK(cudaFuncSetAttribute(self_attn_dq_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_q));
  self_attn_dq_kernel<D><<<grid, BWD_THREADS, smem_q, st>>>(mq, mk, mv, mdo, mkt, lse, delta, dq, n, C, sl2, scale);
  GF_LAUNCH_OK();
  return GF_OK;
}

template <int D>
static int launch_bwd_vjp(const float* q, const float* qt, const float* k, const float* kt, const float* v, const float* vt, const float* dO,
                          const float* dOt, const float* lse, const float* delta, const float* a, const float* at, const float* bk,
                          const float* bkt, const float* cv, const float* cvt, float* row_r, float* row_t, float* gq, float* gk, float* gv,
                          float* gdo, int B, int n, int C, float scale, cudaStream_t st) {
  CUtensorMap mq, mk, mv, mdo, ma, mbk, mcv, mqt, mkt, mvt, mdot, mat, mbkt, mcvt;
  int rc;
  if ((rc = map_nat(&mq, q, B, n, C)) || (rc = map_nat(&mk, k, B, n, C)) || (rc = map_nat(&mv, v, B, n, C)) ||
      (rc = map_nat(&mdo, dO, B, n, C)) || (rc = map_nat(&ma, a, B, n, C)) || (rc = map_nat(&mbk, bk, B, n, C)) ||
      (rc = map_nat(&mcv, cv, B, n, C)) || (rc = map_tr(&mqt, qt, B, n, C, D)) || (rc = map_tr(&mkt, kt, B, n, C, D)) ||
      (rc = map_tr(&mvt, vt, B, n, C, D)) || (rc = map_tr(&mdot, dOt, B, n, C, D)) || (rc = map_tr(&mat, at, B, n, C, D)) ||
      (rc = map_tr(&mbkt, bkt, B, n, C, D)) || (rc = map_tr(&mcvt, cvt, B, n, C, D)))
    return rc;
  const dim3 grid(n / T, C / D, B);
  const float sl2 = scale * LOG2E;
  constexpr int smem_r = VjpRowCfg<D>::SMEM, smem_q = VjpQCfg<D>::SMEM, smem_kv = VjpKvCfg<D>::SMEM;
  GF_CUDA_OK(cudaFuncSetAttribute(self_attn_vjp_rows_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_r));
  self_attn_vjp_rows_kernel<D><<<grid, BWD_THREADS, smem_r, st>>>(mq, mk, mv, mdo, ma, mbk, mcvt, lse, delta, row_r, row_t, gdo, n, C,
                                                                  sl2, scale);
  GF_LAUNCH_OK();
  GF_CUDA_OK(cudaFuncSetAttribute(self_attn_vjp_q_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_q));
  self_attn_vjp_q_kernel<D><<<grid, BWD_THREADS, smem_q, st>>>(mq, mk, mv, mdo, ma, mbk, mcv, mkt, mbkt, mvt, lse, delta, row_r, row_t,
                                                               gq, gdo, n, C, sl2, scale);
  GF_LAUNCH_OK();
  GF_CUDA_OK(cudaFuncSetAttribute(self_attn_vjp_kv_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_kv));
  self_attn_vjp_kv_kernel<D><<<grid, BWD_THREADS, smem_kv, st>>>(mq, mk, mv, mdo, ma, mbk, mcv, mqt, mat, mdot, lse, delta, row_r, row_t,
                                                                 gk, gv, n, C, sl2, scale);
  GF_LAUNCH_OK();
  return GF_OK;
}

}  // namespace sa
}  // namespace gf

extern "C" {

int gf_self_attn_fwd(const float* q, const float* k, const float* vt, float* o, float* lse, int B, int n, int C, int d, float scale,
                     void* stream) {
  using namespace gf::sa;
  const void* ptrs[] = {q, k, vt, o, lse};
  const char* names[] = {"q", "k", "vt", "o", "lse"};
  const int rc = check_args("gf_self_attn_fwd", ptrs, names, 5, B, n, C, d, scale);
  if (rc != GF_OK) return rc;
  return d == 32 ? launch_fwd<32>(q, k, vt, o, lse, B, n, C, scale, (cudaStream_t)stream)
                 : launch_fwd<64>(q, k, vt, o, lse, B, n, C, scale, (cudaStream_t)stream);
}

int gf_self_attn_bwd(const float* q, const float* qt, const float* k, const float* kt, const float* v, const float* o, const float* lse,
                     const float* dO, const float* dOt, float* delta, float* dq, float* dk, float* dv, int B, int n, int C, int d,
                     float scale, void* stream) {
  using namespace gf::sa;
  const void* ptrs[] = {q, qt, k, kt, v, o, lse, dO, dOt, delta, dq, dk, dv};
  const char* names[] = {"q", "qt", "k", "kt", "v", "o", "lse", "dO", "dOt", "delta", "dq", "dk", "dv"};
  const int rc = check_args("gf_self_attn_bwd", ptrs, names, 13, B, n, C, d, scale);
  if (rc != GF_OK) return rc;
  return d == 32 ? launch_bwd<32>(q, qt, k, kt, v, o, lse, dO, dOt, delta, dq, dk, dv, B, n, C, scale, (cudaStream_t)stream)
                 : launch_bwd<64>(q, qt, k, kt, v, o, lse, dO, dOt, delta, dq, dk, dv, B, n, C, scale, (cudaStream_t)stream);
}

int gf_self_attn_bwd_vjp(const float* q, const float* qt, const float* k, const float* kt, const float* v, const float* vt, const float* dO,
                         const float* dOt, const float* lse, const float* delta, const float* a, const float* at, const float* bk,
                         const float* bkt, const float* cv, const float* cvt, float* row_r, float* row_t, float* gq, float* gk, float* gv,
                         float* gdo, int B, int n, int C, int d, float scale, void* stream) {
  using namespace gf::sa;
  const void* ptrs[] = {q, qt, k, kt, v, vt, dO, dOt, lse, delta, a, at, bk, bkt, cv, cvt, row_r, row_t, gq, gk, gv, gdo};
  const char* names[] = {"q", "qt", "k", "kt", "v", "vt", "dO", "dOt", "lse", "delta", "a", "at", "bk", "bkt", "cv", "cvt", "row_r", "row_t",
                         "gq", "gk", "gv", "gdo"};
  const int rc = check_args("gf_self_attn_bwd_vjp", ptrs, names, 22, B, n, C, d, scale);
  if (rc != GF_OK) return rc;
  return d == 32 ? launch_bwd_vjp<32>(q, qt, k, kt, v, vt, dO, dOt, lse, delta, a, at, bk, bkt, cv, cvt, row_r, row_t, gq, gk, gv, gdo, B,
                                      n, C, scale, (cudaStream_t)stream)
                 : launch_bwd_vjp<64>(q, qt, k, kt, v, vt, dO, dOt, lse, delta, a, at, bk, bkt, cv, cvt, row_r, row_t, gq, gk, gv, gdo, B,
                                      n, C, scale, (cudaStream_t)stream);
}

}  // extern "C"
