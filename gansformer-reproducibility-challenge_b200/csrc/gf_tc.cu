// gf_tc.cu -- stage T on the Hopper tensor path: TMA-staged tiles, wgmma (tf32) with register accumulators, per-token
// softmax and LayerNorm on CUDA cores, in-place modulation in shared memory, TMA stores.
//
// Replaces, on the reference side (expected src/training/network.py, not in the checkout): the body of
// transformer_layer (Q projection folded into K', QK^T, softmax, PV), integrate and att_norm.  Same algorithm as
// oracle/folded.py per_token(); operands of both contractions are rounded to TF32 by the tensor cores.
//
// One persistent CTA per SM, 9 warps:
//   warp 8       TMA producer: X slabs (128 tokens x 32 channels, 16 KB, SWIZZLE_128B) into a ring; K'/V^T per image
//   warps 0-3,   two consumer warpgroups; warpgroup g owns token rows [64 g, 64 g + 64) of every tile and runs, for them:
//   warps 4-7      GEMM1  S[64,KP] = X[64,C] . K'^T (wgmma, A and B from shared memory), the LayerNorm statistics of the rows
//                  from the same slabs, softmax in registers (a row lives in the 4 lanes of a quad), then per slab
//                  GEMM2  G[64,32] = P[64,KP] . V^T[32 ch,KP]^T (A = P from registers) and the store side
//                  y = LN(x)*g (+b) [+ noise + bias, leaky-ReLU, tRGB, next style] written in place over its half slab, TMA store.
// Single-pass mode (C <= 256): the tile's slabs stay resident from load to store -> X read once, X' written once from HBM.
// Two-pass mode (C = 512, a tile does not fit): slabs stream through the ring once for GEMM1 + statistics and are fetched
// a second time (L2 hits) for the store side.
#include <stdlib.h>
#include "gf_common.cuh"
#include "gf_tc_common.cuh"

namespace gf {

namespace tc {

constexpr int TILE = 128;                 // tokens per tile
constexpr int HALF = 64;                  // rows of one consumer warpgroup (wgmma M)
constexpr int SLAB_CH = 32;               // channels per slab = one 128-byte swizzle span of fp32
constexpr int SLAB_BYTES = TILE * SLAB_CH * 4;
constexpr int MAX_STAGES = 13;
constexpr int NUM_THREADS = 288;          // warps 0-7 two consumer warpgroups, warp 8 producer
constexpr int PRODUCER_WARP = 8;

struct Params {
  float* att; const float* Rt; const float* Ct;
  int n, H, W, k, Cout, B;
  int norm_layer;            // 1 = LayerNorm over C, 0 = none
  int nstages;
  int nwg;                   // consumer warpgroups with rows: 2, or 1 when an image has at most 64 tokens
  long long total_tiles;
  int tiles_per_image;
  int rows;                  // token rows per tile: TILE, or n when an image is smaller than a tile (8x8 grid)
  // fused epilogue (gf_attn_postop)
  const float* pbias; const float* pnoise; const float* pstrength; long long pnoise_bstride; int pact; float pgain; int has_post;
  const float* in_scale; const float* post_scale; int in_ld, post_ld;   // per-(b,c) load-side / store-side scales
  // fused tRGB (1x1 modulated conv of the layer output to 3 planes): rgb_w [B][3][C] per-sample weights, rgb_out [B][3][n]
  const float* rgb_w; const float* rgb_bias; float* rgb_out;
  int heads, seg_shift;      // multi-head: the softmax runs per segment of (1 << seg_shift) table columns (heads * seg == KP)
  // attention dropout (training): the probabilities are dropped / rescaled with the Philox mask the CUDA-core kernels and the
  // backward draw; 1 - sum(q) re-adds the un-droppable constants cb [Cout] (bo, the 1 of 1 + gain) on the store side
  DropoutArgs dp; const float* cb;
};

// ---------------------------------------------------------------------------------------------------------
// shared-memory carve-up (dynamic smem, 1024-byte aligned base)
// ---------------------------------------------------------------------------------------------------------
struct Bars {
  uint64_t slab_full[MAX_STAGES], slab_empty[MAX_STAGES];
  uint64_t kv_full, kv_free;
  uint64_t sc_full[2], sc_free[2];       // per-image load/store-side scale vectors (double-buffered by image parity)
};

template <int KP, int NS, int MODE>
struct Cfg {
  static constexpr int C = NS * SLAB_CH;
  static constexpr int COUT = MODE == GF_INT_BOTH ? 2 * C : C;
  static constexpr int KP_BYTES = KP * C * 4;            // K' : NS chunks of [KP rows x 128 B]
  static constexpr int V_ROW_BYTES = KP * 4;             // V^T row (one channel): KP latents
  static constexpr int V_BYTES = COUT * V_ROW_BYTES;
  static constexpr int PBIAS_BYTES = C * 4;              // post-op bias vector
  static constexpr int OFF_KP = 0;
  static constexpr int OFF_V = OFF_KP + KP_BYTES;
  static constexpr int OFF_PBIAS = OFF_V + V_BYTES;
  // fused tRGB: C <= 256, and C = 512 with k <= 16 (with k = 32 the tables leave the two-pass ring too few stages for the
  // tRGB weights, so that shape keeps the separate tRGB kernel)
  static constexpr bool RGB_OK = NS <= 8 || KP <= 16;
  static constexpr int NVEC = RGB_OK ? 5 : 2;             // per-image vectors: in_scale, post_scale (+ tRGB weights r / g / b)
  static constexpr int SCALE_BYTES = 2 * NVEC * C * 4;   // [image parity][NVEC][C]
  static constexpr int OFF_SCALE = OFF_PBIAS + PBIAS_BYTES;
  static constexpr int OFF_BARS = OFF_SCALE + SCALE_BYTES;
  static constexpr int OFF_RING = (OFF_BARS + (int)sizeof(Bars) + 1023) / 1024 * 1024;
  static constexpr int FIXED_BYTES = OFF_RING;
};

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

template <int KP, int NS, int MODE, bool TWO_PASS>
__global__ void __launch_bounds__(NUM_THREADS, 1)
token_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmO0, const __grid_constant__ CUtensorMap tmO1,
                const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV, const Params P) {
  using CF = Cfg<KP, NS, MODE>;
  constexpr int C = CF::C;
  constexpr int NJ = KP / 8;                           // 8-column blocks of S / k-blocks of GEMM2
  constexpr int SPT = TWO_PASS ? 2 * NS : NS;          // ring slots a tile consumes
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SWIZZLE_128B atoms need 1024 B alignment
  const uint32_t s_base = smem_u32(smem);
  const uint32_t s_kp = s_base + CF::OFF_KP, s_v = s_base + CF::OFF_V, s_ring = s_base + CF::OFF_RING;
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  float* pbias_s = reinterpret_cast<float*>(smem + CF::OFF_PBIAS);
  const float* scale_s = reinterpret_cast<const float*>(smem + CF::OFF_SCALE);
  const uint32_t s_scale = s_base + CF::OFF_SCALE;
  const bool has_rgb = CF::RGB_OK && P.rgb_out != nullptr;
  const bool has_scales = P.in_scale != nullptr || P.post_scale != nullptr || has_rgb;      // any per-image vector to stage
  constexpr int NV = CF::NVEC;
  if (P.has_post)
    for (int i = threadIdx.x; i < C; i += NUM_THREADS) pbias_s[i] = P.pbias ? P.pbias[i] : 0.f;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // provably warp-uniform
  const int lane = threadIdx.x & 31;
  const int nst = P.nstages;

  // contiguous tile range of this CTA
  const long long tile_beg = __shfl_sync(0xffffffffu, (long long)blockIdx.x * P.total_tiles / gridDim.x, 0);
  const long long tile_end = __shfl_sync(0xffffffffu, (long long)(blockIdx.x + 1) * P.total_tiles / gridDim.x, 0);

  if (warp == PRODUCER_WARP && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmO0); prefetch_tmap(&tmO1); prefetch_tmap(&tmK); prefetch_tmap(&tmV);
    for (int i = 0; i < nst; ++i) { mbar_init(smem_u32(&bars->slab_full[i]), 1); mbar_init(smem_u32(&bars->slab_empty[i]), (uint32_t)P.nwg); }
    mbar_init(smem_u32(&bars->kv_full), 1); mbar_init(smem_u32(&bars->kv_free), (uint32_t)P.nwg);
    for (int i = 0; i < 2; ++i) { mbar_init(smem_u32(&bars->sc_full[i]), 1); mbar_init(smem_u32(&bars->sc_free[i]), (uint32_t)P.nwg); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    // =============================== TMA producer ===============================
    if (lane == 0) {
      uint32_t ctr = 0;        // global ring-slot counter of this CTA
      int img_changes = 0;
      int prev_b = -1;
      for (long long tile = tile_beg; tile < tile_end; ++tile) {
        const int b = (int)(tile / P.tiles_per_image);
        if (b != prev_b) {
          if (prev_b >= 0) mbar_wait(smem_u32(&bars->kv_free), (uint32_t)((img_changes - 1) & 1));
          const uint32_t bar = smem_u32(&bars->kv_full);
          mbar_expect_tx(bar, (uint32_t)(CF::KP_BYTES + CF::V_BYTES));
#pragma unroll
          for (int s = 0; s < NS; ++s) tma_load_2d(s_kp + s * (KP * 128), &tmK, bar, s * SLAB_CH, b * KP);
          constexpr int VROWS = CF::COUT < 256 ? CF::COUT : 256;
#pragma unroll
          for (int r0 = 0; r0 < CF::COUT; r0 += VROWS) tma_load_2d(s_v + r0 * CF::V_ROW_BYTES, &tmV, bar, 0, b * CF::COUT + r0);
          if (has_scales) {
            const int par = img_changes & 1;
            mbar_wait(smem_u32(&bars->sc_free[par]), (uint32_t)(((img_changes >> 1) & 1) ^ 1));
            const uint32_t sb = smem_u32(&bars->sc_full[par]);
            mbar_expect_tx(sb, (uint32_t)((P.in_scale ? C * 4 : 0) + (P.post_scale ? C * 4 : 0) + (has_rgb ? 3 * C * 4 : 0)));
            if (P.in_scale) bulk_load_1d(s_scale + par * NV * C * 4, P.in_scale + (size_t)b * P.in_ld, C * 4, sb);
            if (P.post_scale) bulk_load_1d(s_scale + (par * NV + 1) * C * 4, P.post_scale + (size_t)b * P.post_ld, C * 4, sb);
            if (has_rgb) bulk_load_1d(s_scale + (par * NV + 2) * C * 4, P.rgb_w + (size_t)b * 3 * C, 3 * C * 4, sb);   // r | g | b rows are contiguous
          }
          prev_b = b;
          ++img_changes;
        }
        const int row0 = (int)(tile * P.rows);
        for (int ss = 0; ss < SPT; ++ss, ++ctr) {
          const int s = ss % NS;                     // two-pass: the same slabs are fetched again for the store side
          const int stage = (int)(ctr % (uint32_t)nst);
          const uint32_t phase = (ctr / (uint32_t)nst) & 1u;
          mbar_wait(smem_u32(&bars->slab_empty[stage]), phase ^ 1u);
          const uint32_t bar = smem_u32(&bars->slab_full[stage]);
          mbar_expect_tx(bar, (uint32_t)P.rows * 128u);     // short tile: rows >= P.rows of the slab stay stale (never stored)
          tma_load_2d(s_ring + stage * SLAB_BYTES, &tmX, bar, s * SLAB_CH, row0);
        }
      }
    }
    return;
  }

  // =============================== consumer warpgroups ===============================
  const int wg = warp >> 2;
  if (wg >= P.nwg) return;                         // short images: the second warpgroup has no rows
  const int gid = lane >> 2, qd = lane & 3;        // quad (row pair) and lane inside it
  const int rA = wg * HALF + (warp & 3) * 16 + gid;  // tile rows of this thread: rA and rA + 8
  const bool leader = (warp & 3) == 0 && lane == 0;
  const CUtensorMap* tmO = wg ? &tmO1 : &tmO0;
  const uint32_t half_off = (uint32_t)(wg * HALF * 128);
  const float act_a = P.pact == 1 ? 0.6f * P.pgain : P.pgain, act_b = P.pact == 1 ? 0.4f * P.pgain : 0.f;
  const bool has_noise = P.has_post && P.pnoise != nullptr;
  const float pstr = (has_noise && P.pstrength) ? __ldg(P.pstrength) : 1.f;
  const float rgb_b0 = (has_rgb && P.rgb_bias) ? __ldg(P.rgb_bias) : 0.f, rgb_b1 = (has_rgb && P.rgb_bias) ? __ldg(P.rgb_bias + 1) : 0.f,
              rgb_b2 = (has_rgb && P.rgb_bias) ? __ldg(P.rgb_bias + 2) : 0.f;
  const bool dp_on = P.dp.thr != 0;
  const uint64_t dKp = gmma_desc(s_kp, 1024, LAYOUT_SW128);
  const uint64_t dV = gmma_desc(s_v, 8 * CF::V_ROW_BYTES, KP == 32 ? LAYOUT_SW128 : LAYOUT_SW64);

  int stage = 0; uint32_t ph = 0;                  // ring walker: every fill, in slot order
  int img_changes = 0, imgc = 0;
  int b = (int)(tile_beg / P.tiles_per_image);
  int t_in_img = (int)(tile_beg - (long long)b * P.tiles_per_image);
  bool new_img = true;
  int pending_stage = -1;                          // leader: slab whose store may still be reading shared memory
  for (long long tile = tile_beg; tile < tile_end; ++tile) {
    const int bimg = b, t_cur = t_in_img;
    const bool img_first = t_in_img == 0 || tile == tile_beg;
    if (++t_in_img == P.tiles_per_image) { t_in_img = 0; ++b; }
    const bool img_last = t_in_img == 0;
    const int spar = imgc & 1;
    if (new_img) { mbar_wait(smem_u32(&bars->kv_full), (uint32_t)(img_changes & 1)); ++img_changes; new_img = false; }
    if (has_scales && img_first) mbar_wait(smem_u32(&bars->sc_full[spar]), (uint32_t)((imgc >> 1) & 1));
    const float* isc_img = P.in_scale ? scale_s + spar * NV * C : nullptr;

    // positional logits of this thread's rows and columns (issued before the slab loop: their latency hides under it)
    int tok[2];
    float pos[NJ][4];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      tok[i] = min(t_cur * P.rows + rA + 8 * i, P.n - 1);
      const int h = tok[i] / P.W, w = tok[i] - h * P.W;
      const float* rt = P.Rt + ((size_t)bimg * P.H + h) * KP + 2 * qd;
      const float* ct = P.Ct + ((size_t)bimg * P.W + w) * KP + 2 * qd;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float2 r = __ldg(reinterpret_cast<const float2*>(rt + 8 * j)), c = __ldg(reinterpret_cast<const float2*>(ct + 8 * j));
        pos[j][2 * i] = r.x + c.x; pos[j][2 * i + 1] = r.y + c.y;
      }
    }

    // ---- GEMM1 S = X . K'^T and the LayerNorm statistics (shifted sums; a row's channels are split over its quad)
    const int stage0 = stage; const uint32_t ph0 = ph;
    float sacc[KP / 2];
    float sh[2] = {0.f, 0.f}, sum[2] = {0.f, 0.f}, sumsq[2] = {0.f, 0.f};
#pragma unroll 1
    for (int s = 0; s < NS; ++s) {
      mbar_wait(smem_u32(&bars->slab_full[stage]), ph);
      const uint32_t sa = s_ring + stage * SLAB_BYTES + half_off;
      const uint64_t da = gmma_desc(sa, 1024, LAYOUT_SW128);
      const uint64_t db = dKp + (uint64_t)(s * ((KP * 128) >> 4));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if constexpr (KP == 32) wgmma_ss_n32(sacc, da + kk * 2, db + kk * 2, (s | kk) ? 1u : 0u);
        else wgmma_ss_n16(sacc, da + kk * 2, db + kk * 2, (s | kk) ? 1u : 0u);
      }
      wgmma_commit();
      if (P.norm_layer) {
        const float4* isc = isc_img ? reinterpret_cast<const float4*>(isc_img + s * SLAB_CH) : nullptr;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = rA + 8 * i;
          const uint8_t* slab = smem + CF::OFF_RING + stage * SLAB_BYTES + r * 128;
          if (s == 0) { sh[i] = reinterpret_cast<const float*>(slab + ((0 ^ (r & 7)) << 4))[0]; if (isc) sh[i] *= isc[0].x; }
#pragma unroll
          for (int cc = 0; cc < 2; ++cc) {
            const int c = 2 * qd + cc;
            float4 x = *reinterpret_cast<const float4*>(slab + ((c ^ (r & 7)) << 4));
            if (isc) { const float4 d = isc[c]; x.x *= d.x; x.y *= d.y; x.z *= d.z; x.w *= d.w; }
            const float d0 = x.x - sh[i], d1 = x.y - sh[i], d2 = x.z - sh[i], d3 = x.w - sh[i];
            sum[i] += (d0 + d1) + (d2 + d3);
            sumsq[i] = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, sumsq[i]))));
          }
        }
      }
      if (TWO_PASS) {                              // the pass-1 slab may be recycled once this warpgroup's MMAs read it
        wgmma_wait<0>();
        named_bar_sync(1 + wg, 128);
        if (leader) mbar_arrive(smem_u32(&bars->slab_empty[stage]));
      }
      if (++stage == nst) { stage = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    fence_regs<KP / 2>(sacc);
    float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f};
    if (P.norm_layer) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float md = quad_sum(sum[i]) * (1.f / (float)C);
        const float var = fmaxf(quad_sum(sumsq[i]) * (1.f / (float)C) - md * md, 0.f);
        mean[i] = sh[i] + md;
        rstd[i] = rsqrtf(var + 1e-8f);
      }
    }

    // ---- softmax over the latents (logits in log2 units: gf_fold.cu folds log2 e into K' / Rt / Ct).  sacc[4j + 2i + e] is
    // row rA + 8i, column 8j + 2 qd + e.
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) sacc[4 * j + e] += pos[j][e];
    float qdef[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = rA + 8 * i;
      float* a = (P.att && r < P.rows) ? P.att + ((size_t)bimg * P.n + tok[i]) * P.k : nullptr;
      if (P.heads == 1) {
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < NJ; ++j) mx = fmaxf(mx, fmaxf(sacc[4 * j + 2 * i], sacc[4 * j + 2 * i + 1]));
        mx = quad_max(mx);
        float den = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) { const float v = exp2f(sacc[4 * j + 2 * i + e] - mx); sacc[4 * j + 2 * i + e] = v; den += v; }
        const float inv = 1.f / quad_sum(den);
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            sacc[4 * j + 2 * i + e] *= inv;
            const int c = 8 * j + 2 * qd + e;
            if (a && c < P.k) a[c] = sacc[4 * j + 2 * i + e];
          }
      } else {
        // multi-head: one softmax per segment of table columns (head h owns columns [h * seg, (h + 1) * seg)); segments are
        // multiples of 8 columns, so a thread's column 8j + 2 qd + e lies in segment j >> (seg_shift - 3)
        const int jsh = P.seg_shift - 3;
        // per-block partials, then combined over the blocks of the same segment (compile-time indices: stays in registers)
        float bm[NJ], mx[NJ], bs[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) bm[j] = quad_max(fmaxf(sacc[4 * j + 2 * i], sacc[4 * j + 2 * i + 1]));
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          mx[j] = -INFINITY;
#pragma unroll
          for (int j2 = 0; j2 < NJ; ++j2) if ((j2 >> jsh) == (j >> jsh)) mx[j] = fmaxf(mx[j], bm[j2]);
        }
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          bs[j] = 0.f;
#pragma unroll
          for (int e = 0; e < 2; ++e) { const float v = exp2f(sacc[4 * j + 2 * i + e] - mx[j]); sacc[4 * j + 2 * i + e] = v; bs[j] += v; }
          bs[j] = quad_sum(bs[j]);
        }
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          float den = 0.f;
#pragma unroll
          for (int j2 = 0; j2 < NJ; ++j2) if ((j2 >> jsh) == (j >> jsh)) den += bs[j2];
          const float inv = 1.f / den;
#pragma unroll
          for (int e = 0; e < 2; ++e) sacc[4 * j + 2 * i + e] *= inv;
        }
        if (a) {                                   // attention map = mean over the heads
          const int segj = 1 << jsh;
          const float ih = 1.f / (float)P.heads;
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + 2 * qd + e;
              if (j < segj && c < P.k) {
                float m = 0.f;
#pragma unroll
                for (int j2 = 0; j2 < NJ; ++j2) if ((j2 & (segj - 1)) == j) m += sacc[4 * j2 + 2 * i + e];
                a[c] = m * ih;
              }
            }
        }
      }
      if (dp_on) {
        // attention dropout on the probabilities (the map above is pre-dropout): same Philox stream as token_simt_kernel / the backward
        const unsigned long long seed = P.dp.state[0], step = P.dp.state[1];
        const uint32_t gtok = (uint32_t)((size_t)bimg * P.n + tok[i]);
        float qs = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          float mk[4];
          dropout_mult4(P.dp, seed, step, gtok, 2 * j + (qd >> 1), mk);
#pragma unroll
          for (int e = 0; e < 2; ++e) { sacc[4 * j + 2 * i + e] *= mk[2 * (qd & 1) + e]; qs += sacc[4 * j + 2 * i + e]; }
        }
        qdef[i] = 1.f - quad_sum(qs);
      }
    }
    // P rounded to the nearest TF32 (the tensor core's operand truncation is then exact, see gf_fold.cu: round_tf32), then
    // rearranged from the accumulator layout (columns 2 qd, 2 qd + 1) into the A-operand layout (columns qd, qd + 4)
    uint32_t pa[NJ][4];
    {
      const int srcA = (lane & ~3) | (qd >> 1), srcB = srcA + 2;
      const bool odd = qd & 1;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float v0 = cvt_tf32(sacc[4 * j + 2 * i]), v1 = cvt_tf32(sacc[4 * j + 2 * i + 1]);
          const float a0 = __shfl_sync(0xffffffffu, v0, srcA), a1 = __shfl_sync(0xffffffffu, v1, srcA);
          const float b0 = __shfl_sync(0xffffffffu, v0, srcB), b1 = __shfl_sync(0xffffffffu, v1, srcB);
          pa[j][i] = __float_as_uint(odd ? a1 : a0);          // (row rA + 8i, column 8j + qd)
          pa[j][2 + i] = __float_as_uint(odd ? b1 : b0);      // (row rA + 8i, column 8j + qd + 4)
        }
      }
    }

    // ---- store side, per slab: G = P . V^T (gain | bias), y = LN(x) * g (+ b) [post-op] in place, TMA store of the half slab
    float pnz[2] = {0.f, 0.f};
    if (has_noise)
#pragma unroll
      for (int i = 0; i < 2; ++i) pnz[i] = __ldg(P.pnoise + (size_t)bimg * P.pnoise_bstride + tok[i]) * pstr;
    float rgb[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    const float* psc_img = P.post_scale ? scale_s + (spar * NV + 1) * C : nullptr;
    const float* wr_img = scale_s + (spar * NV + (CF::RGB_OK ? 2 : 0)) * C;        // tRGB weights (read when has_rgb)
    if (!TWO_PASS) { stage = stage0; ph = ph0; }   // single pass: walk this tile's slots again
#pragma unroll 1
    for (int s = 0; s < NS; ++s) {
      if (TWO_PASS) mbar_wait(smem_u32(&bars->slab_full[stage]), ph);
      float gv[16], bv[MODE == GF_INT_BOTH ? 16 : 1];
      const uint64_t dvg = dV + (uint64_t)((s * 32 * CF::V_ROW_BYTES) >> 4);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < NJ; ++kk) wgmma_rs_n32(gv, pa[kk], dvg + kk * 2, kk ? 1u : 0u);
      if constexpr (MODE == GF_INT_BOTH) {
        const uint64_t dvb = dV + (uint64_t)(((C + s * 32) * CF::V_ROW_BYTES) >> 4);
#pragma unroll
        for (int kk = 0; kk < NJ; ++kk) wgmma_rs_n32(bv, pa[kk], dvb + kk * 2, kk ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<16>(gv);
      if constexpr (MODE == GF_INT_BOTH) fence_regs<16>(bv);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = rA + 8 * i;
        const float mr = -mean[i] * rstd[i];
        uint8_t* slab = smem + CF::OFF_RING + stage * SLAB_BYTES + r * 128;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int cl = 8 * j + 2 * qd;                            // channel inside the slab
          const int ch = s * SLAB_CH + cl;
          float2* px = reinterpret_cast<float2*>(slab + ((((cl >> 2) ^ (r & 7))) << 4) + (cl & 3) * 4);
          float2 x = *px;
          float g0 = gv[4 * j + 2 * i], g1 = gv[4 * j + 2 * i + 1];
          float b0 = 0.f, b1 = 0.f;
          if constexpr (MODE == GF_INT_BOTH) { b0 = bv[4 * j + 2 * i]; b1 = bv[4 * j + 2 * i + 1]; }
          if (dp_on) {                             // dropout broke sum q = 1: re-add the constants the fold put into V^T
            const float2 cg = __ldg(reinterpret_cast<const float2*>(P.cb + ch));
            g0 = fmaf(qdef[i], cg.x, g0); g1 = fmaf(qdef[i], cg.y, g1);
            if constexpr (MODE == GF_INT_BOTH) {
              const float2 cbb = __ldg(reinterpret_cast<const float2*>(P.cb + C + ch));
              b0 = fmaf(qdef[i], cbb.x, b0); b1 = fmaf(qdef[i], cbb.y, b1);
            }
          }
          if (isc_img) { const float2 d = *reinterpret_cast<const float2*>(isc_img + ch); x.x *= d.x; x.y *= d.y; }
          const float xn0 = fmaf(x.x, rstd[i], mr), xn1 = fmaf(x.y, rstd[i], mr);
          // modulation with the post-op's per-token noise riding on the same FMA (pnz = 0 without a post-op)
          if constexpr (MODE == GF_INT_MUL) {
            x.x = fmaf(xn0, g0, pnz[i]); x.y = fmaf(xn1, g1, pnz[i]);
          } else if constexpr (MODE == GF_INT_ADD) {
            x.x = (xn0 + pnz[i]) + g0; x.y = (xn1 + pnz[i]) + g1;
          } else {
            x.x = fmaf(xn0, g0, b0 + pnz[i]); x.y = fmaf(xn1, g1, b1 + pnz[i]);
          }
          if (P.has_post) {
            const float2 pb = *reinterpret_cast<const float2*>(pbias_s + ch);
            x.x += pb.x; x.y += pb.y;
            // gain * leaky-ReLU(v) = v * (0.6 gain) + |v| * (0.4 gain)  (linear: act_a = gain, act_b = 0): two instructions
            x.x = fmaf(fabsf(x.x), act_b, x.x * act_a); x.y = fmaf(fabsf(x.y), act_b, x.y * act_a);
            if (has_rgb) {                         // tRGB reads the layer output proper: before the next layer's style scale
              const float2 w0 = *reinterpret_cast<const float2*>(wr_img + ch), w1 = *reinterpret_cast<const float2*>(wr_img + C + ch),
                           w2 = *reinterpret_cast<const float2*>(wr_img + 2 * C + ch);
              rgb[i][0] = fmaf(x.x, w0.x, fmaf(x.y, w0.y, rgb[i][0]));
              rgb[i][1] = fmaf(x.x, w1.x, fmaf(x.y, w1.y, rgb[i][1]));
              rgb[i][2] = fmaf(x.x, w2.x, fmaf(x.y, w2.y, rgb[i][2]));
            }
            if (psc_img) { const float2 q2 = *reinterpret_cast<const float2*>(psc_img + ch); x.x *= q2.x; x.y *= q2.y; }
          }
          *px = x;
        }
      }
      fence_proxy_async();                         // generic-proxy writes -> visible to the TMA (async proxy)
      named_bar_sync(1 + wg, 128);
      if (leader) {
        tma_store_2d(tmO, s_ring + stage * SLAB_BYTES + half_off, s * SLAB_CH, (int)(tile * P.rows) + wg * HALF);
        tma_commit();
        if (pending_stage >= 0) {
          tma_wait_read1();                        // the previous store has finished reading its slab
          mbar_arrive(smem_u32(&bars->slab_empty[pending_stage]));
        }
        pending_stage = stage;
      }
      if (++stage == nst) { stage = 0; ph ^= 1u; }
    }
    if (leader) {                                  // no slab stays held across tiles
      tma_wait_read0();
      mbar_arrive(smem_u32(&bars->slab_empty[pending_stage]));
      pending_stage = -1;
    }
    if (has_rgb) {                                 // a row's channels are split over its quad
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float s0 = quad_sum(rgb[i][0]), s1 = quad_sum(rgb[i][1]), s2 = quad_sum(rgb[i][2]);
        const int r = rA + 8 * i;
        if (qd == 0 && r < P.rows) {
          float* o = P.rgb_out + (size_t)bimg * 3 * P.n + (size_t)t_cur * P.rows + r;
          o[0] = s0 + rgb_b0; o[P.n] = s1 + rgb_b1; o[2 * (size_t)P.n] = s2 + rgb_b2;
        }
      }
    }
    // the named barrier of the last slab has ordered every warp's reads of K' / V^T / the scale vectors before this point
    if (leader && has_scales && img_last) mbar_arrive(smem_u32(&bars->sc_free[spar]));
    if (img_last) ++imgc;
    if (img_last) {
      new_img = true;
      if (leader && tile + 1 < tile_end) mbar_arrive(smem_u32(&bars->kv_free));
    }
  }
  if (leader) tma_wait_all();
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
template <int KP, int NS, int MODE>
static int stages_for(int smem_limit) {
  int st = (smem_limit - Cfg<KP, NS, MODE>::FIXED_BYTES - 1024) / SLAB_BYTES;   // 1024: worst-case base alignment slack
  return st > MAX_STAGES ? MAX_STAGES : st;
}
// single-pass needs the whole tile resident; two-pass only streams (a few slabs of slack keep the pipes busy)
#ifndef GF_TWO_PASS_MIN_NS
#define GF_TWO_PASS_MIN_NS 16
#endif
template <int NS> constexpr bool two_pass_shape() { return NS >= GF_TWO_PASS_MIN_NS; }
template <int NS> constexpr int min_stages() { return two_pass_shape<NS>() ? 4 : NS; }

template <int KP, int NS, int MODE>
static int launch(const Layout& L, const gf_attn_desc* d, const float* X, float* Xout, float* att, float* ws, const gf_attn_postop* post, cudaStream_t st) {
  using CF = Cfg<KP, NS, MODE>;
  constexpr bool TWO = two_pass_shape<NS>();
  int nst = stages_for<KP, NS, MODE>(device_smem_optin());
  if (const char* e = getenv("GF_TC_MAX_STAGES")) { const int v = atoi(e); if (v >= min_stages<NS>() && v < nst) nst = v; }   // tuning aid: ring-depth sensitivity
  if (nst < min_stages<NS>()) { set_error("tensor path: shared memory too small for C=%d KP=%d mode=%d", L.C, KP, MODE); return GF_ERR_UNSUPPORTED; }
  CUtensorMap tmX, tmO0, tmO1, tmK, tmV;
  int rc;
  const uint64_t rows = (uint64_t)L.B * L.n;
  const int trows = L.n < TILE ? L.n : TILE;                  // one image per tile when the grid is smaller than a tile
  // each consumer warpgroup stores its own rows: [0, 64) and [64, trows) of the tile
  const int nwg = trows > HALF ? 2 : 1;
  if ((rc = make_map(&tmX, X, rows, L.C, trows, SLAB_CH, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = make_map(&tmO0, Xout, rows, L.C, trows < HALF ? trows : HALF, SLAB_CH, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = make_map(&tmO1, Xout, rows, L.C, nwg == 2 ? trows - HALF : 8, SLAB_CH, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = make_map(&tmK, ws + L.w_Kp, (uint64_t)L.B * KP, L.C, KP, SLAB_CH, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  const uint32_t vrows = CF::COUT < 256 ? CF::COUT : 256;
  if ((rc = make_map(&tmV, ws + L.w_Vt, (uint64_t)L.B * CF::COUT, KP, vrows, KP, KP == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B))) return rc;
  Params P;
  P.att = att; P.Rt = ws + L.w_Rt; P.Ct = ws + L.w_Ct;
  P.n = L.n; P.H = L.H; P.W = L.W; P.k = L.k; P.Cout = L.Cout; P.B = L.B;
  P.norm_layer = d->norm == GF_NORM_LAYER ? 1 : 0;
  P.nstages = nst;
  P.nwg = nwg;
  P.tiles_per_image = (L.n + TILE - 1) / TILE;
  P.rows = trows;
  P.total_tiles = (long long)L.B * P.tiles_per_image;
  P.has_post = post ? 1 : 0;
  P.pbias = post ? post->bias : nullptr; P.pnoise = post ? post->noise : nullptr; P.pstrength = post ? post->strength : nullptr;
  P.pnoise_bstride = post ? post->noise_bstride : 0; P.pact = post ? post->act : 0; P.pgain = post ? post->gain : 1.f;
  P.in_scale = post ? post->in_scale : nullptr; P.post_scale = post ? post->post_scale : nullptr;
  P.in_ld = post ? post->in_scale_ld : 0; P.post_ld = post ? post->post_scale_ld : 0;
  P.rgb_w = post ? post->rgb_w : nullptr; P.rgb_bias = post ? post->rgb_bias : nullptr; P.rgb_out = post ? post->rgb_out : nullptr;
  P.heads = L.heads; P.seg_shift = L.seg == 8 ? 3 : (L.seg == 16 ? 4 : 5);
  if ((rc = dropout_args(post, &P.dp))) return rc;
  P.cb = ws + L.w_CB;
  const int smem_bytes = CF::FIXED_BYTES + nst * SLAB_BYTES + 1024;
  auto kern = token_tc_kernel<KP, NS, MODE, TWO>;
  GF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  long long grid = device_sms();
  if (grid > P.total_tiles) grid = P.total_tiles;
  kern<<<(unsigned)grid, NUM_THREADS, smem_bytes, st>>>(tmX, tmO0, tmO1, tmK, tmV, P);
  GF_LAUNCH_OK();
  set_path(GF_PATH_WGMMA_TF32);
  return GF_OK;
}

template <int KP, int NS>
static int launch_mode(const Layout& L, const gf_attn_desc* d, const float* X, float* Xout, float* att, float* ws, const gf_attn_postop* post, cudaStream_t st) {
  switch (d->integration) {
    case GF_INT_MUL: return launch<KP, NS, GF_INT_MUL>(L, d, X, Xout, att, ws, post, st);
    case GF_INT_ADD: return launch<KP, NS, GF_INT_ADD>(L, d, X, Xout, att, ws, post, st);
    default: return launch<KP, NS, GF_INT_BOTH>(L, d, X, Xout, att, ws, post, st);
  }
}

template <int KP, int NS>
static bool fits(int integration, int limit) {
  switch (integration) {
    case GF_INT_MUL: return stages_for<KP, NS, GF_INT_MUL>(limit) >= min_stages<NS>();
    case GF_INT_ADD: return stages_for<KP, NS, GF_INT_ADD>(limit) >= min_stages<NS>();
    default: return stages_for<KP, NS, GF_INT_BOTH>(limit) >= min_stages<NS>();
  }
}

template <int KP>
static bool fits_ns(int ns, int integration, int limit) {
  switch (ns) {
    case 2: return fits<KP, 2>(integration, limit);
    case 4: return fits<KP, 4>(integration, limit);
    case 8: return fits<KP, 8>(integration, limit);
    default: return fits<KP, 16>(integration, limit);
  }
}

template <int KP>
static int launch_ns(int ns, const Layout& L, const gf_attn_desc* d, const float* X, float* Xout, float* att, float* ws, const gf_attn_postop* post, cudaStream_t st) {
  switch (ns) {
    case 2: return launch_mode<KP, 2>(L, d, X, Xout, att, ws, post, st);
    case 4: return launch_mode<KP, 4>(L, d, X, Xout, att, ws, post, st);
    case 8: return launch_mode<KP, 8>(L, d, X, Xout, att, ws, post, st);
    default: return launch_mode<KP, 16>(L, d, X, Xout, att, ws, post, st);
  }
}

}  // namespace tc

bool tc_supported(const Layout& L, const gf_attn_desc* d) {
  static const bool disabled = getenv("GF_DISABLE_TC") != nullptr;
  if (disabled) return false;
  if (L.C != 64 && L.C != 128 && L.C != 256 && L.C != 512) return false;
  if (L.n % tc::TILE != 0 && !(L.n < tc::TILE && L.n % 8 == 0)) return false;   // whole tiles, or one short tile per image
  if (d->norm != GF_NORM_LAYER && d->norm != GF_NORM_NONE) return false;
  if ((long long)L.B * L.n > 0x7fffffffll) return false;
  const int limit = tc::device_smem_optin();
  return L.KP == 16 ? tc::fits_ns<16>(L.C / 32, d->integration, limit) : tc::fits_ns<32>(L.C / 32, d->integration, limit);
}

int token_pass_tc(const Layout& L, const gf_attn_desc* d, const float* X, float* Xout, float* att, float* ws, const gf_attn_postop* post, cudaStream_t st) {
  if (L.KP == 16) return tc::launch_ns<16>(L.C / 32, L, d, X, Xout, att, ws, post, st);
  return tc::launch_ns<32>(L.C / 32, L, d, X, Xout, att, ws, post, st);
}

}  // namespace gf
