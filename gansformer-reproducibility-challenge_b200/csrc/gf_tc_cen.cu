// gf_tc_cen.cu -- duplex pass A (latents attend to the grid, softmax over the n grid cells) on the Hopper tensor path.
//
// Replaces, on the reference side (expected src/training/network.py, not in the checkout): the k-means / centroid branch
// of transformer_layer (image -> latents attention).  Algorithm = oracle/folded.py centroid_pass():
//     L[t,j] = x_t . M_j + pos(t,j);   A[j,:] = softmax_t L[:,j];   Xbar[j,:] = sum_t A[j,t] x_t
// streamed once over X with an online softmax, split over `nsplit` CTAs per image whose partials (acc[KP][C], m[KP], l[KP])
// are merged by centroid_merge_kernel (gf_simt.cu).
//
// grid (nsplit, B, C / C2), 5 warps, one 64-token tile per step:
//   warp 4     TMA producer: M of the image once, then the X slabs (64 tokens x 32 channels, SWIZZLE_128B) into a ring.
//   warps 0-3  one consumer warpgroup:
//              GEMM1  S[64 tok, KP] = X . M^T    (wgmma, A = slab, B = M, both K-major in shared memory)
//              while the MMAs run, the slabs of this CTA's channel share are transposed into X^T[C2 ch][64 tok]: GEMM2
//              contracts over tokens, and wgmma takes 32-bit operands K-major only
//              online softmax over the tokens (column maxima across the warpgroup), E = 2^(s - m) rounded to TF32 written
//              as E^T[latent][token] (rows KP .. 63 stay zero), accumulators rescaled in registers when a maximum moves
//              GEMM2  D[64 (KP used), C2] += E^T . X   (wgmma, A = E^T, B = X^T)
// HBM traffic: X read once per channel share.
#include <stdlib.h>
#include "gf_common.cuh"
#include "gf_tc_common.cuh"

namespace gf {
namespace tcc {

using namespace tc;

constexpr int TILE = 64;
constexpr int SLAB_CH = 32;
constexpr int SLAB_BYTES = TILE * SLAB_CH * 4;      // 8 KB
constexpr int MAX_ST = 8;
constexpr int NUM_THREADS = 160;                    // warps 0-3 consumers, warp 4 producer
constexpr int ET_BYTES = 2 * 64 * 128;              // E^T: two 32-token chunks of [64 rows x 128 B]

struct Params {
  const float* Rt; const float* Ct; float* part;
  int n, H, W, k, nsplit, tiles_per_image, nst;
};

struct Bars {
  uint64_t full[MAX_ST], empty[MAX_ST];
  uint64_t m_full;
};

// NS = slabs of GEMM1 (all C channels); NS2 = slabs of GEMM2 handled by this CTA (blockIdx.z selects the channel share)
template <int KP, int NS, int NS2 = (NS > 8 ? NS / 2 : NS)>
struct Cfg {
  static constexpr int C = NS * SLAB_CH;
  static constexpr int C2 = NS2 * SLAB_CH;
  static constexpr int M_BYTES = KP * C * 4;                 // NS chunks of [KP rows x 128 B]
  static constexpr int XT_BYTES = 2 * C2 * 128;              // two 32-token chunks of [C2 rows x 128 B]
  static constexpr int OFF_M = 0;
  static constexpr int OFF_XT = OFF_M + M_BYTES;
  static constexpr int OFF_ET = OFF_XT + XT_BYTES;
  static constexpr int OFF_SMALL = OFF_ET + ET_BYTES;        // red[4][KP], mref[KP], resc[KP]
  static constexpr int SMALL_BYTES = 6 * KP * 4;
  static constexpr int OFF_BARS = (OFF_SMALL + SMALL_BYTES + 15) / 16 * 16;
  static constexpr int OFF_RING = (OFF_BARS + (int)sizeof(Bars) + 1023) / 1024 * 1024;
  static constexpr int FIXED_BYTES = OFF_RING;
};

template <int KP, int NS, int NS2>
__global__ void __launch_bounds__(NUM_THREADS, 1)
centroid_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmM, const Params P) {
  using CF = Cfg<KP, NS, NS2>;
  constexpr int C = CF::C, C2 = CF::C2;
  constexpr int NJ = KP / 8;
  constexpr int NC2 = C2 / 32;                                // 32-channel chunks of the GEMM2 accumulator
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t s_base = smem_u32(smem);
  const uint32_t s_m = s_base + CF::OFF_M, s_xt = s_base + CF::OFF_XT, s_et = s_base + CF::OFF_ET, s_ring = s_base + CF::OFF_RING;
  Bars* bars = reinterpret_cast<Bars*>(smem + CF::OFF_BARS);
  float* red = reinterpret_cast<float*>(smem + CF::OFF_SMALL);      // [4][KP]
  float* mref = red + 4 * KP;                                       // [KP] running maxima (log2 units)
  float* resc = mref + KP;                                          // [KP] rescale factors of this tile
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y, sp = blockIdx.x;
  const int zoff = blockIdx.z * C2;                                 // first channel of this CTA's GEMM2 share
  const int per = (P.tiles_per_image + P.nsplit - 1) / P.nsplit;
  const int tile_beg = sp * per, tile_end = min(P.tiles_per_image, tile_beg + per);
  const int ntiles = tile_end - tile_beg;
  const int nst = P.nst;
  float* part = P.part + ((size_t)b * P.nsplit + sp) * KP * (C + 4);

  if (ntiles <= 0) {                          // empty split: neutral partial
    for (int i = threadIdx.x; i < KP * (C2 + 4); i += NUM_THREADS) {
      const int j = i / (C2 + 4), c = i % (C2 + 4);
      if (c < C2) part[(size_t)j * (C + 4) + zoff + c] = 0.f;
      else if (blockIdx.z == 0) part[(size_t)j * (C + 4) + C + (c - C2)] = (c == C2) ? -INFINITY : 0.f;
    }
    return;
  }

  for (int i = threadIdx.x; i < ET_BYTES / 16; i += NUM_THREADS) reinterpret_cast<float4*>(smem + CF::OFF_ET)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (threadIdx.x < KP) { mref[threadIdx.x] = -INFINITY; resc[threadIdx.x] = 1.f; }
  if (warp == 4 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmM);
    for (int i = 0; i < nst; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 1); }
    mbar_init(smem_u32(&bars->m_full), 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4) {
    // =============================== TMA producer ===============================
    if (lane == 0) {
      const uint32_t mb = smem_u32(&bars->m_full);
      mbar_expect_tx(mb, (uint32_t)CF::M_BYTES);
#pragma unroll
      for (int s = 0; s < NS; ++s) tma_load_2d(s_m + s * (KP * 128), &tmM, mb, s * SLAB_CH, b * KP);
      uint32_t ctr = 0;
      for (int t = tile_beg; t < tile_end; ++t) {
        const int row0 = b * P.n + t * TILE;       // the rows past a short image's end are masked by the consumers
        for (int s = 0; s < NS; ++s, ++ctr) {
          const int stage = (int)(ctr % (uint32_t)nst);
          mbar_wait(smem_u32(&bars->empty[stage]), ((ctr / (uint32_t)nst) & 1u) ^ 1u);
          const uint32_t fb = smem_u32(&bars->full[stage]);
          mbar_expect_tx(fb, (uint32_t)SLAB_BYTES);
          tma_load_2d(s_ring + stage * SLAB_BYTES, &tmX, fb, s * SLAB_CH, row0);
        }
      }
    }
    return;
  }

  // =============================== consumer warpgroup ===============================
  const int w = warp, gid = lane >> 2, qd = lane & 3;
  const int tid = threadIdx.x;
  const bool leader = tid == 0;
  const uint64_t dM = gmma_desc(s_m, 1024, LAYOUT_SW128);
  float acc2[NC2][16];
#pragma unroll
  for (int c = 0; c < NC2; ++c)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc2[c][i] = 0.f;
  float lp[NJ][2];                            // this thread's share of the denominators of its columns
#pragma unroll
  for (int j = 0; j < NJ; ++j) { lp[j][0] = 0.f; lp[j][1] = 0.f; }
  mbar_wait(smem_u32(&bars->m_full), 0);
  int stage = 0; uint32_t ph = 0;
  for (int t = tile_beg; t < tile_end; ++t) {
    // positional logits of this thread's rows (tokens 16 w + gid, + 8) and columns (latents 8 jb + 2 qd + e)
    float pos[NJ][4];
    bool valid[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int tk = t * TILE + 16 * w + gid + 8 * i;
      valid[i] = tk < P.n;
      const int tok = min(tk, P.n - 1);
      const int h = tok / P.W, x = tok - h * P.W;
      const float* rt = P.Rt + ((size_t)b * P.H + h) * KP + 2 * qd;
      const float* ct = P.Ct + ((size_t)b * P.W + x) * KP + 2 * qd;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float2 r = __ldg(reinterpret_cast<const float2*>(rt + 8 * j)), c = __ldg(reinterpret_cast<const float2*>(ct + 8 * j));
        pos[j][2 * i] = r.x + c.x; pos[j][2 * i + 1] = r.y + c.y;
      }
    }
    // ---- GEMM1 over all slabs; the slabs of this CTA's channel share are transposed into X^T meanwhile
    float sacc[KP / 2];
#pragma unroll 1
    for (int s = 0; s < NS; ++s) {
      mbar_wait(smem_u32(&bars->full[stage]), ph);
      const uint32_t sa = s_ring + stage * SLAB_BYTES;
      const uint64_t da = gmma_desc(sa, 1024, LAYOUT_SW128);
      const uint64_t db = dM + (uint64_t)(s * ((KP * 128) >> 4));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        if constexpr (KP == 32) wgmma_ss_n32(sacc, da + kk * 2, db + kk * 2, (s | kk) ? 1u : 0u);
        else wgmma_ss_n16(sacc, da + kk * 2, db + kk * 2, (s | kk) ? 1u : 0u);
      }
      wgmma_commit();
      const int cbase = s * SLAB_CH - zoff;
      if (cbase >= 0 && cbase < C2) {
        // thread: token tok = tid / 2, channels 16 (tid & 1) .. + 15 of the slab -> X^T[channel][token]
        const int tok = tid >> 1, tch = tok >> 5, tin = tok & 31;
        const uint8_t* src = smem + CF::OFF_RING + stage * SLAB_BYTES + tok * 128;
        uint8_t* dstc = smem + CF::OFF_XT + tch * (C2 * 128);
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {
          const int c4 = (tid & 1) * 4 + q4;
          const float4 v = *reinterpret_cast<const float4*>(src + ((c4 ^ (tok & 7)) << 4));
          const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int cl = cbase + c4 * 4 + e;
            *reinterpret_cast<float*>(dstc + cl * 128 + ((((tin >> 2) ^ (cl & 7))) << 4) + (tin & 3) * 4) = vv[e];
          }
        }
      }
      wgmma_wait<0>();
      named_bar_sync(1, 128);
      if (leader) mbar_arrive(smem_u32(&bars->empty[stage]));
      if (++stage == nst) { stage = 0; ph ^= 1u; }
    }
    fence_regs<KP / 2>(sacc);
    // ---- logits (log2 units: log2 e is folded into M / Rt2 / Ct2, gf_fold.cu), column maxima over the tile's tokens
    float cm[NJ][2];
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float& v = sacc[4 * j + 2 * i + e];
          v = valid[i] ? v + pos[j][2 * i + e] : -INFINITY;
        }
        float m = fmaxf(sacc[4 * j + e], sacc[4 * j + 2 + e]);
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
        cm[j][e] = m;
      }
    if (gid == 0)
#pragma unroll
      for (int j = 0; j < NJ; ++j) { red[w * KP + 8 * j + 2 * qd] = cm[j][0]; red[w * KP + 8 * j + 2 * qd + 1] = cm[j][1]; }
    named_bar_sync(1, 128);
    if (tid < KP) {
      const float tm = fmaxf(fmaxf(red[tid], red[KP + tid]), fmaxf(red[2 * KP + tid], red[3 * KP + tid]));
      const float mo = mref[tid];
      float mn = mo, f = 1.f;
      if (tid < P.k && tm > mo) { mn = tm; f = mo == -INFINITY ? 1.f : exp2f(mo - mn); }
      mref[tid] = mn;
      resc[tid] = f;
    }
    named_bar_sync(1, 128);
    // ---- E = 2^(s - m) rounded to TF32 (the tensor core's operand truncation is then exact and the denominators see the same
    //      values), written transposed: E^T[latent][token], K-major SW128, 32-token chunks
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * j + 2 * qd + e;
        const float mj = mref[col];
        lp[j][e] *= resc[col];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int tok = 16 * w + gid + 8 * i, tch = tok >> 5, tin = tok & 31;
          const float sv = sacc[4 * j + 2 * i + e];
          const float ev = (col < P.k && valid[i]) ? cvt_tf32(exp2f(sv - mj)) : 0.f;
          lp[j][e] += ev;
          *reinterpret_cast<float*>(smem + CF::OFF_ET + tch * (64 * 128) + col * 128 + ((((tin >> 2) ^ (col & 7))) << 4) + (tin & 3) * 4) = ev;
        }
      }
    // ---- rescale the accumulators whose maximum moved (rows = latents 16 w + gid, + 8)
    {
      const int j0 = 16 * w + gid, j1 = j0 + 8;
      const float f0 = j0 < KP ? resc[j0] : 1.f, f1 = j1 < KP ? resc[j1] : 1.f;
#pragma unroll
      for (int c = 0; c < NC2; ++c)
#pragma unroll
        for (int jb = 0; jb < 4; ++jb) {
          acc2[c][4 * jb] *= f0; acc2[c][4 * jb + 1] *= f0; acc2[c][4 * jb + 2] *= f1; acc2[c][4 * jb + 3] *= f1;
        }
    }
    fence_proxy_async();                      // E^T and X^T (generic proxy) -> wgmma (async proxy)
    named_bar_sync(1, 128);
    // ---- GEMM2: D += E^T . X over the tile's 64 tokens (8 k-blocks: two 32-token chunks of 4)
#pragma unroll
    for (int c = 0; c < NC2; ++c) fence_regs<16>(acc2[c]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint64_t da = gmma_desc(s_et + (kk >> 2) * (64 * 128) + (kk & 3) * 32, 1024, LAYOUT_SW128);
#pragma unroll
      for (int c = 0; c < NC2; ++c) {
        const uint64_t db = gmma_desc(s_xt + (kk >> 2) * (C2 * 128) + c * (32 * 128) + (kk & 3) * 32, 1024, LAYOUT_SW128);
        wgmma_ss_n32(acc2[c], da, db, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NC2; ++c) fence_regs<16>(acc2[c]);
    named_bar_sync(1, 128);                   // E^T / X^T may be rewritten by the next tile
  }

  // ---- flush: partial accumulators, running maxima and denominators of this split
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v = lp[j][e];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (gid == 0) red[w * KP + 8 * j + 2 * qd + e] = v;
    }
  named_bar_sync(1, 128);
  if (tid < KP && blockIdx.z == 0) {
    const int j = tid;
    part[(size_t)j * (C + 4) + C] = j < P.k ? mref[j] * 0.6931471805599453f : -INFINITY;   // log2 -> natural units
    part[(size_t)j * (C + 4) + C + 1] = red[j] + red[KP + j] + red[2 * KP + j] + red[3 * KP + j];
    part[(size_t)j * (C + 4) + C + 2] = 0.f;
    part[(size_t)j * (C + 4) + C + 3] = 0.f;
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = 16 * w + gid + 8 * i;
    if (j < KP) {
      float* dst = part + (size_t)j * (C + 4) + zoff + 2 * qd;
#pragma unroll
      for (int c = 0; c < NC2; ++c)
#pragma unroll
        for (int jb = 0; jb < 4; ++jb)          // X truncation bias of the tensor core (gf_fold.cu)
          *reinterpret_cast<float2*>(dst + c * 32 + 8 * jb) =
              make_float2(acc2[c][4 * jb + 2 * i] * 1.000352220f, acc2[c][4 * jb + 2 * i + 1] * 1.000352220f);
    }
  }
}

template <int KP, int NS>
static int stages_for(int smem_limit) {
  const int s = (smem_limit - Cfg<KP, NS>::FIXED_BYTES - 1024) / SLAB_BYTES;
  return s > MAX_ST ? MAX_ST : s;
}

template <int KP, int NS>
static int launch(const Layout& L, const float* X, float* ws, cudaStream_t st) {
  using CF = Cfg<KP, NS>;
  constexpr int NS2 = NS > 8 ? NS / 2 : NS;
  const int nst = stages_for<KP, NS>(device_smem_optin());
  if (nst < 2) { set_error("tensor-core centroid pass: shared memory too small for C=%d KP=%d", L.C, KP); return GF_ERR_UNSUPPORTED; }
  CUtensorMap tmX, tmM;
  int rc;
  if ((rc = make_map(&tmX, X, (uint64_t)L.B * L.n, L.C, TILE, SLAB_CH, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = make_map(&tmM, ws + L.w_M, (uint64_t)L.B * KP, L.C, KP, SLAB_CH, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  Params P;
  P.Rt = ws + L.w_Rt2; P.Ct = ws + L.w_Ct2; P.part = ws + L.w_PART;
  P.n = L.n; P.H = L.H; P.W = L.W; P.k = L.k; P.nsplit = L.nsplit_cen; P.tiles_per_image = (L.n + TILE - 1) / TILE;
  P.nst = nst;
  const int smem_bytes = CF::FIXED_BYTES + nst * SLAB_BYTES + 1024;
  auto kern = centroid_tc_kernel<KP, NS, NS2>;
  GF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  kern<<<dim3(L.nsplit_cen, L.B, NS / NS2), NUM_THREADS, smem_bytes, st>>>(tmX, tmM, P);
  GF_LAUNCH_OK();
  return GF_OK;
}

template <int KP, int NS>
static bool fits(int limit) { return stages_for<KP, NS>(limit) >= 2; }

template <int KP>
static bool fits_ns(int ns, int limit) {
  return ns == 2 ? fits<KP, 2>(limit) : ns == 4 ? fits<KP, 4>(limit) : ns == 8 ? fits<KP, 8>(limit) : fits<KP, 16>(limit);
}

template <int KP>
static int launch_ns(int ns, const Layout& L, const float* X, float* ws, cudaStream_t st) {
  return ns == 2 ? launch<KP, 2>(L, X, ws, st) : ns == 4 ? launch<KP, 4>(L, X, ws, st) : ns == 8 ? launch<KP, 8>(L, X, ws, st) : launch<KP, 16>(L, X, ws, st);
}

}  // namespace tcc

bool tc_centroid_supported(const Layout& L, const gf_attn_desc* d) {
  if (d->flags & GF_FLAG_FP32_EXACT) return false;
  if (L.C != 64 && L.C != 128 && L.C != 256 && L.C != 512) return false;   // C = 512: two CTAs share the channels
  if (L.B > 65535 || (long long)L.B * L.n > 0x7fffffffll) return false;
  const int limit = tc::device_smem_optin();
  return L.KP == 16 ? tcc::fits_ns<16>(L.C / 32, limit) : tcc::fits_ns<32>(L.C / 32, limit);
}

int centroid_pass_tc(const Layout& L, const float* X, float* ws, cudaStream_t st) {
  return L.KP == 16 ? tcc::launch_ns<16>(L.C / 32, L, X, ws, st) : tcc::launch_ns<32>(L.C / 32, L, X, ws, st);
}

}  // namespace gf
