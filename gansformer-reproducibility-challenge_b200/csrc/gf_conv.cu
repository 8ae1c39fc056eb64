// gf_conv.cu -- row f1, first kernel: the 3x3 stride-1 convolution of the synthesis layers as a wgmma implicit GEMM (TF32),
// channels-last, no im2col buffer.
//
// Replaces, on the reference side (expected src/training/network.py, not in the checkout): the convolution inside
// modulated_conv2d_layer in its activation-scaling form -- the caller has already multiplied x by the style (the attention
// kernel's store side does that) and applies the demodulation afterwards (the attention kernel's load side) -- so the weights
// are batch-shared and the op is a plain  y[b,h,w,o] = sum_{dy,dx,i} x[b,h+dy-1,w+dx-1,i] * wt[dy*3+dx][o][i]  with zero padding.
//
// GEMM view: M = output pixels (one CTA tile = an 8 x 16 patch = 128 pixels), N = output channels (BN = 64 per tile),
// K = 9 taps x Cin.  Per K step (one tap, 32 input channels):
//   warp 8     TMA producer: the A operand is a 4-D box {32 ch, 16 w, 8 h, 1 b} of x at (h0+dy-1, w0+dx-1) -- out-of-image
//              coordinates are zero-filled by TMA, which IS the padding -- landing as 128 rows x 128 B, SWIZZLE_128B (K-major);
//              the B operand is a 2-D box {32 ch, BN rows} of the packed weights wt[tap] (K-major, SWIZZLE_128B)
//   warps 0-7  two consumer warpgroups, one per 64-pixel half of the patch: 4 x 2 wgmma m64n32k8 (tf32) per step into register
//              accumulators, the stage released one step later; then the tile's outputs go straight from registers to global.
// Persistent grid (one CTA per SM), tiles handed out round-robin with the N tile innermost.
#include <stdlib.h>
#include <string.h>
#include "gf_common.cuh"
#include "gf_tc_common.cuh"
#include "../../include/gf_ops.h"

namespace gf {
namespace cv {

using namespace tc;

constexpr int PH = 8, PW = 16, TILE_M = PH * PW;      // output patch of one tile
constexpr int BK = 32;                               // input channels per K step = one 128-byte swizzle span
constexpr int BN = 64;                               // output channels per tile
constexpr int A_BYTES = TILE_M * BK * 4;             // 16 KB
constexpr int B_BYTES = BN * BK * 4;                 // 8 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int NUM_THREADS = 288;                     // warps 0-7 consumers, warp 8 producer
constexpr int MAX_STAGES = 8;

struct Bars {
  uint64_t full[MAX_STAGES], empty[MAX_STAGES];
};

struct Params {
  int B, H, W, Cin, Cout;
  int tiles_h, tiles_w, tiles_n;       // patches per image column / row, N tiles
  long long total_tiles;
  int nstages;
  float alpha;                         // TF32 truncation-bias compensation of the streamed operand
};

// 4-D tiled load: coordinates {c, w, h, b} (innermost first); out-of-bounds elements are zero-filled
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, float* __restrict__ y, const Params P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t s_base = smem_u32(smem);
  const int nst = P.nstages;
  Bars* bars = reinterpret_cast<Bars*>(smem + (size_t)nst * STAGE_BYTES);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int ksteps = 9 * (P.Cin / BK);

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmW);
    for (int i = 0; i < nst; ++i) { mbar_init(smem_u32(&bars->full[i]), 1); mbar_init(smem_u32(&bars->empty[i]), 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // tile index -> (n tile, patch w, patch h, image); the N tile is innermost so neighbouring CTAs share their input patch in L2
  auto decode = [&](long long t, int& nt, int& pw, int& ph, int& b) {
    nt = (int)(t % P.tiles_n); t /= P.tiles_n;
    pw = (int)(t % P.tiles_w); t /= P.tiles_w;
    ph = (int)(t % P.tiles_h); b = (int)(t / P.tiles_h);
  };

  if (warp == 8) {
    // =============================== TMA producer ===============================
    if (lane == 0) {
      int stage = 0; uint32_t ph_ = 0;
      for (long long t = blockIdx.x; t < P.total_tiles; t += gridDim.x) {
        int nt, pw, ph, b;
        decode(t, nt, pw, ph, b);
        const int h0 = ph * PH, w0 = pw * PW, n0 = nt * BN;
        for (int tap = 0; tap < 9; ++tap) {
          const int dy = tap / 3, dx = tap - dy * 3;
          for (int c0 = 0; c0 < P.Cin; c0 += BK) {
            mbar_wait(smem_u32(&bars->empty[stage]), ph_ ^ 1u);
            const uint32_t fb = smem_u32(&bars->full[stage]);
            mbar_expect_tx(fb, (uint32_t)STAGE_BYTES);
            const uint32_t sa = s_base + (uint32_t)stage * STAGE_BYTES;
            tma_load_4d(sa, &tmX, fb, c0, w0 + dx - 1, h0 + dy - 1, b);           // zero-filled outside the image = the padding
            tma_load_2d(sa + A_BYTES, &tmW, fb, c0, tap * P.Cout + n0);
            if (++stage == nst) { stage = 0; ph_ ^= 1u; }
          }
        }
      }
    }
    return;
  }

  // =============================== consumer warpgroups ===============================
  const int wg = warp >> 2;
  const int gid = lane >> 2, qd = lane & 3;
  const int rA = wg * 64 + (warp & 3) * 16 + gid;             // pixels rA and rA + 8 of the patch: (r / 16, r % 16)
  const bool leader = (warp & 3) == 0 && lane == 0;
  int stage = 0; uint32_t ph_ = 0;
  for (long long t = blockIdx.x; t < P.total_tiles; t += gridDim.x) {
    int nt, pw, ph, b;
    decode(t, nt, pw, ph, b);
    float acc[2][16];
    int prev = -1;
#pragma unroll 1
    for (int ks = 0; ks < ksteps; ++ks) {
      mbar_wait(smem_u32(&bars->full[stage]), ph_);
      const uint32_t sa = s_base + (uint32_t)stage * STAGE_BYTES;
      const uint64_t da = gmma_desc(sa + wg * 64 * 128, 1024, LAYOUT_SW128);
      const uint64_t db = gmma_desc(sa + A_BYTES, 1024, LAYOUT_SW128);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        wgmma_ss_n32(acc[0], da + kk * 2, db + kk * 2, (ks | kk) ? 1u : 0u);
        wgmma_ss_n32(acc[1], da + kk * 2, db + (uint64_t)((32 * 128) >> 4) + kk * 2, (ks | kk) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();                                         // the previous step's MMAs are done: release its stage
      if (prev >= 0) {
        named_bar_sync(1 + wg, 128);
        if (leader) mbar_arrive(smem_u32(&bars->empty[prev]));
      }
      prev = stage;
      if (++stage == nst) { stage = 0; ph_ ^= 1u; }
    }
    wgmma_wait<0>();
    fence_regs<16>(acc[0]); fence_regs<16>(acc[1]);
    named_bar_sync(1 + wg, 128);
    if (leader) mbar_arrive(smem_u32(&bars->empty[prev]));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = rA + 8 * i;
      const int h = ph * PH + (r >> 4), w = pw * PW + (r & 15);
      float* yrow = y + (((size_t)b * P.H + h) * P.W + w) * P.Cout + nt * BN + 2 * qd;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<float2*>(yrow + hf * 32 + 8 * j) =
              make_float2(acc[hf][4 * j + 2 * i] * P.alpha, acc[hf][4 * j + 2 * i + 1] * P.alpha);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
static int make_map_nhwc(CUtensorMap* m, const void* base, int B, int H, int W, int C, int box_c, int box_w, int box_h) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return GF_ERR_CUDA; }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (NHWC 4-D) failed with CUresult %d (B=%d H=%d W=%d C=%d)", (int)r, B, H, W, C); return GF_ERR_CUDA; }
  return GF_OK;
}

static int launch(const float* x, const float* wt, float* y, int B, int H, int W, int Cin, int Cout, cudaStream_t st) {
  CUtensorMap tmX, tmW;
  int rc;
  if ((rc = make_map_nhwc(&tmX, x, B, H, W, Cin, BK, PW, PH))) return rc;
  if ((rc = make_map(&tmW, wt, (uint64_t)9 * Cout, (uint64_t)Cin, BN, BK, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  Params P;
  P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout;
  P.tiles_h = H / PH; P.tiles_w = W / PW; P.tiles_n = Cout / BN;
  P.total_tiles = (long long)B * P.tiles_h * P.tiles_w * P.tiles_n;
  int nst = (device_smem_optin() - (int)sizeof(Bars) - 1024) / STAGE_BYTES;
  if (nst > MAX_STAGES) nst = MAX_STAGES;
  if (nst < 2) { set_error("conv3x3: shared memory too small"); return GF_ERR_UNSUPPORTED; }
  P.nstages = nst;
  P.alpha = 1.000352220f;              // the tensor core truncates x to TF32 (mean relative bias 0.7213 * 2^-11); the weights are pre-rounded
  const int smem_bytes = nst * STAGE_BYTES + (int)sizeof(Bars) + 1024;
  GF_CUDA_OK(cudaFuncSetAttribute(conv3x3_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  long long grid = device_sms();
  if (grid > P.total_tiles) grid = P.total_tiles;
  conv3x3_tc_kernel<<<(unsigned)grid, NUM_THREADS, smem_bytes, st>>>(tmX, tmW, y, P);
  GF_LAUNCH_OK();
  return GF_OK;
}

// w [Cout][Cin][3][3] (PyTorch layout) -> wt [9][Cout][Cin], rounded to the nearest TF32
__global__ void pack_weights_kernel(const float* __restrict__ w, float* __restrict__ wt, int Cout, int Cin, float scale) {
  const size_t total = (size_t)9 * Cout * Cin;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i % Cin);
    const int o = (int)((i / Cin) % Cout);
    const int tap = (int)(i / ((size_t)Cin * Cout));
    wt[i] = round_tf32_rn(w[((size_t)o * Cin + ci) * 9 + tap] * scale);
  }
}

}  // namespace cv
}  // namespace gf

using namespace gf;

extern "C" int gf_conv3x3_pack_weights(const float* w, float* wt, int Cout, int Cin, float scale, void* stream) {
  if (!w || !wt || Cout <= 0 || Cin <= 0) { set_error("gf_conv3x3_pack_weights: bad arguments"); return GF_ERR_INVALID; }
  const size_t total = (size_t)9 * Cout * Cin;
  size_t blocks = (total + 255) / 256;
  if (blocks > (size_t)num_sms() * 16) blocks = (size_t)num_sms() * 16;
  cv::pack_weights_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w, wt, Cout, Cin, scale);
  GF_LAUNCH_OK();
  return GF_OK;
}

extern "C" int gf_conv3x3_nhwc_tf32(const float* x, const float* wt, float* y, int B, int H, int W, int Cin, int Cout, void* stream) {
  if (!x || !wt || !y) { set_error("gf_conv3x3_nhwc_tf32: null pointer"); return GF_ERR_INVALID; }
  if (B <= 0 || H % cv::PH || W % cv::PW || Cin % cv::BK || Cout % 64 || Cin <= 0 || Cout <= 0) {
    set_error("gf_conv3x3_nhwc_tf32: needs H %% 8 == 0, W %% 16 == 0, Cin %% 32 == 0, Cout %% 64 == 0 (got B=%d H=%d W=%d Cin=%d Cout=%d)", B, H, W, Cin, Cout);
    return GF_ERR_UNSUPPORTED;
  }
  if (((uintptr_t)x & 15) || ((uintptr_t)wt & 15) || ((uintptr_t)y & 15)) { set_error("gf_conv3x3_nhwc_tf32: pointers must be 16-byte aligned"); return GF_ERR_INVALID; }
  int rc;
  if ((rc = check_device())) return rc;
  return cv::launch(x, wt, y, B, H, W, Cin, Cout, (cudaStream_t)stream);
}
