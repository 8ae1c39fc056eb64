// gf_conv.cu -- row f1, first kernel: the 3x3 stride-1 convolution of the synthesis layers as a wgmma implicit GEMM (TF32),
// channels-last, no im2col buffer.
//
// Replaces, on the reference side (expected src/training/network.py, not in the checkout): the convolution inside
// modulated_conv2d_layer in its activation-scaling form -- the caller has already multiplied x by the style (the attention
// kernel's store side does that) and applies the demodulation afterwards (the attention kernel's load side) -- so the weights
// are batch-shared and the op is a plain  y[b,h,w,o] = sum_{dy,dx,i} x[b,h+dy-1,w+dx-1,i] * wt[dy*3+dx][o][i]  with zero padding.
//
// GEMM view: M = output pixels (one CTA tile = an 8 x 16 patch = 128 pixels), N = output channels (BN in {64, 128, 256} per tile,
// the widest that divides Cout), K = 9 taps x Cin.  The K loop runs over 32-channel chunks, then the filter column dx, then the
// filter row dy:
//   warp 8     TMA producer.  Per (chunk, dx) ONE activation box {32 ch, 16 w, 10 h, 1 b} of x at (w0+dx-1, h0-1): the patch plus
//              a one-row halo above and below, 160 rows x 128 B, SWIZZLE_128B (K-major); out-of-image coordinates are zero-filled
//              by TMA, which IS the padding.  The three dy taps read it through views starting at rows 0, 16 and 32 (byte offsets
//              0, 2048, 4096: whole 1024-byte swizzle atoms, so the plain descriptor works).  Per tap a {32 ch, BN rows} box of the
//              packed weights wt[dy*3+dx].  Activations and weights have separate rings, each with its own full/empty mbarriers.
//   warps 0-7  two consumer warpgroups, one per 64-pixel half of the patch: per tap 4 x wgmma m64nBNk8 (tf32) into register
//              accumulators (A is read once per instruction); the tap's weight slot is released one tap later, the activation
//              slot after its third tap; then the tile's outputs go straight from registers to global.
// Per 32-channel chunk of a BN = 256 tile this moves 3 x 20 KB + 9 x 32 KB from L2 for 9 x 2 MFLOP (0.018 B/FLOP).
// Persistent grid (one CTA per SM), tiles handed out round-robin with the N tile innermost.
#include <stdlib.h>
#include <string.h>
#include "gf_common.cuh"
#include "gf_tc_common.cuh"
#include "../../include/gf_ops.h"

namespace gf {
namespace cv {

using namespace tc;

constexpr int PH = 8, PW = 16;                       // output patch of one tile (M = 128 pixels)
constexpr int BK = 32;                               // input channels per K step = one 128-byte swizzle span
constexpr int A_ROWS = (PH + 2) * PW;                // activation box: the patch plus one halo row above and below
constexpr int A_BYTES = A_ROWS * BK * 4;             // 20 KB
constexpr int NUM_THREADS = 288;                     // warps 0-7 consumers, warp 8 producer
constexpr int MAX_A = 3, MAX_W = 8;                  // ring depths (activation boxes, weight boxes)

struct Bars {
  uint64_t full_a[MAX_A], empty_a[MAX_A], full_w[MAX_W], empty_w[MAX_W];
};

struct Params {
  int B, H, W, Cin, Cout;
  int tiles_h, tiles_w, tiles_n;       // patches per image column / row, N tiles
  long long total_tiles;
  int na, nw;                          // activation / weight ring slots
  float alpha;                         // TF32 truncation-bias compensation of the streamed operand
};

// 4-D tiled load: coordinates {c, w, h, b} (innermost first); out-of-bounds elements are zero-filled
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv3x3_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, float* __restrict__ y, const Params P) {
  constexpr int W_BYTES = BN * BK * 4;               // one tap's weight box: 8 / 16 / 32 KB
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t s_a = smem_u32(smem);                                  // activation ring
  const uint32_t s_w = s_a + (uint32_t)P.na * A_BYTES;                  // weight ring
  Bars* bars = reinterpret_cast<Bars*>(smem + (size_t)P.na * A_BYTES + (size_t)P.nw * W_BYTES);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmW);
    for (int i = 0; i < P.na; ++i) { mbar_init(smem_u32(&bars->full_a[i]), 1); mbar_init(smem_u32(&bars->empty_a[i]), 2); }
    for (int i = 0; i < P.nw; ++i) { mbar_init(smem_u32(&bars->full_w[i]), 1); mbar_init(smem_u32(&bars->empty_w[i]), 2); }
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
      int sa = 0, sw = 0; uint32_t pa = 0, pw_ = 0;
      for (long long t = blockIdx.x; t < P.total_tiles; t += gridDim.x) {
        int nt, pw, ph, b;
        decode(t, nt, pw, ph, b);
        const int h0 = ph * PH, w0 = pw * PW, n0 = nt * BN;
        for (int c0 = 0; c0 < P.Cin; c0 += BK) {
          for (int dx = 0; dx < 3; ++dx) {
            mbar_wait(smem_u32(&bars->empty_a[sa]), pa ^ 1u);
            const uint32_t fa = smem_u32(&bars->full_a[sa]);
            mbar_expect_tx(fa, (uint32_t)A_BYTES);
            tma_load_4d(s_a + (uint32_t)sa * A_BYTES, &tmX, fa, c0, w0 + dx - 1, h0 - 1, b);   // zero-filled outside the image = the padding
            if (++sa == P.na) { sa = 0; pa ^= 1u; }
            for (int dy = 0; dy < 3; ++dy) {
              mbar_wait(smem_u32(&bars->empty_w[sw]), pw_ ^ 1u);
              const uint32_t fw = smem_u32(&bars->full_w[sw]);
              mbar_expect_tx(fw, (uint32_t)W_BYTES);
              tma_load_2d(s_w + (uint32_t)sw * W_BYTES, &tmW, fw, c0, (dy * 3 + dx) * P.Cout + n0);
              if (++sw == P.nw) { sw = 0; pw_ ^= 1u; }
            }
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
  int sa = 0, sw = 0; uint32_t pa = 0, pw_ = 0;
  for (long long t = blockIdx.x; t < P.total_tiles; t += gridDim.x) {
    int nt, pw, ph, b;
    decode(t, nt, pw, ph, b);
    float acc[BN / 2];
    int prev_w = -1, prev_a = -1;                              // slots of the previous tap, released once its MMAs are done
#pragma unroll 1
    for (int c0 = 0; c0 < P.Cin; c0 += BK) {
#pragma unroll 1
      for (int dx = 0; dx < 3; ++dx) {
        mbar_wait(smem_u32(&bars->full_a[sa]), pa);
        const uint32_t a_view = s_a + (uint32_t)sa * A_BYTES + wg * 64 * 128;   // this warpgroup's 64 rows, before the dy shift
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
          mbar_wait(smem_u32(&bars->full_w[sw]), pw_);
          const uint64_t da = gmma_desc(a_view + dy * PW * 128, 1024, LAYOUT_SW128);
          const uint64_t db = gmma_desc(s_w + (uint32_t)sw * W_BYTES, 1024, LAYOUT_SW128);
          const uint32_t acc0 = (c0 | dx | dy) ? 1u : 0u;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_ss<BN>(acc, da + kk * 2, db + kk * 2, (acc0 | kk) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();                                     // the previous tap's MMAs are done: release its slots
          if (prev_w >= 0) {
            named_bar_sync(1 + wg, 128);
            if (leader) {
              mbar_arrive(smem_u32(&bars->empty_w[prev_w]));
              if (prev_a >= 0) mbar_arrive(smem_u32(&bars->empty_a[prev_a]));
            }
          }
          prev_w = sw;
          prev_a = dy == 2 ? sa : -1;                          // the third tap is the last reader of the activation box
          if (++sw == P.nw) { sw = 0; pw_ ^= 1u; }
        }
        if (++sa == P.na) { sa = 0; pa ^= 1u; }
      }
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(acc);
    named_bar_sync(1 + wg, 128);
    if (leader) {
      mbar_arrive(smem_u32(&bars->empty_w[prev_w]));
      mbar_arrive(smem_u32(&bars->empty_a[prev_a]));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = rA + 8 * i;
      const int h = ph * PH + (r >> 4), w = pw * PW + (r & 15);
      float* yrow = y + (((size_t)b * P.H + h) * P.W + w) * P.Cout + nt * BN + 2 * qd;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        *reinterpret_cast<float2*>(yrow + 8 * j) = make_float2(acc[4 * j + 2 * i] * P.alpha, acc[4 * j + 2 * i + 1] * P.alpha);
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

template <int BN>
static int launch_bn(const float* x, const float* wt, float* y, int B, int H, int W, int Cin, int Cout, cudaStream_t st) {
  constexpr int W_BYTES = BN * BK * 4;
  CUtensorMap tmX, tmW;
  int rc;
  if ((rc = make_map_nhwc(&tmX, x, B, H, W, Cin, BK, PW, PH + 2))) return rc;
  if ((rc = make_map(&tmW, wt, (uint64_t)9 * Cout, (uint64_t)Cin, BN, BK, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  Params P;
  P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout;
  P.tiles_h = H / PH; P.tiles_w = W / PW; P.tiles_n = Cout / BN;
  P.total_tiles = (long long)B * P.tiles_h * P.tiles_w * P.tiles_n;
  const int avail = device_smem_optin() - (int)sizeof(Bars) - 1024;
  P.na = MAX_A;
  P.nw = (avail - P.na * A_BYTES) / W_BYTES;
  if (P.nw > MAX_W) P.nw = MAX_W;
  if (P.nw < 2) { set_error("conv3x3: shared memory too small"); return GF_ERR_UNSUPPORTED; }
  P.alpha = 1.000352220f;              // the tensor core truncates x to TF32 (mean relative bias 0.7213 * 2^-11); the weights are pre-rounded
  const int smem_bytes = P.na * A_BYTES + P.nw * W_BYTES + (int)sizeof(Bars) + 1024;
  GF_CUDA_OK(cudaFuncSetAttribute(conv3x3_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  long long grid = device_sms();
  if (grid > P.total_tiles) grid = P.total_tiles;
  conv3x3_tc_kernel<BN><<<(unsigned)grid, NUM_THREADS, smem_bytes, st>>>(tmX, tmW, y, P);
  GF_LAUNCH_OK();
  return GF_OK;
}

// the widest N tile that divides Cout: 256 for the 512- and 256-channel layers, 128 at Cout = 128, 64 otherwise
static int launch(const float* x, const float* wt, float* y, int B, int H, int W, int Cin, int Cout, cudaStream_t st) {
  if (Cout % 256 == 0) return launch_bn<256>(x, wt, y, B, H, W, Cin, Cout, st);
  if (Cout % 128 == 0) return launch_bn<128>(x, wt, y, B, H, W, Cin, Cout, st);
  return launch_bn<64>(x, wt, y, B, H, W, Cin, Cout, st);
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
  if (B <= 0 || H <= 0 || W <= 0 || H % cv::PH || W % cv::PW || Cin % cv::BK || Cout % 64 || Cin <= 0 || Cout <= 0) {
    set_error("gf_conv3x3_nhwc_tf32: needs positive sizes, H %% 8 == 0, W %% 16 == 0, Cin %% 32 == 0, Cout %% 64 == 0 (got B=%d H=%d W=%d Cin=%d Cout=%d)", B, H, W, Cin, Cout);
    return GF_ERR_UNSUPPORTED;
  }
  if (((uintptr_t)x & 15) || ((uintptr_t)wt & 15) || ((uintptr_t)y & 15)) { set_error("gf_conv3x3_nhwc_tf32: pointers must be 16-byte aligned"); return GF_ERR_INVALID; }
  int rc;
  if ((rc = check_device())) return rc;
  return cv::launch(x, wt, y, B, H, W, Cin, Cout, (cudaStream_t)stream);
}
