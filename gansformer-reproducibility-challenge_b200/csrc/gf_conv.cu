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
// Second kernel: upconv_blur_tc_kernel, the upsampling layers' stride-2 transposed convolution + FIR blur + demodulation (below).
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
// The upsampling layers: stride-2 transposed 3x3 convolution + [1,3,3,1] FIR blur + demodulation in one kernel
// ---------------------------------------------------------------------------------------------------------
// conv_transpose2d with stride 2 (q = 2m + k) splits per dimension into T_even[m] = w[k=0] x[m] + w[k=2] x[m-1] and
// T_odd[m] = w[k=1] x[m].  "Phase position" (r, c) holds T_even[r] and T_odd[r-1] per dimension, so every tap reads x at a shift of
// 0 or -1: per 32-channel chunk two activation boxes (column shift 0 and -1) of 9 rows (the 8 phase rows of a step plus one halo
// row), the row shift being a view at a whole number of swizzle atoms.  The four phase accumulators (ee, eo, oe, oo: row phase,
// column phase) take the taps
//   shift (0,0) -> ee(0,0);  (0,-1) -> ee(0,2), eo(0,1);  (-1,0) -> ee(2,0), oe(1,0);  (-1,-1) -> ee(2,2), eo(2,1), oe(1,2), oo(1,1)
// i.e. nine taps per phase position, the MMA work of a stride-1 3x3 convolution at the low resolution.  The blur, per dimension,
//   y[2i] = T_odd[i-1] + 3 T_even[i] + 3 T_odd[i] + T_even[i+1],  y[2i+1] = T_even[i] + 3 T_odd[i] + 3 T_even[i+1] + T_odd[i+1]  (/8),
// needs phase positions i, i+1, i+2 for output pair i; TMA's zero fill makes T_odd[-1], T_odd[H] and T_even[H+1] zero, which is the
// blur's padding of 1.  Work unit = (image, column strip of 16 phase columns = 14 output column pairs, N tile of 64 channels); it
// walks down the strip 8 phase rows per step and keeps the last two phase rows in shared memory for the next step's vertical blur,
// so only the two-column horizontal halo is recomputed.
// MMA: the taps of one activation shift share their A operand, so they go into as few wgmmas as the accumulators allow.  Two
// fragments of 64 floats per thread, X = [ee, eo] and Y = [oe, oo] (64 channels per phase), and per k8 step six instructions:
//   shift (-1,-1) -> n128 into X (taps 8, 7) and n128 into Y (taps 5, 4);  (0,-1) -> n128 into X (taps 2, 1);
//   (-1,0) -> n64 into X (tap 6) and n64 into Y (tap 3);  (0,0) -> n64 into X (tap 0).
// Every wgmma writes a whole fragment or its first half: one n256 over [oe, ee, eo, oo] with n128 / n64 wgmmas on sub-ranges of it
// makes ptxas serialise all of them (C7511, "insufficient register resources for the wgmma pipeline").  The B operand of an n128 is
// its two taps' 64-row weight boxes placed next to each other (rows of one K-major SWIZZLE_128B matrix, no repacking).  Shift
// (-1,-1) comes first in a chunk, so in the first chunk it initialises both fragments.  Per k8 and warpgroup that is 30 KB of
// shared-memory reads (A 6 x 2 KB, B 9 x 2 KB) for 288 MMA clocks, against 36 KB for nine per-tap n64s.
// Shared memory: the activation ring (4 boxes of 18 KB = two chunks), one weight stage of 72 KB holding a chunk's four shift groups
// at fixed offsets, each group with its own full / empty barrier so its slot is refilled as soon as both warpgroups have finished
// its MMAs, and the epilogue's carry (34 KB) and stage (34 KB): 213 KB of the 227 KB.
// Warps 0-7 are the two consumer warpgroups (setmaxnreg 232), warps 8-11 the producer warpgroup (setmaxnreg 40, one thread issues
// the TMA); ptxas -v: 168 registers at launch, no spill.
// Epilogue per 16-channel slice: the accumulators go to shared memory, warp k blurs output row pair 8 step - 2 + k (horizontal then
// vertical, fixed order, see DESIGN §5) and scales once by alpha * gain * d[b, c].  It does not overlap the next step's MMAs (the
// tensor cores idle meanwhile); a full step's staging does not fit beside the rings, see DESIGN §4.4.
constexpr int U_PC = 16, U_PR = 8;                     // phase columns of a strip, phase rows of a step
constexpr int U_OC = U_PC - 2;                         // complete output column pairs per strip
constexpr int U_BN = 64;                               // output channels per unit: 4 phases x 64 / 2 = 128 accumulators per thread
constexpr int U_A_BYTES = (U_PR + 1) * U_PC * BK * 4;  // activation box {32 ch, 16 w, 9 h}: 18 KB
constexpr int U_W_BYTES = U_BN * BK * 4;               // one tap's weight box: 8 KB
constexpr int U_WS_BYTES = 9 * U_W_BYTES;              // weight stage: the nine taps of a chunk, grouped by shift: 72 KB
constexpr int U_CS = 68;                               // floats per staged phase position: 4 phases x 16 channels + 4 (bank spread)
constexpr int U_NA = 4;                                // activation ring slots (two chunks)
constexpr int U_THREADS = 384;                         // warps 0-7 consumers, warps 8-11 producer warpgroup

struct UBars {
  uint64_t full_a[U_NA], empty_a[U_NA], full_w[4], empty_w[4];
};

struct UParams {
  int B, H, W, Cin, Cout;                // H, W: input (low-resolution) size
  int strips, steps, tiles_n;
  int total_units;
  float ag;                              // alpha * gain
  const float* scale;                    // d [B, Cout]
};

// shift groups in issue order: 0 = shift (-1,-1), 1 = (0,-1), 2 = (-1,0), 3 = (0,0).  Groups 0, 1 read the activation box of column
// shift -1, groups 2, 3 the box of column shift 0; U_GROW 0: row shift -1 (view from box row 0), 1: row shift 0 (from box row 1).
// A group's weight boxes: its U_GNX taps of fragment X (phase ee, then eo), then its taps of fragment Y (oe, then oo); one or two
// taps per fragment make one n64 or n128 wgmma.  tests/test_host_cpu_upconv_v2.py reads these tables.
__device__ constexpr int U_GTAPS[4] = {4, 2, 2, 1};
__device__ constexpr int U_GNX[4] = {2, 2, 1, 1};
__device__ constexpr int U_GTAP[4][4] = {{8, 7, 5, 4}, {2, 1, 0, 0}, {6, 3, 0, 0}, {0, 0, 0, 0}};
__device__ constexpr int U_GOFF[4] = {0, 4, 6, 8};                    // first weight box of the group in the stage
__device__ constexpr int U_GROW[4] = {0, 1, 0, 1};

__device__ __forceinline__ void setmaxnreg_dec40() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void setmaxnreg_inc232() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

__global__ void __launch_bounds__(U_THREADS, 1)
upconv_blur_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, float* __restrict__ y, const UParams P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t s_a = smem_u32(smem);
  const uint32_t s_w = s_a + (uint32_t)U_NA * U_A_BYTES;
  float* carry = reinterpret_cast<float*>(smem + (size_t)U_NA * U_A_BYTES + U_WS_BYTES);                  // [4 slices][2 rows][16][U_CS]
  float* stage = carry + 4 * 2 * U_PC * U_CS;                                                             // [8 rows][16][U_CS]
  UBars* bars = reinterpret_cast<UBars*>(stage + U_PR * U_PC * U_CS);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmW);
    for (int i = 0; i < U_NA; ++i) { mbar_init(smem_u32(&bars->full_a[i]), 1); mbar_init(smem_u32(&bars->empty_a[i]), 2); }
    for (int i = 0; i < 4; ++i) { mbar_init(smem_u32(&bars->full_w[i]), 1); mbar_init(smem_u32(&bars->empty_w[i]), 2); }
    fence_barrier_init();
  }
  __syncthreads();

  // unit index -> (n tile, strip, image); the N tile is innermost so neighbouring CTAs share their input strip in L2
  auto decode = [&](int u, int& nt, int& st, int& b) {
    nt = u % P.tiles_n; u /= P.tiles_n;
    st = u % P.strips; b = u / P.strips;
  };

  if (warp >= 8) {
    // =============================== TMA producer ===============================
    setmaxnreg_dec40();
    if (warp == 8 && lane == 0) {
      int sa = 0; uint32_t pa = 0, pw_ = 0;
      for (int u = blockIdx.x; u < P.total_units; u += gridDim.x) {
        int nt, st, b;
        decode(u, nt, st, b);
        const int j0 = st * U_OC, n0 = nt * U_BN;
        for (int s = 0; s < P.steps; ++s) {
          for (int c0 = 0; c0 < P.Cin; c0 += BK) {
            for (int g = 0; g < 4; ++g) {
              if (g == 0 || g == 2) {                      // box of column shift -1 (groups 0, 1), then 0 (groups 2, 3)
                mbar_wait(smem_u32(&bars->empty_a[sa]), pa ^ 1u);
                const uint32_t fa = smem_u32(&bars->full_a[sa]);
                mbar_expect_tx(fa, (uint32_t)U_A_BYTES);
                tma_load_4d(s_a + (uint32_t)sa * U_A_BYTES, &tmX, fa, c0, j0 - (g == 0), s * U_PR - 1, b);   // zero fill = padding
                if (++sa == U_NA) { sa = 0; pa ^= 1u; }
              }
              mbar_wait(smem_u32(&bars->empty_w[g]), pw_ ^ 1u);
              const uint32_t fw = smem_u32(&bars->full_w[g]);
              mbar_expect_tx(fw, (uint32_t)(U_GTAPS[g] * U_W_BYTES));
              for (int k = 0; k < U_GTAPS[g]; ++k)
                tma_load_2d(s_w + (uint32_t)(U_GOFF[g] + k) * U_W_BYTES, &tmW, fw, c0, U_GTAP[g][k] * P.Cout + n0);
            }
            pw_ ^= 1u;
          }
        }
      }
    }
    return;
  }

  // =============================== consumer warpgroups ===============================
  setmaxnreg_inc232();
  const int wg = warp >> 2;                                    // warp k owns phase row k of the step (M rows 16k .. 16k+15)
  const int gid = lane >> 2, qd = lane & 3;
  const bool leader = (warp & 3) == 0 && lane == 0;
  const int cp = lane & 7, cg = lane >> 3;                     // epilogue: channels 2 cp, 2 cp + 1 of a slice; column pairs cg, cg + 4, ...
  int sa = 0; uint32_t pa = 0, pw_ = 0;
  for (int u = blockIdx.x; u < P.total_units; u += gridDim.x) {
    int nt, st, b;
    decode(u, nt, st, b);
    const int j0 = st * U_OC, n0 = nt * U_BN;
    for (int s = 0; s < P.steps; ++s) {
      float accx[U_BN], accy[U_BN];                            // [ee, eo] and [oe, oo] x 64 channels: two m64n128 fragments
      int prev_a = -1;
      uint32_t a_view = 0;
#pragma unroll 1
      for (int c0 = 0; c0 < P.Cin; c0 += BK) {
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          if (g == 0 || g == 2) {
            mbar_wait(smem_u32(&bars->full_a[sa]), pa);
            a_view = s_a + (uint32_t)sa * U_A_BYTES + wg * 4 * U_PC * 128;     // this warpgroup's 4 phase rows, row shift -1
          }
          mbar_wait(smem_u32(&bars->full_w[g]), pw_);
          const uint64_t da = gmma_desc(a_view + U_GROW[g] * U_PC * 128, 1024, LAYOUT_SW128);
          const uint64_t db = gmma_desc(s_w + (uint32_t)U_GOFF[g] * U_W_BYTES, 1024, LAYOUT_SW128);
          const uint64_t dby = db + (uint64_t)(U_GNX[g] * U_W_BYTES >> 4);         // the group's Y taps follow its X taps
          const int ny = U_GTAPS[g] - U_GNX[g];
          const uint32_t acc0 = (c0 > 0 || g > 0) ? 1u : 0u;  // the first chunk's shift (-1,-1) initialises both fragments
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const uint32_t ac = (acc0 | kk) ? 1u : 0u;
            if (U_GNX[g] == 2) wgmma_ss<128>(accx, da + kk * 2, db + kk * 2, ac);
            else wgmma_ss<64>(accx, da + kk * 2, db + kk * 2, ac);
            if (ny == 2) wgmma_ss<128>(accy, da + kk * 2, dby + kk * 2, ac);
            else if (ny == 1) wgmma_ss<64>(accy, da + kk * 2, dby + kk * 2, ac);
          }
          wgmma_commit();
          wgmma_wait<1>();                                     // the previous group's MMAs are done: release its slots
          if (c0 > 0 || g > 0) {
            named_bar_sync(1 + wg, 128);
            if (leader) {
              mbar_arrive(smem_u32(&bars->empty_w[(g + 3) & 3]));
              if (prev_a >= 0) mbar_arrive(smem_u32(&bars->empty_a[prev_a]));
            }
          }
          prev_a = (g == 1 || g == 3) ? sa : -1;               // last group reading this box
          if (g == 1 || g == 3) { if (++sa == U_NA) { sa = 0; pa ^= 1u; } }
        }
        pw_ ^= 1u;
      }
      wgmma_wait<0>();
      fence_regs<U_BN>(accx);
      fence_regs<U_BN>(accy);
      named_bar_sync(1 + wg, 128);
      if (leader) {
        mbar_arrive(smem_u32(&bars->empty_w[3]));
        mbar_arrive(smem_u32(&bars->empty_a[prev_a]));
      }

      // ---- epilogue: blur + demodulation, 16 channels at a time ----
      const int io = s * U_PR - 2 + warp;                      // output row pair of this warp
#pragma unroll
      for (int sl = 0; sl < U_BN / 16; ++sl) {
        float* my_row = stage + warp * U_PC * U_CS;
#pragma unroll
        for (int ph = 0; ph < 4; ++ph)
#pragma unroll
          for (int jj = 0; jj < 2; ++jj)
#pragma unroll
            for (int i = 0; i < 2; ++i)
              *reinterpret_cast<float2*>(my_row + (gid + 8 * i) * U_CS + ph * 16 + jj * 8 + 2 * qd) =
                  make_float2((ph < 2 ? accx : accy)[32 * (ph & 1) + 4 * (2 * sl + jj) + 2 * i], (ph < 2 ? accx : accy)[32 * (ph & 1) + 4 * (2 * sl + jj) + 2 * i + 1]);
        named_bar_sync(3, 256);
        if (io >= 0 && io < P.H) {
          // staged rows: 10-row index r = 0, 1 -> the previous step's last two phase rows (carry), r >= 2 -> this step's row r - 2
          auto row = [&](int r) -> const float* {
            return (r < 2 ? carry + (sl * 2 + r) * U_PC * U_CS : stage + (r - 2) * U_PC * U_CS) + 2 * cp;
          };
          const int ch = n0 + sl * 16 + 2 * cp;
          const float2 d = __ldg(reinterpret_cast<const float2*>(P.scale + (size_t)b * P.Cout + ch));
          const float2 f = make_float2(P.ag * d.x, P.ag * d.y);
          const int Wo = 2 * P.W;
#pragma unroll 1
          for (int p = cg; p < U_OC && j0 + p < P.W; p += 4) {   // phase column p = output column pair j0 + p
            float* y0 = y + (((size_t)b * 2 * P.H + 2 * io) * Wo + 2 * (j0 + p)) * P.Cout + ch;
            // horizontal: h = A + 3 B + 3 C + D with column phases E[c] = T_even[p + c], O[c] = T_odd[p + c - 1]:
            //   output column 2 (j0 + p):     O[0], E[0], O[1], E[1];  2 (j0 + p) + 1: E[0], O[1], E[1], O[2]
            float2 e0, o0, e1, o1;                             // output rows 2 io (e), 2 io + 1 (o) of both columns
            // five horizontally blurred rows, in the order that fixes the sums: Ho(io), He(io), Ho(io+1), He(io+1), Ho(io+2);
            // vertical: y[2i] = Ho(i) + 3 He(i) + 3 Ho(i+1) + He(i+1),  y[2i+1] = He(i) + 3 Ho(i+1) + 3 He(i+1) + Ho(i+2)
#pragma unroll
            for (int v = 0; v < 5; ++v) {
              // 10-row index of phase row io + v / 2; v = 0, 2, 4: row phase odd (oe, oo), v = 1, 3: even (ee, eo)
              const float* base = row(warp + v / 2) + ((v & 1) ? 0 : 32) + p * U_CS;
              const float2 E0 = *reinterpret_cast<const float2*>(base), O0 = *reinterpret_cast<const float2*>(base + 16);
              const float2 E1 = *reinterpret_cast<const float2*>(base + U_CS), O1 = *reinterpret_cast<const float2*>(base + U_CS + 16);
              const float2 O2 = *reinterpret_cast<const float2*>(base + 2 * U_CS + 16);
              float2 h0, h1;
              h0.x = ((O0.x + 3.f * E0.x) + 3.f * O1.x) + E1.x;
              h0.y = ((O0.y + 3.f * E0.y) + 3.f * O1.y) + E1.y;
              h1.x = ((E0.x + 3.f * O1.x) + 3.f * E1.x) + O2.x;
              h1.y = ((E0.y + 3.f * O1.y) + 3.f * E1.y) + O2.y;
              if (v == 0) { e0 = h0; e1 = h1; }
              else if (v == 1) {
                e0.x += 3.f * h0.x; e0.y += 3.f * h0.y; o0 = h0;
                e1.x += 3.f * h1.x; e1.y += 3.f * h1.y; o1 = h1;
              } else if (v == 2) {
                e0.x += 3.f * h0.x; e0.y += 3.f * h0.y; o0.x += 3.f * h0.x; o0.y += 3.f * h0.y;
                e1.x += 3.f * h1.x; e1.y += 3.f * h1.y; o1.x += 3.f * h1.x; o1.y += 3.f * h1.y;
              } else if (v == 3) {
                e0.x += h0.x; e0.y += h0.y; o0.x += 3.f * h0.x; o0.y += 3.f * h0.y;
                e1.x += h1.x; e1.y += h1.y; o1.x += 3.f * h1.x; o1.y += 3.f * h1.y;
              } else {
                o0.x += h0.x; o0.y += h0.y;
                o1.x += h1.x; o1.y += h1.y;
              }
            }
            *reinterpret_cast<float2*>(y0) = make_float2(e0.x * 0.015625f * f.x, e0.y * 0.015625f * f.y);
            *reinterpret_cast<float2*>(y0 + P.Cout) = make_float2(e1.x * 0.015625f * f.x, e1.y * 0.015625f * f.y);
            *reinterpret_cast<float2*>(y0 + (size_t)Wo * P.Cout) = make_float2(o0.x * 0.015625f * f.x, o0.y * 0.015625f * f.y);
            *reinterpret_cast<float2*>(y0 + (size_t)Wo * P.Cout + P.Cout) = make_float2(o1.x * 0.015625f * f.x, o1.y * 0.015625f * f.y);
          }
        }
        named_bar_sync(3, 256);                                // every read of this slice's carry and stage is done
        if (warp >= U_PR - 2) {                                // the last two phase rows become the next step's carry
          float* crow = carry + (sl * 2 + warp - (U_PR - 2)) * U_PC * U_CS;
#pragma unroll
          for (int ph = 0; ph < 4; ++ph)
#pragma unroll
            for (int jj = 0; jj < 2; ++jj)
#pragma unroll
              for (int i = 0; i < 2; ++i)
                *reinterpret_cast<float2*>(crow + (gid + 8 * i) * U_CS + ph * 16 + jj * 8 + 2 * qd) =
                    make_float2((ph < 2 ? accx : accy)[32 * (ph & 1) + 4 * (2 * sl + jj) + 2 * i], (ph < 2 ? accx : accy)[32 * (ph & 1) + 4 * (2 * sl + jj) + 2 * i + 1]);
        }
      }
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

static int launch_upconv(const float* x, const float* wt, const float* scale, float* y, int B, int H, int W, int Cin, int Cout,
                         float gain, cudaStream_t st) {
  CUtensorMap tmX, tmW;
  int rc;
  if ((rc = make_map_nhwc(&tmX, x, B, H, W, Cin, BK, U_PC, U_PR + 1))) return rc;
  if ((rc = make_map(&tmW, wt, (uint64_t)9 * Cout, (uint64_t)Cin, U_BN, BK, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  UParams P;
  P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout;
  P.strips = (W + U_OC - 1) / U_OC;
  P.steps = (H + 2 + U_PR - 1) / U_PR;            // output row pairs 8 s - 2 .. 8 s + 5 per step, 0 .. H - 1 in all
  P.tiles_n = Cout / U_BN;
  const long long units = (long long)B * P.strips * P.tiles_n;
  if (units > (1ll << 30)) { set_error("upconv3x3_blur: too many work units (%lld)", units); return GF_ERR_UNSUPPORTED; }
  P.total_units = (int)units;
  P.ag = 1.000352220f * gain;                      // alpha: the tensor core truncates x to TF32 (see launch_bn); the weights are pre-rounded
  P.scale = scale;
  // activation ring, weight stage, carry (4 slices x 2 rows), stage, barriers, alignment slack
  const int smem_bytes = U_NA * U_A_BYTES + U_WS_BYTES + 8 * U_PC * U_CS * 4 + U_PR * U_PC * U_CS * 4 + (int)sizeof(UBars) + 1024;
  if (smem_bytes > device_smem_optin()) { set_error("upconv3x3_blur: shared memory too small"); return GF_ERR_UNSUPPORTED; }
  GF_CUDA_OK(cudaFuncSetAttribute(upconv_blur_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  long long grid = device_sms();
  if (grid > P.total_units) grid = P.total_units;
  upconv_blur_tc_kernel<<<(unsigned)grid, U_THREADS, smem_bytes, st>>>(tmX, tmW, y, P);
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
  if (B <= 0 || H <= 0 || W <= 0 || H % cv::PH || W % cv::PW || Cin % cv::BK || Cout % 64 || Cin <= 0 || Cout <= 0) {
    set_error("gf_conv3x3_nhwc_tf32: needs positive sizes, H %% 8 == 0, W %% 16 == 0, Cin %% 32 == 0, Cout %% 64 == 0 (got B=%d H=%d W=%d Cin=%d Cout=%d)", B, H, W, Cin, Cout);
    return GF_ERR_UNSUPPORTED;
  }
  if (((uintptr_t)x & 15) || ((uintptr_t)wt & 15) || ((uintptr_t)y & 15)) { set_error("gf_conv3x3_nhwc_tf32: pointers must be 16-byte aligned"); return GF_ERR_INVALID; }
  int rc;
  if ((rc = check_device())) return rc;
  return cv::launch(x, wt, y, B, H, W, Cin, Cout, (cudaStream_t)stream);
}

extern "C" int gf_upconv3x3_blur_nhwc_tf32(const float* x, const float* wt, const float* scale, float* y, int B, int H, int W, int Cin,
                                           int Cout, float gain, void* stream) {
  if (!x || !wt || !scale || !y) { set_error("gf_upconv3x3_blur_nhwc_tf32: null pointer"); return GF_ERR_INVALID; }
  if (B <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || Cin % cv::BK || Cout % cv::U_BN) {
    set_error("gf_upconv3x3_blur_nhwc_tf32: needs positive sizes, Cin %% 32 == 0, Cout %% 64 == 0 (got B=%d H=%d W=%d Cin=%d Cout=%d)", B, H, W, Cin, Cout);
    return GF_ERR_UNSUPPORTED;
  }
  if (((uintptr_t)x & 15) || ((uintptr_t)wt & 15) || ((uintptr_t)y & 15) || ((uintptr_t)scale & 15)) {
    set_error("gf_upconv3x3_blur_nhwc_tf32: pointers must be 16-byte aligned"); return GF_ERR_INVALID;
  }
  int rc;
  if ((rc = check_device())) return rc;
  return cv::launch_upconv(x, wt, scale, y, B, H, W, Cin, Cout, gain, (cudaStream_t)stream);
}
