// gf_tc_gemm.cu -- small TF32 tensor-core GEMM for the per-image products between the big kernels of a layer:
//     C[M,N] = alpha * A[M,K] . B[K,N] + E[(row % emod), :] + v[:]          (A, B row-major, lda = K, ldb = N)
// used (TF32 mode only) for KPALL = keys . AK + CK, MALL = Y . AM + CM and the duplex centroids Xbar . Wv2 + bv2
// (reference side, expected src/training/network.py: the K / V dense_layer calls of transformer_layer).  M = B*k is a few
// thousand rows, far too few for the CUDA-core SGEMM (gf_fold.cu) to fill the GPU at C = 512.
// One 64 x 64 output tile per CTA (one warpgroup), BK = 32, two shared-memory buffers:
//   all 128 threads stage the next A tile [64 x 32] and the next B tile TRANSPOSED to [64 n x 32 k] (wgmma takes 32-bit
//   operands K-major only; B row-major [K,N] is N-major) into 128-byte-swizzled K-major layouts while the current
//   tile's 8 wgmma m64n32k8 run; the epilogue goes from registers to global (alpha, bias rows).
// Out-of-range rows / columns / k are zero-filled at staging and masked at the store.  Operands are truncated to TF32 by the
// tensor core; alpha carries the mean-truncation compensation of both operands (gf_fold.cu: GF_TF32_TRUNC_COMP).
#include <stdlib.h>
#include "gf_common.cuh"
#include "gf_tc_common.cuh"

namespace gf {
namespace tcg {

using namespace tc;

constexpr int BM = 64, BN = 64, BK = 32;
constexpr int TILE_BYTES = 64 * 128;              // [64 rows x 32 fp32], either operand
constexpr int NUM_THREADS = 128;

__device__ __forceinline__ uint32_t sw_off(int row, int k) {    // K-major SWIZZLE_128B offset of (row, k), k < 32
  return (uint32_t)(row * 128 + ((((k >> 2) ^ (row & 7))) << 4) + (k & 3) * 4);
}

__global__ void __launch_bounds__(NUM_THREADS)
gemm_tc_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ Cm, int ldc,
               int M, int N, int K, float alpha, const float* __restrict__ E, int lde, int emod, const float* __restrict__ v) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t s_base = smem_u32(smem);                      // [buf][A | B]
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, gid = lane >> 2, qd = lane & 3;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int nk = (K + BK - 1) / BK;

  float4 ra[4], rb[4];
  auto load = [&](int kt) {
    const int k0 = kt * BK;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + NUM_THREADS * i;
      const int ar = idx >> 3, ac = (idx & 7) * 4;              // A: row, first k
      ra[i] = (m0 + ar < M && k0 + ac < K) ? __ldg(reinterpret_cast<const float4*>(A + (size_t)(m0 + ar) * K + k0 + ac))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
      const int bk = idx >> 4, bn = (idx & 15) * 4;             // B: k row, first n
      rb[i] = (k0 + bk < K && n0 + bn < N) ? __ldg(reinterpret_cast<const float4*>(B + (size_t)(k0 + bk) * N + n0 + bn))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store = [&](int buf) {
    uint8_t* sa = smem + buf * 2 * TILE_BYTES;
    uint8_t* sb = sa + TILE_BYTES;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + NUM_THREADS * i;
      const int ar = idx >> 3, ac = (idx & 7) * 4;
      *reinterpret_cast<float4*>(sa + sw_off(ar, ac)) = ra[i];
      const int bk = idx >> 4, bn = (idx & 15) * 4;
      *reinterpret_cast<float*>(sb + sw_off(bn, bk)) = rb[i].x;
      *reinterpret_cast<float*>(sb + sw_off(bn + 1, bk)) = rb[i].y;
      *reinterpret_cast<float*>(sb + sw_off(bn + 2, bk)) = rb[i].z;
      *reinterpret_cast<float*>(sb + sw_off(bn + 3, bk)) = rb[i].w;
    }
    fence_proxy_async();                                         // generic-proxy writes -> wgmma (async proxy)
  };

  float acc[2][16];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
  load(0);
  store(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    const uint32_t sa = s_base + buf * 2 * TILE_BYTES, sb = sa + TILE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t da = gmma_desc(sa + kk * 32, 1024, LAYOUT_SW128);
      wgmma_ss_n32(acc[0], da, gmma_desc(sb + kk * 32, 1024, LAYOUT_SW128), 1u);
      wgmma_ss_n32(acc[1], da, gmma_desc(sb + 32 * 128 + kk * 32, 1024, LAYOUT_SW128), 1u);
    }
    wgmma_commit();
    if (kt + 1 < nk) {                                           // the other buffer was released by the barrier of the last step
      load(kt + 1);
      store(buf ^ 1);
    }
    wgmma_wait<0>();
    __syncthreads();
  }
  fence_regs<16>(acc[0]); fence_regs<16>(acc[1]);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = m0 + 16 * w + gid + 8 * i;
    if (row >= M) continue;
    const float* erow = E ? E + (size_t)(row % emod) * lde : nullptr;
    float* crow = Cm + (size_t)row * ldc;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jb = 0; jb < 4; ++jb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = n0 + h * 32 + 8 * jb + 2 * qd + e;
          if (c < N) crow[c] = alpha * acc[h][4 * jb + 2 * i + e] + (erow ? erow[c] : 0.f) + (v ? v[c] : 0.f);
        }
  }
}

}  // namespace tcg

// lda == K and ldb == N (dense row-major operands), rows of A and B 16-byte aligned
bool gemm_tc_ok(int M, int N, int K, const float* A, const float* B, const float* Cm, int ldc) {
  if (M < 1 || N < 32 || K < 4) return false;
  if ((K & 3) || (N & 3)) return false;
  if (((uintptr_t)A & 15) || ((uintptr_t)B & 15) || ((uintptr_t)Cm & 15) || (ldc & 3)) return false;
  return true;
}

int gemm_tc(cudaStream_t st, int M, int N, int K, const float* A, const float* B, float* Cm, int ldc, float alpha,
            const float* E, int lde, int emod, const float* v) {
  using namespace tcg;
  const int smem_bytes = 4 * TILE_BYTES + 1024;
  GF_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  if (emod < 1) emod = 1;
  // both operands are truncated to TF32 by the tensor core: compensate the mean truncation bias of each (0.7213 * 2^-11)
  const float comp = 1.000352220f * 1.000352220f;
  gemm_tc_kernel<<<dim3((N + BN - 1) / BN, (M + BM - 1) / BM), NUM_THREADS, smem_bytes, st>>>(A, B, Cm, ldc, M, N, K, alpha * comp, E, lde, emod, v);
  GF_LAUNCH_OK();
  return GF_OK;
}

}  // namespace gf
