// Backward GEMMs of a linear layer y = x W^T (first pieces of the backward pass, cfg 5), without materialising a transpose:
//   wgrad (A_MN = true):   dW[M, N] (fp32) = A^T B,  A = dY [K, M] bf16 (tokens x out-features), B = X [K, N] (tokens x in-features)
//   dgrad (A_MN = false):  dX[M, N] (fp32) = A B,    A = dY [M, K] bf16 (tokens x out-features, K-major as in the forward GEMM),
//                                                    B = W [K, N] (out-features x in-features: the forward weight as stored)
// In both the B operand -- and in wgrad also A -- is contracted over its SLOW dimension:
// such operands are fed to wgmma as MN-major (transposed) tiles: TMA loads
// [64 tokens x 64 features] boxes (SWIZZLE_128B, 128-byte rows along the feature = M/N dimension) and the matrix descriptors
// carry leading-dimension byte offset = distance between 64-feature blocks, stride = 8 token rows.
// One CTA per 128 x 128 output tile, 4-stage TMA ring over 64-token K blocks, one consumer warpgroup (wgmma m64n128k16 on both
// 64-row halves, fp32 accumulators in registers) that stores straight from the accumulator fragments (dW is weight-sized: the
// epilogue is negligible next to the token-long mainloop).
// Reference arithmetic: torch autograd of nn.Linear (dW = dY^T X), checked in tests/gpu_diag.py.
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace wg {
constexpr int BM = 128, BN = 128, BK = 64, STAGES = 4;
constexpr int SUB = BK * 128;                    // [64 tokens x 64 features] bf16, 8 KB
constexpr int A_BYTES = (BM / 64) * SUB, B_BYTES = (BN / 64) * SUB;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // 32 KB
constexpr int OFF_BAR = STAGES * STAGE_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;
constexpr int THREADS = 256;
}  // namespace wg

template <bool A_MN>
__global__ void __launch_bounds__(wg::THREADS, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, float* __restrict__ out,
               int M, int N, int K, int ldc, int accumulate) {
  using namespace wg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* empty_bar = full_bar + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  // split-K over gridDim.z: the token dimension is long (8192 .. 400k rows) and the output weight-sized, so one CTA per tile would
  // leave most SMs idle; partial sums are added with atomics (the host zeroes the output first unless it accumulates anyway)
  const int k_blocks_all = (K + BK - 1) / BK;   // the K tail is zero-filled by TMA (out-of-bounds rows)
  const int kb_per = (k_blocks_all + gridDim.z - 1) / gridDim.z;
  const int kb0 = blockIdx.z * kb_per;
  const int kb1 = (kb0 + kb_per < k_blocks_all) ? kb0 + kb_per : k_blocks_all;
  const bool atomic_out = gridDim.z > 1;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA); prefetch_tmap(&tmB);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1, 50);
        uint8_t* sa = smem + stage * STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
        if constexpr (A_MN) {
#pragma unroll
          for (int j = 0; j < BM / 64; ++j) tma_load_2d(sa + j * SUB, &tmA, &full_bar[stage], m0 + 64 * j, kb * BK);
        } else {   // K-major A: one [128 rows x 64 K] box
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m0);
        }
#pragma unroll
        for (int j = 0; j < BN / 64; ++j) tma_load_2d(sa + A_BYTES + j * SUB, &tmB, &full_bar[stage], n0 + 64 * j, kb * BK);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
    float acc[2][BN / 2];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase, 51);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES), sb = sa + A_BYTES;
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {  // 16 token rows = 2048 B further down the MN-major tile
        const uint64_t db = make_desc_sw128(sb + kk * 2048, SUB, 1024);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t da = A_MN ? make_desc_sw128(sa + h * SUB + kk * 2048, SUB, 1024) : make_desc_sw128(sa + h * 8192 + kk * 32, 0, 1024);
          wgmma<BN, A_MN ? 1 : 0, 1>(acc[h], da, db, (kb > kb0) || (kk != 0));
        }
      }
      wg_commit();
      wg_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    wg_fence_acc(acc[0]);
    wg_fence_acc(acc[1]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        const int row = m0 + 64 * h + 16 * wq + qr + 8 * rs;
        if (row >= M) continue;
        float* dst = out + (size_t)row * ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + qc;
          if (col >= N) continue;   // N % 8 == 0
          float2 o = make_float2(acc[h][4 * j + 2 * rs], acc[h][4 * j + 2 * rs + 1]);
          if (atomic_out) {
            atomicAdd(dst + col, o.x); atomicAdd(dst + col + 1, o.y);
            continue;
          }
          if (accumulate) {   // gradient accumulation over images / sub-iterations (decoder_train.cu)
            const float2 t = *reinterpret_cast<const float2*>(dst + col);
            o.x += t.x; o.y += t.y;
          }
          *reinterpret_cast<float2*>(dst + col) = o;
        }
      }
    }
  }
}

template <bool A_MN>
static int launch_gemm_mn(const __nv_bfloat16* A, const __nv_bfloat16* B, int M, int N, int K, int lda, int ldb, float* out, int ldc,
                          cudaStream_t stream, int accumulate = 0) {
  using namespace wg;
  if (M <= 0 || N <= 0 || K <= 0) return set_error("gemm_tn: empty problem M=%d N=%d K=%d", M, N, K);
  // an MN-major operand is contracted over its rows: any K works (the K tail is zero-filled); a K-major A needs 16-byte rows
  if (M % 8 || N % 8 || (!A_MN && K % 8) || lda % 8 || ldb % 8 || ldc % 4)
    return set_error("gemm_tn: M, N (and K of a K-major operand), lda, ldb must be multiples of 8, ldc of 4");
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tn_kernel<A_MN>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return set_error("gemm_tn: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap tmA, tmB;   // MN-major operand: rows = contraction index, inner (contiguous) dimension = features, box 64 x 64
  if (A_MN ? make_tmap_bf16_2d(&tmA, A, K, M, lda, BK) : make_tmap_bf16_2d(&tmA, A, M, K, lda, BM)) return -1;
  if (make_tmap_bf16_2d(&tmB, B, K, N, ldb, BK)) return -1;
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN);
  {   // split-K until ~2 CTAs per SM (132 SMs), at least 8 k-blocks per split
    const int k_blocks = (K + BK - 1) / BK, tiles = grid.x * grid.y;
    int splits = (264 + tiles - 1) / tiles;
    if (splits > (k_blocks + 7) / 8) splits = (k_blocks + 7) / 8;
    if (splits < 1) splits = 1;
    const int per = (k_blocks + splits - 1) / splits;
    splits = (k_blocks + per - 1) / per;       // no empty split
    grid.z = splits;
    if (splits > 1 && !accumulate &&
        cudaMemset2DAsync(out, (size_t)ldc * 4, 0, (size_t)N * 4, M, stream) != cudaSuccess)
      return set_error("gemm_tn: memset failed");
  }
  prof_begin(stream, A_MN ? "gemm_tn (wgrad)" : "gemm_nn (dgrad)", 2.0 * M * N * K, (double)K * (M + N) * 2 + (double)M * N * 4);
  gemm_tn_kernel<A_MN><<<grid, THREADS, SMEM_BYTES, stream>>>(tmA, tmB, out, M, N, K, ldc, accumulate);
  prof_end(stream);
  LAUNCH_CHECK("gemm_tn");
  return 0;
}

int launch_gemm_tn(const __nv_bfloat16* A, const __nv_bfloat16* B, int M, int N, int K, int lda, int ldb, float* out, int ldc,
                   cudaStream_t stream, int accumulate) {
  return launch_gemm_mn<true>(A, B, M, N, K, lda, ldb, out, ldc, stream, accumulate);
}
int launch_gemm_nn(const __nv_bfloat16* A, const __nv_bfloat16* B, int M, int N, int K, int lda, int ldb, float* out, int ldc,
                   cudaStream_t stream) {
  return launch_gemm_mn<false>(A, B, M, N, K, lda, ldb, out, ldc, stream);
}

}  // namespace msam
