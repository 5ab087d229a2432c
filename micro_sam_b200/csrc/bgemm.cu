// Batched small-K / small-N GEMM for the attention backward pass (cfg 5): one launch covers every (window | image, head) pair.
//   C[w, h] (M x N, fp32)  (+)=  alpha * op(A[w, h]) * op(B[w, h])
// Operands are bf16 views described by 4-D TMA tensor maps (feature, head, row, outer): a head is a column slice of a packed
// buffer such as qkv [rows, 3 * heads * d], a window is a row slice, and out-of-range features (head_dim 80: columns 80..127 of
// the second 64-column box) or rows (196-token windows in 64-row boxes) are ZERO-FILLED by the TMA unit because they lie outside
// the (feature, row) extents of the map -- which a 2-D map over the packed buffer cannot do (the neighbours are in bounds).
// Each operand is either K-major (contraction along the contiguous feature dimension: S = Q K^T, dP = dO V^T, T = Q R^T) or
// MN-major (contraction along the rows: dV = P^T dO, dK = dS^T Q, dQ = dS K), as in gemm_tn.cu.
// One CTA per 128 x 128 output tile and batch entry; 3-stage TMA ring over 64-wide contraction blocks; one consumer warpgroup
// (wgmma m64n128k16 on both 64-row halves, fp32 accumulators in registers).
// Reference arithmetic: torch autograd of (q @ k^T, softmax, @ v) in oracle/sam_ref.py:Attention; checked in tests/gpu_diag.py.
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace bg {
constexpr int BM = 128, BN = 128, BK = 64, STAGES = 3;
constexpr int SUB = 64 * 128;                    // [64 rows x 64 bf16], 8 KB
constexpr int A_BYTES = 2 * SUB, B_BYTES = 2 * SUB;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;   // 32 KB
constexpr int OFF_BAR = STAGES * STAGE_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 128 + 1024;
constexpr int THREADS = 256;
}  // namespace bg

struct BgParams {
  float* out;             // fp32 [outer, heads, M, ldc]
  long o_wstride, o_hstride;
  int ldc, M, N, K, heads;
  int a_hmul, a_wmul, b_hmul, b_wmul;   // 0: the operand is shared along that batch axis
  float alpha;
  int accumulate;
};

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(bg::THREADS, 1)
bgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const BgParams p) {
  using namespace bg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* empty_bar = full_bar + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int h = blockIdx.z % p.heads, w = blockIdx.z / p.heads;
  const int k_blocks = (p.K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA); prefetch_tmap(&tmB);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      const int ah = h * p.a_hmul, aw = w * p.a_wmul, bh = h * p.b_hmul, bw = w * p.b_wmul;
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1, 60);
        uint8_t* sa = smem + stage * STAGE_BYTES;
        uint8_t* sb = sa + A_BYTES;
        mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
        if constexpr (A_MN) {   // [64 contraction rows x 64 M-features] x 2
          tma_load_4d(sa, &tmA, &full_bar[stage], m0, ah, kb * BK, aw);
          tma_load_4d(sa + SUB, &tmA, &full_bar[stage], m0 + 64, ah, kb * BK, aw);
        } else {                // [128 M-rows x 64 contraction features] as two 64-row boxes
          tma_load_4d(sa, &tmA, &full_bar[stage], kb * BK, ah, m0, aw);
          tma_load_4d(sa + SUB, &tmA, &full_bar[stage], kb * BK, ah, m0 + 64, aw);
        }
        if constexpr (B_MN) {
          tma_load_4d(sb, &tmB, &full_bar[stage], n0, bh, kb * BK, bw);
          tma_load_4d(sb + SUB, &tmB, &full_bar[stage], n0 + 64, bh, kb * BK, bw);
        } else {
          tma_load_4d(sb, &tmB, &full_bar[stage], kb * BK, bh, n0, bw);
          tma_load_4d(sb + SUB, &tmB, &full_bar[stage], kb * BK, bh, n0 + 64, bw);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
    float acc[2][BN / 2];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = 0; kb < k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase, 61);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES), sb = sa + A_BYTES;
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk) {
        // MN-major: 16 contraction rows further = +2048 B, 64-feature blocks SUB apart.  K-major: +32 B inside the 128-B row;
        // the two 64-row boxes are contiguous (8-row groups 1024 B apart)
        const uint64_t db = B_MN ? make_desc_sw128(sb + kk * 2048, SUB, 1024) : make_desc_sw128(sb + kk * 32, 0, 1024);
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint64_t da = A_MN ? make_desc_sw128(sa + hf * SUB + kk * 2048, SUB, 1024) : make_desc_sw128(sa + hf * SUB + kk * 32, 0, 1024);
          wgmma<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[hf], da, db, (kb | kk) != 0);
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
    float* obase = p.out + (long)w * p.o_wstride + (long)h * p.o_hstride;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        const int row = m0 + 64 * hf + 16 * wq + qr + 8 * rs;
        if (row >= p.M) continue;
        float* dst = obase + (size_t)row * p.ldc;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + qc;
          if (col >= p.N) continue;   // N % 4 == 0
          float2 o = make_float2(acc[hf][4 * j + 2 * rs] * p.alpha, acc[hf][4 * j + 2 * rs + 1] * p.alpha);
          if (p.accumulate) {
            const float2 t = *reinterpret_cast<const float2*>(dst + col);
            o.x += t.x; o.y += t.y;
          }
          *reinterpret_cast<float2*>(dst + col) = o;
        }
      }
    }
  }
}

// bf16 4-D view: element (f, h, r, w) at base + f + h * hs + r * rs + w * wst  (strides in elements; hs, rs, wst multiples of 8).
// Box = [64 features x 1 head x 64 rows x 1 outer], SWIZZLE_128B, out-of-bounds elements zero-filled.
static int make_tmap_bf16_4d(CUtensorMap* out, const void* gptr, uint64_t feats, uint64_t heads, uint64_t rows, uint64_t outer,
                             uint64_t hs, uint64_t rs, uint64_t wst) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(gptr) & 15) != 0 || hs % 8 || rs % 8 || wst % 8)
    return set_error("bgemm: operand base / strides must be 16-byte aligned");
  // degenerate axes still need a non-zero, 16-byte-multiple stride
  if (hs == 0) hs = 8;
  if (wst == 0) wst = 8;
  cuuint64_t dims[4] = {feats, heads, rows, outer};
  cuuint64_t strides[3] = {hs * 2, rs * 2, wst * 2};
  cuuint32_t box[4] = {64, 1, 64, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(gptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error("bgemm: cuTensorMapEncodeTiled failed (%d) dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu)", (int)r,
                     (unsigned long long)feats, (unsigned long long)heads, (unsigned long long)rows, (unsigned long long)outer,
                     (unsigned long long)hs, (unsigned long long)rs, (unsigned long long)wst);
  return 0;
}

template <bool A_MN, bool B_MN>
static int launch_bgemm_t(const BGemmArgs& a, cudaStream_t stream) {
  using namespace bg;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(bgemm_kernel<A_MN, B_MN>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return set_error("bgemm: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  // the map extents are the logical (feature, row) extents of ONE batch entry: features = the operand's contiguous dimension
  // (K when K-major, M / N when MN-major), rows = the other one
  CUtensorMap tmA, tmB;
  const uint64_t a_feats = A_MN ? a.M : a.K, a_rows = a.a_rows_valid > 0 ? a.a_rows_valid : (A_MN ? a.K : a.M);
  const uint64_t b_feats = B_MN ? a.N : a.K, b_rows = a.b_rows_valid > 0 ? a.b_rows_valid : (B_MN ? a.K : a.N);
  if (make_tmap_bf16_4d(&tmA, a.A, a_feats, a.a_hstride ? a.heads : 1, a_rows, a.a_wstride ? a.outer : 1, a.a_hstride, a.lda,
                        a.a_wstride)) return -1;
  if (make_tmap_bf16_4d(&tmB, a.B, b_feats, a.b_hstride ? a.heads : 1, b_rows, a.b_wstride ? a.outer : 1, a.b_hstride, a.ldb,
                        a.b_wstride)) return -1;
  BgParams p;
  p.out = a.out; p.o_wstride = a.o_wstride; p.o_hstride = a.o_hstride; p.ldc = a.ldc; p.M = a.M; p.N = a.N; p.K = a.K;
  p.heads = a.heads; p.a_hmul = a.a_hstride ? 1 : 0; p.a_wmul = a.a_wstride ? 1 : 0; p.b_hmul = a.b_hstride ? 1 : 0;
  p.b_wmul = a.b_wstride ? 1 : 0; p.alpha = a.alpha; p.accumulate = a.accumulate;
  dim3 grid((a.M + BM - 1) / BM, (a.N + BN - 1) / BN, a.heads * a.outer);
  prof_begin(stream, "bgemm (attention backward)", 2.0 * a.M * a.N * a.K * a.heads * a.outer,
             ((double)a.M * a.K + (double)a.N * a.K) * 2 * a.heads * a.outer + (double)a.M * a.N * 4 * a.heads * a.outer);
  bgemm_kernel<A_MN, B_MN><<<grid, THREADS, SMEM_BYTES, stream>>>(tmA, tmB, p);
  prof_end(stream);
  LAUNCH_CHECK("bgemm");
  return 0;
}

int launch_bgemm(const BGemmArgs& a, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0 || a.heads <= 0 || a.outer <= 0) return set_error("bgemm: empty problem");
  if (a.N % 4 || a.ldc % 4 || a.lda % 8 || a.ldb % 8) return set_error("bgemm: N, ldc must be multiples of 4, lda / ldb of 8");
  if ((long)a.heads * a.outer > 65535) return set_error("bgemm: %ld batch entries exceed the grid limit", (long)a.heads * a.outer);
  if (a.a_mn) return a.b_mn ? launch_bgemm_t<true, true>(a, stream) : launch_bgemm_t<true, false>(a, stream);
  return a.b_mn ? launch_bgemm_t<false, true>(a, stream) : launch_bgemm_t<false, false>(a, stream);
}

}  // namespace msam
