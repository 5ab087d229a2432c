// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epilogue(A[M,K] * W[N,K]^T)
//   * operands: TMA (SWIZZLE_128B boxes of 64 K-elements) -> shared memory ring (mbarrier full/empty)
//   * math:     one consumer warpgroup per 64-column group of the BN-wide tile; each issues wgmma m64n64k16 for both 64-row
//               halves of the 128-row tile (fp32 accumulators in registers) and keeps one k-block of MMAs in flight while
//               it releases the previous ring slot
//   * epilogue: straight from the accumulator fragments: bias / GELU(erf) / ReLU / residual (fp32 or bf16, row modulus), or a
//               fused LayerNorm over N=256 (row statistics reduced across the quad, then across the four column groups
//               through shared memory) -> fp32 / bf16 stores (a quad writes 16 or 32 contiguous bytes of a row).
// One CTA per SM; tiles are distributed round-robin, N-block fastest so that the CTAs that run concurrently share the
// same A row-block through L2.
//
// Replaces the nn.Linear / 1x1-conv / conv-transpose / patch-embed conv calls inside segment_anything's ImageEncoderViT /
// MaskDecoder that micro_sam reaches through util.py:674 (image_encoder) and SamPredictor.predict_torch (inference.py:248,
// instance_segmentation.py:361).
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;

enum { EPI_PLAIN = 0, EPI_LN256 = 1 };

template <int BN>
struct GemmCfg {
  static constexpr int NG = BN / 64;                    // consumer warpgroups = 64-column groups
  static constexpr int THREADS = 128 + NG * 128;        // warp 0: TMA producer (warps 1-3 idle), then the consumers
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : ((BN == 128) ? 6 : 8);
  static constexpr int OFF_BAR = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024 /*align slack*/;   // + 7 KB static (exch, rowp)
};

struct GemmParams {
  int M, N, K;
  const float* bias;      // [N] or null
  const void* residual;   // fp32 (or bf16 if res_bf16) [res_rows, ldr] or null; row index = row % res_rows
  int res_rows, ldr, res_bf16;
  void* out;
  int ldc;
  int out_fp32;
  int act;                // 0 none, 1 GELU(erf), 2 ReLU
  int act_after_res;      // apply act after the residual add
  const float* ln_gamma;  // fused LayerNorm epilogues
  const float* ln_beta;
  float ln_eps;
};

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// GELU(x) = 0.5 x (1 + erf(x / sqrt 2)) for values that are stored as bf16 or consumed by bf16-operand products:
// erf from Abramowitz-Stegun 7.1.25 (three terms, |abs err| <= 2.5e-5 -- measured 2.6e-5 on the GELU over [-10, 10],
// two orders below the bf16 rounding of the operands it feeds), branch-free with the approximate MUFU ops:
//   erf(|u|) = 1 - P(t) e^{-u^2}, t = 1 / (1 + p |u|)   =>   GELU(x) = max(x, 0) - |x| * (0.5 P(t)) * e^{-x^2 / 2}
// 12 instructions (2 MUFU) instead of ~40 for erff() + IEEE reciprocal.  The fp32-output paths keep erff().
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.47047f * 0.70710678118654752440f, z, 1.0f)));
  float poly = fmaf(0.5f * 0.7478556f, t, 0.5f * -0.0958798f);
  poly = fmaf(poly, t, 0.5f * 0.3480242f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * (x * -0.72134752044448170368f)));  // exp(-x^2/2)
  return fmaf(-z * poly, e, fmaxf(x, 0.0f));
}
__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == 1) return gelu_erf(x);
  if (act == 2) return fmaxf(x, 0.0f);
  return x;
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GemmCfg<BN>::THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int NG = Cfg::NG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  // statically declared so that the compiler emits LDS/STS (not generic LD/ST through the LG path)
  __shared__ __align__(16) float2 exch[2 * 4 * 128];  // EPI_LN256 statistics exchange, double buffered by tile parity
  __shared__ __align__(16) float rowp[768];           // [0,256) bias, [256,512) gamma, [512,768) beta (fused epilogues)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_blocks = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int n_blocks = (p.N + BN - 1) / BN;
  const int k_blocks = (p.K + GEMM_BK - 1) / GEMM_BK;
  const int num_tiles = m_blocks * n_blocks;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NG * 4);  // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  if constexpr (EPI != EPI_PLAIN) {  // N <= 256: per-column parameters -> shared memory (indexed by global column)
    for (int i = threadIdx.x; i < p.N && i < 256; i += Cfg::THREADS) {
      rowp[i] = p.bias ? p.bias[i] : 0.f;
      if constexpr (EPI == EPI_LN256) { rowp[256 + i] = p.ln_gamma[i]; rowp[512 + i] = p.ln_beta[i]; }
    }
  }
  __syncthreads();
  pdl_wait();      // the previous kernel's outputs (A, residual) are complete and visible from here on
  pdl_trigger();

  if (warp == 0) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 1);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * GEMM_BK, m_blk * GEMM_BM);
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * GEMM_BK, n_blk * BN);
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------ consumers: MMA + epilogue of one 64-column group
    const int grp = (warp - 4) >> 2;     // 64-column group of the tile
    const int wq = warp & 3;             // warp inside the warpgroup: fragment rows 16 wq .. 16 wq + 15 of each half
    const int qr = lane >> 2, qc = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int m_blk = tile / n_blocks, n_blk = tile % n_blocks;
      float acc[2][32];
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase, 3);
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES + grp * 64 * 128;
        wg_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          // +32 B per K=16 step inside the 128-B swizzle atom
          const uint64_t db = make_desc_sw128(sb + 32 * k, 0, 1024);
          wgmma<64>(acc[0], make_desc_sw128(sa + 32 * k, 0, 1024), db, (kb | k) != 0);
          wgmma<64>(acc[1], make_desc_sw128(sa + 8192 + 32 * k, 0, 1024), db, (kb | k) != 0);
        }
        wg_commit();
        wg_wait<1>();   // the MMAs of the previous k-block have read their slot
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      wg_fence_acc(acc[0]);
      wg_fence_acc(acc[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      const int colbase = n_blk * BN + grp * 64;
      if constexpr (EPI == EPI_PLAIN) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            const int row = m_blk * GEMM_BM + 64 * h + 16 * wq + qr + 8 * rs;
            if (row >= p.M) continue;
            const float* res_f = nullptr;
            const __nv_bfloat16* res_b = nullptr;
            if (p.residual) {
              const size_t off = (size_t)(row % p.res_rows) * p.ldr;
              if (p.res_bf16) res_b = reinterpret_cast<const __nv_bfloat16*>(p.residual) + off;
              else res_f = reinterpret_cast<const float*>(p.residual) + off;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = colbase + 8 * j + qc;
              if (col >= p.N) continue;   // N % 32 == 0: the pair is entirely inside or outside
              float x0 = acc[h][4 * j + 2 * rs], x1 = acc[h][4 * j + 2 * rs + 1];
              if (p.bias) {
                const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                x0 += b.x; x1 += b.y;
              }
              if (p.act_after_res) {
                // activation applied below, after the residual
              } else if (p.act == 1 && !p.out_fp32) {  // bf16 output: the fast erf is exact to well below the output rounding
                x0 = gelu_fast(x0); x1 = gelu_fast(x1);
              } else if (p.act) {
                x0 = apply_act(x0, p.act); x1 = apply_act(x1, p.act);
              }
              if (res_f) {
                const float2 r = *reinterpret_cast<const float2*>(res_f + col);
                x0 += r.x; x1 += r.y;
              } else if (res_b) {
                const uint32_t r = *reinterpret_cast<const uint32_t*>(res_b + col);
                x0 += __uint_as_float(r << 16); x1 += __uint_as_float(r & 0xffff0000u);
              }
              if (p.act_after_res && p.act) { x0 = apply_act(x0, p.act); x1 = apply_act(x1, p.act); }
              if (p.out_fp32)
                *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + (size_t)row * p.ldc + col) = make_float2(x0, x1);
              else
                *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldc + col) = pack_bf16(x0, x1);
            }
          }
        }
      } else {
        // ---- fused LayerNorm over the full 256-wide row (N == BN == 256): exact two-pass statistics per 64-column group
        // (quad shuffles), combined across the four groups with Chan's formula through shared memory.
        float2* ex = exch + (it & 1) * (NG * 128);
        float mean_r[4], rstd_r[4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            const int rt = 64 * h + 16 * wq + qr + 8 * rs;
            const int row = m_blk * GEMM_BM + rt;
            const bool has_res = p.residual != nullptr && row < p.M;
            const __nv_bfloat16* rp =
                has_res ? reinterpret_cast<const __nv_bfloat16*>(p.residual) + (size_t)(row % p.res_rows) * p.ldr : nullptr;
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = colbase + 8 * j + qc;
              float& x0 = acc[h][4 * j + 2 * rs];
              float& x1 = acc[h][4 * j + 2 * rs + 1];
              x0 += rowp[col]; x1 += rowp[col + 1];
              if (has_res) {
                const uint32_t r = *reinterpret_cast<const uint32_t*>(rp + col);
                x0 += __uint_as_float(r << 16); x1 += __uint_as_float(r & 0xffff0000u);
              }
              s += x0 + x1;
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            const float mean_g = s * (1.0f / 64);
            float q = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float d0 = acc[h][4 * j + 2 * rs] - mean_g, d1 = acc[h][4 * j + 2 * rs + 1] - mean_g;
              q = fmaf(d0, d0, fmaf(d1, d1, q));
            }
            q += __shfl_xor_sync(0xffffffffu, q, 1);
            q += __shfl_xor_sync(0xffffffffu, q, 2);
            if ((lane & 3) == 0) ex[grp * 128 + rt] = make_float2(mean_g, q);
          }
        }
        named_bar_sync(1, NG * 128);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            const int rt = 64 * h + 16 * wq + qr + 8 * rs;
            float mean = 0.f;
            float2 st[NG];
#pragma unroll
            for (int g = 0; g < NG; ++g) { st[g] = ex[g * 128 + rt]; mean += st[g].x; }
            mean *= (1.0f / NG);
            float m2 = 0.f;
#pragma unroll
            for (int g = 0; g < NG; ++g) { const float d = st[g].x - mean; m2 += st[g].y + d * d * 64; }
            mean_r[2 * h + rs] = mean;
            rstd_r[2 * h + rs] = rsqrtf(m2 * (1.0f / (NG * 64)) + p.ln_eps);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            const int row = m_blk * GEMM_BM + 64 * h + 16 * wq + qr + 8 * rs;
            if (row >= p.M) continue;
            const float mean = mean_r[2 * h + rs], rstd = rstd_r[2 * h + rs];
            __nv_bfloat16* orow = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldc;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = colbase + 8 * j + qc;
              const float y0 = (acc[h][4 * j + 2 * rs] - mean) * rstd * rowp[256 + col] + rowp[512 + col];
              const float y1 = (acc[h][4 * j + 2 * rs + 1] - mean) * rstd * rowp[256 + col + 1] + rowp[512 + col + 1];
              *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16(y0, y1);
            }
          }
        }
      }
    }
  }
}

template <int BN, int EPI>
static int launch_gemm_bn(const GemmArgs& a, int num_sms, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e =
        cudaFuncSetAttribute(gemm_bf16_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
    if (e != cudaSuccess) return set_error("gemm: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap tmA, tmB;
  if (make_tmap_bf16_2d(&tmA, a.A, a.M, a.K, a.lda, GEMM_BM)) return -1;
  if (make_tmap_bf16_2d(&tmB, a.W, a.N, a.K, a.ldw, BN)) return -1;
  GemmParams p;
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.bias = a.bias;
  p.residual = a.residual;
  p.res_bf16 = a.res_bf16;
  p.res_rows = a.res_rows > 0 ? a.res_rows : a.M;
  p.ldr = a.ldr > 0 ? a.ldr : a.N;
  p.out = a.out;
  p.ldc = a.ldc > 0 ? a.ldc : a.N;
  p.out_fp32 = a.out_fp32;
  p.act = a.act;
  p.act_after_res = a.act_after_res;
  p.ln_gamma = a.ln_gamma; p.ln_beta = a.ln_beta; p.ln_eps = a.ln_eps;
  const int tiles = ((a.M + GEMM_BM - 1) / GEMM_BM) * ((a.N + BN - 1) / BN);
  const int grid = tiles < num_sms ? tiles : num_sms;
  {
    const double out_b = (double)a.M * a.N * (a.out_fp32 ? 4 : 2);
    const double res_b = a.residual ? (double)(a.res_rows > 0 ? a.res_rows : a.M) * a.N * (a.res_bf16 ? 2 : 4) : 0.0;
    const char* nm = EPI == EPI_LN256 ? "gemm_bf16<256,ln256>"
                     : (a.K >= 512 ? "gemm_bf16 plain K>=512" : "gemm_bf16 plain K<512");
    prof_begin(stream, nm, 2.0 * a.M * a.N * a.K, (double)a.M * a.K * 2 + (double)a.N * a.K * 2 + out_b + res_b);
  }
  launch_pdl(gemm_bf16_kernel<BN, EPI>, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, stream, tmA, tmB, p);
  prof_end(stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("gemm launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

int launch_gemm(const GemmArgs& a, int num_sms, cudaStream_t stream) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return set_error("gemm: empty problem M=%d N=%d K=%d", a.M, a.N, a.K);
  if (a.N % 32 != 0) return set_error("gemm: N=%d must be a multiple of 32", a.N);
  if (a.K % 8 != 0 || a.lda % 8 != 0 || a.ldw % 8 != 0)
    return set_error("gemm: K/lda/ldw must be multiples of 8 (16-byte TMA strides)");
  if (a.epi == EPI_LN256) {
    if (a.N != 256 || a.out_fp32 || !a.ln_gamma || !a.ln_beta || a.act)
      return set_error("gemm: fused LN needs N=256, bf16 out, gamma/beta, no act");
    if (a.residual && !a.res_bf16) return set_error("gemm: fused LN takes a bf16 residual");
    return launch_gemm_bn<256, EPI_LN256>(a, num_sms, stream);
  }
  if (a.epi != EPI_PLAIN) return set_error("gemm: unknown epilogue %d", a.epi);
  if ((a.ldc > 0 ? a.ldc : a.N) % 2 != 0) return set_error("gemm: ldc must be even");
  // BN=256 reads the A tile once per 256 output columns; fall back to 128 / 64 when N is not a multiple (or is small), to
  // avoid wasted columns.
  if (a.N % 256 == 0) return launch_gemm_bn<256, EPI_PLAIN>(a, num_sms, stream);
  if (a.N % 128 == 0) return launch_gemm_bn<128, EPI_PLAIN>(a, num_sms, stream);
  return launch_gemm_bn<64, EPI_PLAIN>(a, num_sms, stream);
}

}  // namespace msam
