// Fused output up-scaling + hyper-network mask product of the mask decoder (MaskDecoder.predict_masks after the
// transformer, restated in oracle/sam_ref.py:  upscaled = GELU(convT2(GELU(LN2d(convT1(src)))));  masks = hyper_in @ upscaled):
//
//   keys tile [128 tokens x 256]  --MMA1-->  D1 [128 x (4 sub-pixels x 64 ch)]        conv-transpose 1 (k2 s2) as a GEMM
//        E1: + bias, LayerNorm2d over the 64 channels of a (token, sub-pixel), GELU  -> A2_s [128 x 64] fp16 in shared memory
//   A2_s  --MMA2-->  D2 [128 x (4 sub-sub-pixels x 32 ch)]  (s = 0..3)               conv-transpose 2 (k2 s2) as a GEMM
//        E2: + bias, GELU, dot product with the prompt's hyper-network vectors (<= 4 masks x 32 ch) -> low-res logits
//
// so neither the 64-channel up-scaled embedding (2 MB per prompt written + read by the two-kernel version) nor the
// 32-channel one ever leaves the SM: per prompt the kernel reads 2 MB of `keys` and writes 0.25 MB per mask.
// The element-wise epilogues -- 3.2 G GELUs per 32x32-grid tile, instruction-issue bound in fp32 -- run in PACKED fp16x2
// arithmetic:
//   GELU(x) = 0.5 x (1 + erf(x / sqrt 2)),  erf(x / sqrt 2) ~ tanh(x (a + b x^2))   (minimax a, b: |err| <= 2.7e-4; with the
//   fp16 rounding of the 6-instruction chain the N(0,1)-weighted rms error is 2.9e-4 -- a quarter of the bf16 rounding the
//   two-kernel version applied when it stored the intermediate), one MUFU (tanh.approx.f16x2) per TWO elements,
// the intermediate operand A2 and the conv-transpose-2 weights are fp16 (11-bit mantissa instead of bf16's 8), the hyper
// product accumulates 2 x 8 fp16x2 FMAs per mask and finishes in fp32.
//
// CTA = 4 warpgroups (warpgroup s: sub-pixel s = D1 columns [64 s, 64 s + 64), its A2_s tile and D2_s; wgmma accumulators in
// registers, epilogues straight from the fragments with row reductions across the quad of lanes that shares a row) + 1 TMA
// warp, persistent over a contiguous range of (prompt, 128-token tile) items.
#include <cuda_fp16.h>

#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace up {
constexpr int STAGES = 2;
constexpr int SUBA = 128 * 128;                 // [128 rows x 64 x 16-bit] SWIZZLE_128B sub-tile (16 KB)
constexpr int SUBW = 256 * 128;                 // conv-transpose-1 weight K-slice [256 x 64] bf16 (32 KB)
constexpr int STAGE_BYTES = SUBA + SUBW;
constexpr int OFF_A2 = STAGES * STAGE_BYTES;    // 4 x [128 x 64] fp16
constexpr int OFF_W2 = OFF_A2 + 4 * SUBA;       // [128 x 64] fp16
constexpr int OFF_BAR = OFF_W2 + SUBA;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
constexpr int THREADS = 512 + 32;
constexpr int TILES = 32;                       // 4096 image tokens / 128
}  // namespace up

struct UpParams {
  int P, nm, m0;
  const float* b1;      // [256] conv-transpose-1 bias per (sub-pixel, channel)
  const float* gamma;   // [64] LayerNorm2d
  const float* beta;
  float eps;
  const float* b2;      // [128] conv-transpose-2 bias per (sub-sub-pixel, channel)
  const float* hyper;   // [P, 4, 32]
  float* out;           // [P, nm, 256, 256]
};

__device__ __forceinline__ __half2 tanh_h2(__half2 x) {
  uint32_t r, a = *reinterpret_cast<uint32_t*>(&x);
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(r) : "r"(a));
  return *reinterpret_cast<__half2*>(&r);
}
__device__ __forceinline__ __half2 gelu_h2(__half2 v) {
  const __half2 a = __floats2half2_rn(0.80015708f, 0.80015708f), b = __floats2half2_rn(0.03470089f, 0.03470089f);
  const __half2 hlf = __floats2half2_rn(0.5f, 0.5f);
  const __half2 t = __hfma2(b, __hmul2(v, v), a);
  const __half2 th = tanh_h2(__hmul2(v, t));
  const __half2 h = __hmul2(v, hlf);
  return __hfma2(h, th, h);
}
__device__ __forceinline__ uint32_t h2u(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }

__global__ void __launch_bounds__(up::THREADS, 1)
upscale_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                     const __grid_constant__ CUtensorMap tmW2, const UpParams p) {
  using namespace up;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* w2_full = empty_bar + STAGES;
  __shared__ __align__(16) float b1_s[256];
  __shared__ __align__(16) __half2 gb_s[64];          // [0,32) gamma pairs, [32,64) beta pairs
  __shared__ __align__(16) __half2 b2_s[64];          // conv-transpose-2 bias pairs, index ss*16 + i

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long total = (long)p.P * TILES;
  const int it_begin = (int)(total * blockIdx.x / gridDim.x), it_end = (int)(total * (blockIdx.x + 1) / gridDim.x);
  const int n_items = it_end - it_begin;

  if (warp == 16 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmW1); prefetch_tmap(&tmW2);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 16); }
    mbar_init(w2_full, 1);
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 256; i += THREADS) b1_s[i] = p.b1[i];
  for (int i = threadIdx.x; i < 32; i += THREADS) {
    gb_s[i] = __floats2half2_rn(p.gamma[2 * i], p.gamma[2 * i + 1]);
    gb_s[32 + i] = __floats2half2_rn(p.beta[2 * i], p.beta[2 * i + 1]);
  }
  for (int i = threadIdx.x; i < 64; i += THREADS) b2_s[i] = __floats2half2_rn(p.b2[2 * i], p.b2[2 * i + 1]);
  __syncthreads();

  if (warp == 16) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0 && n_items > 0) {
      mbar_expect_tx(w2_full, SUBA);
      tma_load_2d(smem + OFF_W2, &tmW2, w2_full, 0, 0);
      int stage = 0;
      uint32_t phase = 0;
      for (int item = it_begin; item < it_end; ++item) {
        const int row0 = (item / TILES) * 4096 + (item % TILES) * 128;
        if (item + 2 < it_end) {  // keys tile of a later item -> L2
          const int pr = ((item + 2) / TILES) * 4096 + ((item + 2) % TILES) * 128;
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_prefetch_2d(&tmX, 64 * j, pr);
        }
        for (int j = 0; j < 4; ++j) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 40);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          tma_load_2d(sa, &tmX, &full_bar[stage], 64 * j, row0);
          tma_load_2d(sa + SUBA, &tmW1, &full_bar[stage], 64 * j, 0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------ warpgroup s = sub-pixel s.  Fragment element i of a thread:
  // row 64 h + 16 wq + qr + 8 ((i >> 1) & 1) of the 64-row half h, column 8 (i >> 2) + qc + (i & 1).
  const int sp = warp >> 2, wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
  const uint32_t a2 = smem_u32(smem + OFF_A2 + sp * SUBA), aw2 = smem_u32(smem + OFF_W2);
  const float inv64 = 1.0f / 64.0f;
  int stage = 0;
  uint32_t phase = 0;
  if (n_items > 0) mbar_wait(w2_full, 0, 45);
  for (int it = 0; it < n_items; ++it) {
    const int item = it_begin + it, pp = item / TILES, rt = item % TILES;
    // ---- MMA1: D1[:, 64 sp .. 64 sp + 64) = keys tile . W1[64 sp .., :]^T
    float d1[2][32];
    for (int j = 0; j < 4; ++j) {
      mbar_wait(&full_bar[stage], phase, 42);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
      const uint64_t db = make_desc_sw128(sa + SUBA + sp * 8192, 0, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma<64>(d1[h], make_desc_sw128(sa + h * 8192, 0, 1024) + 2 * k, db + 2 * k, (j | k) != 0);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(d1[0]);
      wg_fence_acc(d1[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    // ---- E1: (row, sub-pixel sp): + bias, LayerNorm over 64 channels, GELU -> A2_sp (fp16, K-major SW128)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        const int r = 64 * h + 16 * wq + qr + 8 * rs;
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = d1[h][4 * j + 2 * rs + e];
            x += b1_s[64 * sp + 8 * j + qc + e];
            s1 += x;
            s2 = fmaf(x, x, s2);
          }
        }
        s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
        s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
        s2 += __shfl_xor_sync(0xffffffffu, s2, 1);
        s2 += __shfl_xor_sync(0xffffffffu, s2, 2);
        const float mean = s1 * inv64;
        const float var = fmaxf(s2 * inv64 - mean * mean, 0.f);
        const float rstd = rsqrtf(var + p.eps);
        const float shift = -mean * rstd;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + qc;
          const __half2 n2 = __floats2half2_rn(fmaf(d1[h][4 * j + 2 * rs], rstd, shift), fmaf(d1[h][4 * j + 2 * rs + 1], rstd, shift));
          const uint32_t v = h2u(gelu_h2(__hfma2(n2, gb_s[c >> 1], gb_s[32 + (c >> 1)])));
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(a2 + (uint32_t)r * 128u + ((uint32_t)((c >> 3) ^ (r & 7)) << 4) + (uint32_t)(c & 7) * 2u),
                       "r"(v) : "memory");
        }
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(1 + sp, 128);   // the whole A2_sp tile is written before this warpgroup's MMA2 reads it
    // ---- MMA2 + E2 per half of the conv-transpose-2 outputs (sub-sub-pixels ss = 2 hf, 2 hf + 1 = W2 rows [64 hf, +64)):
    // + bias, GELU, hyper product over the 32 channels -> low-res logits
    const int tok0 = rt * 128;
#pragma unroll 1
    for (int hf = 0; hf < 2; ++hf) {
      float d2[2][32];
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          wgmma<64, 0, 0, true>(d2[h], make_desc_sw128(a2 + h * 8192 + 32 * k, 0, 1024), make_desc_sw128(aw2 + hf * 8192 + 32 * k, 0, 1024), k != 0);
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(d2[0]);
      wg_fence_acc(d2[1]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
          const int tok = tok0 + 64 * h + 16 * wq + qr + 8 * rs, ty = tok >> 6, tx = tok & 63;
#pragma unroll
          for (int sl = 0; sl < 2; ++sl) {
            const int ss = 2 * hf + sl;
            // this thread: channel pairs i = 4 jj + qc / 2 (jj < 4) of columns 32 sl + 8 jj + qc
            __half2 gv[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * sl + jj, i = 4 * jj + (qc >> 1);
              gv[jj] = gelu_h2(__hadd2(__floats2half2_rn(d2[h][4 * j + 2 * rs], d2[h][4 * j + 2 * rs + 1]), b2_s[ss * 16 + i]));
            }
            float* o = p.out + (size_t)pp * p.nm * 65536 + (size_t)(4 * ty + 2 * (sp >> 1) + (ss >> 1)) * 256 + 4 * tx + 2 * (sp & 1) + (ss & 1);
            for (int mi = 0; mi < p.nm; ++mi) {
              const float2* hv = reinterpret_cast<const float2*>(p.hyper + ((size_t)pp * 4 + p.m0 + mi) * 32);
              __half2 acc = __floats2half2_rn(0.f, 0.f);
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const float2 w = __ldg(hv + 4 * jj + (qc >> 1));
                acc = __hfma2(gv[jj], __floats2half2_rn(w.x, w.y), acc);
              }
              const float2 f = __half22float2(acc);
              float v = f.x + f.y;
              v += __shfl_xor_sync(0xffffffffu, v, 1);
              v += __shfl_xor_sync(0xffffffffu, v, 2);
              if ((lane & 3) == 0) o[(size_t)mi * 65536] = v;
            }
          }
        }
      }
    }
  }
}

int launch_upscale_fused(const UpscaleFusedArgs& a, int num_sms, cudaStream_t stream) {
  using namespace up;
  if (a.P <= 0 || a.nm < 1 || a.nm > 4 || a.m0 < 0 || a.m0 + a.nm > 4) return set_error("upscale_fused: bad arguments (P=%d nm=%d m0=%d)", a.P, a.nm, a.m0);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(upscale_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return set_error("upscale_fused: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap tmX, tmW1, tmW2;
  if (make_tmap_bf16_2d(&tmX, a.keys, (uint64_t)a.P * 4096, 256, 256, 128)) return -1;
  if (make_tmap_bf16_2d(&tmW1, a.w1, 256, 256, 256, 256)) return -1;
  if (make_tmap_f16_2d(&tmW2, a.w2_f16, 128, 64, 64, 128)) return -1;
  UpParams p;
  p.P = a.P; p.nm = a.nm; p.m0 = a.m0; p.b1 = a.b1; p.gamma = a.gamma; p.beta = a.beta; p.eps = a.eps; p.b2 = a.b2;
  p.hyper = a.hyper; p.out = a.out;
  const long total = (long)a.P * TILES;
  const int grid = total < num_sms ? (int)total : num_sms;
  prof_begin(stream, "upscale_fused (convT1+LN2d+GELU+convT2+GELU+hyper)",
             (double)a.P * 4096 * (2.0 * 256 * 256 + 4 * 2.0 * 128 * 64 + 2.0 * 512 * a.nm),
             (double)a.P * (4096.0 * 256 * 2 + 65536.0 * 4 * a.nm));
  upscale_fused_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(tmX, tmW1, tmW2, p);
  prof_end(stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("upscale_fused launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

}  // namespace msam
