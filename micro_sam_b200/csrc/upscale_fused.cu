// Fused output up-scaling + hyper-network mask product of the mask decoder (MaskDecoder.predict_masks after the
// transformer, restated in oracle/sam_ref.py:  upscaled = GELU(convT2(GELU(LN2d(convT1(src)))));  masks = hyper_in @ upscaled):
//
//   keys [64 tokens x 256]  --MMA1-->  D1 [64 x (4 sub-pixels x 64 ch)]               conv-transpose 1 (k2 s2) as a GEMM
//        E1: + bias, LayerNorm2d over the 64 channels of a (token, sub-pixel), GELU  -> A2_s: fp16 register A fragments
//   A2_s  --MMA2-->  D2 [64 x (4 sub-sub-pixels x 32 ch)]  (s = 0..3)                  conv-transpose 2 (k2 s2) as a GEMM
//        E2: + bias, GELU                                                           -> G_s: fp16 register A fragments
//   G_s   --MMA3-->  [64 x 8] per sub-sub-pixel, against the prompt's hyper-network vectors (<= 4 masks x 32 ch, rows >= nm
//                    zero)                                                          -> low-res logits
//
// so neither the 64-channel up-scaled embedding (2 MB per prompt written + read by the two-kernel version) nor the
// 32-channel one ever leaves the SM: per prompt the kernel reads 2 MB of `keys` and writes 0.25 MB per mask.
// The element-wise epilogues -- 3.2 G GELUs per 32x32-grid tile, instruction-issue bound in fp32 -- run in PACKED fp16x2
// arithmetic:
//   GELU(x) = 0.5 x (1 + erf(x / sqrt 2)),  erf(x / sqrt 2) ~ tanh(x (a + b x^2))   (minimax a, b: |err| <= 2.7e-4; with the
//   fp16 rounding of the 6-instruction chain the N(0,1)-weighted rms error is 2.9e-4 -- a quarter of the bf16 rounding the
//   two-kernel version applied when it stored the intermediate), one MUFU (tanh.approx.f16x2) per TWO elements,
// the intermediate operand A2, the conv-transpose-2 weights and the hyper vectors are fp16 (11-bit mantissa instead of
// bf16's 8); every product accumulates in fp32 on the tensor core.
//
// Work item = (prompt, token row ty) = 64 tokens, whose logits are the complete output rows [4 ty, 4 ty + 4) of every mask
// (4 KB contiguous per mask).  CTA = 2 consumer warpgroups + 1 warpgroup of which warps 8 / 9 issue the TMA loads and
// warps 10 / 11 the TMA stores of consumer warpgroup 0 / 1; persistent over a contiguous range of items, which the two
// consumers take alternately.  Each consumer has its own keys ring and output staging buffer, so the two drift apart and
// one warpgroup's epilogues run while the other's MMAs keep the tensor core busy.  Both conv-transpose weights stay
// resident in shared memory for the whole kernel (loaded once per CTA instead of once per item).  E1 / E2 work straight
// from the accumulator fragments (LayerNorm row reductions across the quad of lanes that shares a row) and hand their
// results to the next MMA as register A operands: a 16-column slice of an accumulator fragment is an m64k16 A fragment.
#include <cuda_fp16.h>

#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace up {
constexpr int TILES = 64;                        // token rows of the 64 x 64 image-token grid = items per prompt
constexpr int SLICE_X = 64 * 128;                // keys K-slice [64 tokens x 64] bf16 SW128 (8 KB)
constexpr int SLICE_W1 = 256 * 128;              // conv-transpose-1 weight K-slice [256 x 64] bf16 SW128 (32 KB)
constexpr int W2_BYTES = 128 * 128;              // conv-transpose-2 weight [128 x 64] fp16 SW128 (16 KB)
constexpr int OFF_W1 = 0;
constexpr int OFF_W2 = OFF_W1 + 4 * SLICE_W1;
constexpr int OFF_HYP = OFF_W2 + W2_BYTES;       // 2 warpgroups x [8 x 64] fp16 SW128 hyper tile (1 KB)
constexpr int OFF_RING = OFF_HYP + 2 * 1024;     // 2 warpgroups x STAGES keys slices
constexpr int PAR_BYTES = 1024 + 256 + 256;      // b1 [256] fp32 | gamma, beta [32 + 32] half2 | b2 [64] half2
constexpr int THREADS = 256 + 128;
constexpr int PF_AHEAD = 4;                      // L2 prefetch distance in items (2 items of the same warpgroup)

template <int NM> struct Layout {
  static constexpr int STAGES = NM <= 3 ? 3 : 2;  // keys ring stages per warpgroup (nm = 4: the staging buffers take the third)
  static constexpr int STG_BYTES = NM * 4 * 256 * 4;  // logit staging [NM][4 rows][256] fp32 per warpgroup
  static constexpr int OFF_STG = OFF_RING + 2 * STAGES * SLICE_X;
  static constexpr int OFF_PAR = OFF_STG + 2 * STG_BYTES;
  static constexpr int OFF_BAR = OFF_PAR + PAR_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "resident weights + rings + staging exceed the shared memory of an SM");
};
}  // namespace up

struct UpParams {
  int P, m0;
  const float* b1;      // [256] conv-transpose-1 bias per (sub-pixel, channel)
  const float* gamma;   // [64] LayerNorm2d
  const float* beta;
  float eps;
  const float* b2;      // [128] conv-transpose-2 bias per (sub-sub-pixel, channel)
  const float* hyper;   // [P, 4, 32]
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

// MMA2 of sub-pixel sp: D2 = A2_sp [64 x 64] . W2^T, A2_sp from registers (k-step k = a2[16 sp + 4 k .. + 4))
__device__ __forceinline__ void up_mma2(float (&d2)[64], const uint32_t (&a2)[64], int sp, uint64_t dw2) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint32_t a[4] = {a2[16 * sp + 4 * k], a2[16 * sp + 4 * k + 1], a2[16 * sp + 4 * k + 2], a2[16 * sp + 4 * k + 3]};
    wgmma_rs<128, 0, true>(d2, a, dw2 + 2 * k, k != 0);
  }
}

template <int NM>
__global__ void __launch_bounds__(up::THREADS, 1)
upscale_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
                     const __grid_constant__ CUtensorMap tmW2, const __grid_constant__ CUtensorMap tmO, const UpParams p) {
  using namespace up;
  using L = Layout<NM>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* full_bar = w_full + 1;              // [g * STAGES + s]
  uint64_t* empty_bar = full_bar + 2 * STAGES;  // [g * STAGES + s]: the 4 warps of warpgroup g arrive
  uint64_t* ofull = empty_bar + 2 * STAGES;     // [g]: staging buffer of warpgroup g written (4 warps arrive)
  uint64_t* oempty = ofull + 2;                 // [g]: its TMA store has read it
  float* b1_s = reinterpret_cast<float*>(smem + L::OFF_PAR);
  __half2* gb_s = reinterpret_cast<__half2*>(smem + L::OFF_PAR + 1024);  // [0,32) gamma pairs, [32,64) beta pairs
  __half2* b2_s = gb_s + 64;                                           // conv-transpose-2 bias pairs, index ss*16 + i

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long total = (long)p.P * TILES;
  const int it_begin = (int)(total * blockIdx.x / gridDim.x), it_end = (int)(total * (blockIdx.x + 1) / gridDim.x);

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmW1); prefetch_tmap(&tmW2); prefetch_tmap(&tmO);
    mbar_init(w_full, 1);
    for (int i = 0; i < 2 * STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    for (int g = 0; g < 2; ++g) { mbar_init(&ofull[g], 4); mbar_init(&oempty[g], 1); }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 256; i += THREADS) b1_s[i] = p.b1[i];
  for (int i = threadIdx.x; i < 32; i += THREADS) {
    gb_s[i] = __floats2half2_rn(p.gamma[2 * i], p.gamma[2 * i + 1]);
    gb_s[32 + i] = __floats2half2_rn(p.beta[2 * i], p.beta[2 * i + 1]);
  }
  for (int i = threadIdx.x; i < 64; i += THREADS) b2_s[i] = __floats2half2_rn(p.b2[2 * i], p.b2[2 * i + 1]);
  __syncthreads();

  if (warp >= 8) {
    // D1 (128 registers) + the A2 fragments (64): the loading warpgroup hands its registers to the two consumers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp < 10 && lane == 0) {
      // ---------------------------------------------------------- TMA loads of consumer warpgroup g = warp - 8
      const int g = warp - 8;
      if (g == 0 && it_begin < it_end) {
        mbar_expect_tx(w_full, 4 * SLICE_W1 + W2_BYTES);
#pragma unroll
        for (int j = 0; j < 4; ++j) tma_load_2d(smem + OFF_W1 + j * SLICE_W1, &tmW1, w_full, 64 * j, 0);
        tma_load_2d(smem + OFF_W2, &tmW2, w_full, 0, 0);
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int item = it_begin + g; item < it_end; item += 2) {
        if (item + PF_AHEAD < it_end) {  // keys of a later item of this warpgroup -> L2
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_prefetch_2d(&tmX, 64 * j, (item + PF_AHEAD) * 64);
        }
        for (int j = 0; j < 4; ++j) {
          mbar_wait(&empty_bar[g * STAGES + stage], phase ^ 1, 40);
          mbar_expect_tx(&full_bar[g * STAGES + stage], SLICE_X);
          tma_load_2d(smem + OFF_RING + (g * STAGES + stage) * SLICE_X, &tmX, &full_bar[g * STAGES + stage], 64 * j, item * 64);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else if (lane == 0) {
      // ---------------------------------------------------------- TMA stores of consumer warpgroup g = warp - 10 (kept out
      // of the consumers' code, where the store instructions make ptxas serialise the wgmma pipeline)
      const int g = warp - 10;
      uint32_t ophase = 0;
      for (int item = it_begin + g; item < it_end; item += 2) {
        mbar_wait(&ofull[g], ophase, 44);
        tma_store_3d(&tmO, smem + L::OFF_STG + g * L::STG_BYTES, 0, 4 * (item % TILES), (item / TILES) * NM);
        tma_store_commit();
        tma_store_wait_read<0>();
        mbar_arrive(&oempty[g]);
        ophase ^= 1;
      }
      tma_store_wait_all();
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");

  // ------------------------------------------------------------ consumer warpgroup g: items it_begin + g, + 2, ...
  // Fragment element i of a thread: token tx = 16 wq + qr + 8 ((i >> 1) & 1) of the item's row, column 8 (i >> 2) + qc + (i & 1).
  const int g = warp >> 2, wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
  const uint32_t ring = smem_u32(smem + OFF_RING) + (uint32_t)(g * STAGES * SLICE_X);
  const uint32_t aw1 = smem_u32(smem + OFF_W1), hyp = smem_u32(smem + OFF_HYP) + (uint32_t)g * 1024u;
  const uint32_t stg = smem_u32(smem + L::OFF_STG) + (uint32_t)(g * L::STG_BYTES);
  const uint64_t dw2 = make_desc_sw128(smem_u32(smem + OFF_W2), 0, 1024), dh = make_desc_sw128(hyp, 0, 1024);
  const float inv64 = 1.0f / 64.0f;
  int stage = 0, cur_p = -1;
  uint32_t phase = 0, ophase = 0;
  if (it_begin + g < it_end) mbar_wait(w_full, 0, 45);
  for (int item = it_begin + g; item < it_end; item += 2) {
    const int pp = item / TILES;
    if (pp != cur_p) {
      // hyper tile B [8 x 64] fp16 SW128: rows m < NM = hyper[pp, m0 + m, 0 .. 32), the rest zero (columns >= 32 are never
      // read).  The first barrier keeps the rewrite behind every warp's wait for the previous prompt's last MMA3; the
      // second makes the whole tile visible to the async proxy before any warp's wgmma reads it.
      named_bar_sync(1 + g, 128);
      const int t = threadIdx.x & 127;
      if (t < 64) {
        const int n = t >> 3, kc = t & 7;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (n < NM && kc < 4) {
          const float4* src = reinterpret_cast<const float4*>(p.hyper + ((size_t)pp * 4 + p.m0 + n) * 32 + 8 * kc);
          const float4 a = __ldg(src), b = __ldg(src + 1);
          v = make_uint4(h2u(__floats2half2_rn(a.x, a.y)), h2u(__floats2half2_rn(a.z, a.w)), h2u(__floats2half2_rn(b.x, b.y)),
                         h2u(__floats2half2_rn(b.z, b.w)));
        }
        st_shared_v4(hyp + (uint32_t)n * 128u + ((uint32_t)(kc ^ n) << 4), v);
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + g, 128);
      cur_p = pp;
    }
    // ---- MMA1: D1 = keys [64 x 256] . W1^T (all 4 sub-pixels); each ring stage is released as soon as its MMAs complete
    float d1[128];
    int prev = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      mbar_wait(&full_bar[g * STAGES + stage], phase, 42);
      const uint64_t da = make_desc_sw128(ring + (uint32_t)(stage * SLICE_X), 0, 1024);
      const uint64_t db = make_desc_sw128(aw1 + (uint32_t)(j * SLICE_W1), 0, 1024);
      wg_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma<256>(d1, da + 2 * k, db + 2 * k, (j | k) != 0);
      wg_commit();
      if (j > 0) {
        wg_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[g * STAGES + prev]);
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    wg_fence_acc(d1);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[g * STAGES + prev]);
    // ---- E1: (token, sub-pixel sp): + bias, LayerNorm over 64 channels, GELU -> fp16 A fragments of MMA2.  Columns
    // 8 j + qc + {0, 1} of sub-pixel sp, rows rs: a2[16 sp + 2 j + rs] (k-step k = j / 2 holds a2[16 sp + 4 k .. + 4))
    uint32_t a2[64];
#pragma unroll
    for (int sp = 0; sp < 4; ++sp) {
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& x = d1[32 * sp + 4 * j + 2 * rs + e];
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
          const __half2 n2 = __floats2half2_rn(fmaf(d1[32 * sp + 4 * j + 2 * rs], rstd, shift), fmaf(d1[32 * sp + 4 * j + 2 * rs + 1], rstd, shift));
          a2[16 * sp + 2 * j + rs] = h2u(gelu_h2(__hfma2(n2, gb_s[c >> 1], gb_s[32 + (c >> 1)])));
        }
      }
    }
    // ---- per sub-pixel sp: MMA2, E2 (+ bias, GELU -> fp16 A fragments), MMA3 against the hyper tile.  MMA2 of sp + 1 is
    // issued behind MMA3 of sp, so it runs while this warpgroup writes sp's logits to the staging buffer.
    float d2[64];
    wg_fence();
    up_mma2(d2, a2, 0, dw2);
    wg_commit();
    mbar_wait(&oempty[g], ophase ^ 1, 46);  // the store warp has read this buffer's previous item
#pragma unroll
    for (int sp = 0; sp < 4; ++sp) {
      wg_wait<0>();
      wg_fence_acc(d2);
      // columns 8 jj + qc + {0, 1} of sub-sub-pixel ss, rows rs: g2[8 ss + 2 jj + rs]
      uint32_t g2[32];
#pragma unroll
      for (int ss = 0; ss < 4; ++ss)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            const int j = 4 * ss + jj;
            g2[8 * ss + 2 * jj + rs] =
                h2u(gelu_h2(__hadd2(__floats2half2_rn(d2[4 * j + 2 * rs], d2[4 * j + 2 * rs + 1]), b2_s[16 * ss + 4 * jj + (qc >> 1)])));
          }
      float d3[4][4];  // [ss]: tokens rs, masks qc + {0, 1}
      wg_fence();
#pragma unroll
      for (int ss = 0; ss < 4; ++ss)
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          const uint32_t a[4] = {g2[8 * ss + 4 * kk], g2[8 * ss + 4 * kk + 1], g2[8 * ss + 4 * kk + 2], g2[8 * ss + 4 * kk + 3]};
          wgmma_rs<8, 0, true>(d3[ss], a, dh + 2 * kk, kk != 0);
        }
      wg_commit();
      if (sp < 3) {
        up_mma2(d2, a2, sp + 1, dw2);
        wg_commit();
        wg_wait<1>();
      } else {
        wg_wait<0>();
      }
#pragma unroll
      for (int ss = 0; ss < 4; ++ss) wg_fence_acc(d3[ss]);
      // logit (mask m, output row 4 ty + 2 (sp >> 1) + (ss >> 1), column 4 tx + 2 (sp & 1) + (ss & 1)) -> staging
      // [m][2 (sp >> 1) + (ss >> 1)][4 tx + 2 (sp & 1) + (ss & 1)]; the ss & 1 pair is one 8-byte store
#pragma unroll
      for (int sh = 0; sh < 2; ++sh)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = qc + e;
            if (m < NM) {
              const uint32_t addr = stg + (uint32_t)(((m * 4 + 2 * (sp >> 1) + sh) * 256 + 4 * (16 * wq + qr + 8 * rs) + 2 * (sp & 1)) * 4);
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(d3[2 * sh][2 * rs + e]), "f"(d3[2 * sh + 1][2 * rs + e])
                           : "memory");
            }
          }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(&ofull[g]);
    ophase ^= 1;
  }
}

// out [P * nm, 256, 256] fp32 as a 3-D tensor map whose box [nm][4][256] is one item's logits
static int make_tmap_logits(CUtensorMap* m, float* out, int P, int nm) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t dims[3] = {256, 256, (cuuint64_t)P * nm};
  cuuint64_t strides[2] = {256 * 4, 65536 * 4};
  cuuint32_t box[3] = {256, 4, (cuuint32_t)nm};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("upscale_fused: cuTensorMapEncodeTiled failed (%d) for the logits (P=%d nm=%d)", (int)r, P, nm);
  return 0;
}

template <int NM>
static int launch_nm(const CUtensorMap& tmX, const CUtensorMap& tmW1, const CUtensorMap& tmW2, const CUtensorMap& tmO,
                     const UpParams& p, int grid, cudaStream_t stream) {
  constexpr int SMEM = up::Layout<NM>::SMEM_BYTES;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(upscale_fused_kernel<NM>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return set_error("upscale_fused: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  upscale_fused_kernel<NM><<<grid, up::THREADS, SMEM, stream>>>(tmX, tmW1, tmW2, tmO, p);
  return 0;
}

int launch_upscale_fused(const UpscaleFusedArgs& a, int num_sms, cudaStream_t stream) {
  using namespace up;
  if (a.P <= 0 || a.nm < 1 || a.nm > 4 || a.m0 < 0 || a.m0 + a.nm > 4) return set_error("upscale_fused: bad arguments (P=%d nm=%d m0=%d)", a.P, a.nm, a.m0);
  CUtensorMap tmX, tmW1, tmW2, tmO;
  if (make_tmap_bf16_2d(&tmX, a.keys, (uint64_t)a.P * 4096, 256, 256, 64)) return -1;
  if (make_tmap_bf16_2d(&tmW1, a.w1, 256, 256, 256, 256)) return -1;
  if (make_tmap_f16_2d(&tmW2, a.w2_f16, 128, 64, 64, 128)) return -1;
  if (make_tmap_logits(&tmO, a.out, a.P, a.nm)) return -1;
  UpParams p;
  p.P = a.P; p.m0 = a.m0; p.b1 = a.b1; p.gamma = a.gamma; p.beta = a.beta; p.eps = a.eps; p.b2 = a.b2; p.hyper = a.hyper;
  const long total = (long)a.P * TILES;
  const int grid = total < num_sms ? (int)total : num_sms;
  prof_begin(stream, "upscale_fused (convT1+LN2d+GELU+convT2+GELU+hyper)",
             (double)a.P * 4096 * (2.0 * 256 * 256 + 4 * 2.0 * 128 * 64 + 2.0 * 512 * a.nm),
             (double)a.P * (4096.0 * 256 * 2 + 65536.0 * 4 * a.nm));
  int rc = 0;
  switch (a.nm) {
    case 1: rc = launch_nm<1>(tmX, tmW1, tmW2, tmO, p, grid, stream); break;
    case 2: rc = launch_nm<2>(tmX, tmW1, tmW2, tmO, p, grid, stream); break;
    case 3: rc = launch_nm<3>(tmX, tmW1, tmW2, tmO, p, grid, stream); break;
    default: rc = launch_nm<4>(tmX, tmW1, tmW2, tmO, p, grid, stream); break;
  }
  prof_end(stream);
  if (rc) return rc;
  LAUNCH_CHECK("upscale_fused");
  return 0;
}

}  // namespace msam
