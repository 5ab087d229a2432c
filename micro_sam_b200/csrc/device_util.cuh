// Small device helpers shared by the kernel files: bf16 packing, float warp reductions, exact GELU and its derivative, ex2,
// bilinear source indices and a block-local bitonic sort.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace msam {

// two floats -> one packed bf16x2 word (round to nearest even), `lo` in the low half
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// the low / high bf16 of a packed word as float (exact)
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// butterfly over all 32 lanes: every lane returns the warp's sum / max
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// GELU(x) = x Phi(x) = 0.5 x (1 + erf(x / sqrt 2))
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// d/dx [x Phi(x)] = Phi(x) + x phi(x).  Two variants on purpose: the fp32 mask_downscaling path of the training decoder
// (decoder_train.cu) uses gelu_erf_grad with expf; the bf16 encoder MLP backward (backward.cu:gelu_bwd) uses
// gelu_erf_grad_fast with __expf.  They round differently, so merging them changes results.
__device__ __forceinline__ float gelu_erf_grad(float x) {
  return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * expf(-0.5f * x * x);
}
__device__ __forceinline__ float gelu_erf_grad_fast(float x) {
  return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * __expf(-0.5f * x * x);
}

// 2^x on the MUFU unit (approximate, flushes denormals)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// PyTorch's upsample_bilinear2d source index (align_corners=False): max(0, (dst + 0.5) * scale - 0.5)
__device__ __forceinline__ void lin_src(int d, float scale, int n, int& i0, int& i1, float& l1) {
  const float s = fmaxf((d + 0.5f) * scale - 0.5f, 0.f);
  i0 = (int)s;
  i1 = i0 + (i0 < n - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

// Bitonic sort of keys [npow2] (a power of two) by the nthreads threads of a block, thread tid striding over the keys;
// descending or ascending.  One __syncthreads() after every merge step, the last of them before the return.
template <bool kDescending>
__device__ __forceinline__ void block_bitonic_sort(unsigned long long* keys, int npow2, int tid, int nthreads) {
  for (int k = 2; k <= npow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < npow2; i += nthreads) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = keys[i], b = keys[l];
          const bool first = (i & k) == 0;
          if (kDescending ? (first ? a < b : a > b) : (first ? a > b : a < b)) { keys[i] = b; keys[l] = a; }
        }
      }
      __syncthreads();
    }
}

}  // namespace msam
