// Mask decoder in training mode (BASELINE.json configs[4]; micro_sam/training/trainable_sam.py:62-114 + sam_trainer.py:131-172):
// MaskDecoder.forward on the prompts of ONE image, keeping the activations, and its backward pass -- gradients of every mask-decoder
// and prompt-encoder parameter plus dL/d(image embedding), which is what the encoder backward pass (encoder_train.cu) consumes.
// Restates oracle/sam_ref.py:MaskDecoder / TwoWayTransformer / DecAttention (the inference kernels t2i_fused / i2t_fused /
// upscale_fused fold projections into each other and keep nothing, so they cannot be differentiated through); checked against torch
// autograd in tests/test_gpu_backward.py.
//
// Structure: a tape.  Every forward op (linear, LayerNorm, add+cast, attention, GELU, ...) runs on the existing kernels -- wgmma
// GEMMs (gemm.cu), the batched attention GEMM (bgemm.cu), LayerNorm -- allocates its output from a per-slot arena
// and pushes its backward closure; backward() replays the closures in reverse.  Tensors carry an fp32 value, an fp32 gradient
// (accumulated: every consumer ADDS) and a bf16 copy (the GEMM operand).  Parameter gradients accumulate across calls (images,
// sub-iterations) until msam_decoder_zero_grads.  Prompts: points and / or boxes, with the dense prompt no_mask_embed or, for mask
// prompts, mask_downscaling(mask) (md_* kernels: fp32, taped by keeping the mask; no gradient w.r.t. the mask itself).  A
// prompt-free batch (semantic training, micro_sam/training/semantic_sam_trainer.py) runs B images as B prompts of 5 tokens in one
// slot, prompt p keyed by image p (src_images_* kernels); its backward writes dL/d embedding per image.
#include "device_util.cuh"
#include "engine.h"

#include <algorithm>
#include <cmath>
#include <functional>

namespace msam {

namespace {

// out_bf16[r, c] = bf16(a[r, c] + b[r % b_rows, c]); b may be null.  n4 = rows * cols / 4
__global__ void add_cast_kernel(const float4* __restrict__ a, const float4* __restrict__ b, long n4, long b_n4, uint2* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = a[i];
  if (b) { const float4 w = b[i % b_n4]; v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
  out[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}
// dst += src (fp32)
__global__ void add_inplace_kernel(float4* __restrict__ dst, const float4* __restrict__ src, long n4) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 d = dst[i];
  const float4 s = src[i];
  d.x += s.x; d.y += s.y; d.z += s.z; d.w += s.w;
  dst[i] = d;
}
// dy_bf16 = bf16(g) [masked by y > 0 when relu_y != null]
__global__ void grad_cast_kernel(const float4* __restrict__ g, const uint2* __restrict__ relu_y, long n4, uint2* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = g[i];
  if (relu_y) {
    const uint2 y = relu_y[i];
    if (!(__uint_as_float(y.x << 16) > 0.f)) v.x = 0.f;
    if (!(__uint_as_float(y.x & 0xffff0000u) > 0.f)) v.y = 0.f;
    if (!(__uint_as_float(y.y << 16) > 0.f)) v.z = 0.f;
    if (!(__uint_as_float(y.y & 0xffff0000u) > 0.f)) v.w = 0.f;
  }
  out[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}
// strided row copy / accumulate: dst[r * dp + c] (+)= src[r * sp + c], c < cols
__global__ void copy_rows_kernel(const float* __restrict__ src, long sp, float* __restrict__ dst, long dp, long rows, int cols, int accumulate) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const long r = i / cols;
  const int c = i % cols;
  const float v = src[r * sp + c];
  if (accumulate) dst[r * dp + c] += v; else dst[r * dp + c] = v;
}
// softmax over the first n_valid entries of fp32 rows (pitch entries each) -> bf16 probabilities (zero beyond n_valid)
__global__ void softmax_rows_kernel(const float* __restrict__ S, long rows, int n_valid, int pitch, __nv_bfloat16* __restrict__ P) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + row * pitch;
  __nv_bfloat16* p = P + row * pitch;
  float m = -INFINITY;
  for (int k = lane; k < n_valid; k += 32) m = fmaxf(m, s[k]);
  m = warp_max(m);
  float l = 0.f;
  for (int k = lane; k < n_valid; k += 32) l += __expf(s[k] - m);
  const float inv = 1.0f / warp_sum(l);
  for (int k = lane; k < pitch; k += 32) p[k] = __float2bfloat16(k < n_valid ? __expf(s[k] - m) * inv : 0.f);
}
// dS = P o (dP - sum_k P dP)
__global__ void ds_rows_kernel(const __nv_bfloat16* __restrict__ P, const float* __restrict__ dP, long rows, int n_valid, int pitch,
                               __nv_bfloat16* __restrict__ dS) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const __nv_bfloat16* p = P + row * pitch;
  const float* dp = dP + row * pitch;
  __nv_bfloat16* ds = dS + row * pitch;
  float del = 0.f;
  for (int k = lane; k < n_valid; k += 32) del += __bfloat162float(p[k]) * dp[k];
  del = warp_sum(del);
  for (int k = lane; k < pitch; k += 32) ds[k] = __float2bfloat16(k < n_valid ? __bfloat162float(p[k]) * (dp[k] - del) : 0.f);
}
// tokens [P, T, 256]: rows 0..4 = output tokens (iou token, 4 mask tokens), rows 5.. = sparse prompt embeddings [P, Ts, 256]
__global__ void assemble_tokens_kernel(const float* __restrict__ out_tokens, const float* __restrict__ sparse, int P, int T, int Ts,
                                       float* __restrict__ tok) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * T * 256) return;
  const int c = i % 256, t = (i / 256) % T;
  const long p = i / (256L * T);
  tok[i] = t < 5 ? out_tokens[t * 256 + c] : sparse[(p * Ts + (t - 5)) * 256 + c];
}
// gradients of the embedding tables behind the tokens: output tokens (rows 0..4) and, per sparse token, the table row emb_index
// selects (0..3 = point_embeddings, 4 = not_a_point_embed; the positional part has no parameters)
__global__ void token_grads_kernel(const float* __restrict__ g_tok, const int* __restrict__ emb_index, int P, int T, int Ts,
                                   float* __restrict__ g_out_tokens, float* __restrict__ g_point_emb, float* __restrict__ g_nap) {
  const int c = threadIdx.x, t = blockIdx.x;   // 256 threads, T blocks
  float s = 0.f;
  if (t < 5) {
    for (int p = 0; p < P; ++p) s += g_tok[((long)p * T + t) * 256 + c];
    g_out_tokens[t * 256 + c] += s;
  } else {
    for (int p = 0; p < P; ++p) {
      const int e = emb_index[p * Ts + (t - 5)];
      const float v = g_tok[((long)p * T + t) * 256 + c];
      if (e >= 0 && e < 4) atomicAdd(g_point_emb + e * 256 + c, v);
      else if (e == 4) atomicAdd(g_nap + c, v);
    }
  }
}
// keys0[p, pix, c] = emb_nchw[c, pix] + no_mask[c]
__global__ void src_broadcast_kernel(const float* __restrict__ emb_nchw, const float* __restrict__ no_mask, int P, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int pix0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) tile[i][threadIdx.x] = emb_nchw[(long)(c0 + i) * 4096 + pix0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const float v = tile[threadIdx.x][i] + no_mask[c0 + threadIdx.x];
    for (int p = 0; p < P; ++p) out[((long)p * 4096 + pix0 + i) * 256 + c0 + threadIdx.x] = v;
  }
}
// d_emb_nchw[c, pix] = sum_p g[p, pix, c];  g_no_mask[c] += sum_{p, pix} g[p, pix, c]
__global__ void src_grad_kernel(const float* __restrict__ g, int P, float* __restrict__ d_emb_nchw, float* __restrict__ g_no_mask) {
  __shared__ float tile[32][33];
  const int pix0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += g[((long)p * 4096 + pix0 + i) * 256 + c0 + threadIdx.x];
    tile[i][threadIdx.x] = s;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) d_emb_nchw[(long)(c0 + i) * 4096 + pix0 + threadIdx.x] = tile[threadIdx.x][i];
  if (threadIdx.y == 0) {
    float s = 0.f;
    for (int i = 0; i < 32; ++i) s += tile[i][threadIdx.x];
    atomicAdd(g_no_mask + c0 + threadIdx.x, s);
  }
}
// Prompt-free batches (one prompt per image): keys0[p, pix, c] = emb_nchw[p, c, pix] + no_mask[c].  grid = (128, 8, P)
__global__ void src_images_kernel(const float* __restrict__ emb_nchw, const float* __restrict__ no_mask, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int pix0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const long p = blockIdx.z;
  const float* e = emb_nchw + p * 256 * 4096;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) tile[i][threadIdx.x] = e[(long)(c0 + i) * 4096 + pix0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    out[(p * 4096 + pix0 + i) * 256 + c0 + threadIdx.x] = tile[threadIdx.x][i] + no_mask[c0 + threadIdx.x];
}
// d_emb_nchw[p, c, pix] = g[p, pix, c] (per image, not summed);  g_no_mask[c] += sum_{p, pix} g[p, pix, c].  grid = (128, 8, P)
__global__ void src_images_grad_kernel(const float* __restrict__ g, float* __restrict__ d_emb_nchw, float* __restrict__ g_no_mask) {
  __shared__ float tile[32][33];
  const int pix0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const long p = blockIdx.z;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) tile[i][threadIdx.x] = g[(p * 4096 + pix0 + i) * 256 + c0 + threadIdx.x];
  __syncthreads();
  float* d = d_emb_nchw + p * 256 * 4096;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) d[(long)(c0 + i) * 4096 + pix0 + threadIdx.x] = tile[threadIdx.x][i];
  if (threadIdx.y == 0) {
    float s = 0.f;
    for (int i = 0; i < 32; ++i) s += tile[i][threadIdx.x];
    atomicAdd(g_no_mask + c0 + threadIdx.x, s);
  }
}
// hyper product output [P, 65536 (pixel order ((i*64+j)*4+s1)*4+s2), 4] <-> low-res masks [P, nm, 256, 256] (masks m0 .. m0 + nm - 1)
__device__ __forceinline__ long up_row(int Y, int X) {
  return ((((long)(Y >> 2) * 64 + (X >> 2)) * 4 + (((Y >> 1) & 1) * 2 + ((X >> 1) & 1))) * 4 + ((Y & 1) * 2 + (X & 1)));
}
__global__ void masks_out_kernel(const float* __restrict__ o4, int P, int nm, int m0, float* __restrict__ low_res) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * nm * 65536) return;
  const int X = i % 256, Y = (i / 256) % 256, m = (i / 65536) % nm;
  const long p = i / (65536L * nm);
  low_res[i] = o4[(p * 65536 + up_row(Y, X)) * 4 + m0 + m];
}
// d_low_res [P, nm, 256, 256] -> bf16 [P, 65536, 8] in pixel order (columns m0 .. m0+nm-1, zero elsewhere)
__global__ void masks_grad_kernel(const float* __restrict__ d_low, int P, int nm, int m0, __nv_bfloat16* __restrict__ out8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * 65536) return;
  const int X = i % 256, Y = (i / 256) % 256;
  const long p = i / 65536;
  float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int m = 0; m < nm; ++m) v[m0 + m] = d_low[((p * nm + m) * 256 + Y) * 256 + X];
  *reinterpret_cast<uint4*>(out8 + (p * 65536 + up_row(Y, X)) * 8) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}

// ------------------------------------------------------------------------------------------------ mask prompts
// PromptEncoder.mask_downscaling: conv 1->4 (k2 s2, 256^2 -> 128^2), LayerNorm2d(4), GELU, conv 4->16 (k2 s2 -> 64^2), LayerNorm2d(16),
// GELU, conv 1x1 16->256, all fp32.  Output pixel (ty, tx) of the 64^2 grid depends on its own 4x4 input patch only.  The ten
// parameters live in one packed fp32 buffer (masters and gradients alike) in upstream order and layout:
constexpr int MD_W1 = 0, MD_B1 = 16, MD_G1 = 20, MD_BE1 = 24, MD_W2 = 28, MD_B2 = 284, MD_G2 = 300, MD_BE2 = 316, MD_W3 = 332,
              MD_B3 = 4428, MD_N = 4684;
constexpr int MD_SMALL = MD_W3;      // parameters of the two strided stages (reduced from md_param_grad_kernel's partials)
constexpr int MD_BIG = MD_N - MD_W3; // W3 + b3 (reduced from md_keys_grad_kernel's partials)
constexpr int MD_PIX_TILE = 128;     // pixels per tile of md_param_grad_kernel (= its block size)
constexpr int MD_GRID2 = 256;        // most blocks of md_param_grad_kernel: partial rows to reduce, independent of the device

// Stages of one output pixel.  Index s = sy * 2 + sx is the stage-1 sub-pixel, k = dy * 2 + dx the position in a 2x2 conv window;
// stage-1 channel c of sub-pixel s sits at c * 4 + s, the order of W2's input index (W2 [o][c][sy][sx]).  LayerNorm2d statistics are
// two-pass (mean first, then the centred sum of squares): an almost constant mask makes the 4 stage-1 channels almost equal, and a
// one-pass E[x^2] - E[x]^2 would cancel.
// Stage 1 at sub-pixel s: m = the 2x2 input window, n = normalised, a = affine (pre-GELU) values of the 4 channels; returns rstd.
__device__ __forceinline__ float md_stage1(const float* __restrict__ mask_p, int pix, int s, const float* W, float m[4], float n[4],
                                           float a[4]) {
  const float* mp = mask_p + (size_t)(4 * (pix >> 6) + 2 * (s >> 1)) * 256 + 4 * (pix & 63) + 2 * (s & 1);
  m[0] = mp[0]; m[1] = mp[1]; m[2] = mp[256]; m[3] = mp[257];
  float y[4], mean = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float acc = W[MD_B1 + c];
#pragma unroll
    for (int k = 0; k < 4; ++k) acc += W[MD_W1 + c * 4 + k] * m[k];
    y[c] = acc;
    mean += acc;
  }
  mean *= 0.25f;
  float var = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) var += (y[c] - mean) * (y[c] - mean);
  const float rstd = rsqrtf(var * 0.25f + 1e-6f);
#pragma unroll
  for (int c = 0; c < 4; ++c) { n[c] = (y[c] - mean) * rstd; a[c] = n[c] * W[MD_G1 + c] + W[MD_BE1 + c]; }
  return rstd;
}
// Stage 2 from the stage-1 GELU outputs h1[c * 4 + s]: n = normalised, a = affine (pre-GELU) values of the 16 channels; returns rstd.
__device__ __forceinline__ float md_stage2(const float h1[16], const float* W, float n[16], float a[16]) {
  float z[16], mean = 0.f;
#pragma unroll
  for (int o = 0; o < 16; ++o) {
    float acc = W[MD_B2 + o];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc += W[MD_W2 + o * 16 + k] * h1[k];
    z[o] = acc;
    mean += acc;
  }
  mean *= (1.0f / 16);
  float var = 0.f;
#pragma unroll
  for (int o = 0; o < 16; ++o) var += (z[o] - mean) * (z[o] - mean);
  const float rstd = rsqrtf(var * (1.0f / 16) + 1e-6f);
#pragma unroll
  for (int o = 0; o < 16; ++o) { n[o] = (z[o] - mean) * rstd; a[o] = n[o] * W[MD_G2 + o] + W[MD_BE2 + o]; }
  return rstd;
}
// the stage-2 GELU outputs h2 of one pixel (forward)
__device__ __forceinline__ void md_pixel(const float* __restrict__ mask_p, int pix, const float* W, float h2[16]) {
  float h1[16];
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    float m[4], n[4], a[4];
    md_stage1(mask_p, pix, s, W, m, n, a);
#pragma unroll
    for (int c = 0; c < 4; ++c) h1[c * 4 + s] = gelu_erf(a[c]);
  }
  float n2[16], a2[16];
  md_stage2(h1, W, n2, a2);
#pragma unroll
  for (int o = 0; o < 16; ++o) h2[o] = gelu_erf(a2[o]);
}

// Forward: out[p, pix, c] = dense_p[c, pix] (+ emb_nchw[c, pix]); h2_out[p, pix, 0..15] = stage-2 output (the 1x1 conv's input,
// kept for its weight gradient).  grid = (4096 / 16, P), block = 256 (thread = output channel; 16 pixels per block).
__global__ void __launch_bounds__(256)
md_forward_kernel(const float* __restrict__ mask, const float* __restrict__ W, const float* __restrict__ emb_nchw,
                  float* __restrict__ out, __nv_bfloat16* __restrict__ out_bf, float* __restrict__ h2_out) {
  __shared__ float sh[16][17];
  const int p = blockIdx.y, pix0 = blockIdx.x * 16, tid = threadIdx.x;
  if (tid < 16) {
    float h2[16];
    md_pixel(mask + (size_t)p * 65536, pix0 + tid, W, h2);
#pragma unroll
    for (int o = 0; o < 16; ++o) { sh[tid][o] = h2[o]; h2_out[((size_t)p * 4096 + pix0 + tid) * 16 + o] = h2[o]; }
  }
  __syncthreads();
  float w[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) w[o] = W[MD_W3 + tid * 16 + o];
  const float b = W[MD_B3 + tid];
  for (int i = 0; i < 16; ++i) {
    float acc = b;
#pragma unroll
    for (int o = 0; o < 16; ++o) acc += w[o] * sh[i][o];
    if (emb_nchw) acc += emb_nchw[(size_t)tid * 4096 + pix0 + i];
    const size_t row = (size_t)p * 4096 + pix0 + i;
    out[row * 256 + tid] = acc;
    if (out_bf) out_bf[row * 256 + tid] = __float2bfloat16(acc);
  }
}

// Backward, part 1: the one pass over g = dL/d keys0 [P, 4096, 256].  Per 16-pixel tile (grid = 256, block = 256, thread = channel):
// d_emb_nchw[c, pix] = sum_p g[p, pix, c] (when non-null), d_h2[p, pix, :] = g[p, pix, :] W3, and this block's partial sums of
// dW3 = sum g^T h2 and db3 = sum g -> part[blockIdx.x][MD_BIG] (reduced by md_reduce_kernel; no atomics).
__global__ void __launch_bounds__(256)
md_keys_grad_kernel(const float* __restrict__ g, const float* __restrict__ h2, const float* __restrict__ W, int P,
                    float* __restrict__ d_emb_nchw, float* __restrict__ d_h2, float* __restrict__ part) {
  __shared__ float gs[16][257];
  __shared__ float hs[16][16];
  __shared__ float w3s[256 * 16];
  const int pix0 = blockIdx.x * 16, tid = threadIdx.x;
  for (int i = tid; i < 256 * 16; i += 256) w3s[i] = W[MD_W3 + i];
  float demb[16], dw[16], db = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) { demb[i] = 0.f; dw[i] = 0.f; }
  for (int p = 0; p < P; ++p) {
    __syncthreads();
    const size_t row0 = (size_t)p * 4096 + pix0;
#pragma unroll 4
    for (int i = 0; i < 16; ++i) gs[i][tid] = g[(row0 + i) * 256 + tid];
    hs[tid >> 4][tid & 15] = h2[row0 * 16 + tid];
    __syncthreads();
    {
      const int i = tid >> 4, o = tid & 15;
      float acc = 0.f;
#pragma unroll 8
      for (int c = 0; c < 256; ++c) acc += gs[i][c] * w3s[c * 16 + o];
      d_h2[row0 * 16 + tid] = acc;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float v = gs[i][tid];
      demb[i] += v;
      db += v;
#pragma unroll
      for (int o = 0; o < 16; ++o) dw[o] += v * hs[i][o];
    }
  }
  if (d_emb_nchw) {
#pragma unroll
    for (int i = 0; i < 16; ++i) d_emb_nchw[(size_t)tid * 4096 + pix0 + i] = demb[i];
  }
  float* pr = part + (size_t)blockIdx.x * MD_BIG;
#pragma unroll
  for (int o = 0; o < 16; ++o) pr[tid * 16 + o] = dw[o];
  pr[4096 + tid] = db;
}

// Backward, part 2: pixel-local GELU', LayerNorm2d backward and the transposed k2s2 convs through both stages (stage values are
// recomputed from the mask).  Block b (MD_PIX_TILE threads, thread = pixel) takes the tiles b, b + gridDim.x, ... of the P * 4096
// pixels; per tile, phase A puts each pixel's terms in shared memory ([term][pixel], row pitch MD_LD so that phase B's reads of
// different terms at one pixel fall in different banks) and phase B sums them over the tile's pixels into one accumulator per
// parameter element and thread -> part[blockIdx.x][MD_SMALL].
constexpr int MD_TERMS = 8 * 16;
constexpr int MD_LD = MD_PIX_TILE + 1;
__global__ void __launch_bounds__(MD_PIX_TILE)
md_param_grad_kernel(const float* __restrict__ mask, const float* __restrict__ d_h2, const float* __restrict__ Wg, int P,
                     float* __restrict__ part) {
  extern __shared__ float sm[];      // [MD_TERMS][MD_LD]
  float* s_m = sm;                   // m[s * 4 + k]
  float* s_dy1 = sm + 16 * MD_LD;    // dL/d stage-1 conv output [c * 4 + s]
  float* s_e1 = sm + 32 * MD_LD;     // dL/d a1 * n1
  float* s_da1 = sm + 48 * MD_LD;    // dL/d a1 (holds a1 itself until the stage-1 backward)
  float* s_h1 = sm + 64 * MD_LD;
  float* s_dz = sm + 80 * MD_LD;     // dL/d stage-2 conv output
  float* s_e2 = sm + 96 * MD_LD;
  float* s_da2 = sm + 112 * MD_LD;
  __shared__ float s_w[MD_SMALL];
  const int tid = threadIdx.x;
  for (int i = tid; i < MD_SMALL; i += MD_PIX_TILE) s_w[i] = Wg[i];
  __syncthreads();
  const float* W = s_w;
  const int ntiles = P * (4096 / MD_PIX_TILE);
  float acc[3] = {0.f, 0.f, 0.f};    // parameter elements tid, tid + 128, tid + 256 (< MD_SMALL)
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int p = tile / (4096 / MD_PIX_TILE), pix = (tile % (4096 / MD_PIX_TILE)) * MD_PIX_TILE + tid;
    {
      const float* mask_p = mask + (size_t)p * 65536;
      float n1[16], rstd1[4], h1[16];
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        float m[4], n[4], a[4];
        rstd1[s] = md_stage1(mask_p, pix, s, W, m, n, a);
#pragma unroll
        for (int k = 0; k < 4; ++k) s_m[(s * 4 + k) * MD_LD + tid] = m[k];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = c * 4 + s;
          n1[j] = n[c];
          h1[j] = gelu_erf(a[c]);
          s_h1[j * MD_LD + tid] = h1[j];
          s_da1[j * MD_LD + tid] = a[c];
        }
      }
      float dz[16];
      {
        float n2[16], a2[16];
        const float rstd2 = md_stage2(h1, W, n2, a2);
        const float* dh = d_h2 + ((size_t)p * 4096 + pix) * 16;
        float mdn = 0.f, mdnn = 0.f;
#pragma unroll
        for (int o = 0; o < 16; ++o) {
          const float da = dh[o] * gelu_erf_grad(a2[o]);
          s_da2[o * MD_LD + tid] = da;
          s_e2[o * MD_LD + tid] = da * n2[o];
          dz[o] = da * W[MD_G2 + o];          // dL/d n2, turned into dL/d z below
          mdn += dz[o];
          mdnn += dz[o] * n2[o];
        }
        mdn *= (1.0f / 16); mdnn *= (1.0f / 16);
#pragma unroll
        for (int o = 0; o < 16; ++o) {
          dz[o] = rstd2 * (dz[o] - mdn - n2[o] * mdnn);
          s_dz[o * MD_LD + tid] = dz[o];
        }
      }
#pragma unroll 4   // fully unrolled, the 16 interleaved erf / exp evaluations need more than 255 registers
      for (int k = 0; k < 16; ++k) {
        float dh1 = 0.f;
#pragma unroll
        for (int o = 0; o < 16; ++o) dh1 += dz[o] * W[MD_W2 + o * 16 + k];
        const float da = dh1 * gelu_erf_grad(s_da1[k * MD_LD + tid]);
        s_da1[k * MD_LD + tid] = da;
        s_e1[k * MD_LD + tid] = da * n1[k];
        s_dy1[k * MD_LD + tid] = da * W[MD_G1 + (k >> 2)];    // dL/d n1, turned into dL/d y1 below
      }
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        float mdn1 = 0.f, mdnn1 = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float dn = s_dy1[(c * 4 + s) * MD_LD + tid];
          mdn1 += dn;
          mdnn1 += dn * n1[c * 4 + s];
        }
        mdn1 *= 0.25f; mdnn1 *= 0.25f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float* d = s_dy1 + (c * 4 + s) * MD_LD + tid;
          *d = rstd1[s] * (*d - mdn1 - n1[c * 4 + s] * mdnn1);
        }
      }
    }
    __syncthreads();
#pragma unroll 1
    for (int q = 0; q < 3; ++q) {
      const int j = tid + q * MD_PIX_TILE;
      if (j >= MD_SMALL) break;
      float sum = 0.f;
      if (j < MD_B1) {                       // W1[c][k] = sum_s dy1[c, s] m[s, k]
        const int c = j >> 2, k = j & 3;
#pragma unroll 4
        for (int i = 0; i < MD_PIX_TILE; ++i)
#pragma unroll
          for (int s = 0; s < 4; ++s) sum += s_dy1[(c * 4 + s) * MD_LD + i] * s_m[(s * 4 + k) * MD_LD + i];
      } else if (j < MD_W2) {                // b1 / gamma1 / beta1: sums over the 4 sub-pixels
        const float* src = j < MD_G1 ? s_dy1 : j < MD_BE1 ? s_e1 : s_da1;
        const int c = (j - MD_B1) & 3;
#pragma unroll 4
        for (int i = 0; i < MD_PIX_TILE; ++i)
#pragma unroll
          for (int s = 0; s < 4; ++s) sum += src[(c * 4 + s) * MD_LD + i];
      } else if (j < MD_B2) {                // W2[o][k] = dz[o] h1[k]
        const int o = (j - MD_W2) >> 4, k = (j - MD_W2) & 15;
#pragma unroll 4
        for (int i = 0; i < MD_PIX_TILE; ++i) sum += s_dz[o * MD_LD + i] * s_h1[k * MD_LD + i];
      } else {                               // b2 / gamma2 / beta2
        const float* src = j < MD_G2 ? s_dz : j < MD_BE2 ? s_e2 : s_da2;
        const int o = (j - MD_B2) & 15;
#pragma unroll 4
        for (int i = 0; i < MD_PIX_TILE; ++i) sum += src[o * MD_LD + i];
      }
      acc[q] += sum;
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int j = tid + q * MD_PIX_TILE;
    if (j < MD_SMALL) part[(size_t)blockIdx.x * MD_SMALL + j] = acc[q];
  }
}

// grads[j] (+)= sum over the partial rows of element j, in a fixed order: one warp per element.
__global__ void md_reduce_kernel(const float* __restrict__ part_small, int rows_small, const float* __restrict__ part_big, int rows_big,
                                 float* __restrict__ grads, int accumulate) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= MD_N) return;
  const bool small = j < MD_SMALL;
  const float* src = small ? part_small + j : part_big + (j - MD_SMALL);
  const int rows = small ? rows_small : rows_big;
  const long pitch = small ? MD_SMALL : MD_BIG;
  float s = 0.f;
  for (int r = lane; r < rows; r += 32) s += src[(long)r * pitch];
  s = warp_sum(s);
  if (lane == 0) grads[j] = accumulate ? grads[j] + s : s;
}

inline int md_grid2(int P) { return std::min(P * (4096 / MD_PIX_TILE), MD_GRID2); }
inline size_t md_scratch_floats(int P) {   // h2, d_h2, partials of both backward kernels
  return (size_t)P * 4096 * 16 * 2 + (size_t)md_grid2(P) * MD_SMALL + (size_t)(4096 / 16) * MD_BIG;
}
struct MdScratch { float *h2, *d_h2, *part_small, *part_big; };
inline MdScratch md_carve(float* base, int P) {
  MdScratch s;
  s.h2 = base;
  s.d_h2 = s.h2 + (size_t)P * 4096 * 16;
  s.part_small = s.d_h2 + (size_t)P * 4096 * 16;
  s.part_big = s.part_small + (size_t)md_grid2(P) * MD_SMALL;
  return s;
}

int md_forward(const float* mask, int P, const float* W, const float* emb_nchw, float* out, __nv_bfloat16* out_bf, const MdScratch& s,
               cudaStream_t st) {
  md_forward_kernel<<<dim3(4096 / 16, P), 256, 0, st>>>(mask, W, emb_nchw, out, out_bf, s.h2);
  LAUNCH_CHECK("md_forward");
  return 0;
}
// g = dL/d keys0 [P * 4096, 256] -> d_emb_nchw (if non-null) and the ten parameter gradients, added to (accumulate) or written over grads
int md_backward(const float* g, const float* mask, int P, const float* W, float* d_emb_nchw, const MdScratch& s, float* grads,
                int accumulate, cudaStream_t st) {
  md_keys_grad_kernel<<<4096 / 16, 256, 0, st>>>(g, s.h2, W, P, d_emb_nchw, s.d_h2, s.part_big);
  LAUNCH_CHECK("md_keys_grad");
  const size_t smem = (size_t)MD_TERMS * MD_LD * 4;
  if (cudaFuncSetAttribute(md_param_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return set_error("md_param_grad: shared-memory attribute failed");
  md_param_grad_kernel<<<md_grid2(P), MD_PIX_TILE, smem, st>>>(mask, s.d_h2, W, P, s.part_small);
  LAUNCH_CHECK("md_param_grad");
  md_reduce_kernel<<<nblk((long)MD_N * 32), 256, 0, st>>>(s.part_small, md_grid2(P), s.part_big, 4096 / 16, grads, accumulate);
  LAUNCH_CHECK("md_reduce");
  return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ data structures
struct Ten {
  float* v = nullptr;            // fp32 value
  float* g = nullptr;            // fp32 gradient (accumulated by the consumers' backward closures)
  __nv_bfloat16* b = nullptr;    // bf16 copy (GEMM operand)
  long rows = 0;
  int cols = 0;
  long n() const { return rows * cols; }
};
// tiles > 1: a conv-transpose as a linear layer over sub-pixel tiles, out = tiles * co columns; bias [out] holds the bias [co] once per
// tile, its gradient gb [co] sums over the tiles
struct DLin { int out = 0, in = 0, tiles = 1; __nv_bfloat16 *w = nullptr, *wT = nullptr; float *bias = nullptr, *gw = nullptr, *gb = nullptr; };
struct DLn { int D = 0; float eps = 1e-5f; float *g = nullptr, *b = nullptr, *gg = nullptr, *gb = nullptr; };
struct DAttn { DLin q, k, v, o; int inner = 0; };
struct DLayer { DAttn self, t2i, i2t; DLn n1, n2, n3, n4; DLin mlp1, mlp2; };

struct DecSlot {
  uint8_t* arena = nullptr;
  size_t cap = 0, used = 0;
  std::vector<std::function<int(cudaStream_t)>> tape;
  int P = 0, T = 0, Ts = 0, nm = 0, m0 = 0;
  bool images = false;               // prompt-free batch: prompt p is image p with no sparse tokens (msam_decoder_train_forward_images)
  Ten low4, iou32, keys0, tok;
  int* emb_index = nullptr;
  __nv_bfloat16* dmask8 = nullptr;
  float* mask = nullptr;             // mask prompts [P, 256, 256] of the last forward, or null (dense prompt = no_mask_embed)
  MdScratch md{};
  bool live = false;
};

struct DecTrain {
  DLayer layer[2];
  DAttn fin;
  DLn nfin, upln;
  DLin ct1, ct2, hyper[4][3], iou[3];
  float *point_emb = nullptr, *not_a_point = nullptr, *no_mask = nullptr, *out_tokens = nullptr;
  float *g_point_emb = nullptr, *g_nap = nullptr, *g_no_mask = nullptr, *g_out_tokens = nullptr;
  DecSlot slot[8];
  // mask_downscaling: packed fp32 masters / gradients (MD_* offsets), created by the first mask-prompt call; registered by the first
  // masked training forward, so that runs without mask prompts never see them
  float *md_w = nullptr, *md_g = nullptr;
  bool md_registered = false;
  bool md_written = false;           // a masked backward added to md_g since the last msam_decoder_zero_grads
  // Since the last msam_decoder_zero_grads: a backward of a prompt-free batch / of a prompted slot has run.  unreached = only
  // prompt-free ones: the IoU head and the sparse-prompt tables then have no gradient, and AdamW skips them (OptParam::skip).
  bool free_written = false, prompted_written = false, unreached = false;
};

namespace {

struct Ctx {
  Engine& e;
  DecTrain& d;
  DecSlot& s;
  cudaStream_t st;
  int err = 0;

  void* take(size_t bytes) {
    const size_t off = (s.used + 255) & ~size_t(255);
    if (off + bytes > s.cap) { err = set_error("decoder training: arena of %zu bytes exhausted (need %zu more)", s.cap, off + bytes - s.cap); return nullptr; }
    s.used = off + bytes;
    return s.arena + off;
  }
  Ten ten(long rows, int cols, bool v, bool g, bool b) {
    Ten t; t.rows = rows; t.cols = cols;
    if (v) t.v = (float*)take((size_t)rows * cols * 4);
    if (g) { t.g = (float*)take((size_t)rows * cols * 4); if (t.g) cudaMemsetAsync(t.g, 0, (size_t)rows * cols * 4, st); }
    if (b) t.b = (__nv_bfloat16*)take((size_t)rows * cols * 2);
    return t;
  }
};

int cast_grad(const float* g, const __nv_bfloat16* relu_y, long n, __nv_bfloat16* out, cudaStream_t st) {
  grad_cast_kernel<<<nblk(n / 4), 256, 0, st>>>((const float4*)g, (const uint2*)relu_y, n / 4, (uint2*)out);
  LAUNCH_CHECK("grad_cast");
  return 0;
}
int add_inplace(float* dst, const float* src, long n, cudaStream_t st) {
  add_inplace_kernel<<<nblk(n / 4), 256, 0, st>>>((float4*)dst, (const float4*)src, n / 4);
  LAUNCH_CHECK("add_inplace");
  return 0;
}

// y = act(x W^T + b) (+ residual).  bf16_out: y.b only (consumed by GEMMs / attention), else y.v fp32.
// backward: dy = y.g [o relu mask]; gW += dy^T x, gb += colsum(dy), x.g += dy W, residual.g += y.g
int op_linear(Ctx& c, const Ten& x, DLin& L, Ten& y, int act, const Ten* residual, bool bf16_out) {
  if (c.err) return -1;
  y = c.ten(x.rows, L.out, !bf16_out, true, bf16_out);
  if (c.err) return -1;
  GemmArgs a;
  a.A = x.b; a.W = L.w; a.M = (int)x.rows; a.N = L.out; a.K = L.in; a.lda = L.in; a.ldw = L.in; a.bias = L.bias; a.act = act;
  if (residual) { a.residual = residual->v; }
  a.out = bf16_out ? (void*)y.b : (void*)y.v; a.out_fp32 = bf16_out ? 0 : 1;
  RUN(launch_gemm(a, c.e.num_sms, c.st));
  Engine* e = &c.e;
  DLin* Lp = &L;
  const Ten xin = x, yout = y;
  const Ten res = residual ? *residual : Ten();
  const bool relu = act == 2;
  __nv_bfloat16* scratch = (__nv_bfloat16*)c.take((size_t)y.rows * L.out * 2);
  if (c.err) return -1;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(cast_grad(yout.g, relu ? yout.b : nullptr, yout.n(), scratch, st));
    RUN(launch_gemm_tn(scratch, xin.b, Lp->out, Lp->in, (int)xin.rows, Lp->out, Lp->in, Lp->gw, Lp->in, st, 1));
    RUN(launch_colsum(scratch, xin.rows * Lp->tiles, Lp->out / Lp->tiles, Lp->gb, st));   // [rows, tiles * co] read as [tiles * rows, co]
    if (xin.g) {
      GemmArgs a;
      a.A = scratch; a.W = Lp->wT; a.M = (int)xin.rows; a.N = Lp->in; a.K = Lp->out; a.lda = Lp->out; a.ldw = Lp->out;
      a.residual = xin.g; a.out = xin.g; a.out_fp32 = 1;
      RUN(launch_gemm(a, e->num_sms, st));
    }
    if (res.g) RUN(add_inplace(res.g, yout.g, yout.n(), st));
    return 0;
  });
  return 0;
}

int op_layernorm(Ctx& c, const Ten& x, DLn& L, Ten& y, bool want_v = true) {
  if (c.err) return -1;
  y = c.ten(x.rows, x.cols, want_v, true, true);
  if (c.err) return -1;
  LnArgs l;
  l.x = x.v; l.rows = (int)x.rows; l.D = x.cols; l.gamma = L.g; l.beta = L.b; l.eps = L.eps; l.out = y.b; l.out_f32 = y.v;
  RUN(launch_layernorm(l, c.st));
  const Ten xin = x, yout = y;
  DLn* Lp = &L;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    return launch_layernorm_bwd(xin.v, (int)xin.rows, xin.cols, Lp->g, Lp->eps, yout.g, 0, 64, 14, 1, xin.g, Lp->gg, Lp->gb, st);
  });
  return 0;
}

// y.b = bf16(a.v + b_v[row % b_rows]) ; backward: a.g += y.g ; b_g += y.g (same row count only)
int op_add_cast(Ctx& c, const Ten& a, const float* b_v, long b_rows, float* b_g, Ten& y) {
  if (c.err) return -1;
  y = c.ten(a.rows, a.cols, false, true, true);
  if (c.err) return -1;
  add_cast_kernel<<<nblk(a.n() / 4), 256, 0, c.st>>>((const float4*)a.v, (const float4*)b_v, a.n() / 4, b_rows * a.cols / 4, (uint2*)y.b);
  LAUNCH_CHECK("add_cast");
  const Ten ain = a, yout = y;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(add_inplace(ain.g, yout.g, yout.n(), st));
    if (b_g) RUN(add_inplace(b_g, yout.g, yout.n(), st));
    return 0;
  });
  return 0;
}

// softmax(q k^T / sqrt(hd)) v per (prompt, head); q [P*Tq, inner], k / v [P*Tk, inner] (bf16 + fp32 gradients) -> o (fp32 + bf16)
int op_attention(Ctx& c, const Ten& q, const Ten& k, const Ten& v, int P, int Tq, int Tk, int inner, int heads, Ten& o) {
  if (c.err) return -1;
  const int hd = inner / heads, pitch = (Tk + 7) & ~7;
  const float scale = 1.0f / sqrtf((float)hd);
  const long nb = (long)P * heads;
  o = c.ten((long)P * Tq, inner, true, true, true);
  float* S = (float*)c.take((size_t)nb * Tq * pitch * 4);
  __nv_bfloat16* Pm = (__nv_bfloat16*)c.take((size_t)nb * Tq * pitch * 2);
  __nv_bfloat16* dS = (__nv_bfloat16*)c.take((size_t)nb * Tq * pitch * 2);
  __nv_bfloat16* dOb = (__nv_bfloat16*)c.take((size_t)P * Tq * inner * 2);
  if (c.err) return -1;
  const long s_h = (long)Tq * pitch, s_w = (long)heads * Tq * pitch;
  BGemmArgs a;
  a.A = q.b; a.B = k.b; a.M = Tq; a.N = pitch; a.K = hd; a.lda = a.ldb = inner; a.a_hstride = a.b_hstride = hd;
  a.a_wstride = (long)Tq * inner; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk;
  a.heads = heads; a.outer = P; a.out = S; a.ldc = pitch; a.o_hstride = s_h; a.o_wstride = s_w; a.alpha = scale;
  RUN(launch_bgemm(a, c.st));
  softmax_rows_kernel<<<nblk(nb * Tq, 8), 256, 0, c.st>>>(S, nb * Tq, Tk, pitch, Pm);
  LAUNCH_CHECK("softmax_rows");
  // O = P V, written head-interleaved [P*Tq, inner]
  a = BGemmArgs();
  a.A = Pm; a.B = v.b; a.b_mn = 1; a.M = Tq; a.N = hd; a.K = pitch; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
  a.b_hstride = hd; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk; a.heads = heads; a.outer = P;
  a.out = o.v; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tq * inner;
  RUN(launch_bgemm(a, c.st));
  RUN(launch_cast_bf16(o.v, o.n(), o.b, c.st));
  const Ten qq = q, kk = k, vv = v, oo = o;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(cast_grad(oo.g, nullptr, oo.n(), dOb, st));
    BGemmArgs a;
    // dV += P^T dO
    a.A = Pm; a.B = dOb; a.a_mn = a.b_mn = 1; a.M = Tk; a.N = hd; a.K = Tq; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
    a.b_hstride = hd; a.b_wstride = (long)Tq * inner; a.heads = heads; a.outer = P;
    a.out = vv.g; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tk * inner; a.accumulate = 1;
    RUN(launch_bgemm(a, st));
    // dP = dO V^T (over S)
    a = BGemmArgs();
    a.A = dOb; a.B = vv.b; a.M = Tq; a.N = pitch; a.K = hd; a.lda = a.ldb = inner; a.a_hstride = a.b_hstride = hd;
    a.a_wstride = (long)Tq * inner; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk;
    a.heads = heads; a.outer = P; a.out = S; a.ldc = pitch; a.o_hstride = s_h; a.o_wstride = s_w;
    RUN(launch_bgemm(a, st));
    ds_rows_kernel<<<nblk(nb * Tq, 8), 256, 0, st>>>(Pm, S, nb * Tq, Tk, pitch, dS);
    LAUNCH_CHECK("ds_rows");
    // dQ += scale dS K
    a = BGemmArgs();
    a.A = dS; a.B = kk.b; a.b_mn = 1; a.M = Tq; a.N = hd; a.K = pitch; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
    a.b_hstride = hd; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk; a.heads = heads; a.outer = P;
    a.out = qq.g; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tq * inner; a.alpha = scale; a.accumulate = 1;
    RUN(launch_bgemm(a, st));
    // dK += scale dS^T Q
    a = BGemmArgs();
    a.A = dS; a.B = qq.b; a.a_mn = a.b_mn = 1; a.M = Tk; a.N = hd; a.K = Tq; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
    a.b_hstride = hd; a.b_wstride = (long)Tq * inner; a.heads = heads; a.outer = P;
    a.out = kk.g; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tk * inner; a.alpha = scale; a.accumulate = 1;
    RUN(launch_bgemm(a, st));
    return 0;
  });
  return 0;
}

// y.b = gelu(x.b); backward: x.g += y.g o gelu'(x)
int op_gelu(Ctx& c, const Ten& x, Ten& y) {
  if (c.err) return -1;
  y = c.ten(x.rows, x.cols, false, true, true);
  __nv_bfloat16* t1 = (__nv_bfloat16*)c.take((size_t)x.n() * 2);
  float* t2 = (float*)c.take((size_t)x.n() * 4);
  if (c.err) return -1;
  RUN(launch_gelu_fwd(x.b, x.n(), y.b, c.st));
  const Ten xin = x, yout = y;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(cast_grad(yout.g, nullptr, yout.n(), t1, st));
    RUN(launch_gelu_bwd(t1, xin.b, xin.n(), t1, st));
    RUN(launch_cast_f32(t1, xin.n(), t2, st));
    return add_inplace(xin.g, t2, xin.n(), st);
  });
  return 0;
}

// rows of a [P, pitch] view <-> compact [P, cols] tensor (token slices)
int op_slice_rows(Ctx& c, const Ten& x, long offset, long pitch, long rows, int cols, Ten& y) {
  if (c.err) return -1;
  y = c.ten(rows, cols, true, true, true);
  if (c.err) return -1;
  copy_rows_kernel<<<nblk(rows * cols), 256, 0, c.st>>>(x.v + offset, pitch, y.v, cols, rows, cols, 0);
  LAUNCH_CHECK("slice_rows");
  RUN(launch_cast_bf16(y.v, y.n(), y.b, c.st));
  const Ten xin = x, yout = y;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    copy_rows_kernel<<<nblk(rows * cols), 256, 0, st>>>(yout.g, cols, xin.g + offset, pitch, rows, cols, 1);
    LAUNCH_CHECK("slice_rows_bwd");
    return 0;
  });
  return 0;
}

int attn_module(Ctx& c, DAttn& A, const Ten& q_in, const Ten& k_in, const Ten& v_in, int P, int Tq, int Tk, const Ten* residual, Ten& out) {
  Ten q, k, v, o;
  RUN(op_linear(c, q_in, A.q, q, 0, nullptr, true));
  RUN(op_linear(c, k_in, A.k, k, 0, nullptr, true));
  RUN(op_linear(c, v_in, A.v, v, 0, nullptr, true));
  RUN(op_attention(c, q, k, v, P, Tq, Tk, A.inner, 8, o));
  return op_linear(c, o, A.o, out, 0, residual, false);
}

}  // namespace

// ------------------------------------------------------------------------------------------------ setup
// registered with the upstream element counts; out_pad > out: the GEMM operands have out_pad rows, the rows beyond out stay zero (their
// gradient rows are sums of zeros)
static int dt_lin(Engine& e, const std::string& key, int out, int in, DLin* L, int out_pad = 0) {
  const auto* w = e.host(key + ".weight", {out, in});
  const auto* b = e.host(key + ".bias", {out});
  if (!w || !b) return -1;
  const int op = out_pad > out ? out_pad : out;
  std::vector<float> wp((size_t)op * in, 0.f), bp(op, 0.f);
  std::copy(w->begin(), w->end(), wp.begin());
  std::copy(b->begin(), b->end(), bp.begin());
  L->out = op; L->in = in;
  CHK(L->w = e.upload_bf16(wp.data(), wp.size()));
  CHK(L->wT = (__nv_bfloat16*)e.dalloc((size_t)op * in * 2));
  RUN(launch_transpose_bf16(L->w, op, in, L->wT, 0));
  CHK(L->bias = e.upload_f32(bp.data(), bp.size()));
  CHK(L->gw = (float*)e.dalloc((size_t)op * in * 4, true));
  CHK(L->gb = (float*)e.dalloc((size_t)op * 4, true));
  OptParam pw, pb;
  pw.key = key + ".weight"; pw.g = L->gw; pw.n = (int64_t)out * in; pw.decoder = true;
  pw.refresh = Refresh::Cast; pw.dst = L->w; pw.dstT = L->wT; pw.rows = op; pw.cols = in;
  pb.key = key + ".bias"; pb.w = L->bias; pb.g = L->gb; pb.n = out; pb.decoder = true;
  CHK(e.train_add(pw, w->data()) && e.train_add(pb));
  return 0;
}
static int dt_ln(Engine& e, const std::string& key, int D, float eps, DLn* L) {
  L->D = D; L->eps = eps;
  CHK(L->g = e.up_f32(key + ".weight", {D}));
  CHK(L->b = e.up_f32(key + ".bias", {D}));
  OptParam p;
  p.n = D; p.decoder = true;
  p.key = key + ".weight"; p.w = L->g; CHK(L->gg = e.train_add(p));
  p.key = key + ".bias"; p.w = L->b; CHK(L->gb = e.train_add(p));
  return 0;
}
static int dt_attn(Engine& e, const std::string& key, int inner, DAttn* A) {
  A->inner = inner;
  RUN(dt_lin(e, key + ".q_proj", inner, 256, &A->q));
  RUN(dt_lin(e, key + ".k_proj", inner, 256, &A->k));
  RUN(dt_lin(e, key + ".v_proj", inner, 256, &A->v));
  return dt_lin(e, key + ".out_proj", 256, inner, &A->o);
}
// ConvTranspose2d(k = 2, s = 2) weight [ci, co, 2, 2] as the GEMM operand [(dy*2+dx)*co + o][ci], registered in this layout under
// "<key>.weight@gemm"; the bias is registered as [co] and refreshed into the 4 tiles the GEMM epilogue reads
static int dt_convT(Engine& e, const std::string& key, int ci, int co, DLin* L) {
  const auto* w = e.host(key + ".weight", {ci, co, 2, 2});
  const auto* b = e.host(key + ".bias", {co});
  if (!w || !b) return -1;
  std::vector<float> wg((size_t)4 * co * ci), bg((size_t)4 * co);
  for (int i = 0; i < ci; ++i)
    for (int o = 0; o < co; ++o)
      for (int s = 0; s < 4; ++s) wg[((size_t)s * co + o) * ci + i] = (*w)[((size_t)i * co + o) * 4 + s];
  for (int s = 0; s < 4; ++s)
    for (int o = 0; o < co; ++o) bg[s * co + o] = (*b)[o];
  L->out = 4 * co; L->in = ci; L->tiles = 4;
  CHK(L->w = e.upload_bf16(wg.data(), wg.size()));
  CHK(L->wT = (__nv_bfloat16*)e.dalloc(wg.size() * 2));
  RUN(launch_transpose_bf16(L->w, 4 * co, ci, L->wT, 0));
  CHK(L->bias = e.upload_f32(bg.data(), bg.size()));
  OptParam pw, pb;
  pw.key = key + ".weight@gemm"; pw.n = (int64_t)wg.size(); pw.decoder = true;
  pw.refresh = Refresh::Cast; pw.dst = L->w; pw.dstT = L->wT; pw.rows = 4 * co; pw.cols = ci;
  pb.key = key + ".bias"; pb.n = co; pb.decoder = true; pb.refresh = Refresh::TileBias4; pb.dst4 = L->bias;
  CHK(L->gw = e.train_add(pw, wg.data()));
  CHK(L->gb = e.train_add(pb, b->data()));
  return 0;
}

int Engine::dec_train_setup() {
  if (dtrain) return 0;
  if (!finalized || !dec) return set_error("decoder training: weights not loaded");
  if (dec_host.empty()) return set_error("decoder training: host copies of the decoder weights are gone");
  host_weights.swap(dec_host);   // host()/up_f32() read host_weights
  dtrain = new DecTrain();
  DecTrain& d = *dtrain;
  int rc = 0;
  auto go = [&]() -> int {
    const std::string m = "mask_decoder.", tr = m + "transformer.";
    for (int l = 0; l < 2; ++l) {
      const std::string p = tr + "layers." + std::to_string(l) + ".";
      DLayer& L = d.layer[l];
      RUN(dt_attn(*this, p + "self_attn", 256, &L.self));
      RUN(dt_attn(*this, p + "cross_attn_token_to_image", 128, &L.t2i));
      RUN(dt_attn(*this, p + "cross_attn_image_to_token", 128, &L.i2t));
      RUN(dt_ln(*this, p + "norm1", 256, 1e-5f, &L.n1));
      RUN(dt_ln(*this, p + "norm2", 256, 1e-5f, &L.n2));
      RUN(dt_ln(*this, p + "norm3", 256, 1e-5f, &L.n3));
      RUN(dt_ln(*this, p + "norm4", 256, 1e-5f, &L.n4));
      RUN(dt_lin(*this, p + "mlp.lin1", 2048, 256, &L.mlp1));
      RUN(dt_lin(*this, p + "mlp.lin2", 256, 2048, &L.mlp2));
    }
    RUN(dt_attn(*this, tr + "final_attn_token_to_image", 128, &d.fin));
    RUN(dt_ln(*this, tr + "norm_final_attn", 256, 1e-5f, &d.nfin));
    RUN(dt_convT(*this, m + "output_upscaling.0", 256, 64, &d.ct1));
    RUN(dt_ln(*this, m + "output_upscaling.1", 64, 1e-6f, &d.upln));
    RUN(dt_convT(*this, m + "output_upscaling.3", 64, 32, &d.ct2));
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 3; ++j)
        RUN(dt_lin(*this, m + "output_hypernetworks_mlps." + std::to_string(i) + ".layers." + std::to_string(j), j == 2 ? 32 : 256, 256, &d.hyper[i][j]));
    for (int j = 0; j < 3; ++j)
      RUN(dt_lin(*this, m + "iou_prediction_head.layers." + std::to_string(j), j == 2 ? 4 : 256, 256, &d.iou[j], 32));
    // embedding tables: the 4 point embeddings and the output tokens (iou token, then the 4 mask tokens) are each one buffer
    std::vector<float> pe(4 * 256), ot(5 * 256);
    for (int i = 0; i < 4; ++i) {
      const auto* w = host("prompt_encoder.point_embeddings." + std::to_string(i) + ".weight", {1, 256});
      CHK(w);
      std::copy(w->begin(), w->end(), pe.begin() + i * 256);
    }
    const auto* it = host(m + "iou_token.weight", {1, 256});
    const auto* mt = host(m + "mask_tokens.weight", {4, 256});
    CHK(it && mt);
    std::copy(it->begin(), it->end(), ot.begin());
    std::copy(mt->begin(), mt->end(), ot.begin() + 256);
    CHK(d.point_emb = upload_f32(pe.data(), pe.size()));
    CHK(d.out_tokens = upload_f32(ot.data(), ot.size()));
    CHK(d.not_a_point = up_f32("prompt_encoder.not_a_point_embed.weight", {1, 256}));
    CHK(d.no_mask = up_f32("prompt_encoder.no_mask_embed.weight", {1, 256}));
    CHK(d.g_point_emb = (float*)dalloc(4 * 256 * 4, true));
    CHK(d.g_out_tokens = (float*)dalloc(5 * 256 * 4, true));
    OptParam p;
    p.decoder = true;
    for (int i = 0; i < 4; ++i) {
      p.key = "prompt_encoder.point_embeddings." + std::to_string(i) + ".weight"; p.w = d.point_emb + i * 256; p.g = d.g_point_emb + i * 256;
      p.n = 256;
      CHK(train_add(p));
    }
    p.key = "prompt_encoder.not_a_point_embed.weight"; p.w = d.not_a_point; p.g = nullptr; p.n = 256; CHK(d.g_nap = train_add(p));
    p.key = m + "iou_token.weight"; p.w = d.out_tokens; p.g = d.g_out_tokens; p.n = 256; CHK(train_add(p));
    p.key = m + "mask_tokens.weight"; p.w = d.out_tokens + 256; p.g = d.g_out_tokens + 256; p.n = 4 * 256; CHK(train_add(p));
    p.key = "prompt_encoder.no_mask_embed.weight"; p.w = d.no_mask; p.g = nullptr; p.n = 256; CHK(d.g_no_mask = train_add(p));
    // what a prompt-free batch cannot reach (its loss ignores the IoU predictions; no sparse tokens): torch leaves their .grad None
    // after such backwards only, and AdamW skips them (mask_downscaling is skipped through md_written)
    for (OptParam& q : opt)
      if (q.key.rfind(m + "iou_prediction_head.", 0) == 0 || q.key.rfind("prompt_encoder.point_embeddings.", 0) == 0 ||
          q.key == "prompt_encoder.not_a_point_embed.weight")
        q.skip = &d.unreached;
    return 0;
  };
  rc = go();
  host_weights.swap(dec_host);
  if (rc == 0 && cudaDeviceSynchronize() != cudaSuccess) rc = set_error("decoder training setup: %s", cudaGetErrorString(cudaGetLastError()));
  if (rc) { delete dtrain; dtrain = nullptr; }
  return rc;
}

namespace {
struct MdTensor { const char* key; int off; std::initializer_list<int64_t> shape; };
const MdTensor kMdTensors[10] = {
    {"0.weight", MD_W1, {4, 1, 2, 2}},  {"0.bias", MD_B1, {4}},  {"1.weight", MD_G1, {4}},  {"1.bias", MD_BE1, {4}},
    {"3.weight", MD_W2, {16, 4, 2, 2}}, {"3.bias", MD_B2, {16}}, {"4.weight", MD_G2, {16}}, {"4.bias", MD_BE2, {16}},
    {"6.weight", MD_W3, {256, 16, 1, 1}}, {"6.bias", MD_B3, {256}}};
const std::string kMdPrefix = "prompt_encoder.mask_downscaling.";
int64_t md_numel(const MdTensor& t) { int64_t n = 1; for (int64_t d : t.shape) n *= d; return n; }
}  // namespace

// fp32 masters of mask_downscaling (from the host copies) and a zeroed gradient buffer; nothing is registered yet
int Engine::md_setup() {
  RUN(dec_train_setup());
  DecTrain& d = *dtrain;
  if (d.md_w) return 0;
  std::vector<float> w(MD_N);
  host_weights.swap(dec_host);
  int rc = 0;
  for (const MdTensor& t : kMdTensors) {
    const auto* h = host(kMdPrefix + t.key, t.shape);
    if (!h) { rc = -1; break; }
    std::copy(h->begin(), h->end(), w.begin() + t.off);
  }
  host_weights.swap(dec_host);
  if (rc) return rc;
  CHK(d.md_w = upload_f32(w.data(), w.size()));
  CHK(d.md_g = (float*)dalloc((size_t)MD_N * 4, true));
  return 0;
}

// the ten tensors join the registry (after every tensor registered before); AdamW updates them only after a
// masked backward has written their gradient since the last msam_decoder_zero_grads (torch.optim.AdamW skips a parameter whose grad
// is None), with their own step count
int Engine::md_register() {
  RUN(md_setup());
  DecTrain& d = *dtrain;
  if (d.md_registered) return 0;
  for (const MdTensor& t : kMdTensors) {
    OptParam p;
    p.key = kMdPrefix + t.key; p.w = d.md_w + t.off; p.g = d.md_g + t.off; p.n = md_numel(t); p.written = &d.md_written; p.decoder = true;
    CHK(train_add(p));
  }
  d.md_registered = true;
  return 0;
}

int Engine::op_mask_downscaling_train(const float* mask, int P, const float* d_dense, float* dense_out, float* grads_out,
                                      cudaStream_t st) {
  if (P <= 0) return set_error("msam_op_mask_downscaling_train: P = %d", P);
  RUN(md_setup());
  const float* W = dtrain->md_w;
  float* scratch = nullptr;
  if (cudaMallocAsync((void**)&scratch, md_scratch_floats(P) * 4, st) != cudaSuccess)
    return set_error("msam_op_mask_downscaling_train: cudaMallocAsync failed");
  const MdScratch s = md_carve(scratch, P);
  int rc = md_forward(mask, P, W, nullptr, dense_out, nullptr, s, st);
  if (!rc) rc = md_backward(d_dense, mask, P, W, nullptr, s, grads_out, 0, st);
  cudaFreeAsync(scratch, st);
  return rc;
}

// ------------------------------------------------------------------------------------------------ forward
int Engine::decoder_train_forward(int slot, const float* emb_nchw, const float* sparse, const int* emb_index, int Ts, int P,
                                  const float* mask_in, int multimask, float* low_res, float* iou, cudaStream_t st) {
  if (slot < 0 || slot >= 8) return set_error("decoder training: slot %d outside [0, 8)", slot);
  if (P <= 0 || Ts <= 0 || !sparse || !emb_index) return set_error("decoder training: needs sparse prompt embeddings (points and / or boxes)");
  if (5 + Ts > 64) return set_error("decoder training: %d tokens per prompt exceeds the supported 64", 5 + Ts);
  return dec_train_run(slot, emb_nchw, sparse, emb_index, Ts, P, mask_in, false, multimask, low_res, iou, st);
}

int Engine::decoder_train_forward_images(int slot, const float* emb_nchw, int B, int multimask, float* low_res, float* iou,
                                         cudaStream_t st) {
  if (slot < 0 || slot >= 8) return set_error("decoder training: slot %d outside [0, 8)", slot);
  if (B <= 0) return set_error("decoder training: B = %d images", B);
  return dec_train_run(slot, emb_nchw, nullptr, nullptr, 0, B, nullptr, true, multimask, low_res, iou, st);
}

// The tape of one slot.  images = false: P prompts of ONE image (Ts sparse tokens each, dense prompt no_mask_embed or
// mask_downscaling(mask_in)); images = true: P images with no prompt (T = 5 output tokens, dense prompt no_mask_embed), prompt p
// reading image p.  Every op after the keys is per prompt either way.
int Engine::dec_train_run(int slot, const float* emb_nchw, const float* sparse, const int* emb_index, int Ts, int P,
                          const float* mask_in, bool images, int multimask, float* low_res, float* iou, cudaStream_t st) {
  RUN(dec_train_setup());
  if (mask_in) RUN(md_register());
  DecTrain& d = *dtrain;
  DecSlot& s = d.slot[slot];
  const int T = 5 + Ts;
  const long Rt = (long)P * T, Ri = (long)P * 4096;
  {   // arena: ~ 110 fp32-equivalents of [P*4096, 256] cover the image-side tensors of both layers + the upscaling path
    size_t need = (size_t)Ri * 256 * 4 * 64 + ((size_t)64 << 20);
    if (mask_in) need += ((size_t)P * 65536 + md_scratch_floats(P)) * 4 + 1024;
    if (s.cap < need) {
      if (s.arena) cudaFree(s.arena);
      s.arena = nullptr; s.cap = 0;
      if (cudaMalloc(&s.arena, need) != cudaSuccess) return set_error("decoder training: cudaMalloc of %zu bytes failed", need);
      s.cap = need;
    }
  }
  s.used = 0; s.tape.clear(); s.live = false; s.mask = nullptr;
  s.P = P; s.T = T; s.Ts = Ts; s.nm = multimask ? 3 : 1; s.m0 = multimask ? 1 : 0; s.images = images; s.emb_index = nullptr;
  Ctx c{*this, d, s, st};
  if (Ts > 0) {
    s.emb_index = (int*)c.take((size_t)P * Ts * 4);
    if (c.err) return -1;
    if (cudaMemcpyAsync(s.emb_index, emb_index, (size_t)P * Ts * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("decoder training: copy failed");
  }
  // tokens and image-side source
  Ten tok = c.ten(Rt, 256, true, true, true);
  Ten keys0 = c.ten(Ri, 256, true, true, true);
  if (c.err) return -1;
  assemble_tokens_kernel<<<nblk(Rt * 256), 256, 0, st>>>(d.out_tokens, sparse, P, T, Ts, tok.v);
  LAUNCH_CHECK("assemble_tokens");
  RUN(launch_cast_bf16(tok.v, tok.n(), tok.b, st));
  if (mask_in) {   // dense prompt = mask_downscaling(mask); the mask is kept: the backward pass recomputes the stages from it
    s.mask = (float*)c.take((size_t)P * 65536 * 4);
    float* scratch = (float*)c.take(md_scratch_floats(P) * 4);
    if (c.err) return -1;
    s.md = md_carve(scratch, P);
    if (cudaMemcpyAsync(s.mask, mask_in, (size_t)P * 65536 * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return set_error("decoder training: copy failed");
    RUN(md_forward(s.mask, P, d.md_w, emb_nchw, keys0.v, keys0.b, s.md, st));
  } else if (images) {
    src_images_kernel<<<dim3(128, 8, P), dim3(32, 8), 0, st>>>(emb_nchw, d.no_mask, keys0.v);
    LAUNCH_CHECK("src_images");
    RUN(launch_cast_bf16(keys0.v, keys0.n(), keys0.b, st));
  } else {
    src_broadcast_kernel<<<dim3(128, 8), dim3(32, 8), 0, st>>>(emb_nchw, d.no_mask, P, keys0.v);
    LAUNCH_CHECK("src_broadcast");
    RUN(launch_cast_bf16(keys0.v, keys0.n(), keys0.b, st));
  }
  s.tok = tok; s.keys0 = keys0;
  const float* pos = dec_pos();     // dense positional encoding, token-major [4096, 256] (no parameters)
  Ten Q = tok, K = keys0;
  for (int l = 0; l < 2; ++l) {
    DLayer& L = d.layer[l];
    Ten a, Q1, Q2, Q3, qin, kin, h;
    // self attention
    if (l == 0) {
      RUN(attn_module(c, L.self, Q, Q, Q, P, T, T, nullptr, a));
    } else {
      RUN(op_add_cast(c, Q, tok.v, Rt, tok.g, qin));
      RUN(attn_module(c, L.self, qin, qin, Q, P, T, T, &Q, a));
    }
    RUN(op_layernorm(c, a, L.n1, Q1));
    // token -> image
    RUN(op_add_cast(c, Q1, tok.v, Rt, tok.g, qin));
    RUN(op_add_cast(c, K, pos, 4096, nullptr, kin));
    RUN(attn_module(c, L.t2i, qin, kin, K, P, T, 4096, &Q1, a));
    RUN(op_layernorm(c, a, L.n2, Q2));
    // MLP
    RUN(op_linear(c, Q2, L.mlp1, h, 2, nullptr, true));
    RUN(op_linear(c, h, L.mlp2, a, 0, &Q2, false));
    RUN(op_layernorm(c, a, L.n3, Q3));
    // image -> token
    RUN(op_add_cast(c, Q3, tok.v, Rt, tok.g, qin));
    RUN(attn_module(c, L.i2t, kin, qin, Q3, P, 4096, T, &K, a));
    Ten K1;
    RUN(op_layernorm(c, a, L.n4, K1));
    Q = Q3; K = K1;
  }
  Ten qin, kin, a, hs;
  RUN(op_add_cast(c, Q, tok.v, Rt, tok.g, qin));
  RUN(op_add_cast(c, K, pos, 4096, nullptr, kin));
  RUN(attn_module(c, d.fin, qin, kin, K, P, T, 4096, &Q, a));
  RUN(op_layernorm(c, a, d.nfin, hs));
  // upscaling: convT1 -> LayerNorm2d -> GELU -> convT2 -> GELU, all as row-wise ops on [pixel, sub-pixel] rows
  Ten u1, y1, a1, u2, up;
  RUN(op_linear(c, K, d.ct1, u1, 0, nullptr, false));                  // [Ri, 4 * 64]
  Ten u1r = u1; u1r.rows = Ri * 4; u1r.cols = 64;
  RUN(op_layernorm(c, u1r, d.upln, y1, false));                         // [Ri * 4, 64]
  RUN(op_gelu(c, y1, a1));
  RUN(op_linear(c, a1, d.ct2, u2, 0, nullptr, true));                  // [Ri * 4, 4 * 32]
  RUN(op_gelu(c, u2, up));                                              // rows of 32 channels: [Ri * 16, 32]
  // hyper-network MLPs on the mask tokens, IoU head on the IoU token
  Ten hyper = c.ten((long)P * 8, 32, true, true, true);                 // [P, 8 (4 used), 32]
  if (c.err) return -1;
  if (cudaMemsetAsync(hyper.v, 0, (size_t)hyper.n() * 4, st) != cudaSuccess) return set_error("decoder training: memset failed");
  for (int i = 0; i < 4; ++i) {
    Ten x, h1, h2, h3;
    RUN(op_slice_rows(c, hs, (long)(1 + i) * 256, (long)T * 256, P, 256, x));
    RUN(op_linear(c, x, d.hyper[i][0], h1, 2, nullptr, true));
    RUN(op_linear(c, h1, d.hyper[i][1], h2, 2, nullptr, true));
    RUN(op_linear(c, h2, d.hyper[i][2], h3, 0, nullptr, false));       // [P, 32]
    copy_rows_kernel<<<nblk((long)P * 32), 256, 0, st>>>(h3.v, 32, hyper.v + i * 32, 8 * 32, P, 32, 0);
    LAUNCH_CHECK("hyper_gather");
    const Ten h3c = h3, hyc = hyper;
    const int ii = i, PP = P;
    s.tape.push_back([=](cudaStream_t st2) -> int {
      copy_rows_kernel<<<nblk((long)PP * 32), 256, 0, st2>>>(hyc.g + ii * 32, 8 * 32, h3c.g, 32, PP, 32, 1);
      LAUNCH_CHECK("hyper_scatter");
      return 0;
    });
  }
  RUN(launch_cast_bf16(hyper.v, hyper.n(), hyper.b, st));
  {
    Ten x, h1, h2;
    RUN(op_slice_rows(c, hs, 0, (long)T * 256, P, 256, x));
    RUN(op_linear(c, x, d.iou[0], h1, 2, nullptr, true));
    RUN(op_linear(c, h1, d.iou[1], h2, 2, nullptr, true));
    RUN(op_linear(c, h2, d.iou[2], s.iou32, 0, nullptr, false));       // [P, 32], columns 0..3 real
    copy_rows_kernel<<<nblk((long)P * s.nm), 256, 0, st>>>(s.iou32.v + s.m0, 32, iou, s.nm, P, s.nm, 0);
    LAUNCH_CHECK("iou_out");
  }
  // masks = hyper @ upscaled: per prompt [65536 x 32] x [32 x 4]
  s.low4 = c.ten((long)P * 65536, 4, true, false, false);
  s.dmask8 = (__nv_bfloat16*)c.take((size_t)P * 65536 * 8 * 2);
  if (c.err) return -1;
  {
    BGemmArgs g;
    g.A = up.b; g.B = hyper.b; g.M = 65536; g.N = 4; g.K = 32; g.lda = 32; g.ldb = 32; g.a_wstride = 65536L * 32; g.b_wstride = 8 * 32;
    g.b_rows_valid = 4; g.heads = 1; g.outer = P; g.out = s.low4.v; g.ldc = 4; g.o_wstride = 65536L * 4;
    RUN(launch_bgemm(g, st));
    masks_out_kernel<<<nblk((long)P * s.nm * 65536), 256, 0, st>>>(s.low4.v, P, s.nm, s.m0, low_res);
    LAUNCH_CHECK("masks_out");
    const Ten upc = up, hyc = hyper;
    __nv_bfloat16* dm = s.dmask8;
    const int PP = P;
    s.tape.push_back([=](cudaStream_t st2) -> int {   // dmask8 was filled by decoder_train_backward
      BGemmArgs g;
      // d up += dmask hyper
      g.A = dm; g.B = hyc.b; g.b_mn = 1; g.M = 65536; g.N = 32; g.K = 8; g.lda = 8; g.ldb = 32; g.a_wstride = 65536L * 8; g.b_wstride = 8 * 32;
      g.heads = 1; g.outer = PP; g.out = upc.g; g.ldc = 32; g.o_wstride = 65536L * 32; g.accumulate = 1;
      RUN(launch_bgemm(g, st2));
      // d hyper += dmask^T up
      g = BGemmArgs();
      g.A = dm; g.B = upc.b; g.a_mn = g.b_mn = 1; g.M = 8; g.N = 32; g.K = 65536; g.lda = 8; g.ldb = 32; g.a_wstride = 65536L * 8;
      g.b_wstride = 65536L * 32; g.heads = 1; g.outer = PP; g.out = hyc.g; g.ldc = 32; g.o_wstride = 8 * 32; g.accumulate = 1;
      return launch_bgemm(g, st2);
    });
  }
  if (c.err) return -1;
  s.live = true;
  return 0;
}

// ------------------------------------------------------------------------------------------------ backward
int Engine::decoder_train_backward(int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, cudaStream_t st) {
  if (!dtrain || slot < 0 || slot >= 8 || !dtrain->slot[slot].live) return set_error("decoder training: no saved forward pass in slot %d", slot);
  DecTrain& d = *dtrain;
  DecSlot& s = d.slot[slot];
  const int P = s.P;
  if (d_low_res) {
    masks_grad_kernel<<<nblk((long)P * 65536), 256, 0, st>>>(d_low_res, P, s.nm, s.m0, s.dmask8);
    LAUNCH_CHECK("masks_grad");
  } else if (cudaMemsetAsync(s.dmask8, 0, (size_t)P * 65536 * 16, st) != cudaSuccess) {
    return set_error("decoder training: memset failed");
  }
  if (d_iou) {
    copy_rows_kernel<<<nblk((long)P * s.nm), 256, 0, st>>>(d_iou, s.nm, s.iou32.g + s.m0, 32, P, s.nm, 1);
    LAUNCH_CHECK("iou_grad");
  }
  for (auto it = s.tape.rbegin(); it != s.tape.rend(); ++it) RUN((*it)(st));
  token_grads_kernel<<<s.T, 256, 0, st>>>(s.tok.g, s.emb_index, P, s.T, s.Ts, d.g_out_tokens, d.g_point_emb, d.g_nap);
  LAUNCH_CHECK("token_grads");
  if (s.mask) {
    RUN(md_backward(s.keys0.g, s.mask, P, d.md_w, d_emb_nchw, s.md, d.md_g, 1, st));
    d.md_written = true;
  } else if (s.images) {
    src_images_grad_kernel<<<dim3(128, 8, P), dim3(32, 8), 0, st>>>(s.keys0.g, d_emb_nchw, d.g_no_mask);
    LAUNCH_CHECK("src_images_grad");
  } else {
    src_grad_kernel<<<dim3(128, 8), dim3(32, 8), 0, st>>>(s.keys0.g, P, d_emb_nchw, d.g_no_mask);
    LAUNCH_CHECK("src_grad");
  }
  (s.images ? d.free_written : d.prompted_written) = true;
  d.unreached = d.free_written && !d.prompted_written;
  s.live = false;   // gradients of the activations are consumed: one backward per forward
  return 0;
}

void Engine::dec_train_free() {
  if (!dtrain) return;
  for (DecSlot& s : dtrain->slot)
    if (s.arena) cudaFree(s.arena);
  delete dtrain;
  dtrain = nullptr;
}

int Engine::decoder_zero_grads(cudaStream_t st) {
  if (!dtrain) return 0;
  for (const OptParam& p : opt)
    if (p.decoder && cudaMemsetAsync(p.g, 0, (size_t)p.n * 4, st) != cudaSuccess) return set_error("decoder training: memset failed");
  dtrain->md_written = dtrain->free_written = dtrain->prompted_written = dtrain->unreached = false;
  return 0;
}

int Engine::dec_train_refresh_prompt_tables(cudaStream_t st) {
  return dtrain ? dec_set_prompt_tables(dtrain->point_emb, dtrain->not_a_point, st) : 0;
}

}  // namespace msam
