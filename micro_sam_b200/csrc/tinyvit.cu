// MobileSAM's TinyViT image encoder (`vit_t`, micro_sam/util.py:35-43,436-441) on sm_90a.  Restated in oracle/tinyvit_ref.py.
//   stem        conv3x3/2 (3->32) + BN + GELU  [direct kernel, fused Sam.preprocess]  ->  conv3x3/2 (32->64) + BN  [im2col + GEMM]
//   stage 0     2 x MBConv @256^2 (1x1 64->256 GELU | dw3x3 GELU | 1x1 256->64 + shortcut, GELU)  ->  PatchMerging 64->128 /2
//   stage 1-3   TinyViTBlock: window attention (7 / 14 / 7, head_dim 32, learned bias table) + dw3x3 local conv + MLP,
//               PatchMerging 128->160 /2, 160->320 /1
//   neck        conv1x1 -> LN2d -> conv3x3 -> LN2d (shared with the ViT path)
// Everything 1x1 / dense is the wgmma GEMM of gemm.cu with BatchNorm folded into weight + bias at load time; the
// depth-wise convolutions, the window LayerNorm (zero pad tokens BEFORE the norm -> pad rows = LN bias) and the small-window
// attention are HBM-bound CUDA-core kernels.  Activations: bf16 NHWC in the conv stage, fp32 token-major residual stream after.
#include "device_util.cuh"
#include "engine.h"

#include <cmath>

namespace msam {

namespace {

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { f[2 * i] = bf16_lo(w[i]); f[2 * i + 1] = bf16_hi(w[i]); }
}

// ---------------------------------------------------------------------------------------------------------------
// Stem conv 1: Sam.preprocess ((x - mean) / std, zero pad to img x img) + conv3x3 stride 2 pad 1 (3 -> 32) + folded BN + GELU.
// Source uint8 HWC [B, h, w, 3] or preprocessed fp32 NCHW [B, 3, img, img].  One thread = one output pixel x 8 channels.
// w: [27][32] (tap-major: (ky*3+kx)*3 + c), b: [32].  out: bf16 NHWC [B, img/2, img/2, 32].
__global__ void tv_stem1_kernel(const uint8_t* __restrict__ u8, const float* __restrict__ f32, int B, int h, int w, int img,
                                float m0, float m1, float m2, float s0, float s1, float s2, const float* __restrict__ wt,
                                const float* __restrict__ bias, __nv_bfloat16* __restrict__ out) {
  const int ho = img / 2;
  const long total = (long)B * ho * ho * 4;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = idx & 3;
  const long pix = idx >> 2;
  const int ox = pix % ho, oy = (pix / ho) % ho;
  const int b = pix / ((long)ho * ho);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = __ldg(bias + cg * 8 + i);
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int y = oy * 2 + ky - 1;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int x = ox * 2 + kx - 1;
      float v[3] = {0.f, 0.f, 0.f};
      if (y >= 0 && x >= 0 && y < img && x < img) {
        if (f32) {
#pragma unroll
          for (int c = 0; c < 3; ++c) v[c] = __ldg(f32 + (((long)b * 3 + c) * img + y) * img + x);
        } else if (y < h && x < w) {
          const uint8_t* p = u8 + (((long)b * h + y) * w + x) * 3;
          v[0] = ((float)p[0] - m0) / s0; v[1] = ((float)p[1] - m1) / s1; v[2] = ((float)p[2] - m2) / s2;
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* wr = wt + ((ky * 3 + kx) * 3 + c) * 32 + cg * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(v[c], __ldg(wr + i), acc[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = gelu_erf(acc[i]);
  *reinterpret_cast<uint4*>(out + pix * 32 + cg * 8) =
      make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
}

// im2col for a 3x3 / pad 1 conv with stride on bf16 NHWC [B, Hin, Hin, C]: out[opix][(ky*3+kx)*C + c].  One thread = 8 channels.
__global__ void tv_im2col_kernel(const __nv_bfloat16* __restrict__ x, int B, int Hin, int C, int stride,
                                 __nv_bfloat16* __restrict__ out) {
  const int Ho = Hin / stride, c8 = C / 8;
  const long total = (long)B * Ho * Ho * 9 * c8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = idx % c8;
  const int k = (idx / c8) % 9;
  const long pix = idx / (9 * c8);
  const int ox = pix % Ho, oy = (pix / Ho) % Ho;
  const long b = pix / ((long)Ho * Ho);
  const int sy = oy * stride + k / 3 - 1, sx = ox * stride + k % 3 - 1;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (sy >= 0 && sy < Hin && sx >= 0 && sx < Hin) v = *reinterpret_cast<const uint4*>(x + ((b * Hin + sy) * Hin + sx) * C + cc * 8);
  *reinterpret_cast<uint4*>(out + pix * 9 * C + (long)k * C + cc * 8) = v;
}

// Depth-wise conv3x3 pad 1 (stride 1 / 2) + folded BN (+ GELU) on NHWC.  bf16 variant: one thread = 8 channels of one output
// pixel; fp32 variant (token residual stream): 4 channels.  w: [9][C] fp32, b: [C].
__global__ void tv_dwconv_bf16_kernel(const __nv_bfloat16* __restrict__ x, int B, int Hin, int C, int stride,
                                      const float* __restrict__ wt, const float* __restrict__ bias, int act,
                                      __nv_bfloat16* __restrict__ out) {
  const int Ho = Hin / stride, c8 = C / 8;
  const long total = (long)B * Ho * Ho * c8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = idx % c8;
  const long pix = idx / c8;
  const int ox = pix % Ho, oy = (pix / Ho) % Ho;
  const long b = pix / ((long)Ho * Ho);
  float acc[8];
  {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + cc * 8)), b1 = __ldg(reinterpret_cast<const float4*>(bias + cc * 8 + 4));
    acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w; acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int sy = oy * stride + k / 3 - 1, sx = ox * stride + k % 3 - 1;
    if (sy < 0 || sy >= Hin || sx < 0 || sx >= Hin) continue;
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(x + ((b * Hin + sy) * Hin + sx) * C + cc * 8), v);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(wt + (long)k * C + cc * 8));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(wt + (long)k * C + cc * 8 + 4));
    acc[0] = fmaf(v[0], w0.x, acc[0]); acc[1] = fmaf(v[1], w0.y, acc[1]); acc[2] = fmaf(v[2], w0.z, acc[2]); acc[3] = fmaf(v[3], w0.w, acc[3]);
    acc[4] = fmaf(v[4], w1.x, acc[4]); acc[5] = fmaf(v[5], w1.y, acc[5]); acc[6] = fmaf(v[6], w1.z, acc[6]); acc[7] = fmaf(v[7], w1.w, acc[7]);
  }
  if (act) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = gelu_erf(acc[i]);
  }
  *reinterpret_cast<uint4*>(out + pix * C + cc * 8) =
      make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
}

__global__ void tv_dwconv_f32_kernel(const float* __restrict__ x, int B, int Hin, int C, const float* __restrict__ wt,
                                     const float* __restrict__ bias, float* __restrict__ out) {
  const int c4 = C / 4;
  const long total = (long)B * Hin * Hin * c4;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = idx % c4;
  const long pix = idx / c4;
  const int ox = pix % Hin, oy = (pix / Hin) % Hin;
  const long b = pix / ((long)Hin * Hin);
  float4 acc = __ldg(reinterpret_cast<const float4*>(bias + cc * 4));
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int sy = oy + k / 3 - 1, sx = ox + k % 3 - 1;
    if (sy < 0 || sy >= Hin || sx < 0 || sx >= Hin) continue;
    const float4 v = *reinterpret_cast<const float4*>(x + ((b * Hin + sy) * Hin + sx) * C + cc * 4);
    const float4 w = __ldg(reinterpret_cast<const float4*>(wt + (long)k * C + cc * 4));
    acc.x = fmaf(v.x, w.x, acc.x); acc.y = fmaf(v.y, w.y, acc.y); acc.z = fmaf(v.z, w.z, acc.z); acc.w = fmaf(v.w, w.w, acc.w);
  }
  *reinterpret_cast<float4*>(out + pix * C + cc * 4) = acc;
}

// LayerNorm + window partition with TinyViT's padding rule: the zero pad tokens are appended BEFORE attn.norm, so a pad row
// is LayerNorm(0) = beta.  One warp per OUTPUT row of the window-partitioned layout [(b*nw*nw + wy*nw + wx) * ws*ws + ty*ws + tx].
constexpr int TV_LN_V4 = 3;  // D <= 384
__global__ void tv_ln_window_kernel(const float* __restrict__ x, int B, int H, int D, int ws, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ out) {
  const int nw = (H + ws - 1) / ws, N = ws * ws;
  const long rows = (long)B * nw * nw * N;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int t = warp % N;
  const long win = warp / N;
  const int wx = win % nw, wy = (win / nw) % nw;
  const long b = win / ((long)nw * nw);
  const int y = wy * ws + t / ws, xx = wx * ws + t % ws;
  const int nv = D >> 2;
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  __nv_bfloat16* orow = out + warp * D;
  if (y >= H || xx >= H) {
    for (int k = lane; k < nv; k += 32) {
      const float4 bb = __ldg(b4 + k);
      *reinterpret_cast<uint2*>(orow + 4 * k) = make_uint2(pack_bf16(bb.x, bb.y), pack_bf16(bb.z, bb.w));
    }
    return;
  }
  const float4* src = reinterpret_cast<const float4*>(x + ((b * H + y) * H + xx) * D);
  float4 v[TV_LN_V4];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < TV_LN_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) { v[i] = src[k]; sum += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
  }
  const float mean = warp_sum(sum) / (float)D;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < TV_LN_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) {
      const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + bq * bq) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)D + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
#pragma unroll
  for (int i = 0; i < TV_LN_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) {
      const float4 g = __ldg(g4 + k), bb = __ldg(b4 + k);
      *reinterpret_cast<uint2*>(orow + 4 * k) =
          make_uint2(pack_bf16((v[i].x - mean) * rstd * g.x + bb.x, (v[i].y - mean) * rstd * g.y + bb.y),
                     pack_bf16((v[i].z - mean) * rstd * g.z + bb.z, (v[i].w - mean) * rstd * g.w + bb.w));
    }
  }
}

// TinyViT window attention, head_dim 32, N = ws*ws keys (49 or 196), bias[h][|dy|*ws + |dx|].
// qkv: bf16 [(windows) * N, heads * 96], per head [q | k | v]; out: bf16 [B*H*H, heads*32] in image token order (pad queries dropped).
// One CTA per (window, head); K / V staged in shared memory as fp32; one thread per query row, online softmax over the keys
// in chunks of 4 (shared-memory reads are warp broadcasts).
template <int WS>
__global__ void __launch_bounds__(WS == 7 ? 64 : 224)
tv_attn_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ bias_tab, int heads, int H, float scale,
               __nv_bfloat16* __restrict__ out) {
  constexpr int N = WS * WS, HD = 32, NP = (N + 3) & ~3;
  extern __shared__ float tv_smem[];   // K | V | bias row
  float* sK = tv_smem;
  float* sV = tv_smem + NP * HD;
  float* sB = tv_smem + 2 * NP * HD;
  const int head = blockIdx.y;
  const long win = blockIdx.x;
  const int nw = (H + WS - 1) / WS;
  const int ld = heads * 96;
  const __nv_bfloat16* base = qkv + win * N * (long)ld + head * 96;
  for (int i = threadIdx.x; i < NP * 4; i += blockDim.x) {   // 4 x 16-byte chunks per row for K and for V
    const int row = i >> 2, ch = i & 3;
    float k8[8] = {0, 0, 0, 0, 0, 0, 0, 0}, v8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (row < N) {
      unpack8(*reinterpret_cast<const uint4*>(base + (long)row * ld + 32 + ch * 8), k8);
      unpack8(*reinterpret_cast<const uint4*>(base + (long)row * ld + 64 + ch * 8), v8);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) { sK[row * HD + ch * 8 + e] = k8[e]; sV[row * HD + ch * 8 + e] = v8[e]; }
  }
  for (int i = threadIdx.x; i < N; i += blockDim.x) sB[i] = __ldg(bias_tab + (long)head * N + i);
  __syncthreads();
  const int t = threadIdx.x;
  if (t >= N) return;
  float q[HD], acc[HD];
#pragma unroll
  for (int ch = 0; ch < 4; ++ch) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(base + (long)t * ld + ch * 8), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) q[ch * 8 + e] = f[e] * scale;
  }
#pragma unroll
  for (int i = 0; i < HD; ++i) acc[i] = 0.f;
  const int qy = t / WS, qx = t % WS;
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < N; j0 += 4) {
    float s[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = j0 + jj;
      float d = 0.f;
      const float4* kr = reinterpret_cast<const float4*>(sK + j * HD);
#pragma unroll
      for (int i = 0; i < HD / 4; ++i) {
        const float4 kk = kr[i];
        d = fmaf(q[4 * i], kk.x, d); d = fmaf(q[4 * i + 1], kk.y, d); d = fmaf(q[4 * i + 2], kk.z, d); d = fmaf(q[4 * i + 3], kk.w, d);
      }
      if (j < N) {
        const int ky = j / WS, kx = j % WS;
        const int dy = qy > ky ? qy - ky : ky - qy, dx = qx > kx ? qx - kx : kx - qx;
        s[jj] = d + sB[dy * WS + dx];
      } else {
        s[jj] = -INFINITY;
      }
    }
    const float mn = fmaxf(fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3])), m);
    const float corr = __expf(m - mn);   // m = -inf on the first chunk -> 0
    l *= corr;
#pragma unroll
    for (int i = 0; i < HD; ++i) acc[i] *= corr;
    m = mn;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const float p = __expf(s[jj] - m);
      l += p;
      const float4* vr = reinterpret_cast<const float4*>(sV + (j0 + jj) * HD);
#pragma unroll
      for (int i = 0; i < HD / 4; ++i) {
        const float4 vv = vr[i];
        acc[4 * i] = fmaf(p, vv.x, acc[4 * i]); acc[4 * i + 1] = fmaf(p, vv.y, acc[4 * i + 1]);
        acc[4 * i + 2] = fmaf(p, vv.z, acc[4 * i + 2]); acc[4 * i + 3] = fmaf(p, vv.w, acc[4 * i + 3]);
      }
    }
  }
  const int wx = win % nw, wy = (win / nw) % nw;
  const long b = win / ((long)nw * nw);
  const int y = wy * WS + qy, x = wx * WS + qx;
  if (y >= H || x >= H) return;
  const float inv = 1.0f / l;
  __nv_bfloat16* orow = out + ((b * H + y) * H + x) * (long)(heads * HD) + head * HD;
#pragma unroll
  for (int ch = 0; ch < 4; ++ch)
    *reinterpret_cast<uint4*>(orow + ch * 8) =
        make_uint4(pack_bf16(acc[ch * 8] * inv, acc[ch * 8 + 1] * inv), pack_bf16(acc[ch * 8 + 2] * inv, acc[ch * 8 + 3] * inv),
                   pack_bf16(acc[ch * 8 + 4] * inv, acc[ch * 8 + 5] * inv), pack_bf16(acc[ch * 8 + 6] * inv, acc[ch * 8 + 7] * inv));
}

}  // namespace

// ------------------------------------------------------------------------------------------------ launches
int launch_tv_stem1(const uint8_t* u8, const float* f32, int B, int h, int w, int img, const float* wt, const float* bias,
                    __nv_bfloat16* out, cudaStream_t st) {
  static const float mean[3] = {123.675f, 116.28f, 103.53f}, stdv[3] = {58.395f, 57.12f, 57.375f};
  const int ho = img / 2;
  const long total = (long)B * ho * ho * 4;
  prof_begin(st, "tinyvit stem conv1", 2.0 * B * ho * ho * 27 * 32, (double)B * ((double)img * img * 3 + (double)ho * ho * 32 * 2));
  tv_stem1_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(u8, f32, B, h, w, img, mean[0], mean[1], mean[2], stdv[0],
                                                                stdv[1], stdv[2], wt, bias, out);
  prof_end(st);
  LAUNCH_CHECK("stem conv1");
  return 0;
}

int launch_tv_im2col(const __nv_bfloat16* x, int B, int Hin, int C, int stride, __nv_bfloat16* out, cudaStream_t st) {
  const long tc = (long)B * (Hin / stride) * (Hin / stride) * 9 * (C / 8);
  tv_im2col_kernel<<<(unsigned)((tc + 255) / 256), 256, 0, st>>>(x, B, Hin, C, stride, out);
  LAUNCH_CHECK("stem im2col");
  return 0;
}

int launch_tv_dwconv_bf16(const __nv_bfloat16* x, int B, int Hin, int C, int stride, const float* w, const float* b, int act,
                          __nv_bfloat16* out, cudaStream_t st) {
  const long total = (long)B * (Hin / stride) * (Hin / stride) * (C / 8);
  prof_begin(st, "tinyvit dwconv3x3 (bf16)", 0.0, (double)B * Hin * Hin * C * 2 + (double)total * 16);
  tv_dwconv_bf16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, B, Hin, C, stride, w, b, act, out);
  prof_end(st);
  LAUNCH_CHECK("dwconv");
  return 0;
}

int launch_tv_dwconv_f32(const float* x, int B, int Hin, int C, const float* w, const float* b, float* out, cudaStream_t st) {
  const long total = (long)B * Hin * Hin * (C / 4);
  tv_dwconv_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, B, Hin, C, w, b, out);
  LAUNCH_CHECK("local conv");
  return 0;
}

int launch_tv_ln_window(const float* x, int B, int H, int D, int ws, const float* gamma, const float* beta, float eps,
                        __nv_bfloat16* out, cudaStream_t st) {
  const int nw = (H + ws - 1) / ws;
  const long warps = (long)B * nw * nw * ws * ws;   // one warp per window-partitioned row
  tv_ln_window_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(x, B, H, D, ws, gamma, beta, eps, out);
  LAUNCH_CHECK("window layernorm");
  return 0;
}

int launch_tv_attention(const __nv_bfloat16* qkv, const float* bias_tab, int B, int H, int ws, int heads, __nv_bfloat16* out,
                        cudaStream_t st) {
  const int N = ws * ws, nw = (H + ws - 1) / ws;
  const long Mw = (long)B * nw * nw * N, M = (long)B * H * H;
  const float scale = 1.0f / sqrtf(32.0f);
  prof_begin(st, "tinyvit window attention", 4.0 * B * nw * nw * heads * (double)N * N * 32,
             (double)Mw * heads * 96 * 2 + (double)M * heads * 32 * 2);
  constexpr int SM7 = (2 * 52 * 32 + 49) * 4, SM14 = (2 * 196 * 32 + 196) * 4;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(tv_attn_kernel<14>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM14) != cudaSuccess)
      return set_error("tinyvit attention: cudaFuncSetAttribute failed");
    attr_set = true;
  }
  if (ws == 7) tv_attn_kernel<7><<<dim3(B * nw * nw, heads), 64, SM7, st>>>(qkv, bias_tab, heads, H, scale, out);
  else tv_attn_kernel<14><<<dim3(B * nw * nw, heads), 224, SM14, st>>>(qkv, bias_tab, heads, H, scale, out);
  prof_end(st);
  LAUNCH_CHECK("window attention");
  return 0;
}

// ------------------------------------------------------------------------------------------------ weights
namespace {

struct FoldedConv {
  std::vector<float> w;  // [out][in_per_group * k * k], scaled by gamma / sqrt(var + eps)
  std::vector<float> b;  // [out]
};

}  // namespace

// Conv2d_BN (keys <p>.c.weight, <p>.bn.{weight,bias,running_mean,running_var}) with the eval-mode BatchNorm folded in.
static int fold_conv_bn(Engine& e, const std::string& p, int out, int inner, FoldedConv* f) {
  const auto* w = e.host(p + ".c.weight", {out, inner});
  const auto* g = e.host(p + ".bn.weight", {out});
  const auto* b = e.host(p + ".bn.bias", {out});
  const auto* mu = e.host(p + ".bn.running_mean", {out});
  const auto* var = e.host(p + ".bn.running_var", {out});
  if (!w || !g || !b || !mu || !var) return -1;
  f->w.resize((size_t)out * inner);
  f->b.resize(out);
  for (int o = 0; o < out; ++o) {
    const float s = (*g)[o] / std::sqrt((*var)[o] + 1e-5f);
    for (int i = 0; i < inner; ++i) f->w[(size_t)o * inner + i] = (*w)[(size_t)o * inner + i] * s;
    f->b[o] = (*b)[o] - (*mu)[o] * s;
  }
  return 0;
}

static int up_pointwise(Engine& e, const std::string& p, int out, int in, TvConv* c) {  // 1x1 Conv2d_BN -> GEMM operand [out, in]
  FoldedConv f;
  if (fold_conv_bn(e, p, out, in, &f)) return -1;
  CHK(c->w = e.upload_bf16(f.w.data(), f.w.size()));
  CHK(c->b = e.upload_f32(f.b.data(), f.b.size()));
  return 0;
}
static int up_depthwise(Engine& e, const std::string& p, int C, TvConv* c) {  // dw 3x3 Conv2d_BN -> [9][C] fp32
  FoldedConv f;
  if (fold_conv_bn(e, p, C, 9, &f)) return -1;
  std::vector<float> r((size_t)9 * C);
  for (int ch = 0; ch < C; ++ch)
    for (int k = 0; k < 9; ++k) r[(size_t)k * C + ch] = f.w[(size_t)ch * 9 + k];
  CHK(c->wf = e.upload_f32(r.data(), r.size()));
  CHK(c->b = e.upload_f32(f.b.data(), f.b.size()));
  return 0;
}
static int up_merge(Engine& e, const std::string& p, int dim, int out, TvMerge* m) {
  if (up_pointwise(e, p + "conv1", out, dim, &m->conv1)) return -1;
  if (up_depthwise(e, p + "conv2", out, &m->conv2)) return -1;
  if (up_pointwise(e, p + "conv3", out, out, &m->conv3)) return -1;
  return 0;
}

int Engine::finalize_tinyvit() {
  static const int dims[4] = {64, 128, 160, 320}, depths[4] = {2, 2, 6, 2}, nheads[4] = {2, 4, 5, 10}, wsz[4] = {7, 7, 14, 7};
  const std::string e = "image_encoder.";
  {  // stem
    FoldedConv f;
    if (fold_conv_bn(*this, e + "patch_embed.seq.0", 32, 27, &f)) return -1;
    std::vector<float> r(27 * 32);   // [ (ky*3+kx)*3 + c ][ out ]  from [out][c][ky][kx]
    for (int o = 0; o < 32; ++o)
      for (int c = 0; c < 3; ++c)
        for (int k = 0; k < 9; ++k) r[(size_t)(k * 3 + c) * 32 + o] = f.w[(size_t)o * 27 + c * 9 + k];
    CHK(tv.stem1.wf = upload_f32(r.data(), r.size()));
    CHK(tv.stem1.b = upload_f32(f.b.data(), f.b.size()));
    if (fold_conv_bn(*this, e + "patch_embed.seq.2", 64, 32 * 9, &f)) return -1;
    std::vector<float> g((size_t)64 * 288);   // GEMM operand [out][(ky*3+kx)*32 + c]
    for (int o = 0; o < 64; ++o)
      for (int c = 0; c < 32; ++c)
        for (int k = 0; k < 9; ++k) g[(size_t)o * 288 + k * 32 + c] = f.w[(size_t)o * 288 + c * 9 + k];
    CHK(tv.stem2.w = upload_bf16(g.data(), g.size()));
    CHK(tv.stem2.b = upload_f32(f.b.data(), f.b.size()));
  }
  for (int i = 0; i < 2; ++i) {
    const std::string p = e + "layers.0.blocks." + std::to_string(i) + ".";
    if (up_pointwise(*this, p + "conv1", 256, 64, &tv.mb[i].conv1)) return -1;
    if (up_depthwise(*this, p + "conv2", 256, &tv.mb[i].conv2)) return -1;
    if (up_pointwise(*this, p + "conv3", 64, 256, &tv.mb[i].conv3)) return -1;
  }
  if (up_merge(*this, e + "layers.0.downsample.", 64, 128, &tv.merge[0])) return -1;
  for (int s = 1; s < 4; ++s) {
    const int D = dims[s], N = wsz[s] * wsz[s];
    tv.stage[s].dim = D; tv.stage[s].heads = nheads[s]; tv.stage[s].ws = wsz[s];
    tv.stage[s].blocks.resize(depths[s]);
    for (int i = 0; i < depths[s]; ++i) {
      TvBlock& b = tv.stage[s].blocks[i];
      const std::string p = e + "layers." + std::to_string(s) + ".blocks." + std::to_string(i) + ".";
      CHK(b.an_g = up_f32(p + "attn.norm.weight", {D}));
      CHK(b.an_b = up_f32(p + "attn.norm.bias", {D}));
      CHK(b.qkv_w = up_bf16(p + "attn.qkv.weight", {3 * D, D}));
      CHK(b.qkv_b = up_f32(p + "attn.qkv.bias", {3 * D}));
      CHK(b.bias_tab = up_f32(p + "attn.attention_biases", {nheads[s], N}));
      CHK(b.proj_w = up_bf16(p + "attn.proj.weight", {D, D}));
      CHK(b.proj_b = up_f32(p + "attn.proj.bias", {D}));
      if (up_depthwise(*this, p + "local_conv", D, &b.local)) return -1;
      CHK(b.mn_g = up_f32(p + "mlp.norm.weight", {D}));
      CHK(b.mn_b = up_f32(p + "mlp.norm.bias", {D}));
      CHK(b.fc1_w = up_bf16(p + "mlp.fc1.weight", {4 * D, D}));
      CHK(b.fc1_b = up_f32(p + "mlp.fc1.bias", {4 * D}));
      CHK(b.fc2_w = up_bf16(p + "mlp.fc2.weight", {D, 4 * D}));
      CHK(b.fc2_b = up_f32(p + "mlp.fc2.bias", {D}));
    }
    if (s < 3 && up_merge(*this, e + "layers." + std::to_string(s) + ".downsample.", D, dims[s + 1], &tv.merge[s])) return -1;
  }
  const int C = cfg.out_chans, D = 320;
  CHK(enc.neck_conv1 = up_bf16(e + "neck.0.weight", {C, D, 1, 1}));
  CHK(enc.neck_ln1_g = up_f32(e + "neck.1.weight", {C}));
  CHK(enc.neck_ln1_b = up_f32(e + "neck.1.bias", {C}));
  {
    const auto* w = host(e + "neck.2.weight", {C, C, 3, 3});
    CHK(w);
    std::vector<float> r((size_t)C * 9 * C);
    for (int o = 0; o < C; ++o)
      for (int c = 0; c < C; ++c)
        for (int k = 0; k < 9; ++k) r[((size_t)o * 9 + k) * C + c] = (*w)[((size_t)o * C + c) * 9 + k];
    CHK(enc.neck_conv2 = upload_bf16(r.data(), r.size()));
  }
  CHK(enc.neck_ln2_g = up_f32(e + "neck.3.weight", {C}));
  CHK(enc.neck_ln2_b = up_f32(e + "neck.3.bias", {C}));
  return 0;
}

int Engine::alloc_tinyvit_ws() {
  const size_t B = cfg.max_batch, C = cfg.out_chans, T = 4096;
  CHK(tv.s1 = (__nv_bfloat16*)dalloc(B * 512 * 512 * 32 * 2));
  CHK(tv.col = (__nv_bfloat16*)dalloc(B * 65536 * 288 * 2));
  CHK(tv.a0 = (__nv_bfloat16*)dalloc(B * 65536 * 64 * 2));
  CHK(tv.a1 = (__nv_bfloat16*)dalloc(B * 65536 * 64 * 2));
  CHK(tv.h1 = (__nv_bfloat16*)dalloc(B * 65536 * 256 * 2));    // MBConv hidden; later fc1 output / merge conv1 output
  CHK(tv.h2 = (__nv_bfloat16*)dalloc(B * 65536 * 256 * 2));
  CHK(tv.x = (float*)dalloc(B * 16384 * 128 * 4));              // >= 4096 * 320
  CHK(tv.x2 = (float*)dalloc(B * 16384 * 128 * 4));
  CHK(tv.xw = (__nv_bfloat16*)dalloc(B * 17689 * 128 * 2));      // >= 4900 * 320
  CHK(tv.qkv = (__nv_bfloat16*)dalloc(B * 17689 * 384 * 2));     // >= 4900 * 960
  CHK(tv.attn = (__nv_bfloat16*)dalloc(B * 16384 * 128 * 2));
  CHK(tv.xn = (__nv_bfloat16*)dalloc(B * 16384 * 128 * 2));
  CHK(ws.neck1 = (float*)dalloc(B * T * C * 4));
  CHK(ws.neck1b = (__nv_bfloat16*)dalloc(B * T * C * 2));
  CHK(ws.neck_col = (__nv_bfloat16*)dalloc(B * T * 9 * C * 2));
  CHK(ws.neck2 = (float*)dalloc(B * T * C * 4));
  return 0;
}

// ------------------------------------------------------------------------------------------------ forward
static int tv_gemm(Engine& e, const __nv_bfloat16* A, const __nv_bfloat16* W, int M, int N, int K, const float* bias, int act,
                   const void* residual, int res_bf16, int act_after_res, void* out, int out_fp32, cudaStream_t st) {
  GemmArgs a;
  a.A = A; a.W = W; a.M = M; a.N = N; a.K = K; a.lda = K; a.ldw = K; a.bias = bias; a.act = act;
  a.residual = residual; a.res_bf16 = res_bf16; a.act_after_res = act_after_res; a.out = out; a.out_fp32 = out_fp32;
  return launch_gemm(a, e.num_sms, st);
}

static int tv_merge(Engine& e, const TvMerge& m, const __nv_bfloat16* in, int nb, int Hin, int dim, int out_dim, int stride,
                    float* x_out, cudaStream_t st) {
  const int Min = nb * Hin * Hin, Ho = Hin / stride, Mo = nb * Ho * Ho;
  if (tv_gemm(e, in, m.conv1.w, Min, out_dim, dim, m.conv1.b, 1, nullptr, 0, 0, e.tv.h1, 0, st)) return -1;
  if (launch_tv_dwconv_bf16(e.tv.h1, nb, Hin, out_dim, stride, m.conv2.wf, m.conv2.b, 1, e.tv.h2, st)) return -1;
  return tv_gemm(e, e.tv.h2, m.conv3.w, Mo, out_dim, out_dim, m.conv3.b, 0, nullptr, 0, 0, x_out, 1, st);
}

int Engine::encode_tinyvit(const uint8_t* u8, const float* f32, int B, int hh, int ww, float* out, cudaStream_t st,
                           int stop_after, float* x_out) {
  if (!finalized) return set_error("msam_encode: weights not finalized");
  if (B <= 0) return set_error("msam_encode: empty batch");
  const int img = cfg.image_size, C = cfg.out_chans;
  if (u8 && (hh > img || ww > img || hh <= 0 || ww <= 0)) return set_error("msam_encode_u8: image %dx%d exceeds %d", hh, ww, img);
  for (int b0 = 0; b0 < B; b0 += cfg.max_batch) {
    const int nb = (B - b0 < cfg.max_batch) ? (B - b0) : cfg.max_batch;
    const uint8_t* u8p = u8 ? u8 + (size_t)b0 * hh * ww * 3 : nullptr;
    const float* f32p = f32 ? f32 + (size_t)b0 * 3 * img * img : nullptr;
    if (launch_tv_stem1(u8p, f32p, nb, hh, ww, img, tv.stem1.wf, tv.stem1.b, tv.s1, st)) return -1;
    if (launch_tv_im2col(tv.s1, nb, 512, 32, 2, tv.col, st)) return -1;
    if (tv_gemm(*this, tv.col, tv.stem2.w, nb * 65536, 64, 288, tv.stem2.b, 0, nullptr, 0, 0, tv.a0, 0, st)) return -1;
    int stage_idx = 0;   // stop_after counts: 1 = after layers.0 (incl. its downsample), 2 / 3 / 4 = after layers.1 / 2 / 3
    __nv_bfloat16 *cur = tv.a0, *nxt = tv.a1;
    for (int i = 0; i < 2; ++i) {   // MBConv @ 256 x 256, 64 channels
      const int M = nb * 65536;
      if (tv_gemm(*this, cur, tv.mb[i].conv1.w, M, 256, 64, tv.mb[i].conv1.b, 1, nullptr, 0, 0, tv.h1, 0, st)) return -1;
      if (launch_tv_dwconv_bf16(tv.h1, nb, 256, 256, 1, tv.mb[i].conv2.wf, tv.mb[i].conv2.b, 1, tv.h2, st)) return -1;
      if (tv_gemm(*this, tv.h2, tv.mb[i].conv3.w, M, 64, 256, tv.mb[i].conv3.b, 1, cur, 1, 1, nxt, 0, st)) return -1;
      __nv_bfloat16* t = cur; cur = nxt; nxt = t;
    }
    if (tv_merge(*this, tv.merge[0], cur, nb, 256, 64, 128, 2, tv.x, st)) return -1;
    ++stage_idx;
    int H = 128;
    for (int s = 1; s < 4 && !(stop_after >= 0 && stage_idx >= stop_after); ++s) {
      const TvStage& S = tv.stage[s];
      const int D = S.dim, wsz = S.ws, N = wsz * wsz, nw = (H + wsz - 1) / wsz;
      const int M = nb * H * H, Mw = nb * nw * nw * N;
      for (const TvBlock& b : S.blocks) {
        if (launch_tv_ln_window(tv.x, nb, H, D, wsz, b.an_g, b.an_b, 1e-5f, tv.xw, st)) return -1;
        if (tv_gemm(*this, tv.xw, b.qkv_w, Mw, 3 * D, D, b.qkv_b, 0, nullptr, 0, 0, tv.qkv, 0, st)) return -1;
        if (launch_tv_attention(tv.qkv, b.bias_tab, nb, H, wsz, S.heads, tv.attn, st)) return -1;
        if (tv_gemm(*this, tv.attn, b.proj_w, M, D, D, b.proj_b, 0, tv.x, 0, 0, tv.x2, 1, st)) return -1;
        if (launch_tv_dwconv_f32(tv.x2, nb, H, D, b.local.wf, b.local.b, tv.x, st)) return -1;
        LnArgs l;
        l.x = tv.x; l.rows = M; l.D = D; l.gamma = b.mn_g; l.beta = b.mn_b; l.eps = 1e-5f; l.out = tv.xn;
        if (launch_layernorm(l, st)) return -1;
        if (tv_gemm(*this, tv.xn, b.fc1_w, M, 4 * D, D, b.fc1_b, 1, nullptr, 0, 0, tv.h1, 0, st)) return -1;
        if (tv_gemm(*this, tv.h1, b.fc2_w, M, D, 4 * D, b.fc2_b, 0, tv.x, 0, 0, tv.x, 1, st)) return -1;
      }
      if (s < 3) {
        static const int dims[4] = {64, 128, 160, 320};
        const int stride = (dims[s + 1] == 320) ? 1 : 2;
        if (launch_cast_bf16(tv.x, (long)M * D, tv.xn, st)) return -1;
        if (tv_merge(*this, tv.merge[s], tv.xn, nb, H, D, dims[s + 1], stride, tv.x, st)) return -1;
        H /= stride;
      }
      ++stage_idx;
    }
    if (stop_after >= 0) {   // parity localisation: the fp32 token stream after `stop_after` stages
      static const int dims[5] = {64, 128, 160, 320, 320};
      const int sidx = stop_after > 4 ? 4 : stop_after;
      const size_t n = (size_t)nb * H * H * dims[sidx];
      if (cudaMemcpyAsync(x_out + (size_t)b0 * H * H * dims[sidx], tv.x, n * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return set_error("encode_blocks: copy failed");
      continue;
    }
    // neck: conv1x1 -> LN2d -> conv3x3 (im2col GEMM) -> LN2d (NCHW out), as the ViT path
    const int T = 4096, M = nb * T, D = 320;
    if (launch_cast_bf16(tv.x, (long)M * D, tv.xn, st)) return -1;
    if (tv_gemm(*this, tv.xn, enc.neck_conv1, M, C, D, nullptr, 0, nullptr, 0, 0, ws.neck1, 1, st)) return -1;
    {
      LnArgs l;
      l.x = ws.neck1; l.rows = M; l.D = C; l.gamma = enc.neck_ln1_g; l.beta = enc.neck_ln1_b; l.eps = 1e-6f; l.out = ws.neck1b;
      if (launch_layernorm(l, st)) return -1;
    }
    if (launch_im2col3x3(ws.neck1b, nb, 64, C, ws.neck_col, st)) return -1;
    if (tv_gemm(*this, ws.neck_col, enc.neck_conv2, M, C, 9 * C, nullptr, 0, nullptr, 0, 0, ws.neck2, 1, st)) return -1;
    if (launch_layernorm2d_nchw(ws.neck2, nb, T, enc.neck_ln2_g, enc.neck_ln2_b, 1e-6f, out + (size_t)b0 * C * T, st)) return -1;
  }
  return 0;
}

}  // namespace msam
