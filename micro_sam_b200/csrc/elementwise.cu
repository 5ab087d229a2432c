// HBM-bound helper kernels of the encoder path: preprocess+patchify, LayerNorm (row / window-partitioned / NCHW),
// fp32->bf16 casts, 3x3 im2col.  All are simple coalesced streaming kernels; the heavy lifting is in gemm.cu /
// attention.cu.
#include "kernels.h"
#include "ptx.cuh"

namespace msam {

// ---------------------------------------------------------------------------------------------------------------
// Sam.preprocess + PatchEmbed im2col.  Output A[b*g*g + ty*g + tx][c*256 + py*16 + px] (bf16), matching the flattened
// Conv2d weight [D, 3*16*16].  Source is either uint8 HWC (h x w <= img x img; normalise + zero-pad fused:
// (x - mean) / std inside, 0 outside == F.pad after normalisation, trainable_sam.py:24-47) or an already
// preprocessed fp32 NCHW tensor (what ImageEncoderViT.forward receives, util.py:674).
// One thread = one (token, channel, patch row): 16 pixels -> 32 bytes out.
__global__ void patchify_kernel(const uint8_t* __restrict__ u8, const float* __restrict__ f32, int B, int h, int w,
                                int img, float m0, float m1, float m2, float s0, float s1, float s2,
                                __nv_bfloat16* __restrict__ out) {
  const int g = img / 16;
  const long total = (long)B * g * g * 3 * 16;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int py = idx % 16;
  const int c = (idx / 16) % 3;
  const long tok = idx / 48;
  const int tx = tok % g, ty = (tok / g) % g;
  const int b = tok / ((long)g * g);
  const int y = ty * 16 + py, x0 = tx * 16;
  float v[16];
  if (f32) {
    const float4* src = reinterpret_cast<const float4*>(f32 + (((long)b * 3 + c) * img + y) * img + x0);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 t = __ldg(src + i);
      v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
  } else {
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2);
    const float stdv = c == 0 ? s0 : (c == 1 ? s1 : s2);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int x = x0 + i;
      v[i] = (y < h && x < w) ? ((float)u8[(((long)b * h + y) * w + x) * 3 + c] - mean) / stdv : 0.f;
    }
  }
  uint4 o0, o1;
  o0.x = pack_bf16(v[0], v[1]); o0.y = pack_bf16(v[2], v[3]); o0.z = pack_bf16(v[4], v[5]); o0.w = pack_bf16(v[6], v[7]);
  o1.x = pack_bf16(v[8], v[9]); o1.y = pack_bf16(v[10], v[11]); o1.z = pack_bf16(v[12], v[13]); o1.w = pack_bf16(v[14], v[15]);
  uint4* dst = reinterpret_cast<uint4*>(out + tok * 768 + c * 256 + py * 16);
  dst[0] = o0;
  dst[1] = o1;
}

int launch_patchify(const uint8_t* u8, const float* f32, int B, int h, int w, int img, const float* mean,
                    const float* stdv, __nv_bfloat16* out, cudaStream_t stream) {
  const int g = img / 16;
  const long total = (long)B * g * g * 48;
  patchify_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(u8, f32, B, h, w, img, mean[0], mean[1], mean[2],
                                                                    stdv[0], stdv[1], stdv[2], out);
  LAUNCH_CHECK("patchify");
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm over the last dim of fp32 rows -> bf16 (and optionally a second bf16 output with `add` [add_rows, D]
// broadcast-added after the affine: used by the decoder for keys + positional encoding).  One warp per row, row held in
// registers, two-pass (mean, then centred variance) like torch.  mode 1 scatters rows into the window-partitioned
// layout [(b*wpr*wpr + wy*wpr + wx) * ws*ws + ty*ws + tx] (pad rows of `out` are pre-zeroed and never written).
constexpr int LN_MAX_V4 = 10;  // D <= 1280

__global__ void layernorm_rows_kernel(const float* __restrict__ x, int rows, int D, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ out,
                                      int mode, int grid, int ws, const float* __restrict__ add, int add_rows,
                                      __nv_bfloat16* __restrict__ out2, float* __restrict__ out_f32, int act) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  pdl_wait();
  pdl_trigger();
  if (warp >= rows) return;
  const float4* src = reinterpret_cast<const float4*>(x + (long)warp * D);
  const int nv = D >> 2;
  float4 v[LN_MAX_V4];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) {
      v[i] = src[k];
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(sum) / (float)D;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)D + eps);

  long orow = warp;
  if (mode == 1) {
    const int gg = grid * grid;
    const int b = warp / gg, t = warp % gg, y = t / grid, xx = t % grid;
    const int wpr = (grid + ws - 1) / ws;
    orow = ((long)(b * wpr + y / ws) * wpr + xx / ws) * (ws * ws) + (y % ws) * ws + (xx % ws);
  }
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  const float4* a4 = add ? reinterpret_cast<const float4*>(add + (long)(warp % add_rows) * D) : nullptr;
#pragma unroll
  for (int i = 0; i < LN_MAX_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) {
      const float4 g = __ldg(g4 + k), bb = __ldg(b4 + k);
      float4 r;
      r.x = (v[i].x - mean) * rstd * g.x + bb.x;
      r.y = (v[i].y - mean) * rstd * g.y + bb.y;
      r.z = (v[i].z - mean) * rstd * g.z + bb.z;
      r.w = (v[i].w - mean) * rstd * g.w + bb.w;
      if (act == 1) { r.x = gelu_erf(r.x); r.y = gelu_erf(r.y); r.z = gelu_erf(r.z); r.w = gelu_erf(r.w); }
      if (out) *reinterpret_cast<uint2*>(out + orow * D + 4 * k) = make_uint2(pack_bf16(r.x, r.y), pack_bf16(r.z, r.w));
      if (out_f32) *reinterpret_cast<float4*>(out_f32 + orow * D + 4 * k) = r;
      if (out2) {
        const float4 a = __ldg(a4 + k);
        *reinterpret_cast<uint2*>(out2 + orow * D + 4 * k) = make_uint2(pack_bf16(r.x + a.x, r.y + a.y), pack_bf16(r.z + a.z, r.w + a.w));
      }
    }
  }
}

int launch_layernorm(const LnArgs& a, cudaStream_t stream) {
  if (a.D % 4 != 0 || a.D > LN_MAX_V4 * 128) return set_error("layernorm: unsupported D=%d", a.D);
  if (a.rows <= 0) return 0;
  const int warps_per_block = 8;
  const unsigned blocks = (unsigned)((a.rows + warps_per_block - 1) / warps_per_block);
  prof_begin(stream, "layernorm_rows", 0.0, (double)a.rows * a.D * (4 + (a.out ? 2 : 0) + (a.out2 ? 2 : 0) + (a.out_f32 ? 4 : 0)));
  launch_pdl(layernorm_rows_kernel, dim3(blocks), dim3(warps_per_block * 32), 0, stream, a.x, a.rows, a.D, a.gamma, a.beta, a.eps,
             a.out, a.window_mode, a.grid, a.ws, a.add, a.add_rows, a.out2, a.out_f32, a.act);
  prof_end(stream);
  LAUNCH_CHECK("layernorm");
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Final neck LayerNorm2d: fp32 rows [B*T, C=256] (token-major) -> fp32 NCHW [B, C, T] (T = 64*64), normalising over C.
// Block = 32 consecutive tokens; 8 warps x 4 tokens each; transposed through shared memory so the NCHW stores are
// 128-byte coalesced.
__global__ void layernorm2d_nchw_kernel(const float* __restrict__ x, int T, const float* __restrict__ gamma,
                                        const float* __restrict__ beta, float eps, float* __restrict__ out) {
  constexpr int C = 256;
  __shared__ float tile[C][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long tok0 = (long)blockIdx.x * 32;
  for (int t = warp * 4; t < warp * 4 + 4; ++t) {
    const float4* src = reinterpret_cast<const float4*>(x + (tok0 + t) * C);
    const float4 a = src[lane], b = src[lane + 32];
    const float mean = warp_sum((a.x + a.y) + (a.z + a.w) + (b.x + b.y) + (b.z + b.w)) / C;
    float d[8] = {a.x - mean, a.y - mean, a.z - mean, a.w - mean, b.x - mean, b.y - mean, b.z - mean, b.w - mean};
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) sq += d[i] * d[i];
    const float rstd = rsqrtf(warp_sum(sq) / C + eps);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = (i < 4) ? (4 * lane + i) : (128 + 4 * lane + (i - 4));
      tile[c][t] = d[i] * rstd * __ldg(gamma + c) + __ldg(beta + c);
    }
  }
  __syncthreads();
  const long b = tok0 / T, t0 = tok0 % T;
  for (int c = warp; c < C; c += 8) out[((long)b * C + c) * T + t0 + lane] = tile[c][lane];
}

int launch_layernorm2d_nchw(const float* x, int B, int T, const float* gamma, const float* beta, float eps, float* out,
                            cudaStream_t stream) {
  if (T % 32 != 0) return set_error("layernorm2d: T=%d must be a multiple of 32", T);
  layernorm2d_nchw_kernel<<<(unsigned)((long)B * T / 32), 256, 0, stream>>>(x, T, gamma, beta, eps, out);
  LAUNCH_CHECK("layernorm2d");
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void cast_bf16_kernel(const float* __restrict__ x, long n4, __nv_bfloat16* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = reinterpret_cast<const float4*>(x)[i];
  reinterpret_cast<uint2*>(out)[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}
int launch_cast_bf16(const float* x, long n, __nv_bfloat16* out, cudaStream_t stream) {
  if (n % 4 != 0) return set_error("cast: n must be a multiple of 4");
  const long n4 = n / 4;
  if (n4 == 0) return 0;
  cast_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(x, n4, out);
  LAUNCH_CHECK("cast");
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// im2col for the neck's 3x3 / pad 1 conv on token-major bf16 [B, g, g, C]: out[tok][(ky*3+kx)*C + c].
// One thread = 8 channels (16 B).
__global__ void im2col3x3_kernel(const __nv_bfloat16* __restrict__ x, int B, int g, int C,
                                 __nv_bfloat16* __restrict__ out) {
  const int c8 = C / 8;
  const long total = (long)B * g * g * 9 * c8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = idx % c8;
  const int k = (idx / c8) % 9;
  const long tok = idx / (9 * c8);
  const int xx = tok % g, y = (tok / g) % g;
  const long b = tok / ((long)g * g);
  const int sy = y + k / 3 - 1, sx = xx + k % 3 - 1;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (sy >= 0 && sy < g && sx >= 0 && sx < g)
    v = *reinterpret_cast<const uint4*>(x + ((b * g + sy) * g + sx) * C + cc * 8);
  *reinterpret_cast<uint4*>(out + tok * 9 * C + (long)k * C + cc * 8) = v;
}
int launch_im2col3x3(const __nv_bfloat16* x, int B, int g, int C, __nv_bfloat16* out, cudaStream_t stream) {
  const long total = (long)B * g * g * 9 * (C / 8);
  im2col3x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, B, g, C, out);
  LAUNCH_CHECK("im2col");
  return 0;
}

}  // namespace msam
