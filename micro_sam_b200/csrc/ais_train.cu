// Training of the AIS decoder (torch_em's UNETR decoder as micro-sam trains it, DESIGN.md section 2): the backward pass of every
// decoder layer, the norms (of inference and training alike) and the distance-based Dice loss.  Every reduction runs in a fixed
// order, so two identical steps give bit-identical gradients.
//   ais_wgrad_kernel     : 3x3 / 1x1 weight gradient dW[co, tap, ci] = sum_p dY[p, co] X[p + tap, ci], an implicit GEMM on wgmma
//                          with K over the pixels.  A k-block is one 64 x 2-pixel box of dY and of X (shifted by the tap) read
//                          through the 4-D tensor maps of ais_conv_kernel: TMA's zero fill is the padding, the K tail and the
//                          pixels past the image, and the channels past C0 come from the second source's map.  Split-K over
//                          CTAs, each split writes its own fp32 partial, reduced over the splits in order.
//   ais_nt_*             : InstanceNorm (per image and channel) and BatchNorm in training mode (per channel over the batch):
//                          fp64 chunk partials (or those of ais_conv_kernel's epilogue), a finalize in a fixed order, an apply
//                          pass; the backward pass has the same shape.
//   ais_up2_bwd_kernel   : adjoint of bilinear x2 (align_corners=False) as a gather: every input pixel sums the <= 4 x 4 outputs
//                          that read it, so no atomics.
//   ais_s2d_kernel       : space-to-depth of dY, the input of the 2x2 / stride 2 transposed convolution's backward GEMMs.
//   ais_head_bwd_*       : out_conv (1x1 to 3 channels) + sigmoid backward.
//   ais_rsz_bwd_*        : adjoint of the crop + bilinear resize of postprocess_masks, one gather per axis.
//   ais_dl_*             : per-channel sums of the distance-based Dice loss and its backward pass.
// The data gradient of a convolution is ais_conv_kernel itself (ais.cu), run on dY with the weights rotated by 180 degrees.
#include <algorithm>
#include <cmath>

#include "device_util.cuh"
#include "engine.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace msam {
namespace {

// ------------------------------------------------------------------------------------------------ weight gradient
// One CTA: 64 * MH output channels x 64 * NB input channels of one tap.  Each k-block is a {64 ch, 64 x, 2 y, 1 image} box
// (128 pixel rows of 128 B, SWIZZLE_128B): an MN-major wgmma operand contracted over its 128 rows.  Warp 0 loads, the
// second warpgroup issues wgmma m64n(64 NB)k16 on each 64-channel half of dY.
constexpr int WG_BOX = 128 * 128;   // bytes of one 128-pixel x 64-channel box

template <int MH, int NB>
struct WgCfg {
  static constexpr int A_BYTES = MH * WG_BOX, STAGE_BYTES = (MH + NB) * WG_BOX;
  static constexpr int STAGES = 196608 / STAGE_BYTES;
  static constexpr int OFF_BAR = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};

struct WgParams {
  int C0, Cin, ks, tiles_x, tiles, kb_total, kb_per, ldw, Cout;
  float* part;   // [splits][Cout][ldw], ldw = ks * ks * Cin
};

template <int MH, int NB>
__global__ void __launch_bounds__(256, 1)
ais_wgrad_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tm0,
                 const __grid_constant__ CUtensorMap tm1, const WgParams p) {
  using Cfg = WgCfg<MH, NB>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * 64 * MH;
  const int ntap = p.Cin / (64 * NB);
  const int tap = blockIdx.y / ntap, n0 = (blockIdx.y - tap * ntap) * 64 * NB;
  const int dy = p.ks == 3 ? tap / 3 - 1 : 0, dx = p.ks == 3 ? tap % 3 - 1 : 0;
  const int kb0 = blockIdx.z * p.kb_per, kb1 = min(kb0 + p.kb_per, p.kb_total);

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmY);
    prefetch_tmap(&tm0);
    prefetch_tmap(&tm1);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        const int b = kb / p.tiles, t = kb - b * p.tiles;
        const int x0 = (t % p.tiles_x) * 64, y0 = (t / p.tiles_x) * 2;
        mbar_wait(&empty_bar[stage], phase ^ 1, 60);
        uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
#pragma unroll
        for (int h = 0; h < MH; ++h) tma_load_4d(sa + h * WG_BOX, &tmY, &full_bar[stage], m0 + 64 * h, x0, y0, b);
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          const int c = n0 + 64 * j;
          uint8_t* dst = sa + Cfg::A_BYTES + j * WG_BOX;
          if (c < p.C0) tma_load_4d(dst, &tm0, &full_bar[stage], c, x0 + dx, y0 + dy, b);
          else tma_load_4d(dst, &tm1, &full_bar[stage], c - p.C0, x0 + dx, y0 + dy, b);
        }
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
    float acc[MH][NB * 32];
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase, 61);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES), sb = sa + Cfg::A_BYTES;
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {   // 16 pixel rows = 2048 B further down both MN-major tiles
        const uint64_t db = make_desc_sw128(sb + kk * 2048, WG_BOX, 1024);
#pragma unroll
        for (int h = 0; h < MH; ++h)
          wgmma<NB * 64, 1, 1>(acc[h], make_desc_sw128(sa + h * WG_BOX + kk * 2048, WG_BOX, 1024), db, (kb > kb0) || (kk != 0));
      }
      wg_commit();
      wg_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
#pragma unroll
    for (int h = 0; h < MH; ++h) wg_fence_acc(acc[h]);
    float* out = p.part + (size_t)blockIdx.z * p.Cout * p.ldw + (size_t)tap * p.Cin + n0;
#pragma unroll
    for (int h = 0; h < MH; ++h) {
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        float* dst = out + (size_t)(m0 + 64 * h + 16 * wq + qr + 8 * rs) * p.ldw;
#pragma unroll
        for (int j = 0; j < NB * 8; ++j)
          *reinterpret_cast<float2*>(dst + 8 * j + qc) = make_float2(acc[h][4 * j + 2 * rs], acc[h][4 * j + 2 * rs + 1]);
      }
    }
  }
}

// out[i] = sum over the splits s = 0, 1, ... of part[s][i], in that order
__global__ void ais_split_sum_kernel(const float* __restrict__ part, int splits, long n, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = part[i];
  for (int k = 1; k < splits; ++k) s += part[(size_t)k * n + i];
  out[i] = s;
}

struct WgPlan {
  int MH, NB, ctas, splits, per, kb_total, tiles_x, tiles;
};

WgPlan wgrad_plan(int Cout, int Cin, int B, int H, int W, int ks) {
  WgPlan q;
  q.MH = Cout % 128 == 0 ? 2 : 1;
  q.NB = Cin % 128 == 0 ? 2 : 1;
  q.tiles_x = (W + 63) / 64;
  q.tiles = q.tiles_x * ((H + 1) / 2);
  q.kb_total = B * q.tiles;
  q.ctas = (Cout / (64 * q.MH)) * ks * ks * (Cin / (64 * q.NB));
  int splits = (264 + q.ctas - 1) / q.ctas;   // about two waves of one CTA per SM (198 KB of shared memory each), at least 8 k-blocks per split; shapes only
  splits = std::min(splits, (q.kb_total + 7) / 8);
  splits = std::max(splits, 1);
  q.per = (q.kb_total + splits - 1) / splits;
  q.splits = (q.kb_total + q.per - 1) / q.per;   // no empty split
  return q;
}

template <int MH, int NB>
int launch_wgrad_cfg(const CUtensorMap& ty, const CUtensorMap& t0, const CUtensorMap& t1, const WgParams& p, dim3 grid,
                     cudaStream_t st) {
  if (cudaFuncSetAttribute(ais_wgrad_kernel<MH, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, WgCfg<MH, NB>::SMEM_BYTES) !=
      cudaSuccess)
    return set_error("ais wgrad: cudaFuncSetAttribute failed");
  ais_wgrad_kernel<MH, NB><<<grid, 256, WgCfg<MH, NB>::SMEM_BYTES, st>>>(ty, t0, t1, p);
  return 0;
}

// ------------------------------------------------------------------------------------------------ norms
constexpr int NT_CHUNK = 1024;   // pixels per partial sum

// Partial sums over a chunk of image b's pixels, channel c, in fp64:
//   dy == null (statistics):  s0 = sum x,  s1 = sum x^2
//   dy != null (backward):    g = dy (times [out > 0] when `out` is given), s0 = sum g,  s1 = sum g (x - mean) rstd  (x == null:
//                             s1 = 0; the bias gradient)
template <typename TD>
__global__ void ais_nt_partial_kernel(const __nv_bfloat16* __restrict__ x, int ldx, const TD* __restrict__ dy, int ldd,
                                      const __nv_bfloat16* __restrict__ out, const float* __restrict__ mean,
                                      const float* __restrict__ rstd, int per_image, int HW, int C, int nchunk,
                                      double* __restrict__ part) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const int p0 = ch * NT_CHUNK, p1 = min(HW, p0 + NT_CHUNK);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int gi = (per_image ? b * C : 0) + c;
    const float mu = mean ? mean[gi] : 0.f, rs = rstd ? rstd[gi] : 0.f;
    double s0 = 0.0, s1 = 0.0;
    for (int q = p0; q < p1; ++q) {
      const size_t pix = (size_t)b * HW + q;
      if (!dy) {
        const double v = (double)__bfloat162float(x[pix * ldx + c]);
        s0 += v;
        s1 += v * v;
        continue;
      }
      float g = (float)dy[pix * ldd + c];
      if (out && !(__bfloat162float(out[pix * C + c]) > 0.f)) g = 0.f;
      s0 += (double)g;
      if (x) s1 += (double)(g * ((__bfloat162float(x[pix * ldx + c]) - mu) * rs));
    }
    double* o = part + (((size_t)b * nchunk + ch) * C + c) * 2;
    o[0] = s0;
    o[1] = s1;
  }
}

// One block per group (image and channel, or channel): thread t sums the group's chunk partials t, t + 256, ... in order (for
// BatchNorm every image's chunks, in image order), then a fixed tree over the threads.  Thread 0: mean / rstd of the biased
// variance (when wanted), scale / shift of the affine apply, and BatchNorm's running statistics as torch updates them (momentum,
// unbiased variance).
__global__ void __launch_bounds__(256) ais_nt_finalize_kernel(const double* __restrict__ part, int B, int HW, int C, int nchunk,
                                                              int per_image, float eps, const float* gamma, const float* beta,
                                                              float momentum, float* run_mean, float* run_var,
                                                              float* __restrict__ mean, float* __restrict__ rstd,
                                                              float* __restrict__ scale, float* __restrict__ shift) {
  __shared__ double rs[256], rss[256];
  const int i = blockIdx.x, c = i % C;
  const int n = per_image ? nchunk : B * nchunk;   // the group's chunks: part[b][chunk] with b * nchunk + chunk from k0 on
  const size_t k0 = per_image ? (size_t)(i / C) * nchunk : 0;
  double s = 0.0, ss = 0.0;
  for (int k = threadIdx.x; k < n; k += 256) {
    const double* p = part + ((k0 + k) * C + c) * 2;
    s += p[0];
    ss += p[1];
  }
  rs[threadIdx.x] = s;
  rss[threadIdx.x] = ss;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      rs[threadIdx.x] += rs[threadIdx.x + o];
      rss[threadIdx.x] += rss[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x) return;
  const double cnt = per_image ? (double)HW : (double)HW * B;
  const double mu = rs[0] / cnt, var = fmax(rss[0] / cnt - mu * mu, 0.0);
  const double r = 1.0 / sqrt(var + (double)eps);
  const double g = gamma ? (double)gamma[c] : 1.0, bt = beta ? (double)beta[c] : 0.0;
  scale[i] = (float)(g * r);
  shift[i] = (float)(bt - mu * g * r);
  if (mean) {
    mean[i] = (float)mu;
    rstd[i] = (float)r;
  }
  if (run_mean) {
    run_mean[c] = (float)((1.0 - momentum) * (double)run_mean[c] + momentum * mu);
    run_var[c] = (float)((1.0 - momentum) * (double)run_var[c] + momentum * var * cnt / fmax(cnt - 1.0, 1.0));
  }
}

// y = x * scale + shift (per image and channel, or per channel), optionally ReLU; bf16 NHWC, 8 channels per thread
__global__ void ais_nt_apply_kernel(const __nv_bfloat16* __restrict__ x, int HW, int C, long total8, const float* __restrict__ scale,
                                    const float* __restrict__ shift, int per_image, int relu, __nv_bfloat16* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  const long e = i * 8;
  const int c = (int)(e % C), b = (int)(e / ((long)HW * C));
  const uint4 v = *reinterpret_cast<const uint4*>(x + e);
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int g = (per_image ? b * C : 0) + c + 2 * k;
    float lo = bf16_lo(w[k]) * scale[g] + shift[g], hi = bf16_hi(w[k]) * scale[g + 1] + shift[g + 1];
    if (relu) {
      lo = fmaxf(lo, 0.f);
      hi = fmaxf(hi, 0.f);
    }
    o[k] = pack_bf16(lo, hi);
  }
  *reinterpret_cast<uint4*>(out + e) = make_uint4(o[0], o[1], o[2], o[3]);
}

// Backward coefficients per group: coef = {gamma rstd, mean(g), mean(g xhat)}; per channel, in image order, the parameter
// gradients dgamma = sum g xhat and dbeta = sum g (either may be null).
__global__ void ais_nt_bwd_finalize_kernel(const double* __restrict__ part, int B, int HW, int C, int nchunk, int per_image,
                                           const float* gamma, const float* __restrict__ rstd, float* __restrict__ coef,
                                           float* dgamma, float* dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double tg = 0.0, tgx = 0.0;
  for (int b = 0; b < B; ++b) {
    double s0 = 0.0, s1 = 0.0;
    for (int ch = 0; ch < nchunk; ++ch) {
      const double* p = part + (((size_t)b * nchunk + ch) * C + c) * 2;
      s0 += p[0];
      s1 += p[1];
    }
    tg += s0;
    tgx += s1;
    if (per_image && coef) {
      float* k = coef + ((size_t)b * C + c) * 3;
      k[0] = (gamma ? gamma[c] : 1.f) * rstd[b * C + c];
      k[1] = (float)(s0 / HW);
      k[2] = (float)(s1 / HW);
    }
  }
  if (!per_image && coef) {
    coef[c * 3] = (gamma ? gamma[c] : 1.f) * rstd[c];
    coef[c * 3 + 1] = (float)(tg / ((double)HW * B));
    coef[c * 3 + 2] = (float)(tgx / ((double)HW * B));
  }
  if (dgamma) dgamma[c] = (float)tgx;
  if (dbeta) dbeta[c] = (float)tg;
}

// dx = gamma rstd (g - mean(g) - xhat mean(g xhat)), g = dy [* (out > 0)]; in_mask: times [x > 0] (the ReLU before the norm).
// out_mode 0: bf16 store, 1: fp32 store, 2: fp32 add.  One thread per (pixel, channel).
template <typename TD>
__global__ void ais_nt_bwd_apply_kernel(const __nv_bfloat16* __restrict__ x, int ldx, const TD* __restrict__ dy, int ldd,
                                        const __nv_bfloat16* __restrict__ out, const float* __restrict__ mean,
                                        const float* __restrict__ rstd, const float* __restrict__ coef, int per_image, int in_mask,
                                        int HW, int C, long n, void* dx, int ldo, int out_mode) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const long pix = i / C;
  const int b = (int)(pix / HW);
  const int gi = (per_image ? b * C : 0) + c;
  const float xv = __bfloat162float(x[pix * ldx + c]);
  float g = (float)dy[pix * ldd + c];
  if (out && !(__bfloat162float(out[pix * C + c]) > 0.f)) g = 0.f;
  const float* k = coef + (size_t)gi * 3;
  float v = k[0] * (g - k[1] - ((xv - mean[gi]) * rstd[gi]) * k[2]);
  if (in_mask && !(xv > 0.f)) v = 0.f;
  const size_t o = pix * ldo + c;
  if (out_mode == 0) reinterpret_cast<__nv_bfloat16*>(dx)[o] = __float2bfloat16(v);
  else if (out_mode == 1) reinterpret_cast<float*>(dx)[o] = v;
  else reinterpret_cast<float*>(dx)[o] += v;
}

// ------------------------------------------------------------------------------------------------ samplers
// weight of source index i in the bilinear interpolation of destination index d (align_corners=False)
__device__ __forceinline__ float lin_weight(int d, float scale, int n, int i) {
  int i0, i1;
  float l1;
  lin_src(d, scale, n, i0, i1, l1);
  return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}

// adjoint of ais_up2_kernel: dx [B, H, W, C] from dy [B, 2H, 2W, C], both bf16; output rows 2y - 1 .. 2y + 2 read row y
__global__ void ais_up2_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int B, int H, int W, int C, __nv_bfloat16* __restrict__ dx) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int C8 = C / 8;
  if (i >= (long)B * H * W * C8) return;
  const int c = (int)(i % C8) * 8;
  const long p = i / C8;
  const int x = (int)(p % W), y = (int)((p / W) % H), b = (int)(p / ((long)H * W));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int oy = max(2 * y - 1, 0); oy <= min(2 * y + 2, 2 * H - 1); ++oy) {
    const float wy = lin_weight(oy, 0.5f, H, y);
    if (wy == 0.f) continue;
    for (int ox = max(2 * x - 1, 0); ox <= min(2 * x + 2, 2 * W - 1); ++ox) {
      const float w = wy * lin_weight(ox, 0.5f, W, x);
      if (w == 0.f) continue;
      const uint4 q = *reinterpret_cast<const uint4*>(dy + (((size_t)b * 2 * H + oy) * 2 * W + ox) * C + c);
      const uint32_t a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        acc[2 * k] += w * bf16_lo(a[k]);
        acc[2 * k + 1] += w * bf16_hi(a[k]);
      }
    }
  }
  *reinterpret_cast<uint4*>(dx + p * C + c) =
      make_uint4(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]), pack_bf16(acc[4], acc[5]), pack_bf16(acc[6], acc[7]));
}

// out[b, y, x, (i * 2 + j) * C + c] = dy[b, 2y + i, 2x + j, c]: the transposed convolution's output as the GEMM's columns
__global__ void ais_s2d_kernel(const __nv_bfloat16* __restrict__ dy, int B, int H, int W, int C, __nv_bfloat16* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int C8 = C / 8;
  if (i >= (long)B * H * W * 4 * C8) return;
  const int c = (int)(i % C8) * 8, ij = (int)((i / C8) % 4);
  const long p = i / (4 * C8);
  const int x = (int)(p % W), y = (int)((p / W) % H), b = (int)(p / ((long)H * W));
  *reinterpret_cast<uint4*>(out + p * 4 * C + ij * C + c) =
      *reinterpret_cast<const uint4*>(dy + (((size_t)b * 2 * H + 2 * y + (ij >> 1)) * 2 * W + 2 * x + (ij & 1)) * C + c);
}

// acc (fp32) += x (bf16)
__global__ void ais_add_bf16_kernel(float* __restrict__ acc, const __nv_bfloat16* __restrict__ x, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) acc[i] += __bfloat162float(x[i]);
}

// g (bf16) *= [out > 0]: the ReLU of the layer that wrote out
__global__ void ais_relu_mask_kernel(__nv_bfloat16* __restrict__ g, const __nv_bfloat16* __restrict__ out, long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(__bfloat162float(out[i]) > 0.f)) g[i] = __float2bfloat16(0.f);
}

// ------------------------------------------------------------------------------------------------ head
// per pixel: ds_k = dmaps_k s_k (1 - s_k) (s = the sigmoid maps), dh_c = sum_k ds_k w[k, c] times [h_c > 0] (bf16)
__global__ void ais_head_bwd_kernel(const __nv_bfloat16* __restrict__ h, int B, int HW, int C, const float* __restrict__ w,
                                    const float* __restrict__ maps, const float* __restrict__ dmaps, float* __restrict__ ds,
                                    __nv_bfloat16* __restrict__ dh) {
  __shared__ float sw[3 * 512];
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long)B * HW) return;
  const long b = p / HW, q = p % HW;
  float d[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float s = maps[(b * 3 + k) * HW + q];
    d[k] = dmaps[(b * 3 + k) * HW + q] * s * (1.f - s);
    ds[p * 3 + k] = d[k];
  }
  for (int c = 0; c < C; ++c) {
    const float v = d[0] * sw[c] + d[1] * sw[C + c] + d[2] * sw[2 * C + c];
    dh[p * C + c] = __float2bfloat16(__bfloat162float(h[p * C + c]) > 0.f ? v : 0.f);
  }
}

// partials over NT_CHUNK pixels: part[chunk][k][C + 1] = {sum ds_k h_c (c < C), sum ds_k}
__global__ void ais_head_wgrad_partial_kernel(const __nv_bfloat16* __restrict__ h, long P, int C, const float* __restrict__ ds,
                                              double* __restrict__ part) {
  const long p0 = (long)blockIdx.x * NT_CHUNK, p1 = min(P, p0 + NT_CHUNK);
  for (int c = threadIdx.x; c <= C; c += blockDim.x) {
    double s[3] = {0.0, 0.0, 0.0};
    for (long p = p0; p < p1; ++p) {
      const double v = c < C ? (double)__bfloat162float(h[p * C + c]) : 1.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) s[k] += (double)ds[p * 3 + k] * v;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) part[((size_t)blockIdx.x * 3 + k) * (C + 1) + c] = s[k];
  }
}

__global__ void ais_head_wgrad_finalize_kernel(const double* __restrict__ part, int nchunk, int C, float* __restrict__ dw,
                                               float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * (C + 1)) return;
  double s = 0.0;
  for (int ch = 0; ch < nchunk; ++ch) s += part[(size_t)ch * 3 * (C + 1) + i];
  const int k = i / (C + 1), c = i % (C + 1);
  if (c < C) dw[k * C + c] = (float)s;
  else db[k] = (float)s;
}

// ------------------------------------------------------------------------------------------------ crop + resize backward
// along x: t[r, x] = sum_ox w(ox, x) dout[r, ox] for x < iw (the forward's source width)
__global__ void ais_rsz_bwd_x_kernel(const float* __restrict__ dout, long rows, int ow, int iw, float* __restrict__ t) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * iw) return;
  const int x = (int)(i % iw);
  const long r = i / iw;
  const float sc = (float)iw / (float)ow;
  const int o0 = max(0, (int)floorf((x - 0.5f) / sc - 0.5f) - 1), o1 = min(ow - 1, (int)ceilf((x + 1.5f) / sc - 0.5f) + 1);
  float s = 0.f;
  for (int o = o0; o <= o1; ++o) {
    const float w = lin_weight(o, sc, iw, x);
    if (w != 0.f) s += w * dout[r * ow + o];
  }
  t[i] = s;
}

// along y, with the crop's adjoint: d[pl, y, x] = sum_oy w(oy, y) t[pl, oy, x] inside [ih, iw], 0 outside
__global__ void ais_rsz_bwd_y_kernel(const float* __restrict__ t, int P, int Hs, int Ws, int ih, int iw, int oh,
                                     float* __restrict__ d) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * Hs * Ws) return;
  const int x = (int)(i % Ws), y = (int)((i / Ws) % Hs);
  const long pl = i / ((long)Hs * Ws);
  float s = 0.f;
  if (x < iw && y < ih) {
    const float sc = (float)ih / (float)oh;
    const int o0 = max(0, (int)floorf((y - 0.5f) / sc - 0.5f) - 1), o1 = min(oh - 1, (int)ceilf((y + 1.5f) / sc - 0.5f) + 1);
    for (int o = o0; o <= o1; ++o) {
      const float w = lin_weight(o, sc, ih, y);
      if (w != 0.f) s += w * t[(pl * oh + o) * iw + x];
    }
  }
  d[i] = s;
}

// ------------------------------------------------------------------------------------------------ distance-based Dice loss
// Channel k of prediction x and target y (fp32 [B, 3, HW]); with mask, channels 1 and 2 of both are multiplied by y_0.
// part[b][chunk][k][3] = {sum x y, sum x^2, sum y^2} over the chunk, reduced by a fixed tree of 256 threads.
constexpr int DL_CHUNK = 4096;

__device__ __forceinline__ float dl_mask(const float* y, long b, int HW, long q, int k, int mask) {
  return (mask && k > 0) ? y[(b * 3) * HW + q] : 1.f;
}

__global__ void __launch_bounds__(256) ais_dl_partial_kernel(const float* __restrict__ x, const float* __restrict__ y, int HW,
                                                             int nchunk, int mask, double* __restrict__ part) {
  __shared__ double red[256][9];
  const int b = blockIdx.y, ch = blockIdx.x;
  const long q0 = (long)ch * DL_CHUNK, q1 = min((long)HW, q0 + DL_CHUNK);
  double s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (long q = q0 + threadIdx.x; q < q1; q += 256) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float m = dl_mask(y, b, HW, q, k, mask);
      const double xv = (double)(x[((long)b * 3 + k) * HW + q] * m), yv = (double)(y[((long)b * 3 + k) * HW + q] * m);
      s[3 * k] += xv * yv;
      s[3 * k + 1] += xv * xv;
      s[3 * k + 2] += yv * yv;
    }
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) red[threadIdx.x][j] = s[j];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o)
      for (int j = 0; j < 9; ++j) red[threadIdx.x][j] += red[threadIdx.x + o][j];
    __syncthreads();
  }
  if (threadIdx.x < 9) part[((size_t)b * nchunk + ch) * 9 + threadIdx.x] = red[0][threadIdx.x];
}

__global__ void ais_dl_finalize_kernel(const double* __restrict__ part, int n, double* __restrict__ stats) {
  const int j = threadIdx.x;
  if (j >= 9) return;
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += part[(size_t)i * 9 + j];
  stats[j] = s;
}

// dx_k = m_k (dN_k y'_k + 2 dXX_k x'_k) for the upstream gradients coef[k] = {dL/d sum x'y', dL/d sum x'^2}
__global__ void ais_dl_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, int B, int HW, int mask,
                                  const float* __restrict__ coef, float* __restrict__ dx) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)B * 3 * HW) return;
  const long q = i % HW, bk = i / HW;
  const int k = (int)(bk % 3);
  const long b = bk / 3;
  const float m = dl_mask(y, b, HW, q, k, mask);
  dx[i] = m * (coef[2 * k] * (y[i] * m) + 2.f * coef[2 * k + 1] * (x[i] * m));
}

int64_t nt_ws_bytes(int B, int HW, int C) {
  return (int64_t)up256((size_t)B * ((HW + NT_CHUNK - 1) / NT_CHUNK) * C * 16) + (int64_t)up256((size_t)B * C * 12);
}

}  // namespace
}  // namespace msam

using namespace msam;

extern "C" {

int64_t msam_ais_wgrad_workspace(int Cout, int C0, int C1, int B, int H, int W, int ks) {
  if (Cout <= 0 || Cout % 64 || C0 <= 0 || C0 % 64 || C1 < 0 || C1 % 64 || B <= 0 || H <= 0 || W <= 0 || (ks != 1 && ks != 3))
    return -1;
  const WgPlan q = wgrad_plan(Cout, C0 + C1, B, H, W, ks);
  return (int64_t)q.splits * Cout * ks * ks * (C0 + C1) * 4;
}

int msam_op_ais_wgrad(const void* dy, int Cout, const void* x0, int C0, const void* x1, int C1, int B, int H, int W, int ks, void* ws,
                      int64_t ws_bytes, float* dw, void* stream) {
  if (!dy || !x0 || !dw || !ws || (C1 > 0 && !x1)) return set_error("msam_op_ais_wgrad: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || (long)B * ((W + 63) / 64) * ((H + 1) / 2) >= (1l << 31))
    return set_error("msam_op_ais_wgrad: B=%d, H=%d, W=%d", B, H, W);
  if (C0 <= 0 || C0 % 64 || C1 < 0 || C1 % 64 || Cout <= 0 || Cout % 64)
    return set_error("msam_op_ais_wgrad: Cout=%d, C0=%d, C1=%d (multiples of 64, C1 may be 0)", Cout, C0, C1);
  if (ks != 1 && ks != 3) return set_error("msam_op_ais_wgrad: kernel size %d (1 or 3)", ks);
  const int64_t need = msam_ais_wgrad_workspace(Cout, C0, C1, B, H, W, ks);
  if (ws_bytes < need) return set_error("msam_op_ais_wgrad: workspace of %lld bytes, %lld needed", (long long)ws_bytes, (long long)need);
  if (!al16(dy) || !al16(x0) || (x1 && !al16(x1)) || ((uintptr_t)dw & 7) || ((uintptr_t)ws & 15))
    return set_error("msam_op_ais_wgrad: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int Cin = C0 + C1;
  const WgPlan q = wgrad_plan(Cout, Cin, B, H, W, ks);
  CUtensorMap ty, t0, t1;
  RUN(make_tmap_nhwc(&ty, dy, B, H, W, Cout));
  RUN(make_tmap_nhwc(&t0, x0, B, H, W, C0));
  if (C1 > 0) RUN(make_tmap_nhwc(&t1, x1, B, H, W, C1));
  else t1 = t0;
  WgParams p{C0, Cin, ks, q.tiles_x, q.tiles, q.kb_total, q.per, ks * ks * Cin, Cout, (float*)ws};
  const dim3 grid(Cout / (64 * q.MH), ks * ks * (Cin / (64 * q.NB)), q.splits);
  const double M = (double)B * H * W, n = (double)Cout * ks * ks * Cin;
  prof_begin(st, ks == 3 ? "ais wgrad 3x3" : "ais wgrad 1x1", 2.0 * M * n, 2.0 * M * (Cout + Cin) * ks * ks + 8.0 * q.splits * n);
  int rc;
  if (q.MH == 2) rc = q.NB == 2 ? launch_wgrad_cfg<2, 2>(ty, t0, t1, p, grid, st) : launch_wgrad_cfg<2, 1>(ty, t0, t1, p, grid, st);
  else rc = q.NB == 2 ? launch_wgrad_cfg<1, 2>(ty, t0, t1, p, grid, st) : launch_wgrad_cfg<1, 1>(ty, t0, t1, p, grid, st);
  RUN(rc);
  LAUNCH_CHECK("ais wgrad");
  ais_split_sum_kernel<<<nblk((long)n), 256, 0, st>>>((const float*)ws, q.splits, (long)n, dw);
  prof_end(st);
  LAUNCH_CHECK("ais wgrad split sum");
  return 0;
}

int64_t msam_ais_norm_workspace(int B, int HW, int C) {
  if (B <= 0 || HW <= 0 || C <= 0) return -1;
  return nt_ws_bytes(B, HW, C);
}

static int nt_check(const char* fn, int B, int HW, int C, void* ws, int64_t ws_bytes) {
  if (B <= 0 || HW <= 0 || C <= 0 || C % 8 || (long)B * HW * C >= (1l << 40))
    return set_error("%s: B=%d, HW=%d, C=%d (C a multiple of 8)", fn, B, HW, C);
  if (!ws || ((uintptr_t)ws & 255)) return set_error("%s: null or misaligned workspace", fn);
  if (ws_bytes < nt_ws_bytes(B, HW, C))
    return set_error("%s: workspace of %lld bytes, %lld needed", fn, (long long)ws_bytes, (long long)nt_ws_bytes(B, HW, C));
  return 0;
}

int msam_op_ais_norm_forward(const void* x, int B, int HW, int C, int per_image, const double* stats, int nchunk, const float* gamma,
                             const float* beta, float eps, int relu, float momentum, float* run_mean, float* run_var, void* ws,
                             int64_t ws_bytes, float* mean, float* rstd, void* out, void* stream) {
  if (!x || !out) return set_error("msam_op_ais_norm_forward: null argument");
  RUN(nt_check("msam_op_ais_norm_forward", B, HW, C, ws, ws_bytes));
  if (stats && nchunk <= 0) return set_error("msam_op_ais_norm_forward: %d statistics chunks", nchunk);
  if ((gamma == nullptr) != (beta == nullptr) || (mean == nullptr) != (rstd == nullptr) || (run_mean == nullptr) != (run_var == nullptr) ||
      (run_mean && per_image))
    return set_error("msam_op_ais_norm_forward: gamma / beta, mean / rstd and the running statistics go in pairs (running ones for "
                     "BatchNorm only)");
  if (!al16(x) || !al16(out) || ((uintptr_t)stats & 7)) return set_error("msam_op_ais_norm_forward: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int own = (HW + NT_CHUNK - 1) / NT_CHUNK;
  double* part = (double*)ws;
  float* scale = (float*)((char*)ws + up256((size_t)B * own * C * 16));
  float* shift = scale + (size_t)B * C;
  // the inference decoder's InstanceNorms keep no mean / rstd; their labels match its kernel tables
  const char* label = !per_image ? "ais batchnorm (train)" : mean ? "ais instnorm (train)"
                                 : stats ? "ais instnorm (conv statistics)" : "ais instnorm";
  prof_begin(st, label, 0.0, (stats ? 4.0 : 6.0) * B * HW * C);
  if (!stats) {
    ais_nt_partial_kernel<float><<<dim3(own, B), C < 256 ? C : 256, 0, st>>>((const __nv_bfloat16*)x, C, nullptr, 0, nullptr, nullptr,
                                                                           nullptr, per_image, HW, C, own, part);
    LAUNCH_CHECK("ais norm partials");
    stats = part;
    nchunk = own;
  }
  ais_nt_finalize_kernel<<<per_image ? B * C : C, 256, 0, st>>>(stats, B, HW, C, nchunk, per_image, eps, gamma, beta, momentum,
                                                                run_mean, run_var, mean, rstd, scale, shift);
  LAUNCH_CHECK("ais norm finalize");
  const long t8 = (long)B * HW * C / 8;
  ais_nt_apply_kernel<<<nblk(t8), 256, 0, st>>>((const __nv_bfloat16*)x, HW, C, t8, scale, shift, per_image, relu, (__nv_bfloat16*)out);
  prof_end(st);
  LAUNCH_CHECK("ais norm apply");
  return 0;
}

int msam_op_ais_norm_backward(const void* x, int ldx, const void* dy, int dy_f32, int ldd, const void* relu_out, int B, int HW, int C,
                              int per_image, const float* gamma, const float* mean, const float* rstd, int in_mask, void* ws,
                              int64_t ws_bytes, void* dx, int out_mode, int ldo, float* dgamma, float* dbeta, void* stream) {
  if (!x || !dy || !mean || !rstd || !dx) return set_error("msam_op_ais_norm_backward: null argument");
  RUN(nt_check("msam_op_ais_norm_backward", B, HW, C, ws, ws_bytes));
  if (ldx < C || ldd < C || ldo < C || out_mode < 0 || out_mode > 2)
    return set_error("msam_op_ais_norm_backward: strides %d, %d, %d for %d channels, output mode %d", ldx, ldd, ldo, C, out_mode);
  if ((uintptr_t)x & 1 || (uintptr_t)dy & (dy_f32 ? 3 : 1) || (uintptr_t)dx & (out_mode ? 3 : 1))
    return set_error("msam_op_ais_norm_backward: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = (HW + NT_CHUNK - 1) / NT_CHUNK;
  double* part = (double*)ws;
  float* coef = (float*)((char*)ws + up256((size_t)B * nchunk * C * 16));
  const __nv_bfloat16 *xb = (const __nv_bfloat16*)x, *ob = (const __nv_bfloat16*)relu_out;
  const int thr = C < 256 ? C : 256;
  const long n = (long)B * HW * C;
  prof_begin(st, per_image ? "ais instnorm backward" : "ais batchnorm backward", 0.0, 10.0 * n);
  if (dy_f32) ais_nt_partial_kernel<float><<<dim3(nchunk, B), thr, 0, st>>>(xb, ldx, (const float*)dy, ldd, ob, mean, rstd, per_image, HW, C, nchunk, part);
  else ais_nt_partial_kernel<__nv_bfloat16><<<dim3(nchunk, B), thr, 0, st>>>(xb, ldx, (const __nv_bfloat16*)dy, ldd, ob, mean, rstd, per_image, HW, C, nchunk, part);
  LAUNCH_CHECK("ais norm backward partials");
  ais_nt_bwd_finalize_kernel<<<nblk(C, 128), 128, 0, st>>>(part, B, HW, C, nchunk, per_image, gamma, rstd, coef, dgamma, dbeta);
  LAUNCH_CHECK("ais norm backward finalize");
  if (dy_f32) ais_nt_bwd_apply_kernel<float><<<nblk(n), 256, 0, st>>>(xb, ldx, (const float*)dy, ldd, ob, mean, rstd, coef, per_image, in_mask, HW, C, n, dx, ldo, out_mode);
  else ais_nt_bwd_apply_kernel<__nv_bfloat16><<<nblk(n), 256, 0, st>>>(xb, ldx, (const __nv_bfloat16*)dy, ldd, ob, mean, rstd, coef, per_image, in_mask, HW, C, n, dx, ldo, out_mode);
  prof_end(st);
  LAUNCH_CHECK("ais norm backward apply");
  return 0;
}

int msam_op_ais_chan_sum(const void* g, int B, int HW, int C, void* ws, int64_t ws_bytes, float* out, void* stream) {
  if (!g || !out) return set_error("msam_op_ais_chan_sum: null argument");
  RUN(nt_check("msam_op_ais_chan_sum", B, HW, C, ws, ws_bytes));
  if ((uintptr_t)g & 1) return set_error("msam_op_ais_chan_sum: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = (HW + NT_CHUNK - 1) / NT_CHUNK;
  ais_nt_partial_kernel<__nv_bfloat16><<<dim3(nchunk, B), C < 256 ? C : 256, 0, st>>>(
      nullptr, C, (const __nv_bfloat16*)g, C, nullptr, nullptr, nullptr, 0, HW, C, nchunk, (double*)ws);
  LAUNCH_CHECK("ais channel sum partials");
  ais_nt_bwd_finalize_kernel<<<nblk(C, 128), 128, 0, st>>>((const double*)ws, B, HW, C, nchunk, 0, nullptr, nullptr, nullptr, nullptr, out);
  LAUNCH_CHECK("ais channel sum");
  return 0;
}

int msam_op_ais_upsample2_backward(const void* dy, int B, int H, int W, int C, void* dx, void* stream) {
  if (!dy || !dx) return set_error("msam_op_ais_upsample2_backward: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || (long)B * 4 * H * W * C >= (1l << 40))
    return set_error("msam_op_ais_upsample2_backward: B=%d, H=%d, W=%d, C=%d (C a multiple of 8)", B, H, W, C);
  if (!al16(dy) || !al16(dx)) return set_error("msam_op_ais_upsample2_backward: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin(st, "ais upsample x2 backward", 0.0, 10.0 * B * H * W * C);
  ais_up2_bwd_kernel<<<nblk((long)B * H * W * (C / 8)), 256, 0, st>>>((const __nv_bfloat16*)dy, B, H, W, C, (__nv_bfloat16*)dx);
  prof_end(st);
  LAUNCH_CHECK("ais upsample x2 backward");
  return 0;
}

int msam_op_ais_space_to_depth(const void* dy, int B, int H, int W, int C, void* out, void* stream) {
  if (!dy || !out) return set_error("msam_op_ais_space_to_depth: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || (long)B * 4 * H * W * C >= (1l << 40))
    return set_error("msam_op_ais_space_to_depth: B=%d, H=%d, W=%d, C=%d (C a multiple of 8)", B, H, W, C);
  if (!al16(dy) || !al16(out)) return set_error("msam_op_ais_space_to_depth: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  ais_s2d_kernel<<<nblk((long)B * H * W * C / 2), 256, 0, st>>>((const __nv_bfloat16*)dy, B, H, W, C, (__nv_bfloat16*)out);
  LAUNCH_CHECK("ais space to depth");
  return 0;
}

int msam_op_ais_add_bf16(float* acc, const void* x, int64_t n, void* stream) {
  if (!acc || !x) return set_error("msam_op_ais_add_bf16: null argument");
  if (n <= 0) return set_error("msam_op_ais_add_bf16: %lld elements", (long long)n);
  ais_add_bf16_kernel<<<nblk(n), 256, 0, (cudaStream_t)stream>>>(acc, (const __nv_bfloat16*)x, n);
  LAUNCH_CHECK("ais add");
  return 0;
}

int msam_op_ais_relu_mask(void* g, const void* out, int64_t n, void* stream) {
  if (!g || !out) return set_error("msam_op_ais_relu_mask: null argument");
  if (n <= 0) return set_error("msam_op_ais_relu_mask: %lld elements", (long long)n);
  ais_relu_mask_kernel<<<nblk(n), 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)g, (const __nv_bfloat16*)out, n);
  LAUNCH_CHECK("ais relu mask");
  return 0;
}

int64_t msam_ais_head_backward_workspace(int B, int HW, int C) {
  if (B <= 0 || HW <= 0 || C <= 0) return -1;
  const long P = (long)B * HW;
  return (int64_t)up256((size_t)P * 12) + (int64_t)((P + NT_CHUNK - 1) / NT_CHUNK) * 3 * (C + 1) * 8;
}

int msam_op_ais_head_backward(const void* h, int B, int HW, int C, const float* w, const float* maps, const float* dmaps, void* ws,
                              int64_t ws_bytes, void* dh, float* dw, float* db, void* stream) {
  if (!h || !w || !maps || !dmaps || !ws || !dh || !dw || !db) return set_error("msam_op_ais_head_backward: null argument");
  if (B <= 0 || HW <= 0 || C <= 0 || C % 8 || C > 512 || (long)B * HW >= (1l << 31))
    return set_error("msam_op_ais_head_backward: B=%d, HW=%d, C=%d (C a multiple of 8, at most 512)", B, HW, C);
  if (ws_bytes < msam_ais_head_backward_workspace(B, HW, C)) return set_error("msam_op_ais_head_backward: workspace too small");
  if (((uintptr_t)ws & 255) || ((uintptr_t)h & 1) || ((uintptr_t)dh & 1)) return set_error("msam_op_ais_head_backward: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const long P = (long)B * HW;
  const int nchunk = (int)((P + NT_CHUNK - 1) / NT_CHUNK);
  float* ds = (float*)ws;
  double* part = (double*)((char*)ws + up256((size_t)P * 12));
  prof_begin(st, "ais out_conv + sigmoid backward", 12.0 * P * C, 4.0 * P * C + 24.0 * P);
  ais_head_bwd_kernel<<<nblk(P), 256, 0, st>>>((const __nv_bfloat16*)h, B, HW, C, w, maps, dmaps, ds, (__nv_bfloat16*)dh);
  LAUNCH_CHECK("ais head backward");
  ais_head_wgrad_partial_kernel<<<nchunk, 128, 0, st>>>((const __nv_bfloat16*)h, P, C, ds, part);
  LAUNCH_CHECK("ais head wgrad partials");
  ais_head_wgrad_finalize_kernel<<<nblk(3 * (C + 1)), 256, 0, st>>>(part, nchunk, C, dw, db);
  prof_end(st);
  LAUNCH_CHECK("ais head wgrad");
  return 0;
}

int msam_op_ais_resize_backward(const float* dout, int P, int Hs, int Ws, int ih, int iw, int oh, int ow, float* tmp, float* dsrc,
                                void* stream) {
  if (!dout || !tmp || !dsrc) return set_error("msam_op_ais_resize_backward: null argument");
  if (P <= 0 || Hs <= 0 || Ws <= 0 || ih <= 0 || iw <= 0 || ih > Hs || iw > Ws || oh <= 0 || ow <= 0 ||
      (long)P * oh * ow >= (1l << 40) || (long)P * Hs * Ws >= (1l << 40))
    return set_error("msam_op_ais_resize_backward: P=%d, source %dx%d, crop %dx%d, output %dx%d", P, Hs, Ws, ih, iw, oh, ow);
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin(st, "ais crop + resize backward", 0.0, 8.0 * P * oh * ow + 8.0 * P * Hs * Ws);
  ais_rsz_bwd_x_kernel<<<nblk((long)P * oh * iw), 256, 0, st>>>(dout, (long)P * oh, ow, iw, tmp);
  LAUNCH_CHECK("ais resize backward (x)");
  ais_rsz_bwd_y_kernel<<<nblk((long)P * Hs * Ws), 256, 0, st>>>(tmp, P, Hs, Ws, ih, iw, oh, dsrc);
  prof_end(st);
  LAUNCH_CHECK("ais resize backward (y)");
  return 0;
}

int64_t msam_ais_dist_loss_workspace(int B, int HW) {
  if (B <= 0 || HW <= 0) return -1;
  return (int64_t)B * ((HW + DL_CHUNK - 1) / DL_CHUNK) * 9 * 8;
}

int msam_op_ais_dist_loss_stats(const float* x, const float* y, int B, int HW, int mask, void* ws, int64_t ws_bytes, double* stats,
                                void* stream) {
  if (!x || !y || !ws || !stats) return set_error("msam_op_ais_dist_loss_stats: null argument");
  if (B <= 0 || HW <= 0 || (long)B * 3 * HW >= (1l << 40)) return set_error("msam_op_ais_dist_loss_stats: B=%d, HW=%d", B, HW);
  if (ws_bytes < msam_ais_dist_loss_workspace(B, HW) || ((uintptr_t)ws & 7))
    return set_error("msam_op_ais_dist_loss_stats: workspace too small or misaligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int nchunk = (HW + DL_CHUNK - 1) / DL_CHUNK;
  ais_dl_partial_kernel<<<dim3(nchunk, B), 256, 0, st>>>(x, y, HW, nchunk, mask, (double*)ws);
  LAUNCH_CHECK("ais distance loss partials");
  ais_dl_finalize_kernel<<<1, 32, 0, st>>>((const double*)ws, B * nchunk, stats);
  LAUNCH_CHECK("ais distance loss statistics");
  return 0;
}

int msam_op_ais_dist_loss_backward(const float* x, const float* y, int B, int HW, int mask, const float* coef, float* dx, void* stream) {
  if (!x || !y || !coef || !dx) return set_error("msam_op_ais_dist_loss_backward: null argument");
  if (B <= 0 || HW <= 0 || (long)B * 3 * HW >= (1l << 40)) return set_error("msam_op_ais_dist_loss_backward: B=%d, HW=%d", B, HW);
  ais_dl_bwd_kernel<<<nblk((long)B * 3 * HW), 256, 0, (cudaStream_t)stream>>>(x, y, B, HW, mask, coef, dx);
  LAUNCH_CHECK("ais distance loss backward");
  return 0;
}

}  // extern "C"
