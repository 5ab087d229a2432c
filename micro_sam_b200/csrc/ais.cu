// Decoder-based automatic instance segmentation (micro-sam's InstanceSegmentationWithDecoder, instance_segmentation.py:
// 688-735 and 1081-1173) on the device.
//
// UNETR decoder layers, bf16 NHWC activations, fp32 accumulation:
//   ais_conv_kernel     : implicit-GEMM convolution (3x3 pad 1 or 1x1) on wgmma, warp-specialised TMA / mbarrier ring.  The
//                         GEMM row is an output pixel, the K loop walks (tap, 64-channel slice) over up to two sources' 4-D
//                         tensor maps, so a channel concatenation is read in place and TMA's zero fill is the padding.
//                         Epilogue: bias (BatchNorm folded into the weights on the host), ReLU or the 2x2 / stride 2
//                         transposed-convolution scatter, and per-(image, channel) partial sums for the InstanceNorm after it.
//   InstanceNorm2d      : the ais_nt_* norm kernels of ais_train.cu (msam_op_ais_norm_forward), fed the epilogue's partial sums.
//                         It cannot be folded into the next convolution: its zero padding would pick up the shift.
//   ais_up2_kernel      : bilinear x2, align_corners=False (the interpolation upsampler; its conv1x1 runs before it, at the
//                         low resolution, because bilinear taps sum to 1).
//   ais_head_kernel     : out_conv (1x1 to 3 channels) + sigmoid, fp32 planes.
//   ais_resize_kernel   : crop to input_size, then bilinear to original_size (postprocess_masks).
// Post-processing (generate), one fp32 [H, W] image:
//   gaussian smoothing in fp64 (mirror border, no FMA), thresholds, 8-connected marker components numbered in raster order,
//   the seeded-watershed rule of DESIGN.md section 2 as two monotone fixpoints (tile-local iterations in shared memory, global
//   sweeps until a device flag stays clear), then the size filter with sequential renumbering.
#include <climits>
#include <cmath>

#include "device_util.cuh"
#include "engine.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace msam {
namespace {

// ------------------------------------------------------------------------------------------------ implicit-GEMM convolution
// One CTA computes a 128-pixel x BN-column tile: 64 x 2 pixels of one image (TMA box {64 ch, 64 x, 2 y, 1 image} of the 4-D map
// (C, W, H, B), rows of 128 B in the SWIZZLE_128B layout of a K-major wgmma operand) against BN weight rows ([N][K], K-major).
// A k-block is one (tap, 64-channel slice); its box sits at (x0 + dx - 1, y0 + dy - 1), so TMA's zero fill of out-of-image
// coordinates is the convolution's zero padding, and the slices past C0 come from the second source's map.  Warp 0 issues
// the loads into a ring of STAGES slots (full / empty mbarriers, as gemm_bf16_kernel); each consumer warpgroup owns 64
// columns and both 64-row halves (wgmma m64n64k16).
constexpr int CV_TX = 64, CV_TY = 2, CV_BK = 64;

template <int BN>
struct ConvCfg {
  static constexpr int NG = BN / 64;
  static constexpr int THREADS = 128 + NG * 128;
  static constexpr int A_BYTES = CV_TX * CV_TY * CV_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + BN * CV_BK * 2;
  static constexpr int STAGES = BN == 128 ? 5 : 8;
  static constexpr int OFF_BAR = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024 /*align slack*/;
};

struct ConvParams {
  int C0, C1, H, W, ks, N, Cout, relu, transposed, tiles_x, tiles_y;
  const float* bias;     // [Cout]
  __nv_bfloat16* out;    // [B, H, W, Cout], or [B, 2H, 2W, Cout] when transposed (column (i * 2 + j) * Cout + co)
  double* stats;         // null, or [B][(N / Cout) * tiles][Cout][2]: sum and sum of squares of the stored bf16 outputs
};

template <int BN>
__global__ void __launch_bounds__(ConvCfg<BN>::THREADS, 1)
ais_conv_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
                const __grid_constant__ CUtensorMap tmW, const ConvParams p) {
  using Cfg = ConvCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  __shared__ float red[Cfg::NG][4][64][2];   // per-warp column sums of the statistics epilogue

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.tiles_x * p.tiles_y;
  const int b = blockIdx.x / tiles, t = blockIdx.x % tiles;
  const int x0 = (t % p.tiles_x) * CV_TX, y0 = (t / p.tiles_x) * CV_TY;
  const int n0 = blockIdx.y * BN;
  const int kpt = (p.C0 + p.C1) / CV_BK, KB = p.ks * p.ks * kpt;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tm0);
    prefetch_tmap(&tm1);
    prefetch_tmap(&tmW);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], Cfg::NG * 4);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {   // TMA producer
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < KB; ++kb) {
        const int tap = kb / kpt, c = (kb - tap * kpt) * CV_BK;
        const int dy = p.ks == 3 ? tap / 3 - 1 : 0, dx = p.ks == 3 ? tap % 3 - 1 : 0;
        mbar_wait(&empty_bar[stage], phase ^ 1, 1);
        uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
        if (c < p.C0) tma_load_4d(sa, &tm0, &full_bar[stage], c, x0 + dx, y0 + dy, b);
        else tma_load_4d(sa, &tm1, &full_bar[stage], c - p.C0, x0 + dx, y0 + dy, b);
        tma_load_2d(sa + Cfg::A_BYTES, &tmW, &full_bar[stage], kb * CV_BK, n0);   // K row tap * (C0 + C1) + c = kb * 64
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    const int grp = (warp - 4) >> 2, wq = warp & 3;
    const int qr = lane >> 2, qc = 2 * (lane & 3);
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    float acc[2][32];
    for (int kb = 0; kb < KB; ++kb) {
      mbar_wait(&full_bar[stage], phase, 3);
      const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
      const uint32_t sb = sa + Cfg::A_BYTES + grp * 64 * 128;
      wg_fence();
#pragma unroll
      for (int k = 0; k < CV_BK / 16; ++k) {
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

    // epilogue: bias, ReLU, bf16 store; statistics of the stored values
    const int ncol = n0 + grp * 64;
    const int ij = ncol / p.Cout, cob = ncol - ij * p.Cout;
    float s[16], ss[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) s[i] = ss[i] = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        const int row = 64 * h + 16 * wq + qr + 8 * rs;
        const int x = x0 + (row & 63), y = y0 + (row >> 6);
        const bool valid = x < p.W && y < p.H;
        const size_t obase = p.transposed
            ? (((size_t)b * 2 * p.H + 2 * y + (ij >> 1)) * 2 * p.W + 2 * x + (ij & 1)) * p.Cout
            : (((size_t)b * p.H + y) * p.W + x) * p.Cout;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int co = cob + 8 * j + qc;
          float v0 = acc[h][4 * j + 2 * rs] + p.bias[co], v1 = acc[h][4 * j + 2 * rs + 1] + p.bias[co + 1];
          if (p.relu) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          const uint32_t w = pack_bf16(v0, v1);
          if (valid) {
            *reinterpret_cast<uint32_t*>(p.out + obase + co) = w;
            const float r0 = bf16_lo(w), r1 = bf16_hi(w);
            s[2 * j] += r0;
            ss[2 * j] += r0 * r0;
            s[2 * j + 1] += r1;
            ss[2 * j + 1] += r1 * r1;
          }
        }
      }
    }
    if (p.stats) {   // fixed reduction order: lanes of one column (xor 4, 8, 16), then the 4 warps in order, in fp64
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
          ss[i] += __shfl_xor_sync(0xffffffffu, ss[i], o);
        }
      }
      if (lane < 4) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int col = 8 * (i >> 1) + 2 * lane + (i & 1);
          red[grp][wq][col][0] = s[i];
          red[grp][wq][col][1] = ss[i];
        }
      }
      named_bar_sync(1 + grp, 128);
      const int tg = threadIdx.x - 128 - 128 * grp;
      if (tg < 64) {
        double S = 0.0, SS = 0.0;
        for (int w = 0; w < 4; ++w) {
          S += (double)red[grp][w][tg][0];
          SS += (double)red[grp][w][tg][1];
        }
        const int nch = (p.N / p.Cout) * tiles, chunk = ij * tiles + t;
        double* o = p.stats + (((size_t)b * nch + chunk) * p.Cout + cob + tg) * 2;
        o[0] = S;
        o[1] = SS;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ bilinear x2, head, resize
__global__ void ais_up2_kernel(const __nv_bfloat16* __restrict__ x, int B, int H, int W, int C, __nv_bfloat16* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int C8 = C / 8;
  if (i >= (long)B * 4 * H * W * C8) return;
  const int c = (int)(i % C8) * 8;
  const long p = i / C8;
  const int ox = (int)(p % (2 * W)), oy = (int)((p / (2 * W)) % (2 * H)), b = (int)(p / (4l * H * W));
  int y0, y1, x0, x1;
  float ly, lx;
  lin_src(oy, 0.5f, H, y0, y1, ly);
  lin_src(ox, 0.5f, W, x0, x1, lx);
  const __nv_bfloat16* base = x + (size_t)b * H * W * C + c;
  const uint4 q00 = *reinterpret_cast<const uint4*>(base + ((size_t)y0 * W + x0) * C);
  const uint4 q01 = *reinterpret_cast<const uint4*>(base + ((size_t)y0 * W + x1) * C);
  const uint4 q10 = *reinterpret_cast<const uint4*>(base + ((size_t)y1 * W + x0) * C);
  const uint4 q11 = *reinterpret_cast<const uint4*>(base + ((size_t)y1 * W + x1) * C);
  const uint32_t a00[4] = {q00.x, q00.y, q00.z, q00.w}, a01[4] = {q01.x, q01.y, q01.z, q01.w};
  const uint32_t a10[4] = {q10.x, q10.y, q10.z, q10.w}, a11[4] = {q11.x, q11.y, q11.z, q11.w};
  const float hy = 1.f - ly, hx = 1.f - lx;
  uint32_t o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float lo = hy * (hx * bf16_lo(a00[k]) + lx * bf16_lo(a01[k])) + ly * (hx * bf16_lo(a10[k]) + lx * bf16_lo(a11[k]));
    const float hi = hy * (hx * bf16_hi(a00[k]) + lx * bf16_hi(a01[k])) + ly * (hx * bf16_hi(a10[k]) + lx * bf16_hi(a11[k]));
    o[k] = pack_bf16(lo, hi);
  }
  *reinterpret_cast<uint4*>(out + p * C + c) = make_uint4(o[0], o[1], o[2], o[3]);
}

// out_conv (1x1, C -> 3) + sigmoid: bf16 NHWC [B, HW, C] -> fp32 planes [B, 3, HW]; C <= 512, C % 8 == 0
__global__ void ais_head_kernel(const __nv_bfloat16* __restrict__ x, int B, int HW, int C, const float* __restrict__ w,
                                const float* __restrict__ bias, float* __restrict__ out) {
  __shared__ float sw[3 * 512];
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long)B * HW) return;
  float s0 = bias[0], s1 = bias[1], s2 = bias[2];
  const __nv_bfloat16* xp = x + p * C;
  for (int c = 0; c < C; c += 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xp + c);
    const uint32_t q[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float f = (k & 1) ? bf16_hi(q[k >> 1]) : bf16_lo(q[k >> 1]);
      s0 += sw[c + k] * f;
      s1 += sw[C + c + k] * f;
      s2 += sw[2 * C + c + k] * f;
    }
  }
  const long b = p / HW, q = p % HW;
  out[(b * 3 + 0) * HW + q] = 1.f / (1.f + expf(-s0));
  out[(b * 3 + 1) * HW + q] = 1.f / (1.f + expf(-s1));
  out[(b * 3 + 2) * HW + q] = 1.f / (1.f + expf(-s2));
}

// planes [P, Hs, Ws] cropped to [ih, iw] and resized (bilinear, align_corners=False) to [P, oh, ow]
__global__ void ais_resize_kernel(const float* __restrict__ x, int P, int Hs, int Ws, int ih, int iw, int oh, int ow,
                                  float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * oh * ow) return;
  const int ox = (int)(i % ow), oy = (int)((i / ow) % oh), pl = (int)(i / ((long)oh * ow));
  int y0, y1, x0, x1;
  float ly, lx;
  lin_src(oy, (float)ih / (float)oh, ih, y0, y1, ly);
  lin_src(ox, (float)iw / (float)ow, iw, x0, x1, lx);
  const float* s = x + (size_t)pl * Hs * Ws;
  const float hy = 1.f - ly, hx = 1.f - lx;
  out[i] = hy * (hx * s[y0 * Ws + x0] + lx * s[y0 * Ws + x1]) + ly * (hx * s[y1 * Ws + x0] + lx * s[y1 * Ws + x1]);
}

// ------------------------------------------------------------------------------------------------ post-processing
constexpr int MAX_TAPS = 129;

__device__ __forceinline__ int mirror(int i, int n) {   // scipy mode 'mirror': reflect about the edge pixel, no repeat
  if (n == 1) return 0;
  const int p = 2 * n - 2;
  i %= p;
  if (i < 0) i += p;
  return i < n ? i : p - i;
}

// one separable pass in fp64 without FMA contraction, taps summed from -r to r starting at 0.0 (the order ais_ref uses)
template <typename Tin, typename Tout>
__global__ void ais_smooth_kernel(const Tin* __restrict__ in, int H, int W, int axis, const double* __restrict__ taps, int r,
                                  Tout* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int x = i % W, y = i / W;
  double acc = 0.0;
  for (int k = -r; k <= r; ++k) {
    const int j = axis == 0 ? mirror(y + k, H) * W + x : y * W + mirror(x + k, W);
    acc = __dadd_rn(acc, __dmul_rn(taps[k + r], (double)in[j]));
  }
  out[i] = (Tout)acc;
}

// fg = fg_s > t_fg; marker = cd_s < t_cd && bd_s < t_bd && fg, as an int32 0/1 image for the component labelling
__global__ void ais_masks_kernel(const float* __restrict__ fg, const float* __restrict__ cd, const float* __restrict__ bd, int n,
                                 float t_fg, float t_cd, float t_bd, uint8_t* __restrict__ fmask, int* __restrict__ marker) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool f = fg[i] > t_fg;
  fmask[i] = f;
  marker[i] = f && cd[i] < t_cd && bd[i] < t_bd;
}

// seeds: B = h, label = component id; other foreground pixels: B = +inf, label = INT_MAX; background: B = +inf, label = 0
__global__ void ais_ws_init_kernel(const int* __restrict__ parent, const uint8_t* __restrict__ fmask, const float* __restrict__ h,
                                   const int* __restrict__ scan, const int* __restrict__ boffs, int n, float* __restrict__ Bv,
                                   int* __restrict__ lab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = parent[i];
  if (r >= 0) {
    Bv[i] = h[i];
    lab[i] = scan[r] + boffs[r >> 10];
  } else {
    Bv[i] = INFINITY;
    lab[i] = fmask[i] ? INT_MAX : 0;
  }
}

constexpr int WS_T = 32;   // tile edge; 256 threads, 4 pixels each

// B(p) = max(h(p), min over foreground 4-neighbours B(q)) for foreground non-seed p, iterated in the tile until it is stable
__global__ void __launch_bounds__(256) ais_ws_barrier_kernel(const float* __restrict__ h, const uint8_t* __restrict__ fmask,
                                                             const int* __restrict__ parent, int H, int W, float* Bv, int* flag) {
  __shared__ float sb[WS_T + 2][WS_T + 2];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int gx0 = blockIdx.x * WS_T, gy0 = blockIdx.y * WS_T;
  for (int k = threadIdx.x; k < (WS_T + 2) * (WS_T + 2); k += 256) {
    const int ly = k / (WS_T + 2), lx = k % (WS_T + 2), gy = gy0 + ly - 1, gx = gx0 + lx - 1;
    sb[ly][lx] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? Bv[gy * W + gx] : INFINITY;
  }
  float hv[4];
  bool act[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int gy = gy0 + ty + 8 * q, gx = gx0 + tx;
    const bool in = gy < H && gx < W;
    const int i = gy * W + gx;
    act[q] = in && fmask[i] && parent[i] < 0;
    hv[q] = act[q] ? h[i] : 0.f;
  }
  __syncthreads();
  volatile float(*vb)[WS_T + 2] = sb;
  while (true) {
    bool ch = false;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!act[q]) continue;
      const int ly = ty + 8 * q + 1, lx = tx + 1;
      const float m = fminf(fminf(vb[ly - 1][lx], vb[ly + 1][lx]), fminf(vb[ly][lx - 1], vb[ly][lx + 1]));
      const float v = fmaxf(hv[q], m);
      if (v < vb[ly][lx]) {
        vb[ly][lx] = v;
        ch = true;
      }
    }
    if (!__syncthreads_or(ch)) break;
  }
  bool wrote = false;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int gy = gy0 + ty + 8 * q, gx = gx0 + tx;
    if (act[q] && sb[ty + 8 * q + 1][tx + 1] < Bv[gy * W + gx]) {
      Bv[gy * W + gx] = sb[ty + 8 * q + 1][tx + 1];
      wrote = true;
    }
  }
  if (__syncthreads_or(wrote) && threadIdx.x == 0) *flag = 1;
}

// label(p) = min(label(p), min label over the foreground 4-neighbours of minimal B), for reached non-seed p
__global__ void __launch_bounds__(256) ais_ws_label_kernel(const float* __restrict__ Bv, const uint8_t* __restrict__ fmask,
                                                           const int* __restrict__ parent, int H, int W, int* lab, int* flag) {
  __shared__ float sb[WS_T + 2][WS_T + 2];
  __shared__ int sl[WS_T + 2][WS_T + 2];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int gx0 = blockIdx.x * WS_T, gy0 = blockIdx.y * WS_T;
  for (int k = threadIdx.x; k < (WS_T + 2) * (WS_T + 2); k += 256) {
    const int ly = k / (WS_T + 2), lx = k % (WS_T + 2), gy = gy0 + ly - 1, gx = gx0 + lx - 1;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    sb[ly][lx] = in ? Bv[gy * W + gx] : INFINITY;
    sl[ly][lx] = in ? lab[gy * W + gx] : 0;
  }
  __syncthreads();
  bool act[4];
  int dirs[4];   // bit d set: neighbour d (N, S, W, E) has the minimal B
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int gy = gy0 + ty + 8 * q, gx = gx0 + tx, ly = ty + 8 * q + 1, lx = tx + 1;
    const bool in = gy < H && gx < W;
    act[q] = in && fmask[gy * W + gx] && parent[gy * W + gx] < 0 && sb[ly][lx] < INFINITY;
    const float bn[4] = {sb[ly - 1][lx], sb[ly + 1][lx], sb[ly][lx - 1], sb[ly][lx + 1]};
    const float m = fminf(fminf(bn[0], bn[1]), fminf(bn[2], bn[3]));
    dirs[q] = (bn[0] == m) | ((bn[1] == m) << 1) | ((bn[2] == m) << 2) | ((bn[3] == m) << 3);
  }
  volatile int(*vl)[WS_T + 2] = sl;
  while (true) {
    bool ch = false;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!act[q]) continue;
      const int ly = ty + 8 * q + 1, lx = tx + 1;
      int v = vl[ly][lx];
      if (dirs[q] & 1) v = min(v, vl[ly - 1][lx]);
      if (dirs[q] & 2) v = min(v, vl[ly + 1][lx]);
      if (dirs[q] & 4) v = min(v, vl[ly][lx - 1]);
      if (dirs[q] & 8) v = min(v, vl[ly][lx + 1]);
      if (v < vl[ly][lx]) {
        vl[ly][lx] = v;
        ch = true;
      }
    }
    if (!__syncthreads_or(ch)) break;
  }
  bool wrote = false;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int gy = gy0 + ty + 8 * q, gx = gx0 + tx;
    if (act[q] && sl[ty + 8 * q + 1][tx + 1] < lab[gy * W + gx]) {
      lab[gy * W + gx] = sl[ty + 8 * q + 1][tx + 1];
      wrote = true;
    }
  }
  if (__syncthreads_or(wrote) && threadIdx.x == 0) *flag = 1;
}

__global__ void ais_count_kernel(const int* __restrict__ lab, int n, int* __restrict__ cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = lab[i];
  if (l > 0 && l != INT_MAX) atomicAdd(cnt + l, 1);
}

__global__ void ais_keep_kernel(const int* __restrict__ cnt, int n_ids, int min_size, int* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_ids) return;
  keep[i] = i > 0 && cnt[i] >= min_size;
}

// unreached pixels (INT_MAX) -> 0; with the size filter, ids -> their rank among the kept ids
__global__ void ais_final_kernel(int* lab, int n, const int* __restrict__ keep, const int* __restrict__ scan,
                                 const int* __restrict__ boffs, int filter) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int l = lab[i];
  if (l == INT_MAX) l = 0;
  if (filter && l > 0) l = keep[l] ? scan[l] + boffs[l >> 10] : 0;
  lab[i] = l;
}

// area and bounding box [x0, y0, x1, y1] (inclusive) of every id
__global__ void ais_props_kernel(const int* __restrict__ lab, int H, int W, int* __restrict__ props) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int l = lab[i];
  if (l <= 0) return;
  int* p = props + 5 * (l - 1);
  atomicAdd(p, 1);
  atomicMin(p + 1, i % W);
  atomicMin(p + 2, i / W);
  atomicMax(p + 3, i % W);
  atomicMax(p + 4, i / W);
}

__global__ void ais_props_init_kernel(int* props, int n_ids) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_ids) return;
  int* p = props + 5 * i;
  p[0] = 0;
  p[1] = p[2] = INT_MAX;
  p[3] = p[4] = -1;
}

int gaussian_taps(const double* taps, int r, double* dev, cudaStream_t st) {
  if (r < 0 || 2 * r + 1 > MAX_TAPS) return set_error("msam_ais_postprocess: smoothing radius %d (at most %d)", r, MAX_TAPS / 2);
  if (r > 0 && !taps) return set_error("msam_ais_postprocess: null taps");
  if (r > 0 && cudaMemcpyAsync(dev, taps, sizeof(double) * (2 * r + 1), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return set_error("msam_ais_postprocess: uploading the smoothing taps failed");
  return 0;
}

// the smoothed map: r == 0 copies
int smooth(const float* in, int H, int W, const double* taps, int r, double* tmp, float* out, cudaStream_t st) {
  const int n = H * W;
  if (r == 0) {
    if (cudaMemcpyAsync(out, in, sizeof(float) * n, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return set_error("msam_ais_postprocess: copy failed");
    return 0;
  }
  ais_smooth_kernel<float, double><<<nblk(n), 256, 0, st>>>(in, H, W, 0, taps, r, tmp);
  LAUNCH_CHECK("ais smooth (axis 0)");
  ais_smooth_kernel<double, float><<<nblk(n), 256, 0, st>>>(tmp, H, W, 1, taps, r, out);
  LAUNCH_CHECK("ais smooth (axis 1)");
  return 0;
}

struct PostWs {
  double *tmp, *taps;
  float *fg, *cd, *bd, *Bv;
  uint8_t* fmask;
  int *parent, *flag, *scan, *bsums, *lab, *cnt, *keep, *scan2, *bsums2, *dflag;
};

// carves the workspace at `base` (null: only the size is wanted)
size_t post_ws(int H, int W, char* base, PostWs* w) {
  const size_t n = (size_t)H * W, nb = (n + 1 + 1023) / 1024 + 4096;
  size_t o = 0;
  auto carve = [&](size_t bytes) { char* p = base ? base + o : nullptr; o += up256(bytes); return p; };
  PostWs t;
  t.tmp = (double*)carve(8 * n);
  t.taps = (double*)carve(8 * 2 * MAX_TAPS);
  t.fg = (float*)carve(4 * n);
  t.cd = (float*)carve(4 * n);
  t.bd = (float*)carve(4 * n);
  t.Bv = (float*)carve(4 * n);
  t.fmask = (uint8_t*)carve(n);
  t.parent = (int*)carve(4 * n);
  t.flag = (int*)carve(4 * n);
  t.scan = (int*)carve(4 * n);
  t.bsums = (int*)carve(4 * nb);
  t.cnt = (int*)carve(4 * (n + 1));
  t.keep = (int*)carve(4 * (n + 1));
  t.scan2 = (int*)carve(4 * (n + 1));
  t.bsums2 = (int*)carve(4 * nb);
  t.dflag = (int*)carve(4);
  if (w) *w = t;
  return o;
}

}  // namespace

// 4-D map (C, W, H, B) of a bf16 NHWC tensor, box {64 ch, 64 x, 2 y, 1}, SWIZZLE_128B, out-of-bounds elements zero
int make_tmap_nhwc(CUtensorMap* m, const void* x, int B, int H, int W, int C) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {CV_BK, CV_TX, CV_TY, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("ais conv: cuTensorMapEncodeTiled failed (%d) for [%d, %d, %d, %d]", (int)r, B, H, W, C);
  return 0;
}

template <int BN>
int launch_conv_bn(const CUtensorMap& t0, const CUtensorMap& t1, const CUtensorMap& tw, const ConvParams& p, int B,
                   cudaStream_t st) {
  // set on every launch: the attribute belongs to the current device, and the call is cheap next to the kernel
  if (cudaFuncSetAttribute(ais_conv_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, ConvCfg<BN>::SMEM_BYTES) !=
      cudaSuccess)
    return set_error("ais conv: cudaFuncSetAttribute failed");
  ais_conv_kernel<BN><<<dim3(B * p.tiles_x * p.tiles_y, p.N / BN), ConvCfg<BN>::THREADS, ConvCfg<BN>::SMEM_BYTES, st>>>(t0, t1, tw, p);
  return 0;
}

int launch_ais_conv(const __nv_bfloat16* x0, int C0, const __nv_bfloat16* x1, int C1, int B, int H, int W, int ks,
                    const __nv_bfloat16* w, const float* bias, int Cout, int relu, int transposed, __nv_bfloat16* out,
                    double* stats, cudaStream_t st) {
  const int N = transposed ? 4 * Cout : Cout, K = ks * ks * (C0 + C1);
  ConvParams p{C0, C1, H, W, ks, N, Cout, relu, transposed, (W + CV_TX - 1) / CV_TX, (H + CV_TY - 1) / CV_TY, bias, out, stats};
  CUtensorMap t0, t1, tw;
  RUN(make_tmap_nhwc(&t0, x0, B, H, W, C0));
  if (C1 > 0) RUN(make_tmap_nhwc(&t1, x1, B, H, W, C1));
  else t1 = t0;
  const int BN = N % 128 == 0 ? 128 : 64;
  RUN(make_tmap_bf16_2d(&tw, w, N, K, K, BN));
  const long M = (long)B * H * W;
  prof_begin(st, ks == 3 ? "ais conv3x3" : (transposed ? "ais convT2x2" : "ais conv1x1"), 2.0 * M * N * K,
             2.0 * M * (C0 + C1) + 2.0 * N * K + 2.0 * M * N);
  RUN(BN == 128 ? launch_conv_bn<128>(t0, t1, tw, p, B, st) : launch_conv_bn<64>(t0, t1, tw, p, B, st));
  prof_end(st);
  LAUNCH_CHECK("ais conv");
  return 0;
}

int conv_stats_count(int B, int H, int W, int Cout, int transposed) {   // doubles
  return B * (transposed ? 4 : 1) * ((W + CV_TX - 1) / CV_TX) * ((H + CV_TY - 1) / CV_TY) * Cout * 2;
}

}  // namespace msam

using namespace msam;

extern "C" {

int64_t msam_ais_conv_stats_size(int B, int H, int W, int Cout, int transposed) {
  if (B <= 0 || H <= 0 || W <= 0 || Cout <= 0) return -1;
  return (int64_t)conv_stats_count(B, H, W, Cout, transposed) * 8;
}

int msam_op_ais_conv(const void* x0, int C0, const void* x1, int C1, int B, int H, int W, int ks, const void* w_bf16,
                     const float* bias, int Cout, int relu, int transposed, void* out, double* stats, void* stream) {
  if (!x0 || !w_bf16 || !bias || !out || (C1 > 0 && !x1)) return set_error("msam_op_ais_conv: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || (long)B * H * W * (transposed ? 4 : 1) >= (1l << 31) ||
      (long)B * ((W + CV_TX - 1) / CV_TX) * ((H + CV_TY - 1) / CV_TY) >= (1l << 31))
    return set_error("msam_op_ais_conv: B=%d, H=%d, W=%d", B, H, W);
  if (C0 <= 0 || C0 % 64 || C1 < 0 || C1 % 64)
    return set_error("msam_op_ais_conv: C0=%d, C1=%d (positive / non-negative multiples of 64)", C0, C1);
  if (Cout <= 0 || Cout % 64) return set_error("msam_op_ais_conv: Cout=%d (a multiple of 64)", Cout);
  if (ks != 1 && ks != 3) return set_error("msam_op_ais_conv: kernel size %d (1 or 3)", ks);
  if (transposed && ks != 1) return set_error("msam_op_ais_conv: the transposed convolution is a 1x1 GEMM (ks=1)");
  if (!al16(x0) || (x1 && !al16(x1)) || !al16(w_bf16) || ((uintptr_t)out & 3) || ((uintptr_t)bias & 3) ||
      ((uintptr_t)stats & 7))
    return set_error("msam_op_ais_conv: misaligned pointer");
  return launch_ais_conv((const __nv_bfloat16*)x0, C0, (const __nv_bfloat16*)x1, C1, B, H, W, ks, (const __nv_bfloat16*)w_bf16,
                         bias, Cout, relu != 0, transposed != 0, (__nv_bfloat16*)out, stats, (cudaStream_t)stream);
}

int msam_op_ais_upsample2(const void* x, int B, int H, int W, int C, void* out, void* stream) {
  if (!x || !out) return set_error("msam_op_ais_upsample2: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 || (long)B * 4 * H * W * C >= (1l << 40))
    return set_error("msam_op_ais_upsample2: B=%d, H=%d, W=%d, C=%d (C a multiple of 8)", B, H, W, C);
  if (!al16(x) || !al16(out)) return set_error("msam_op_ais_upsample2: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin(st, "ais upsample x2", 0.0, 10.0 * B * H * W * C);
  ais_up2_kernel<<<nblk((long)B * 4 * H * W * (C / 8)), 256, 0, st>>>((const __nv_bfloat16*)x, B, H, W, C, (__nv_bfloat16*)out);
  prof_end(st);
  LAUNCH_CHECK("ais upsample x2");
  return 0;
}

int msam_op_ais_head(const void* x, int B, int HW, int C, const float* w, const float* bias, float* out, void* stream) {
  if (!x || !w || !bias || !out) return set_error("msam_op_ais_head: null argument");
  if (B <= 0 || HW <= 0 || C <= 0 || C % 8 || C > 512 || (long)B * HW >= (1l << 31))
    return set_error("msam_op_ais_head: B=%d, HW=%d, C=%d (C a multiple of 8, at most 512)", B, HW, C);
  if (!al16(x)) return set_error("msam_op_ais_head: misaligned pointer");
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin(st, "ais out_conv + sigmoid", 6.0 * B * HW * C, 2.0 * B * HW * C + 12.0 * B * HW);
  ais_head_kernel<<<nblk((long)B * HW), 256, 0, st>>>((const __nv_bfloat16*)x, B, HW, C, w, bias, out);
  prof_end(st);
  LAUNCH_CHECK("ais head");
  return 0;
}

int msam_op_ais_resize(const float* x, int P, int Hs, int Ws, int ih, int iw, int oh, int ow, float* out, void* stream) {
  if (!x || !out) return set_error("msam_op_ais_resize: null argument");
  if (P <= 0 || Hs <= 0 || Ws <= 0 || ih <= 0 || iw <= 0 || ih > Hs || iw > Ws || oh <= 0 || ow <= 0 ||
      (long)P * oh * ow >= (1l << 40))
    return set_error("msam_op_ais_resize: P=%d, source %dx%d, crop %dx%d, output %dx%d", P, Hs, Ws, ih, iw, oh, ow);
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin(st, "ais crop + resize", 0.0, 8.0 * P * oh * ow);
  ais_resize_kernel<<<nblk((long)P * oh * ow), 256, 0, st>>>(x, P, Hs, Ws, ih, iw, oh, ow, out);
  prof_end(st);
  LAUNCH_CHECK("ais resize");
  return 0;
}

int64_t msam_ais_postprocess_workspace(int H, int W) {
  if (H <= 0 || W <= 0 || (long)H * W >= (1l << 30)) return -1;
  return (int64_t)post_ws(H, W, nullptr, nullptr);
}

int msam_ais_postprocess(const float* fg, const float* cd, const float* bd, int H, int W, const double* taps_fg, int r_fg,
                         const double* taps_d, int r_d, float t_fg, float t_cd, float t_bd, int min_size, void* ws,
                         int64_t ws_bytes, int32_t* labels, int* n_ids, int* sweeps, void* stream) {
  if (!fg || !cd || !bd || !ws || !labels || !n_ids || !sweeps) return set_error("msam_ais_postprocess: null argument");
  const int64_t need = msam_ais_postprocess_workspace(H, W);
  if (need < 0) return set_error("msam_ais_postprocess: image %d x %d", H, W);
  if (ws_bytes < need) return set_error("msam_ais_postprocess: workspace of %lld bytes, %lld needed", (long long)ws_bytes, (long long)need);
  if ((uintptr_t)ws & 255) return set_error("msam_ais_postprocess: workspace not 256-byte aligned");
  if (min_size < 0) return set_error("msam_ais_postprocess: min_size %d", min_size);
  cudaStream_t st = (cudaStream_t)stream;
  PostWs w;
  post_ws(H, W, (char*)ws, &w);
  w.lab = labels;   // the labels are computed in place
  RUN(gaussian_taps(taps_fg, r_fg, w.taps, st));
  RUN(gaussian_taps(taps_d, r_d, w.taps + MAX_TAPS, st));
  const int n = H * W;
  prof_begin(st, "ais smoothing", 0.0, 24.0 * n);
  RUN(smooth(fg, H, W, w.taps, r_fg, w.tmp, w.fg, st));
  RUN(smooth(cd, H, W, w.taps + MAX_TAPS, r_d, w.tmp, w.cd, st));
  RUN(smooth(bd, H, W, w.taps + MAX_TAPS, r_d, w.tmp, w.bd, st));
  prof_end(st);
  prof_begin(st, "ais markers", 0.0, 0.0);
  ais_masks_kernel<<<nblk(n), 256, 0, st>>>(w.fg, w.cd, w.bd, n, t_fg, t_cd, t_bd, w.fmask, w.flag);
  LAUNCH_CHECK("ais masks");
  // 8-connected marker components (roots in raster order); the sizes go to cnt and the unread background count to dflag,
  // both rewritten before their own use below, and flag changes from the marker image to the root flags
  RUN(post_label_components(w.flag, H, W, w.parent, w.cnt, w.dflag, st, H, 1));
  RUN(post_flag_components(n, w.parent, w.cnt, 0, w.flag, st));
  RUN(post_inclusive_scan(w.flag, n, w.scan, w.bsums, st));
  ais_ws_init_kernel<<<nblk(n), 256, 0, st>>>(w.parent, w.fmask, w.bd, w.scan, w.bsums, n, w.Bv, w.lab);
  LAUNCH_CHECK("ais watershed init");
  prof_end(st);
  int ids = 0;
  if (cudaMemcpyAsync(&ids, w.scan + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess) return set_error("copy failed");
  int boff = 0;
  if (cudaMemcpyAsync(&boff, w.bsums + ((n - 1) >> 10), sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess)
    return set_error("copy failed");
  if (cudaStreamSynchronize(st) != cudaSuccess) return set_error("msam_ais_postprocess: %s", cudaGetErrorString(cudaGetLastError()));
  ids += boff;
  const dim3 tg((W + WS_T - 1) / WS_T, (H + WS_T - 1) / WS_T);
  const int max_sweeps = n + 2;   // every sweep that changes something settles at least one more pixel for good
  int nsw = 0;
  for (int pass = 0; pass < 2; ++pass) {
    prof_begin(st, pass == 0 ? "ais watershed barrier" : "ais watershed label", 0.0, 0.0);
    for (int it = 0;; ++it) {
      if (it > max_sweeps) return set_error("msam_ais_postprocess: the watershed did not converge in %d sweeps", max_sweeps);
      int f = 0;
      if (cudaMemsetAsync(w.dflag, 0, sizeof(int), st) != cudaSuccess) return set_error("memset failed");
      if (pass == 0)
        ais_ws_barrier_kernel<<<tg, 256, 0, st>>>(w.bd, w.fmask, w.parent, H, W, w.Bv, w.dflag);
      else
        ais_ws_label_kernel<<<tg, 256, 0, st>>>(w.Bv, w.fmask, w.parent, H, W, w.lab, w.dflag);
      LAUNCH_CHECK("ais watershed sweep");
      ++nsw;
      if (cudaMemcpyAsync(&f, w.dflag, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
          cudaStreamSynchronize(st) != cudaSuccess)
        return set_error("msam_ais_postprocess: %s", cudaGetErrorString(cudaGetLastError()));
      if (!f) break;
    }
    prof_end(st);
  }
  prof_begin(st, "ais size filter", 0.0, 0.0);
  const int filter = min_size > 0 && ids > 0;
  if (filter) {
    if (cudaMemsetAsync(w.cnt, 0, sizeof(int) * (ids + 1), st) != cudaSuccess) return set_error("msam_ais_postprocess: memset failed");
    ais_count_kernel<<<nblk(n), 256, 0, st>>>(w.lab, n, w.cnt);
    LAUNCH_CHECK("ais count");
    ais_keep_kernel<<<nblk(ids + 1), 256, 0, st>>>(w.cnt, ids, min_size, w.keep);
    LAUNCH_CHECK("ais keep");
    RUN(post_inclusive_scan(w.keep, ids + 1, w.scan2, w.bsums2, st));
  }
  ais_final_kernel<<<nblk(n), 256, 0, st>>>(w.lab, n, w.keep, w.scan2, w.bsums2, filter);
  LAUNCH_CHECK("ais final labels");
  prof_end(st);
  if (filter) {
    int a = 0, c = 0;
    if (cudaMemcpyAsync(&a, w.scan2 + ids, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(&c, w.bsums2 + (ids >> 10), sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
      return set_error("msam_ais_postprocess: %s", cudaGetErrorString(cudaGetLastError()));
    ids = a + c;
  }
  *n_ids = ids;
  *sweeps = nsw;
  return 0;
}

int msam_ais_props(const int32_t* labels, int H, int W, int n_ids, int32_t* props, void* stream) {
  if (!labels || !props) return set_error("msam_ais_props: null argument");
  if (H <= 0 || W <= 0 || n_ids < 0 || (long)H * W >= (1l << 31)) return set_error("msam_ais_props: H=%d, W=%d, n_ids=%d", H, W, n_ids);
  if (n_ids == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  ais_props_init_kernel<<<nblk(n_ids), 256, 0, st>>>(props, n_ids);
  LAUNCH_CHECK("ais props init");
  ais_props_kernel<<<nblk((long)H * W), 256, 0, st>>>(labels, H, W, props);
  LAUNCH_CHECK("ais props");
  return 0;
}

}  // extern "C"
