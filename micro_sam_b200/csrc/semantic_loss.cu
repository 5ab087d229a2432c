// Loss of micro-sam's semantic fine-tuning (micro_sam/training/semantic_sam_trainer.py:11-86: CustomDiceLoss + CrossEntropyLoss on
// the full-resolution multi-class logits) and its adjoint, straight from the low-res logits [B, C, 256, 256].
//
// Per pixel (b, y, x) of the original_size grid the C logits z_c = Sam.postprocess_masks(low_res)[b, c, y, x] are evaluated with the
// interpolation code of postgeom.cuh (the two stages' taps computed once per pixel, shared by the C channels) and never written.
// With p = softmax(z) and the label l = labels[b, y, x]:
//   stats[3c + 0] = sum p_c [l == c]      stats[3c + 1] = sum p_c^2      stats[3c + 2] = sum [l == c]
//   stats[3C + 0] = sum over l in [0, C) of -log p_l = logsumexp(z) - z_l       stats[3C + 1] = |{l in [0, C)}|
//   stats[3C + 2] = |{l outside [0, C), l != -100}|
// over the whole batch.  Label -100 (nn.CrossEntropyLoss's ignore_index) is in no class and out of the cross entropy; any other
// label outside [0, C) is counted in stats[3C + 2] (the host refuses the loss then, as torch refuses such a target).
//
// Stats: one grid-stride pass, per-thread fp64 sums (counts in int), a fixed-order warp / CTA reduction into one partial row
// per CTA, then one CTA sums the rows in order.  No float atomics: repeats are bit-identical.
//
// Backward, w.r.t. the sums (d_stats in the layout of stats; only the entries 3c, 3c + 1 and 3C are read):
//   g_k  = dL/d(sum p_k t_k) t_k + 2 dL/d(sum p_k^2) p_k
//   dz_k = p_k (g_k - sum_j p_j g_j) + dL/d(ce sum) (p_k - [k == l])        (second term only for l in [0, C))
// written per pixel, then the transpose of the two bilinear stages as four separable gathers (original -> input_size along x,
// then y; the crop of the 1024 grid -> 256 along x, then y).  Every output element of a gather sums its taps in ascending
// source order, so d_low_res is written (not accumulated), deterministically, and is zero where no pixel reads the logit.
#include <algorithm>
#include <climits>
#include <cmath>

#include "../../include/msam_b200.h"
#include "kernels.h"
#include "postgeom.cuh"

namespace msam {
namespace {

constexpr int SL_THREADS = 256;
constexpr int SL_MAX_GRID = 1056;   // 8 CTAs per SM of an H100 SXM; fixed, so the partial rows do not depend on the device
constexpr int SL_MAX_C = 15;
constexpr int SL_IGNORE = -100;

// The taps of one original_size pixel: the 2 x 2 stage-1 positions of the second interpolation (one position when it is the
// identity) and, per position, the 2 x 2 low-res taps.  Values equal full_res() term by term.
struct PixTaps {
  Interp y2, x2;            // second stage (unused when identity2)
  Interp y1[2], x1[2];      // first stage at the rows y2.i0 / y2.i1 and columns x2.i0 / x2.i1
};
__device__ __forceinline__ void pix_taps(const PostGeom& g, int y, int x, PixTaps& t) {
  if (g.identity2) {
    t.y1[0] = interp_axis(y, g.s1, g.lr);
    t.x1[0] = interp_axis(x, g.s1, g.lr);
    return;
  }
  t.y2 = interp_axis(y, g.s2y, g.in_h);
  t.x2 = interp_axis(x, g.s2x, g.in_w);
  t.y1[0] = interp_axis(t.y2.i0, g.s1, g.lr); t.y1[1] = interp_axis(t.y2.i1, g.s1, g.lr);
  t.x1[0] = interp_axis(t.x2.i0, g.s1, g.lr); t.x1[1] = interp_axis(t.x2.i1, g.s1, g.lr);
}
__device__ __forceinline__ float stage1_taps(const float* __restrict__ lr, const Interp& iy, const Interp& ix) {
  const float* r0 = lr + iy.i0 * 256;
  const float* r1 = lr + iy.i1 * 256;
  return bilerp(__ldg(r0 + ix.i0), __ldg(r0 + ix.i1), __ldg(r1 + ix.i0), __ldg(r1 + ix.i1), iy, ix);
}
__device__ __forceinline__ float logit_at(const float* __restrict__ lr, const PostGeom& g, const PixTaps& t) {
  if (g.identity2) return stage1_taps(lr, t.y1[0], t.x1[0]);
  return bilerp(stage1_taps(lr, t.y1[0], t.x1[0]), stage1_taps(lr, t.y1[0], t.x1[1]), stage1_taps(lr, t.y1[1], t.x1[0]),
                stage1_taps(lr, t.y1[1], t.x1[1]), t.y2, t.x2);
}

__device__ __forceinline__ int load_label(const void* labels, int label64, long q) {
  if (label64) {
    const long long v = static_cast<const long long*>(labels)[q];
    return (v < INT_MIN || v > INT_MAX) ? INT_MIN : (int)v;   // INT_MIN: out of range, and not the ignore index
  }
  return static_cast<const int*>(labels)[q];
}

// z -> p = softmax(z) in place; returns logsumexp(z)
template <int NC>
__device__ __forceinline__ float softmax_inplace(float (&z)[NC]) {
  float m = z[0];
#pragma unroll
  for (int c = 1; c < NC; ++c) m = fmaxf(m, z[c]);
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) { z[c] = expf(z[c] - m); s += z[c]; }
  const float inv = 1.f / s;
#pragma unroll
  for (int c = 0; c < NC; ++c) z[c] *= inv;
  return m + logf(s);
}

template <int NC>
__device__ __forceinline__ void pixel_logits(const float* __restrict__ low_res, const PostGeom& g, int b, int y, int x, float (&z)[NC]) {
  PixTaps t;
  pix_taps(g, y, x, t);
  const float* lr = low_res + (size_t)b * NC * 65536;
#pragma unroll
  for (int c = 0; c < NC; ++c) z[c] = logit_at(lr + (size_t)c * 65536, g, t);
}

template <int NC>
__global__ void __launch_bounds__(SL_THREADS) sl_stats_kernel(const float* __restrict__ low_res, const void* __restrict__ labels,
                                                              int label64, PostGeom g, long npix, double* __restrict__ part) {
  constexpr int K = 3 * NC + 3;
  double pt[NC], pp[NC], ce = 0.0;
  int nt[NC], nce = 0, nbad = 0;
#pragma unroll
  for (int c = 0; c < NC; ++c) { pt[c] = 0.0; pp[c] = 0.0; nt[c] = 0; }
  const long hw = (long)g.out_h * g.out_w;
  for (long q = (long)blockIdx.x * SL_THREADS + threadIdx.x; q < npix; q += (long)gridDim.x * SL_THREADS) {
    const int b = (int)(q / hw);
    const long r = q - (long)b * hw;
    const int y = (int)(r / g.out_w), x = (int)(r - (long)y * g.out_w);
    float z[NC];
    pixel_logits<NC>(low_res, g, b, y, x, z);
    const int l = load_label(labels, label64, q);
    float zl = 0.f;
#pragma unroll
    for (int c = 0; c < NC; ++c) zl = (c == l) ? z[c] : zl;
    const float lse = softmax_inplace<NC>(z);
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const double p = (double)z[c];
      pp[c] += p * p;
      if (c == l) { pt[c] += p; nt[c] += 1; }
    }
    if (l >= 0 && l < NC) { ce += (double)(lse - zl); nce += 1; }
    else if (l != SL_IGNORE) nbad += 1;
  }
  // fixed-order reduction: warp butterfly, then the 8 warps in order
  __shared__ double red[SL_THREADS / 32][K];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    double a = pt[c], bb = pp[c];
    int n = nt[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o); bb += __shfl_xor_sync(0xffffffffu, bb, o); n += __shfl_xor_sync(0xffffffffu, n, o);
    }
    if (lane == 0) { red[w][3 * c] = a; red[w][3 * c + 1] = bb; red[w][3 * c + 2] = (double)n; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ce += __shfl_xor_sync(0xffffffffu, ce, o); nce += __shfl_xor_sync(0xffffffffu, nce, o); nbad += __shfl_xor_sync(0xffffffffu, nbad, o);
  }
  if (lane == 0) { red[w][3 * NC] = ce; red[w][3 * NC + 1] = (double)nce; red[w][3 * NC + 2] = (double)nbad; }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < SL_THREADS / 32; ++i) s += red[i][threadIdx.x];
    part[(size_t)blockIdx.x * K + threadIdx.x] = s;
  }
}

__global__ void sl_finalize_kernel(const double* __restrict__ part, int n, int K, double* __restrict__ stats) {
  const int j = threadIdx.x;
  if (j >= K) return;
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += part[(size_t)i * K + j];
  stats[j] = s;
}

template <int NC>
__global__ void __launch_bounds__(SL_THREADS) sl_dz_kernel(const float* __restrict__ low_res, const void* __restrict__ labels,
                                                           int label64, PostGeom g, long npix, const double* __restrict__ d_stats,
                                                           float* __restrict__ dz) {
  const long q = (long)blockIdx.x * SL_THREADS + threadIdx.x;
  if (q >= npix) return;
  const long hw = (long)g.out_h * g.out_w;
  const int b = (int)(q / hw);
  const long r = q - (long)b * hw;
  const int y = (int)(r / g.out_w), x = (int)(r - (long)y * g.out_w);
  float p[NC];
  pixel_logits<NC>(low_res, g, b, y, x, p);
  softmax_inplace<NC>(p);
  const int l = load_label(labels, label64, q);
  float gk[NC], sg = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    gk[c] = 2.f * (float)d_stats[3 * c + 1] * p[c] + ((c == l) ? (float)d_stats[3 * c] : 0.f);
    sg = fmaf(p[c], gk[c], sg);
  }
  const float dce = (l >= 0 && l < NC) ? (float)d_stats[3 * NC] : 0.f;
  float* out = dz + (size_t)b * NC * hw + r;
#pragma unroll
  for (int c = 0; c < NC; ++c) out[(size_t)c * hw] = p[c] * (gk[c] - sg) + dce * (p[c] - ((c == l) ? 1.f : 0.f));
}

// Adjoint of interp_axis along one axis: in [n_outer, n_dst, inner] -> out [n_outer, n_src, inner],
//   out[o, i, r] = sum over d in [0, n_dst) of (weight of source i in interp_axis(d, scale, n_src)) * in[o, d, r].
// A source i is read by the d whose first tap i0 is i - 1 or i, i.e. whose unclamped source coordinate lies in [i - 1, i + 1);
// the window below holds those d with a margin of 2 (every candidate's weight is recomputed exactly, so the margin only costs
// zero terms), and reaches the ends where interp_axis clamps.
__global__ void __launch_bounds__(256) sl_axis_adjoint_kernel(const float* __restrict__ in, long n_outer, int n_dst, int inner,
                                                              int n_src, float scale, float* __restrict__ out) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_outer * n_src * inner) return;
  const int rr = (int)(idx % inner);
  const long oi = idx / inner;
  const int i = (int)(oi % n_src);
  const long o = oi / n_src;
  const double inv = 1.0 / (double)scale;
  int lo = (int)floor(((double)i - 0.5) * inv - 0.5) - 2;
  int hi = (int)ceil(((double)i + 1.5) * inv - 0.5) + 2;
  if (lo < 0) lo = 0;
  if (hi > n_dst - 1 || i == n_src - 1) hi = n_dst - 1;
  const float* src = in + (size_t)o * n_dst * inner + rr;
  float acc = 0.f;
  for (int d = lo; d <= hi; ++d) {
    const Interp t = interp_axis(d, scale, n_src);
    const float w = (t.i0 == i ? t.l0 : 0.f) + (t.i1 == i ? t.l1 : 0.f);
    if (w != 0.f) acc = fmaf(w, __ldg(src + (size_t)d * inner), acc);
  }
  out[idx] = acc;
}

int sl_gather(const float* in, long n_outer, int n_dst, int inner, int n_src, float scale, float* out, cudaStream_t st) {
  sl_axis_adjoint_kernel<<<nblk(n_outer * n_src * inner), 256, 0, st>>>(in, n_outer, n_dst, inner, n_src, scale, out);
  LAUNCH_CHECK("semantic loss backward (bilinear adjoint)");
  return 0;
}

long sl_grid(long npix) { return std::min<long>((npix + SL_THREADS - 1) / SL_THREADS, SL_MAX_GRID); }

int sl_check(const char* fn, const float* low_res, const void* labels, int label_dtype, int B, int C, int in_h, int in_w, int H, int W,
             const void* p3, const void* ws, int64_t ws_bytes, int backward, PostGeom* g) {
  if (!low_res || !labels || !p3 || !ws) return set_error("%s: null argument", fn);
  if (C < 1 || C > SL_MAX_C) return set_error("%s: C=%d classes (1..%d are supported)", fn, C, SL_MAX_C);
  if (label_dtype != 0 && label_dtype != 1) return set_error("%s: label_dtype %d (0 int32, 1 int64)", fn, label_dtype);
  if (B <= 0 || (long)H * W >= (1l << 31) || (long)B * C * H * W >= (1l << 40))
    return set_error("%s: B=%d, C=%d, original %dx%d", fn, B, C, H, W);
  if (make_geom(in_h, in_w, H, W, g)) return -1;
  if (((uintptr_t)ws & 255) || ws_bytes < msam_semantic_loss_workspace(B, C, in_h, in_w, H, W, backward))
    return set_error("%s: workspace too small or not 256-byte aligned", fn);
  return 0;
}

template <int NC>
void launch_stats(const float* lr, const void* labels, int label64, const PostGeom& g, long npix, double* part, cudaStream_t st) {
  sl_stats_kernel<NC><<<(unsigned)sl_grid(npix), SL_THREADS, 0, st>>>(lr, labels, label64, g, npix, part);
}
template <int NC>
void launch_dz(const float* lr, const void* labels, int label64, const PostGeom& g, long npix, const double* ds, float* dz,
               cudaStream_t st) {
  sl_dz_kernel<NC><<<nblk(npix, SL_THREADS), SL_THREADS, 0, st>>>(lr, labels, label64, g, npix, ds, dz);
}

#define SL_DISPATCH(C, FN, ...)                                                                                  \
  switch (C) {                                                                                                   \
    case 1: FN<1>(__VA_ARGS__); break;   case 2: FN<2>(__VA_ARGS__); break;   case 3: FN<3>(__VA_ARGS__); break;    \
    case 4: FN<4>(__VA_ARGS__); break;   case 5: FN<5>(__VA_ARGS__); break;   case 6: FN<6>(__VA_ARGS__); break;    \
    case 7: FN<7>(__VA_ARGS__); break;   case 8: FN<8>(__VA_ARGS__); break;   case 9: FN<9>(__VA_ARGS__); break;    \
    case 10: FN<10>(__VA_ARGS__); break; case 11: FN<11>(__VA_ARGS__); break; case 12: FN<12>(__VA_ARGS__); break;  \
    case 13: FN<13>(__VA_ARGS__); break; case 14: FN<14>(__VA_ARGS__); break; default: FN<15>(__VA_ARGS__); break;  \
  }

}  // namespace
}  // namespace msam

using namespace msam;

extern "C" {

int64_t msam_semantic_loss_workspace(int B, int C, int in_h, int in_w, int H, int W, int backward) {
  if (B <= 0 || C < 1 || C > SL_MAX_C || in_h <= 0 || in_w <= 0 || H <= 0 || W <= 0) return -1;
  const long npix = (long)B * H * W;
  size_t bytes = up256((size_t)sl_grid(npix) * (3 * C + 3) * 8);
  if (backward) {
    const size_t bc = (size_t)B * C;
    bytes += up256(bc * std::max((size_t)H * W, (size_t)in_h * in_w) * 4);
    bytes += up256(bc * std::max((size_t)H * in_w, (size_t)in_h * 256) * 4);
  }
  return (int64_t)bytes;
}

int msam_semantic_loss_stats(const float* low_res, const void* labels, int label_dtype, int B, int C, int in_h, int in_w, int H, int W,
                             void* ws, int64_t ws_bytes, double* stats, void* stream) {
  PostGeom g;
  if (sl_check("msam_semantic_loss_stats", low_res, labels, label_dtype, B, C, in_h, in_w, H, W, stats, ws, ws_bytes, 0, &g)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const long npix = (long)B * H * W;
  double* part = (double*)ws;
  prof_begin(st, "semantic_loss_stats", 0.0, (double)B * C * 65536.0 * 4 + (double)npix * (label_dtype ? 8 : 4));
  SL_DISPATCH(C, launch_stats, low_res, labels, label_dtype, g, npix, part, st);
  if (launch_check("semantic loss statistics (partials)")) { prof_end(st); return -1; }
  sl_finalize_kernel<<<1, 64, 0, st>>>(part, (int)sl_grid(npix), 3 * C + 3, stats);
  prof_end(st);
  LAUNCH_CHECK("semantic loss statistics");
  return 0;
}

int msam_semantic_loss_backward(const float* low_res, const void* labels, int label_dtype, const double* d_stats, int B, int C, int in_h,
                                int in_w, int H, int W, void* ws, int64_t ws_bytes, float* d_low_res, void* stream) {
  PostGeom g;
  if (sl_check("msam_semantic_loss_backward", low_res, labels, label_dtype, B, C, in_h, in_w, H, W, d_stats, ws, ws_bytes, 1, &g))
    return -1;
  if (!d_low_res) return set_error("msam_semantic_loss_backward: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const long npix = (long)B * H * W, bc = (long)B * C;
  char* base = (char*)ws + up256((size_t)sl_grid(npix) * (3 * C + 3) * 8);
  float* bufA = (float*)base;
  float* bufB = (float*)(base + up256((size_t)bc * std::max((size_t)H * W, (size_t)in_h * in_w) * 4));
  prof_begin(st, "semantic_loss_backward", 0.0,
             (double)bc * 65536.0 * 8 + (double)npix * (label_dtype ? 8 : 4) + 8.0 * bc * ((double)H * W + (double)in_h * 256) +
                 (g.identity2 ? 0.0 : 8.0 * bc * ((double)H * in_w + (double)in_h * in_w)));
  SL_DISPATCH(C, launch_dz, low_res, labels, label_dtype, g, npix, d_stats, bufA, st);
  if (launch_check("semantic loss backward (per-pixel adjoint)")) { prof_end(st); return -1; }
  const float* s1in = bufA;   // d loss / d (cropped 1024 grid) [bc, in_h, in_w]
  int rc = 0;
  if (!g.identity2) {
    rc = sl_gather(bufA, bc * H, W, 1, in_w, g.s2x, bufB, st);              // x: original -> input_size
    if (!rc) rc = sl_gather(bufB, bc, H, in_w, in_h, g.s2y, bufA, st);      // y
  }
  if (!rc) rc = sl_gather(s1in, bc * in_h, in_w, 1, 256, g.s1, bufB, st);   // x: cropped 1024 grid -> 256
  if (!rc) rc = sl_gather(bufB, bc, in_h, 256, 256, g.s1, d_low_res, st);   // y
  prof_end(st);
  return rc;
}

}  // extern "C"
