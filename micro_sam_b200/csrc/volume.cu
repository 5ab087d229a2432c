// Mask -> prompt derivation of segment_from_mask on the device (micro_sam/prompt_based_segmentation.py:28-140), used by
// multi_dimensional_segmentation.segment_mask_in_volume to carry an object from one slice to the next without a host round
// trip of the mask:
//   stats     : pixel count, bounding box and coordinate sums of a uint8 0/1 mask (one pass, integer atomics)
//   finish    : _process_box (box_extension, clipping, np.round = half-to-even) and ResizeLongestSide(1024).apply_boxes
//   logits    : _compute_logits_from_mask -- torch's CPU antialiased bilinear resize to the longest side 256, reproduced
//               operation by operation (weights in fp32 from the triangle filter, horizontal pass first, then the vertical
//               pass with the accumulation torch's AVX512 build performs), zero padding, +-log((1-eps)/eps) at > 0.5
//   points    : _compute_points_from_mask on the extended box crop -- outer boundary, exact EDT (integer squared distances,
//               sqrt in fp64), scipy's gaussian_filter(sigma=1) (reflect, radius 4, fp64 sums, fp32 after each axis), then
//               the first argmax of the inner field or _peak_local_max(inner, 3) + _peak_local_max(outer, 5)
//   iou       : util.compute_iou's intersection and union counts
//   shift     : scipy.ndimage.shift(order=0) of a mask by the tracking annotator's motion model (track_from_prompts)
// Every floating-point operation whose rounding matters is written with an explicit-rounding intrinsic, so nvcc's FMA
// contraction cannot change a result.
#include <algorithm>
#include <climits>
#include <cmath>
#include <utility>

#include "device_util.cuh"
#include "engine.h"

namespace msam {
namespace {

constexpr int kMaxSide = 8192;       // longest mask side
constexpr int kMaxTaps = 72;         // resize taps per output pixel (2 * ceil(in / out) + 1); shapes that need more are refused
constexpr int kMaxCand = 8192;       // peak candidates per field (sorted in shared memory)
constexpr int kStats = 12;           // int64 stats: count, sum_y, sum_x, y0, x0, y1, x1 (mask box), bx0, by0, bx1, by1, n_points

// scipy.ndimage._filters._gaussian_kernel1d(1.0, 0, 4): the centre weight and the weights at distance 1..4
__constant__ double kGauss[5] = {0x1.9884a307594fbp-2, 0x1.ef8eb9ad499bap-3, 0x1.ba4b99d1799abp-5, 0x1.22724cb7eb269p-8,
                                 0x1.18a9c4fd536c6p-13};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// workspace layout (bytes), see mask_prompts_workspace
struct Ws {
  int32_t* g;          // column distances [ch * cw]
  float *f0, *f1, *f2; // EDT, after the axis-0 pass, smoothed field
  float* rmax;         // row maxima of the peak filter
  float* tmp;          // horizontal resize pass [H * 256]
  unsigned long long* cand;   // [2][kMaxCand] candidate keys
  int32_t* ctr;        // [0] boundary pixels, [1..2] candidates (inner, outer), [3..4] kept, [5] overflow, [6] field min bits x2
  int32_t* kept;       // [2][kMaxCand] kept pixel indices
};
Ws carve(void* base, int H, int W) {
  char* p = (char*)base;
  const size_t f = align256((size_t)4 * H * W);
  Ws w;
  w.g = (int32_t*)p; p += f;
  w.f0 = (float*)p; p += f;
  w.f1 = (float*)p; p += f;
  w.f2 = (float*)p; p += f;
  w.rmax = (float*)p; p += f;
  w.tmp = (float*)p; p += align256((size_t)4 * H * 256);
  w.cand = (unsigned long long*)p; p += 8 * 2 * kMaxCand;
  w.kept = (int32_t*)p; p += 4 * 2 * kMaxCand;
  w.ctr = (int32_t*)p;
  return w;
}

__global__ void stats_init_kernel(int64_t* st, int32_t* ctr) {
  const int t = threadIdx.x;
  if (t < kStats) st[t] = (t == 3 || t == 4) ? LLONG_MAX : (t == 5 || t == 6) ? -1 : 0;
  if (ctr && t < 16) ctr[t] = t == 6 || t == 7 ? 0x7f800000 : 0;   // +inf bits for the field minima
}

__global__ void stats_kernel(const uint8_t* __restrict__ m, int H, int W, int ld, int64_t* st) {
  long long cnt = 0, sy = 0, sx = 0, y0 = LLONG_MAX, x0 = LLONG_MAX, y1 = -1, x1 = -1;
  const long total = (long)H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i % W);
    if (m[(long)y * ld + x] == 1) {
      ++cnt; sy += y; sx += x;
      y0 = min(y0, (long long)y); x0 = min(x0, (long long)x); y1 = max(y1, (long long)y); x1 = max(x1, (long long)x);
    }
  }
  for (int o = 16; o; o >>= 1) {
    cnt += __shfl_down_sync(0xffffffffu, cnt, o); sy += __shfl_down_sync(0xffffffffu, sy, o); sx += __shfl_down_sync(0xffffffffu, sx, o);
    y0 = min(y0, __shfl_down_sync(0xffffffffu, y0, o)); x0 = min(x0, __shfl_down_sync(0xffffffffu, x0, o));
    y1 = max(y1, __shfl_down_sync(0xffffffffu, y1, o)); x1 = max(x1, __shfl_down_sync(0xffffffffu, x1, o));
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicAdd((unsigned long long*)&st[0], (unsigned long long)cnt);
    atomicAdd((unsigned long long*)&st[1], (unsigned long long)sy);
    atomicAdd((unsigned long long*)&st[2], (unsigned long long)sx);
    atomicMin((long long*)&st[3], y0); atomicMin((long long*)&st[4], x0);
    atomicMax((long long*)&st[5], y1); atomicMax((long long*)&st[6], x1);
  }
}

// get_preprocess_shape in fp64 without contraction
__device__ __forceinline__ void preprocess_shape(int h, int w, int long_side, int* nh, int* nw) {
  const double scale = __ddiv_rn((double)long_side, (double)max(h, w));
  *nh = (int)__dadd_rn(__dmul_rn((double)h, scale), 0.5);
  *nw = (int)__dadd_rn(__dmul_rn((double)w, scale), 0.5);
}

// _process_box + apply_boxes: st[3..6] = (y0, x0, ymax, xmax) -> python box (y0, x0, y1 = ymax + 1, x1 = xmax + 1)
__global__ void finish_kernel(int H, int W, double ext, int64_t* st, float* box1024) {
  if (st[0] == 0) {
    st[3] = st[4] = st[5] = st[6] = st[7] = st[8] = st[9] = st[10] = 0;
    if (box1024) box1024[0] = box1024[1] = box1024[2] = box1024[3] = 0.f;
    return;
  }
  const long long y0 = st[3], x0 = st[4], y1 = st[5] + 1, x1 = st[6] + 1;
  st[5] = y1; st[6] = x1;
  double ey = 0.0, ex = 0.0;
  if (ext >= 1.0) { ey = ex = ext; }
  else if (ext != 0.0) { ey = __dmul_rn(ext, (double)(y1 - y0)); ex = __dmul_rn(ext, (double)(x1 - x0)); }
  const double b[4] = {fmax(__dsub_rn((double)x0, ex), 0.0), fmax(__dsub_rn((double)y0, ey), 0.0),
                       fmin(__dadd_rn((double)x1, ex), (double)W), fmin(__dadd_rn((double)y1, ey), (double)H)};
  int nh, nw;
  preprocess_shape(H, W, 1024, &nh, &nw);
  const double sx = __ddiv_rn((double)nw, (double)W), sy = __ddiv_rn((double)nh, (double)H);
  for (int k = 0; k < 4; ++k) {
    const double r = rint(b[k]);   // np.round: half to even
    st[7 + k] = (long long)r;
    if (box1024) box1024[k] = __double2float_rn(__dmul_rn(r, (k & 1) ? sy : sx));
  }
}

// torch's antialiased triangle-filter weights of output index i for a resize in -> out (UpSampleKernel.cpp,
// _compute_indices_min_size_weights_aa, all in fp32 with the fp64 promotions of the C++ expressions)
__device__ int aa_weights(int in, int out, int i, float* w, int* xmin_out) {
  const float scale = __fdiv_rn((float)in, (float)out);
  const float support = scale >= 1.f ? scale : 1.f;
  const int maxsz = (int)ceilf(support) * 2 + 1;
  const float invscale = scale >= 1.f ? __double2float_rn(__ddiv_rn(1.0, (double)scale)) : 1.f;
  const float center = __double2float_rn(__dmul_rn((double)scale, (double)i + 0.5));
  const long long xmin = max((long long)__dadd_rn((double)__fsub_rn(center, support), 0.5), 0LL);
  long long xsize = min((long long)__dadd_rn((double)__fadd_rn(center, support), 0.5), (long long)in) - xmin;
  xsize = max(0LL, min(xsize, (long long)maxsz));   // maxsz <= kMaxTaps, checked on the host
  float tot = 0.f;
  for (int j = 0; j < xsize; ++j) {
    float x = __double2float_rn(__dmul_rn(__dadd_rn((double)__fsub_rn((float)(j + xmin), center), 0.5), (double)invscale));
    x = fabsf(x);
    const float v = x < 1.f ? __double2float_rn(__dsub_rn(1.0, (double)x)) : 0.f;
    w[j] = v;
    tot = __fadd_rn(tot, v);
  }
  if (tot != 0.f)
    for (int j = 0; j < xsize; ++j) w[j] = __fdiv_rn(w[j], tot);
  *xmin_out = (int)xmin;
  return (int)xsize;
}

// horizontal pass on the 0/1 mask: tmp[y, ox] (products are exact, the sum runs in index order)
__global__ void resize_h_kernel(const uint8_t* __restrict__ m, int H, int W, int ld, int tw, float* tmp) {
  const long total = (long)H * tw;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / tw), ox = (int)(i % tw);
    float w[kMaxTaps];
    int x0;
    const int n = aa_weights(W, tw, ox, w, &x0);
    const uint8_t* row = m + (long)y * ld + x0;
    float acc = __fmul_rn(row[0] == 1 ? 1.f : 0.f, w[0]);
    for (int j = 1; j < n; ++j) acc = __fadd_rn(acc, row[j] == 1 ? w[j] : 0.f);
    tmp[i] = acc;
  }
}

// vertical pass + threshold + padding -> logits [256, 256].  src is the horizontal pass (th_src rows of pitch tw) or, when
// the width is unchanged, the mask itself.  torch's vertical loop adds the products of taps 1 .. 4q unfused and contracts
// the remaining (n - 1) % 4 into FMAs (measured against torch's CPU kernel; see tests/test_volume_cpu.py).
__global__ void logits_kernel(const uint8_t* __restrict__ m, int ld, const float* __restrict__ tmp, int H, int W, int th, int tw,
                              float hi, float* logits) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 65536; i += gridDim.x * blockDim.x) {
    const int oy = i >> 8, ox = i & 255;
    float v = 0.f;
    if (oy < th && ox < tw) {
      auto src = [&](int y) -> float { return tmp ? tmp[(long)y * tw + ox] : (m[(long)y * ld + ox] == 1 ? 1.f : 0.f); };
      if (th == H) {
        v = src(oy);
      } else {
        float w[kMaxTaps];
        int y0;
        const int n = aa_weights(H, th, oy, w, &y0);
        const int unfused = ((n - 1) / 4) * 4;
        v = __fmul_rn(src(y0), w[0]);
        for (int j = 1; j < n; ++j)
          v = (j - 1 < unfused) ? __fadd_rn(v, __fmul_rn(src(y0 + j), w[j])) : __fmaf_rn(src(y0 + j), w[j], v);
      }
    }
    logits[i] = v > 0.5f ? hi : -hi;
  }
}

// crop of the extended box: st[7..10] = (bx0, by0, bx1, by1)
struct Crop { int y0, x0, h, w; };
__device__ __forceinline__ Crop crop_of(const int64_t* st) {
  return Crop{(int)st[8], (int)st[7], (int)(st[10] - st[8]), (int)(st[9] - st[7])};
}
__device__ __forceinline__ bool in_mask(const uint8_t* m, int ld, const Crop& c, int y, int x) {
  return y >= 0 && x >= 0 && y < c.h && x < c.w && m[(long)(c.y0 + y) * ld + c.x0 + x] != 0;   // crop.astype(bool)
}

// outer boundary (binary_dilation(crop) & ~crop, border 0) and the 1-D distance along each column to the nearest boundary
// pixel (INT_MAX / 2 = none)
__global__ void edt_cols_kernel(const uint8_t* __restrict__ m, int ld, const int64_t* st, int32_t* g, int32_t* ctr) {
  if (st[0] == 0) return;
  const Crop c = crop_of(st);
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= c.w) return;
  auto bnd = [&](int y) {
    return !in_mask(m, ld, c, y, x) && (in_mask(m, ld, c, y - 1, x) || in_mask(m, ld, c, y + 1, x) || in_mask(m, ld, c, y, x - 1) ||
                                        in_mask(m, ld, c, y, x + 1));
  };
  int d = INT_MAX / 2, nb = 0;
  for (int y = 0; y < c.h; ++y) {
    if (bnd(y)) { d = 0; ++nb; } else if (d < INT_MAX / 2) ++d;
    g[(long)y * c.w + x] = d;
  }
  d = INT_MAX / 2;
  for (int y = c.h - 1; y >= 0; --y) {
    const int cur = g[(long)y * c.w + x];
    if (cur == 0) d = 0; else if (d < INT_MAX / 2) ++d;
    if (d < cur) g[(long)y * c.w + x] = d;
  }
  if (nb) atomicAdd(&ctr[0], nb);
}

// exact squared distance along each row, min over x' of g(x')^2 + (x - x')^2, by Meijster's linear-time lower envelope of
// parabolas (one thread per row; sv / tv hold the envelope's sites and start columns), then sqrt in fp64, rounded to fp32.
// Columns without a boundary pixel get g = h + w, farther than any real distance.  Without any boundary pixel scipy measures
// to the virtual feature (-1, 0).
__device__ __forceinline__ long long floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

__global__ void edt_rows_kernel(const int64_t* st, const int32_t* __restrict__ g, const int32_t* ctr, int32_t* sv_all, int32_t* tv_all,
                                float* f0) {
  if (st[0] == 0) return;
  const Crop c = crop_of(st);
  const int y = blockIdx.x * blockDim.x + threadIdx.x;
  if (y >= c.h) return;
  const long row = (long)y * c.w;
  float* out = f0 + row;
  if (ctr[0] == 0) {
    for (int x = 0; x < c.w; ++x) out[x] = __double2float_rn(__dsqrt_rn((double)((long long)(y + 1) * (y + 1) + (long long)x * x)));
    return;
  }
  const int32_t* gr = g + row;
  int32_t *sv = sv_all + row, *tv = tv_all + row;
  const long long inf = (long long)c.h + c.w;
  auto gg = [&](int i) -> long long { const long long v = gr[i] < INT_MAX / 2 ? gr[i] : inf; return v * v; };
  auto f = [&](long long x, int i) -> long long { return (x - i) * (x - i) + gg(i); };
  int q = 0;
  sv[0] = 0; tv[0] = 0;
  for (int u = 1; u < c.w; ++u) {
    while (q >= 0 && f(tv[q], sv[q]) > f(tv[q], u)) --q;
    if (q < 0) {
      q = 0; sv[0] = u;
    } else {
      const long long i = sv[q];
      const long long wsep = 1 + floor_div((long long)u * u - i * i + gg(u) - gg((int)i), 2 * (u - i));
      if (wsep < c.w) { ++q; sv[q] = u; tv[q] = (int)wsep; }
    }
  }
  for (int u = c.w - 1; u >= 0; --u) {
    out[u] = __double2float_rn(__dsqrt_rn((double)f(u, sv[q])));
    if (u == tv[q]) --q;
  }
}

// scipy 'reflect' (half-sample symmetric) index for any overshoot
__device__ __forceinline__ int reflect(int i, int n) {
  const int p = 2 * n;
  i %= p;
  if (i < 0) i += p;
  return i < n ? i : p - 1 - i;
}

// one axis of gaussian_filter1d: scipy's symmetric correlation, out = x0 * w0, then += (x[-k] + x[+k]) * w_k for k = 4 .. 1,
// in fp64, rounded to fp32
__global__ void gauss_kernel(const int64_t* st, const float* __restrict__ in, float* out, int axis) {
  if (st[0] == 0) return;
  const Crop c = crop_of(st);
  const long total = (long)c.h * c.w;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / c.w), x = (int)(i % c.w);
    auto at = [&](int k) -> double {
      return axis == 0 ? (double)in[(long)reflect(y + k, c.h) * c.w + x] : (double)in[(long)y * c.w + reflect(x + k, c.w)];
    };
    double acc = __dmul_rn(at(0), kGauss[0]);
    for (int k = 4; k >= 1; --k) acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(at(-k), at(k)), kGauss[k]));
    out[i] = __double2float_rn(acc);
  }
}

// inner (which = 0: the field on the mask) or outer (1: off the mask) field
__device__ __forceinline__ float field_at(const uint8_t* m, int ld, const Crop& c, const float* f2, int which, int y, int x) {
  const bool in = in_mask(m, ld, c, y, x);
  return (which == 0) == in ? f2[(long)y * c.w + x] : 0.f;
}

// first argmax in C order of the inner field (values are >= 0, so their bit patterns order like the values)
__global__ void argmax_kernel(const uint8_t* __restrict__ m, int ld, const int64_t* st, const float* f2, unsigned long long* best) {
  if (st[0] == 0) return;
  const Crop c = crop_of(st);
  const long total = (long)c.h * c.w;
  unsigned long long k = 0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const float v = field_at(m, ld, c, f2, 0, (int)(i / c.w), (int)(i % c.w));
    k = max(k, ((unsigned long long)__float_as_uint(v) << 32) | (0xffffffffu - (uint32_t)i));
  }
  for (int o = 16; o; o >>= 1) k = max(k, __shfl_down_sync(0xffffffffu, k, o));
  if ((threadIdx.x & 31) == 0) atomicMax(best, k);
}

// row maxima over [x - d, x + d] (mode 'nearest' = clamped) and the field minima
__global__ void peak_rows_kernel(const uint8_t* __restrict__ m, int ld, const int64_t* st, const float* f2, int which, int d, float* rmax,
                                 int32_t* ctr) {
  if (st[0] == 0) return;
  const Crop c = crop_of(st);
  const long total = (long)c.h * c.w;
  uint32_t mn = 0x7f800000u;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / c.w), x = (int)(i % c.w);
    float r = 0.f;
    for (int k = -d; k <= d; ++k) r = fmaxf(r, field_at(m, ld, c, f2, which, y, min(max(x + k, 0), c.w - 1)));
    rmax[i] = r;
    mn = min(mn, __float_as_uint(field_at(m, ld, c, f2, which, y, x)));
  }
  for (int o = 16; o; o >>= 1) mn = min(mn, __shfl_down_sync(0xffffffffu, mn, o));
  if ((threadIdx.x & 31) == 0) atomicMin((unsigned*)&ctr[6 + which], mn);
}

// candidates: the column maximum of the row maxima equals the pixel and the pixel exceeds the field minimum
__global__ void peak_cand_kernel(const uint8_t* __restrict__ m, int ld, const int64_t* st, const float* f2, int which, int d,
                                 const float* rmax, int32_t* ctr, unsigned long long* cand) {
  if (st[0] == 0) return;
  const Crop c = crop_of(st);
  const long total = (long)c.h * c.w;
  const float mn = __uint_as_float((uint32_t)ctr[6 + which]);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / c.w), x = (int)(i % c.w);
    const float v = field_at(m, ld, c, f2, which, y, x);
    if (!(v > mn)) continue;
    float r = 0.f;
    for (int k = -d; k <= d; ++k) r = fmaxf(r, rmax[(long)min(max(y + k, 0), c.h - 1) * c.w + x]);
    if (r == v) {
      const int slot = atomicAdd(&ctr[1 + which], 1);
      if (slot < kMaxCand) cand[(long)which * kMaxCand + slot] = ((unsigned long long)__float_as_uint(v) << 32) | (0xffffffffu - (uint32_t)i);
      else ctr[5] = 1;
    }
  }
}

// one block per field: sort the candidates strongest first (ties in C order) and thin them greedily (Chebyshev > d)
__global__ void peak_thin_kernel(const int64_t* st, int32_t* ctr, unsigned long long* cand_all, int32_t* kept_all) {
  extern __shared__ unsigned long long s_k[];
  if (st[0] == 0) return;
  const int which = blockIdx.x, d = which == 0 ? 3 : 5;
  const Crop c = crop_of(st);
  const int n = min(ctr[1 + which], kMaxCand);
  int np2 = 1;
  while (np2 < n) np2 <<= 1;
  const unsigned long long* cand = cand_all + (long)which * kMaxCand;
  for (int i = threadIdx.x; i < np2; i += blockDim.x) s_k[i] = i < n ? cand[i] : 0ull;
  __syncthreads();
  block_bitonic_sort<true>(s_k, np2, threadIdx.x, blockDim.x);
  int32_t* kept = kept_all + (long)which * kMaxCand;
  __shared__ int s_nk;
  __shared__ int s_ok;
  if (threadIdx.x == 0) s_nk = 0;
  __syncthreads();
  for (int q = 0; q < n; ++q) {
    const int p = (int)(0xffffffffu - (uint32_t)(s_k[q] & 0xffffffffu));
    const int py = p / c.w, px = p % c.w;
    if (threadIdx.x == 0) s_ok = 1;
    __syncthreads();
    for (int t = threadIdx.x; t < s_nk; t += blockDim.x) {
      const int o = kept[t];
      if (max(abs(o / c.w - py), abs(o % c.w - px)) <= d) s_ok = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_ok) kept[s_nk++] = p;
    __syncthreads();
  }
  if (threadIdx.x == 0) ctr[3 + which] = s_nk;
}

// points (x, y) in the 1024 frame (apply_coords: fp64, then fp32), labels, count
__global__ void points_out_kernel(int H, int W, int mode, const int64_t* st_c, int64_t* st, const int32_t* ctr,
                                  const unsigned long long* best, const int32_t* kept, int max_points, float* pts, float* lbl) {
  if (threadIdx.x != 0) return;
  if (st_c[0] == 0) { st[11] = 0; return; }
  const Crop c = crop_of(st_c);
  int nh, nw;
  preprocess_shape(H, W, 1024, &nh, &nw);
  const double sx = __ddiv_rn((double)nw, (double)W), sy = __ddiv_rn((double)nh, (double)H);
  int n = 0;
  auto put = [&](int p, float label) {
    if (n < max_points) {
      pts[2 * n] = __double2float_rn(__dmul_rn((double)(c.x0 + p % c.w), sx));
      pts[2 * n + 1] = __double2float_rn(__dmul_rn((double)(c.y0 + p / c.w), sy));
      lbl[n] = label;
    }
    ++n;
  };
  if (mode == 1) {
    put((int)(0xffffffffu - (uint32_t)(*best & 0xffffffffu)), 1.f);
  } else {
    for (int k = 0; k < ctr[3]; ++k) put(kept[k], 1.f);
    for (int k = 0; k < ctr[4]; ++k) put(kept[kMaxCand + k], 0.f);
  }
  st[11] = ctr[5] ? -1 : n;   // -1: more than kMaxCand peak candidates
}

__global__ void iou_kernel(const uint8_t* __restrict__ a, int lda, const uint8_t* __restrict__ b, int ldb, int H, int W, int64_t* out) {
  long long inter = 0, uni = 0;
  const long total = (long)H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / W), x = (int)(i % W);
    const bool p = a[(long)y * lda + x] == 1, q = b[(long)y * ldb + x] == 1;
    inter += p && q; uni += p || q;
  }
  for (int o = 16; o; o >>= 1) { inter += __shfl_down_sync(0xffffffffu, inter, o); uni += __shfl_down_sync(0xffffffffu, uni, o); }
  if ((threadIdx.x & 31) == 0 && uni) {
    atomicAdd((unsigned long long*)&out[0], (unsigned long long)inter);
    atomicAdd((unsigned long long*)&out[1], (unsigned long long)uni);
  }
}

// scipy.ndimage.shift(src, (dy, dx), order=0, prefilter=False, mode='constant', cval=0): per axis x = o - s in fp64; the
// pixel is 0 unless 0 <= x <= n - 1 on both axes (a NaN shift fails the test everywhere), else src[floor(x + 0.5)]
__device__ __forceinline__ int shift_src(int o, double s, int n) {
  const double x = __dsub_rn((double)o, s);
  return x >= 0.0 && x <= (double)(n - 1) ? (int)floor(__dadd_rn(x, 0.5)) : -1;
}

// rows over blockIdx.y (the source row is resolved once per row), columns over x
__global__ void shift_kernel(const uint8_t* __restrict__ src, int ld_src, uint8_t* __restrict__ dst, int ld_dst, int H, int W, double dy,
                             double dx) {
  for (int y = blockIdx.y; y < H; y += gridDim.y) {
    const int sy = shift_src(y, dy, H);
    for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < W; x += gridDim.x * blockDim.x) {
      const int sx = shift_src(x, dx, W);
      dst[(long)y * ld_dst + x] = (sy >= 0 && sx >= 0) ? src[(long)sy * ld_src + sx] : 0;
    }
  }
}

int grid_for(long n) { return (int)std::max<long>(1, std::min<long>((n + 255) / 256, 2048)); }

}  // namespace

int64_t mask_prompts_workspace(int H, int W) {
  return (int64_t)(5 * align256((size_t)4 * H * W) + align256((size_t)4 * H * 256)) + 8 * 2 * kMaxCand + 4 * 2 * kMaxCand + 64;
}

int mask_prompts(const uint8_t* mask, int H, int W, int ld, double box_extension, int want_logits, int point_mode, int max_points,
                 void* workspace, int64_t ws_bytes, int64_t* stats, float* box1024, float* logits, float* points, float* labels,
                 float* field, cudaStream_t st) {
  if (H <= 0 || W <= 0 || H > kMaxSide || W > kMaxSide || ld < W || point_mode < 0 || point_mode > 2 || box_extension < 0 ||
      (point_mode && max_points < 1))
    return set_error("mask_prompts: bad arguments H=%d W=%d (<= %d) ld=%d point_mode=%d max_points=%d box_extension=%g", H, W, kMaxSide,
                     ld, point_mode, max_points, box_extension);
  if (ws_bytes < mask_prompts_workspace(H, W))
    return set_error("mask_prompts: workspace of %lld bytes, need %lld", (long long)ws_bytes, (long long)mask_prompts_workspace(H, W));
  const Ws w = carve(workspace, H, W);
  const long hw = (long)H * W;
  stats_init_kernel<<<1, 32, 0, st>>>(stats, w.ctr);
  LAUNCH_CHECK("mask_prompts_init");
  stats_kernel<<<grid_for(hw), 256, 0, st>>>(mask, H, W, ld, stats);
  LAUNCH_CHECK("mask_prompts_stats");
  finish_kernel<<<1, 1, 0, st>>>(H, W, box_extension, stats, box1024);
  LAUNCH_CHECK("mask_prompts_box");
  if (want_logits) {
    // get_preprocess_shape(H, W, 256) on the host: x86-64 fp64 without contraction, as numpy computes it
    const double scale = 256 * 1.0 / std::max(H, W);
    const int th = (int)(H * scale + 0.5), tw = (int)(W * scale + 0.5);
    const float hi = (float)std::log((1 - 1e-3) / 1e-3);
    // torch's tap count per output pixel, 2 * ceil(scale) + 1 with scale = in / out in fp32: every tap must fit, or the logits
    // would no longer be torch's (e.g. 8192 x 111 resizes its width 111 -> 3, scale 37)
    for (const auto& io : {std::make_pair(H, th), std::make_pair(W, tw)}) {
      if (io.first == io.second) continue;
      const float sc = (float)io.first / (float)io.second;
      const int taps = sc >= 1.f ? (int)std::ceil(sc) * 2 + 1 : 3;
      if (io.second <= 0 || taps > kMaxTaps)
        return set_error("mask_prompts: the mask-prompt resize of %d x %d needs %d taps per pixel (at most %d)", H, W, taps, kMaxTaps);
    }
    const float* tmp = nullptr;
    if (tw != W) {
      resize_h_kernel<<<grid_for((long)H * tw), 256, 0, st>>>(mask, H, W, ld, tw, w.tmp);
      LAUNCH_CHECK("mask_prompts_resize_h");
      tmp = w.tmp;
    }
    logits_kernel<<<256, 256, 0, st>>>(mask, ld, tmp, H, W, th, tw, hi, logits);
    LAUNCH_CHECK("mask_prompts_logits");
  }
  if (point_mode) {
    edt_cols_kernel<<<(W + 127) / 128, 128, 0, st>>>(mask, ld, stats, w.g, w.ctr);
    LAUNCH_CHECK("mask_prompts_edt_cols");
    // f1 and rmax are free until the Gaussian and the peak search: they hold the envelopes of the row pass
    edt_rows_kernel<<<(H + 63) / 64, 64, 0, st>>>(stats, w.g, w.ctr, (int32_t*)w.f1, (int32_t*)w.rmax, w.f0);
    LAUNCH_CHECK("mask_prompts_edt_rows");
    gauss_kernel<<<grid_for(hw), 256, 0, st>>>(stats, w.f0, w.f1, 0);
    LAUNCH_CHECK("mask_prompts_gauss0");
    gauss_kernel<<<grid_for(hw), 256, 0, st>>>(stats, w.f1, w.f2, 1);
    LAUNCH_CHECK("mask_prompts_gauss1");
    unsigned long long* best = (unsigned long long*)(w.ctr + 8);
    if (point_mode == 1) {
      cudaMemsetAsync(best, 0, 8, st);
      argmax_kernel<<<grid_for(hw), 256, 0, st>>>(mask, ld, stats, w.f2, best);
      LAUNCH_CHECK("mask_prompts_argmax");
    } else {
      for (int which = 0; which < 2; ++which) {
        const int d = which == 0 ? 3 : 5;
        peak_rows_kernel<<<grid_for(hw), 256, 0, st>>>(mask, ld, stats, w.f2, which, d, w.rmax, w.ctr);
        LAUNCH_CHECK("mask_prompts_peak_rows");
        peak_cand_kernel<<<grid_for(hw), 256, 0, st>>>(mask, ld, stats, w.f2, which, d, w.rmax, w.ctr, w.cand);
        LAUNCH_CHECK("mask_prompts_peak_cand");
      }
      const int smem = 8 * kMaxCand;
      cudaFuncSetAttribute(peak_thin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      peak_thin_kernel<<<2, 512, smem, st>>>(stats, w.ctr, w.cand, w.kept);
      LAUNCH_CHECK("mask_prompts_peak_thin");
    }
    points_out_kernel<<<1, 32, 0, st>>>(H, W, point_mode, stats, stats, w.ctr, best, w.kept, max_points, points, labels);
    LAUNCH_CHECK("mask_prompts_points");
    if (field)
      if (cudaMemcpyAsync(field, w.f2, (size_t)4 * hw, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return set_error("mask_prompts: field copy failed");
  } else {
    cudaMemsetAsync(stats + 11, 0, 8, st);
  }
  return 0;
}

int mask_iou_counts(const uint8_t* a, int lda, const uint8_t* b, int ldb, int H, int W, int64_t* counts, cudaStream_t st) {
  if (H <= 0 || W <= 0 || lda < W || ldb < W) return set_error("mask_iou_counts: bad arguments H=%d W=%d lda=%d ldb=%d", H, W, lda, ldb);
  if (cudaMemsetAsync(counts, 0, 16, st) != cudaSuccess) return set_error("mask_iou_counts: memset failed");
  iou_kernel<<<grid_for((long)H * W), 256, 0, st>>>(a, lda, b, ldb, H, W, counts);
  LAUNCH_CHECK("mask_iou_counts");
  return 0;
}

int shift_mask(const uint8_t* src, int ld_src, uint8_t* dst, int ld_dst, int H, int W, double dy, double dx, cudaStream_t st) {
  if (H <= 0 || W <= 0 || ld_src < W || ld_dst < W)
    return set_error("shift_mask: bad arguments H=%d W=%d ld_src=%d ld_dst=%d", H, W, ld_src, ld_dst);
  shift_kernel<<<dim3(std::min((W + 255) / 256, 64), std::min(H, 65535)), 256, 0, st>>>(src, ld_src, dst, ld_dst, H, W, dy, dx);
  LAUNCH_CHECK("shift_mask");
  return 0;
}

}  // namespace msam
