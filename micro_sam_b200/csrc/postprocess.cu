// Mask post-processing of automatic mask generation / batched inference, without ever materialising the full
// resolution logits (SURVEY.md 7-6): everything is recomputed from the 256x256 low-res logits.
//   mask_stats   : Sam.postprocess_masks (bilinear 256->1024, crop, bilinear -> original size, align_corners=False)
//                  fused with calculate_stability_score, thresholding, batched_mask_to_box and area
//                  (instance_segmentation.py:229-255, inference.py:137-151, _vendored.py:33-85)
//   upsample     : the same interpolation, materialised on request (predict_torch's `masks` output / rle export)
//   filter_nms   : AMGBase._postprocess_batch (instance_segmentation.py:99-132): pred-IoU / stability / crop-edge
//                  filters + torchvision-semantics greedy box NMS, one CTA
//   paint        : mask_data_to_segmentation's painting loop (util.py:1799-1829)
#include "engine.h"
#include "postgeom.cuh"

namespace msam {

// Lazy evaluation (AMG): the statistics of a mask are only needed once it passes the predicted-IoU filter of generate(), so
// initialize() can leave them pending; a launch with `lazy.done != nullptr` skips masks that are already done or that the
// filter rejects (iou_pred > thresh fails; thresh <= 0 = no filter, as in AMGBase._postprocess_batch) and marks the rest.
struct LazyStats {
  const float* iou;
  float iou_thresh;
  uint8_t* done;
};
__device__ __forceinline__ bool lazy_skip(const LazyStats& z, long mi) {
  if (!z.done) return false;
  if (z.done[mi]) return true;
  return z.iou_thresh > 0.f && !(z.iou[mi] > z.iou_thresh);
}

// One CTA per mask.  stats: cnt(v > thr+off), cnt(v > thr-off), area = cnt(v > thr), bbox of (v > thr).
__global__ void __launch_bounds__(256)
mask_stats_kernel(const float* __restrict__ low_res, PostGeom g, float thr, const float* __restrict__ thr_arr, float off,
                  int32_t* __restrict__ boxes, float* __restrict__ stability, int32_t* __restrict__ area, LazyStats lazy) {
  const long mi = blockIdx.x;
  if (lazy_skip(lazy, mi)) return;
  if (thr_arr) thr = thr_arr[mi];  // per-mask threshold (mask_threshold="auto", inference.py:137-151)
  const float* lr = low_res + mi * g.lr * g.lr;
  int hi = 0, lo = 0, ar = 0, x0 = 1 << 30, y0 = 1 << 30, x1 = -1, y1 = -1;
  const float t_hi = thr + off, t_lo = thr - off;
  for (int y = threadIdx.x >> 5; y < g.out_h; y += 8) {
    for (int x = threadIdx.x & 31; x < g.out_w; x += 32) {
      const float v = full_res(lr, g, y, x);
      hi += v > t_hi;
      lo += v > t_lo;
      if (v > thr) {
        ++ar;
        x0 = min(x0, x); x1 = max(x1, x); y0 = min(y0, y); y1 = max(y1, y);
      }
    }
  }
  __shared__ int red[7][8];
  int vals[7] = {hi, lo, ar, x0, y0, x1, y1};
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    int v = vals[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int w = __shfl_xor_sync(0xffffffffu, v, o);
      v = (k < 3) ? v + w : ((k == 3 || k == 4) ? min(v, w) : max(v, w));
    }
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int r[7];
    for (int k = 0; k < 7; ++k) {
      int v = red[k][0];
      for (int w = 1; w < 8; ++w) v = (k < 3) ? v + red[k][w] : ((k == 3 || k == 4) ? min(v, red[k][w]) : max(v, red[k][w]));
      r[k] = v;
    }
    stability[mi] = (float)r[0] / (float)r[1];  // 0/0 -> NaN like torch; NaN fails ">= thresh" downstream
    area[mi] = r[2];
    if (lazy.done) lazy.done[mi] = 1;
    const bool empty = r[2] == 0;
    boxes[mi * 4 + 0] = empty ? 0 : r[3];
    boxes[mi * 4 + 1] = empty ? 0 : r[4];
    boxes[mi * 4 + 2] = empty ? 0 : r[5];
    boxes[mi * 4 + 3] = empty ? 0 : r[6];
  }
}

// Fast path of mask_stats for the common geometry input_size == original_size == (1024, 1024) (4x up-sampling).
// Thread j owns the 4 output columns 4j..4j+3 (taps: low-res columns j-1, j, j+1); rows are walked pair by pair of
// low-res rows (4 output rows per pair, weights 1/8, 3/8, 5/8, 7/8; the clamped border rows are handled apart).  The
// horizontal interpolation is done once per row pair; the per-pixel work is one FMUL + FFMA for the value and, per
// threshold, one FADD + IMAD.HI that adds the sign bit of (t - v) to the counter (v > t  <=>  sign(t - v) = 1) -- all on
// the FMA pipe, because a setp / iadd / sel per pixel (27 instructions per pixel) is bound by the ALU pipe.  Same interp_axis / bilerp arithmetic as the generic kernel: bit-identical results.
// grid = n_masks, block = 512 (two row ranges x 256 low-res columns).
__global__ void __launch_bounds__(512)
mask_stats_x4_kernel(const float* __restrict__ low_res, PostGeom g, float thr, const float* __restrict__ thr_arr, float off,
                     int32_t* __restrict__ boxes, float* __restrict__ stability, int32_t* __restrict__ area, LazyStats lazy) {
  const long mi = blockIdx.x;
  if (lazy_skip(lazy, mi)) return;
  if (thr_arr) thr = thr_arr[mi];
  const float* lr = low_res + mi * 65536;
  const int j = threadIdx.x & 255, part = threadIdx.x >> 8;
  Interp ix[4];
  int k0[4], k1[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    ix[r] = interp_axis(4 * j + r, g.s1, 256);
    k0[r] = ix[r].i0 - j + 1;  // which of the cached columns (j-1, j, j+1) is tap 0 / tap 1
    k1[r] = ix[r].i1 - j + 1;
  }
  const int cm = max(j - 1, 0), cp = min(j + 1, 255);
  const float t_hi = thr + off, t_lo = thr - off;
  unsigned hi = 0, lo = 0, ar = 0, colbits[4] = {0u, 0u, 0u, 0u};
  int y0 = 1 << 30, y1 = -1;
  float hA[4], hB[4];
  // horizontally interpolated values of low-res rows (i0, i1) for this thread's 4 output columns
  auto load_pair = [&](int i0, int i1) {
    const float* r0 = lr + i0 * 256;
    const float* r1 = lr + i1 * 256;
    const float A[3] = {__ldg(r0 + cm), __ldg(r0 + j), __ldg(r0 + cp)};
    const float B[3] = {__ldg(r1 + cm), __ldg(r1 + j), __ldg(r1 + cp)};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float a0 = k0[r] == 0 ? A[0] : (k0[r] == 1 ? A[1] : A[2]);
      const float a1 = k1[r] == 0 ? A[0] : (k1[r] == 1 ? A[1] : A[2]);
      const float b0 = k0[r] == 0 ? B[0] : (k0[r] == 1 ? B[1] : B[2]);
      const float b1 = k1[r] == 0 ? B[0] : (k1[r] == 1 ? B[1] : B[2]);
      hA[r] = ix[r].l0 * a0 + ix[r].l1 * a1;
      hB[r] = ix[r].l0 * b0 + ix[r].l1 * b1;
    }
  };
  auto row = [&](int y, float l0, float l1) {
    unsigned any = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float v = l0 * hA[r] + l1 * hB[r];
      const unsigned bt = __float_as_uint(thr - v);   // sign bit set  <=>  v > thr
      hi += __umulhi(__float_as_uint(t_hi - v), 2u);
      lo += __umulhi(__float_as_uint(t_lo - v), 2u);
      ar += __umulhi(bt, 2u);
      colbits[r] |= bt;
      any |= bt;
    }
    if (any >> 31) { y0 = min(y0, y); y1 = max(y1, y); }
  };
  if (part == 0) {  // rows 0, 1: source index clamped to 0 (weights 1, 0 on rows 0, 1)
    const Interp e0 = interp_axis(0, g.s1, 256);
    load_pair(e0.i0, e0.i1);
    row(0, e0.l0, e0.l1);
    const Interp e1 = interp_axis(1, g.s1, 256);
    row(1, e1.l0, e1.l1);
  }
  // interior: output rows 4*i + 2 .. 4*i + 5 interpolate low-res rows (i, i+1) with weights k/8, k = 1, 3, 5, 7.
  // Bilinear values are convex combinations of their taps: when the 6 taps of this thread's 4 x 4 pixel block are all above
  // the highest threshold (or all below the lowest) by more than the rounding slack of the three lerps, every comparison of
  // the block is decided without evaluating a pixel.  Only blocks that straddle a mask boundary take the per-pixel path, so
  // the result stays bit-identical while the typical mask costs ~8x fewer instructions.
  const int i_begin = part == 0 ? 0 : 128, i_end = part == 0 ? 128 : 255;
  float B0 = __ldg(lr + i_begin * 256 + cm), B1 = __ldg(lr + i_begin * 256 + j), B2 = __ldg(lr + i_begin * 256 + cp);
  int skip_test = 0;  // after a block that needed the per-pixel path the test is skipped for the next 3 (noisy masks: ~no overhead)
  for (int i = i_begin; i < i_end; ++i) {
    const float A0 = B0, A1 = B1, A2 = B2;
    const float* r1 = lr + (i + 1) * 256;
    B0 = __ldg(r1 + cm); B1 = __ldg(r1 + j); B2 = __ldg(r1 + cp);
    const int y = 4 * i + 2;
    if (skip_test == 0) {
      const float mn = fminf(fminf(fminf(A0, A1), fminf(A2, B0)), fminf(B1, B2));
      const float mx = fmaxf(fmaxf(fmaxf(A0, A1), fmaxf(A2, B0)), fmaxf(B1, B2));
      const float slack = 1e-5f * fmaxf(fabsf(mn), fabsf(mx));
      if (mx < t_lo - slack) continue;  // every pixel is below every threshold
      if (mn > t_hi + slack) {          // every pixel is above every threshold
        hi += 16; lo += 16; ar += 16;
        colbits[0] = colbits[1] = colbits[2] = colbits[3] = 0x80000000u;
        y0 = min(y0, y); y1 = max(y1, y + 3);
        continue;
      }
      skip_test = 3;
    } else {
      --skip_test;
    }
    const float A[3] = {A0, A1, A2};
    const float B[3] = {B0, B1, B2};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float a0 = k0[r] == 0 ? A[0] : (k0[r] == 1 ? A[1] : A[2]);
      const float a1 = k1[r] == 0 ? A[0] : (k1[r] == 1 ? A[1] : A[2]);
      const float b0 = k0[r] == 0 ? B[0] : (k0[r] == 1 ? B[1] : B[2]);
      const float b1 = k1[r] == 0 ? B[0] : (k1[r] == 1 ? B[1] : B[2]);
      hA[r] = ix[r].l0 * a0 + ix[r].l1 * a1;
      hB[r] = ix[r].l0 * b0 + ix[r].l1 * b1;
    }
    row(y, 0.875f, 0.125f);
    row(y + 1, 0.625f, 0.375f);
    row(y + 2, 0.375f, 0.625f);
    row(y + 3, 0.125f, 0.875f);
  }
  if (part == 1) {  // rows 1022, 1023: both taps are low-res row 255
    const Interp e0 = interp_axis(1022, g.s1, 256);
    load_pair(e0.i0, e0.i1);
    row(1022, e0.l0, e0.l1);
    const Interp e1 = interp_axis(1023, g.s1, 256);
    row(1023, e1.l0, e1.l1);
  }
  int x0 = 1 << 30, x1 = -1;
#pragma unroll
  for (int r = 0; r < 4; ++r)
    if (colbits[r] >> 31) { x0 = min(x0, 4 * j + r); x1 = max(x1, 4 * j + r); }
  __shared__ int red[7][16];
  int vals[7] = {(int)hi, (int)lo, (int)ar, x0, y0, x1, y1};
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    int v = vals[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int w = __shfl_xor_sync(0xffffffffu, v, o);
      v = (k < 3) ? v + w : ((k == 3 || k == 4) ? min(v, w) : max(v, w));
    }
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int r[7];
    for (int k = 0; k < 7; ++k) {
      int v = red[k][0];
      for (int w = 1; w < 16; ++w) v = (k < 3) ? v + red[k][w] : ((k == 3 || k == 4) ? min(v, red[k][w]) : max(v, red[k][w]));
      r[k] = v;
    }
    stability[mi] = (float)r[0] / (float)r[1];
    area[mi] = r[2];
    if (lazy.done) lazy.done[mi] = 1;
    const bool empty = r[2] == 0;
    boxes[mi * 4 + 0] = empty ? 0 : r[3];
    boxes[mi * 4 + 1] = empty ? 0 : r[4];
    boxes[mi * 4 + 2] = empty ? 0 : r[5];
    boxes[mi * 4 + 3] = empty ? 0 : r[6];
  }
}

// Materialise selected masks: logits (fp32) and/or thresholded (uint8 0/1), each [n_sel, out_h, out_w].
__global__ void upsample_kernel(const float* __restrict__ low_res, const int32_t* __restrict__ sel, PostGeom g,
                                float thr, const float* __restrict__ thr_arr, float* __restrict__ logits,
                                uint8_t* __restrict__ bin) {
  const long k = blockIdx.y;
  const long mi = sel ? sel[k] : k;
  if (thr_arr) thr = thr_arr[mi];
  const float* lr = low_res + mi * g.lr * g.lr;
  const long npx = (long)g.out_h * g.out_w;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long)gridDim.x * blockDim.x) {
    const int y = i / g.out_w, x = i % g.out_w;
    const float v = full_res(lr, g, y, x);
    if (logits) logits[k * npx + i] = v;
    if (bin) bin[k * npx + i] = v > thr;
  }
}

// Paint `n_sel` masks (given in painting order) into a uint32 label image at (oy, ox) offsets of a larger canvas.
// exclusive = 1: the first mask covering a pixel wins (merge_exclusively=True); 0: the last one wins (AMG).
__global__ void paint_kernel(const float* __restrict__ low_res, const int32_t* __restrict__ sel,
                             const int32_t* __restrict__ boxes /*xyxy per mask id*/, const int32_t* __restrict__ seg_ids,
                             int n_sel, PostGeom g, float thr, const float* __restrict__ thr_arr, int exclusive,
                             uint32_t* __restrict__ label, int ld_label) {
  extern __shared__ int32_t sbox[];  // [n_sel][4]
  for (int i = threadIdx.x; i < n_sel * 4; i += blockDim.x) sbox[i] = boxes[(long)sel[i / 4] * 4 + (i % 4)];
  __syncthreads();
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= g.out_w) return;
  uint32_t lab = 0;
  for (int k = 0; k < n_sel; ++k) {
    if (x < sbox[4 * k] || x > sbox[4 * k + 2] || y < sbox[4 * k + 1] || y > sbox[4 * k + 3]) continue;
    const float v = full_res(low_res + (long)sel[k] * g.lr * g.lr, g, y, x);
    if (v > (thr_arr ? thr_arr[sel[k]] : thr)) {
      lab = (uint32_t)seg_ids[k];
      if (exclusive) break;
    }
  }
  if (lab) label[(long)y * ld_label + x] = lab;
}

// ---------------------------------------------------------------------------------------------------------------
// Fused AMG filter + greedy box NMS (single CTA).  keep[] receives indices in descending-score order.  Up to NMS_MAX
// candidates the sort keys / boxes / alive flags live in shared memory; larger inputs (points_per_side 64, the cross-tile NMS
// of a large tiled image) run the same algorithm on a global-memory workspace (L2 resident, slower but unbounded).
constexpr int NMS_MAX = 8192;

struct NmsParams {
  int n;
  float iou_thresh, stab_thresh, nms_thresh;
  int use_filters;
  float crop[4], orig[4];  // xyxy
  float edge_atol;
};

__device__ __forceinline__ uint32_t orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(1024)
filter_nms_kernel(const int32_t* __restrict__ boxes, const float* __restrict__ scores, const float* __restrict__ stab,
                  NmsParams p, int32_t* __restrict__ keep, int32_t* __restrict__ n_keep, unsigned long long* gws) {
  extern __shared__ unsigned long long skey_smem[];  // [npow2] sort keys, then reused
  unsigned long long* skey = gws ? gws : skey_smem;
  __shared__ int s_cnt, s_cur;
  int npow2 = 1;
  while (npow2 < p.n) npow2 <<= 1;
  float* bx = reinterpret_cast<float*>(skey + npow2);  // [n][4] boxes in sorted order
  uint8_t* alive = reinterpret_cast<uint8_t*>(bx + 4 * (size_t)p.n);
  const int tid = threadIdx.x, nt = blockDim.x;

  for (int i = tid; i < npow2; i += nt) {
    unsigned long long key = 0;  // sorts last
    if (i < p.n) {
      bool ok = true;
      const float b0 = (float)boxes[4 * i], b1 = (float)boxes[4 * i + 1], b2 = (float)boxes[4 * i + 2], b3 = (float)boxes[4 * i + 3];
      if (p.use_filters) {
        if (p.iou_thresh > 0.f) ok = ok && (scores[i] > p.iou_thresh);
        if (p.stab_thresh > 0.f) ok = ok && (stab[i] >= p.stab_thresh);
        // is_box_near_crop_edge: boxes are in crop coordinates
        const float u[4] = {b0 + p.crop[0], b1 + p.crop[1], b2 + p.crop[0], b3 + p.crop[1]};
        bool near = false;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const bool nc = fabsf(u[c] - p.crop[c]) <= p.edge_atol, ni = fabsf(u[c] - p.orig[c]) <= p.edge_atol;
          near = near || (nc && !ni);
        }
        ok = ok && !near;
      }
      if (ok) key = ((unsigned long long)orderable(scores[i]) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)i);
    }
    skey[i] = key;
  }
  __syncthreads();
  // bitonic sort, descending
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < npow2; i += nt) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = skey[i], b = skey[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? (a < b) : (a > b)) { skey[i] = b; skey[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0) { s_cnt = 0; }
  __syncthreads();
  // candidates are the non-zero keys at the front
  int ncand = 0;
  {
    int lo = 0, hi = p.n;  // keys are sorted descending; find the first zero key
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (skey[mid] != 0ull) lo = mid + 1; else hi = mid; }
    ncand = lo;
  }
  for (int i = tid; i < ncand; i += nt) {
    const int idx = (int)(0xFFFFFFFFu - (uint32_t)(skey[i] & 0xFFFFFFFFull));
    bx[4 * i] = (float)boxes[4 * idx]; bx[4 * i + 1] = (float)boxes[4 * idx + 1];
    bx[4 * i + 2] = (float)boxes[4 * idx + 2]; bx[4 * i + 3] = (float)boxes[4 * idx + 3];
    alive[i] = 1;
  }
  __syncthreads();
  int cur = 0;
  while (true) {
    // next alive candidate (all threads scan identically; alive[] only changes between barriers)
    while (cur < ncand && !alive[cur]) ++cur;
    if (cur >= ncand) break;
    if (tid == 0) {
      keep[s_cnt] = (int)(0xFFFFFFFFu - (uint32_t)(skey[cur] & 0xFFFFFFFFull));
      ++s_cnt;
    }
    const float ax0 = bx[4 * cur], ay0 = bx[4 * cur + 1], ax1 = bx[4 * cur + 2], ay1 = bx[4 * cur + 3];
    const float aarea = (ax1 - ax0) * (ay1 - ay0);
    __syncthreads();  // everyone has read alive[cur] / bx before anyone updates alive[]
    for (int j = cur + 1 + tid; j < ncand; j += nt) {
      if (!alive[j]) continue;
      const float xx0 = fmaxf(ax0, bx[4 * j]), yy0 = fmaxf(ay0, bx[4 * j + 1]);
      const float xx1 = fminf(ax1, bx[4 * j + 2]), yy1 = fminf(ay1, bx[4 * j + 3]);
      const float w = fmaxf(0.f, xx1 - xx0), h = fmaxf(0.f, yy1 - yy0);
      const float inter = w * h;
      const float barea = (bx[4 * j + 2] - bx[4 * j]) * (bx[4 * j + 3] - bx[4 * j + 1]);
      const float ovr = inter / (aarea + barea - inter);
      if (ovr > p.nms_thresh) alive[j] = 0;
    }
    ++cur;
    __syncthreads();
  }
  __syncthreads();
  if (tid == 0) *n_keep = s_cnt;
  (void)s_cur;
}

#define LAUNCH_CHECK(name)                                                                        \
  do {                                                                                            \
    cudaError_t e_ = cudaGetLastError();                                                          \
    if (e_ != cudaSuccess) return set_error(name " launch failed: %s", cudaGetErrorString(e_)); \
    count_launch();                                                                               \
  } while (0)

int post_mask_stats(const float* low_res, int n, int in_h, int in_w, int out_h, int out_w, float thr, float off,
                    int32_t* boxes, float* stability, int32_t* area, cudaStream_t st, bool force_generic,
                    const float* thr_arr, const float* lazy_iou, float lazy_iou_thresh, uint8_t* lazy_done) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  if (n <= 0) return 0;
  const LazyStats lazy{lazy_iou, lazy_iou_thresh, lazy_done};
  prof_begin(st, "mask_stats", 0.0, (double)n * (65536.0 * 4 + 24));
  if (g.identity2 && in_h == 1024 && in_w == 1024 && !force_generic) {
    mask_stats_x4_kernel<<<n, 512, 0, st>>>(low_res, g, thr, thr_arr, off, boxes, stability, area, lazy);
  } else {
    mask_stats_kernel<<<n, 256, 0, st>>>(low_res, g, thr, thr_arr, off, boxes, stability, area, lazy);
  }
  prof_end(st);
  LAUNCH_CHECK("mask_stats");
  return 0;
}

int post_upsample(const float* low_res, const int32_t* sel, int n_sel, int in_h, int in_w, int out_h, int out_w, float thr,
                  float* logits, uint8_t* bin, cudaStream_t st, const float* thr_arr) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  if (n_sel <= 0) return 0;
  const long npx = (long)out_h * out_w;
  int bx = (int)((npx + 255) / 256);
  if (bx > 1024) bx = 1024;
  for (int k0 = 0; k0 < n_sel; k0 += 32768) {  // gridDim.y limit
    const int nk = (n_sel - k0 < 32768) ? n_sel - k0 : 32768;
    upsample_kernel<<<dim3(bx, nk), 256, 0, st>>>(low_res + (sel ? 0 : (long)k0 * 65536), sel ? sel + k0 : nullptr, g, thr,
                                                  thr_arr ? thr_arr + (sel ? 0 : k0) : nullptr, logits ? logits + (long)k0 * npx : nullptr, bin ? bin + (long)k0 * npx : nullptr);
    LAUNCH_CHECK("upsample");
  }
  return 0;
}

int post_paint(const float* low_res, const int32_t* sel, const int32_t* boxes, const int32_t* seg_ids, int n_sel, int in_h,
               int in_w, int out_h, int out_w, float thr, int exclusive, uint32_t* label, int ld_label, cudaStream_t st,
               const float* thr_arr) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  if (n_sel <= 0) return 0;
  if ((size_t)n_sel * 16 > 200 * 1024) return set_error("paint: too many masks (%d)", n_sel);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(paint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr = true;
  }
  paint_kernel<<<dim3((out_w + 255) / 256, out_h), 256, (size_t)n_sel * 16, st>>>(low_res, sel, boxes, seg_ids, n_sel, g, thr,
                                                                                  thr_arr, exclusive, label, ld_label);
  LAUNCH_CHECK("paint");
  return 0;
}

int post_filter_nms(const int32_t* boxes, const float* scores, const float* stab, int n, int use_filters, float iou_thresh,
                    float stab_thresh, float nms_thresh, const int32_t* crop_box, const int32_t* orig_box, int32_t* keep,
                    int32_t* n_keep, cudaStream_t st) {
  if (n > (1 << 22)) return set_error("filter_nms: n=%d exceeds %d", n, 1 << 22);
  if (n <= 0) {
    cudaMemsetAsync(n_keep, 0, 4, st);
    return 0;
  }
  NmsParams p;
  p.n = n; p.iou_thresh = iou_thresh; p.stab_thresh = stab_thresh; p.nms_thresh = nms_thresh; p.use_filters = use_filters;
  for (int i = 0; i < 4; ++i) { p.crop[i] = crop_box ? (float)crop_box[i] : 0.f; p.orig[i] = orig_box ? (float)orig_box[i] : 0.f; }
  p.edge_atol = 20.f;
  int npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  const size_t smem = (size_t)npow2 * 8 + (size_t)n * 16 + n + 16;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(filter_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    attr = true;
  }
  unsigned long long* gws = nullptr;
  if (n > NMS_MAX && cudaMallocAsync(reinterpret_cast<void**>(&gws), smem, st) != cudaSuccess)
    return set_error("filter_nms: workspace allocation of %zu bytes failed", smem);
  prof_begin(st, "filter_nms", 0.0, (double)n * 28);
  filter_nms_kernel<<<1, 1024, gws ? 0 : smem, st>>>(boxes, scores, stab, p, keep, n_keep, gws);
  prof_end(st);
  if (gws) cudaFreeAsync(gws, st);
  LAUNCH_CHECK("filter_nms");
  return 0;
}

}  // namespace msam

// =================================================================================================================
// util._to_image (util.py:618-651) on the device: per-channel min-max normalisation to uint8 with the reference's exact
// float32 arithmetic:  y = x - min;  y = y / (max(y) + 1e-7f);  u8 = trunc(y * 255).   (max(x - min) == fl(max - min)
// because float subtraction/rounding is monotonic.)  Input: H x W x C (C = 1, 2, 3; C > 3 uses the first three),
// dtype 0 = u8, 1 = u16, 2 = f32, 3 = i16, 4 = f64.  Output H x W x 3 uint8 (gray replicated, 2 channels + zero).
namespace msam {

__device__ __forceinline__ float load_as_f32(const void* p, int dtype, long i) {
  switch (dtype) {
    case 0: return (float)reinterpret_cast<const uint8_t*>(p)[i];
    case 1: return (float)reinterpret_cast<const uint16_t*>(p)[i];
    case 2: return reinterpret_cast<const float*>(p)[i];
    case 3: return (float)reinterpret_cast<const int16_t*>(p)[i];
    default: return (float)reinterpret_cast<const double*>(p)[i];
  }
}
__device__ __forceinline__ uint32_t f2ord(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// mm[2*c] = min (ordered-uint encoding), mm[2*c+1] = max
__global__ void to_image_minmax_kernel(const void* __restrict__ src, int dtype, long npix, int C, int cuse,
                                       uint32_t* __restrict__ mm) {
  uint32_t mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u};
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long)gridDim.x * blockDim.x) {
    for (int c = 0; c < cuse; ++c) {
      const uint32_t o = f2ord(load_as_f32(src, dtype, i * C + c));
      mn[c] = min(mn[c], o);
      mx[c] = max(mx[c], o);
    }
  }
  for (int c = 0; c < cuse; ++c) {
    uint32_t a = mn[c], b = mx[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a = min(a, __shfl_xor_sync(0xffffffffu, a, o));
      b = max(b, __shfl_xor_sync(0xffffffffu, b, o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin(&mm[2 * c], a);
      atomicMax(&mm[2 * c + 1], b);
    }
  }
}

__global__ void to_image_apply_kernel(const void* __restrict__ src, int dtype, long npix, int C, int cuse,
                                      const uint32_t* __restrict__ mm, uint8_t* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  uint8_t px[3] = {0, 0, 0};
  for (int c = 0; c < cuse; ++c) {
    const float mn = ord2f(mm[2 * c]), mx = ord2f(mm[2 * c + 1]);
    const float den = __fadd_rn(__fsub_rn(mx, mn), 1e-7f);
    const float y = __fsub_rn(load_as_f32(src, dtype, i * C + c), mn);
    px[c] = (uint8_t)(int)__fmul_rn(__fdiv_rn(y, den), 255.0f);
  }
  if (cuse == 1) px[1] = px[2] = px[0];
  out[3 * i] = px[0]; out[3 * i + 1] = px[1]; out[3 * i + 2] = px[2];
}

int post_to_image(const void* src, int dtype, int h, int w, int c, uint8_t* out, uint32_t* scratch6, cudaStream_t st) {
  if (dtype < 0 || dtype > 4 || c < 1 || h <= 0 || w <= 0) return set_error("to_image: bad arguments");
  const int cuse = c > 3 ? 3 : c;
  const long npix = (long)h * w;
  static const uint32_t init[6] = {0xffffffffu, 0u, 0xffffffffu, 0u, 0xffffffffu, 0u};
  cudaMemcpyAsync(scratch6, init, sizeof(init), cudaMemcpyHostToDevice, st);
  int blocks = (int)((npix + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  to_image_minmax_kernel<<<blocks, 256, 0, st>>>(src, dtype, npix, c, cuse, scratch6);
  LAUNCH_CHECK("to_image_minmax");
  to_image_apply_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(src, dtype, npix, c, cuse, scratch6, out);
  LAUNCH_CHECK("to_image_apply");
  return 0;
}

// =================================================================================================================
// Loss statistics of the fine-tuning step (training/sam_trainer.py:122-172, _compute_iou + _compute_loss): for every
// predicted mask m of object o the five sums over the H x W pixels that the dice loss (torch_em DiceLoss(reduce_channel=
// None) on sigmoid(masks)) and the IoU regression target need --
//   out[mi] = { sum sigmoid(v) t,  sum sigmoid(v)^2,  sum t,  |{v > 0} and t|,  |{v > 0} or t| }      (t = target in {0,1})
// -- computed straight from the 256 x 256 low-res logits: v = Sam.postprocess_masks(low_res) is evaluated per pixel
// (same interpolation code as mask_stats) and never written.  One CTA per predicted mask; target of mask mi = targets[mi / M].
__global__ void __launch_bounds__(256)
mask_loss_stats_kernel(const float* __restrict__ low_res, const uint8_t* __restrict__ targets, int M, PostGeom g,
                       float* __restrict__ out) {
  const long mi = blockIdx.x;
  const float* lr = low_res + mi * g.lr * g.lr;
  const uint8_t* tg = targets + (mi / M) * (long)g.out_h * g.out_w;
  float s_pt = 0.f, s_pp = 0.f;
  int s_t = 0, s_and = 0, s_or = 0;
  for (int y = threadIdx.x >> 5; y < g.out_h; y += 8) {
    for (int x = threadIdx.x & 31; x < g.out_w; x += 32) {
      const float v = full_res(lr, g, y, x);
      const int t = tg[(long)y * g.out_w + x] != 0;
      const float p = 1.0f / (1.0f + __expf(-v));
      s_pt += t ? p : 0.f;
      s_pp = fmaf(p, p, s_pp);
      const int b = v > 0.f;  // sigmoid(v) > 0.5
      s_t += t; s_and += b & t; s_or += b | t;
    }
  }
  __shared__ float redf[2][8];
  __shared__ int redi[3][8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s_pt += __shfl_xor_sync(0xffffffffu, s_pt, o); s_pp += __shfl_xor_sync(0xffffffffu, s_pp, o);
    s_t += __shfl_xor_sync(0xffffffffu, s_t, o); s_and += __shfl_xor_sync(0xffffffffu, s_and, o);
    s_or += __shfl_xor_sync(0xffffffffu, s_or, o);
  }
  if ((threadIdx.x & 31) == 0) {
    const int w = threadIdx.x >> 5;
    redf[0][w] = s_pt; redf[1][w] = s_pp; redi[0][w] = s_t; redi[1][w] = s_and; redi[2][w] = s_or;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    int c = 0, d = 0, e = 0;
    for (int w = 0; w < 8; ++w) { a += redf[0][w]; b += redf[1][w]; c += redi[0][w]; d += redi[1][w]; e += redi[2][w]; }
    out[mi * 5 + 0] = a; out[mi * 5 + 1] = b; out[mi * 5 + 2] = (float)c; out[mi * 5 + 3] = (float)d; out[mi * 5 + 4] = (float)e;
  }
}

// Adjoint of mask_loss_stats_kernel w.r.t. the low-res logits: the loss reaches them only through  pt = sum sigmoid(v) t  and
// pp = sum sigmoid(v)^2  (the counts are piecewise constant), so with a = dL/dpt, b = dL/dpp per predicted mask
//   dL/dv(y, x) = (a t + 2 b p) p (1 - p),  p = sigmoid(v),
// scattered to the low-res taps with the weights of the two bilinear stages (the transpose of full_res()).  d_low_res is
// ACCUMULATED into with atomics (zero it first).
__device__ __forceinline__ void stage1_scatter(float* __restrict__ dlr, const PostGeom& g, int Y, int X, float w) {
  const Interp iy = interp_axis(Y, g.s1, g.lr), ix = interp_axis(X, g.s1, g.lr);
  atomicAdd(dlr + iy.i0 * g.lr + ix.i0, w * iy.l0 * ix.l0);
  atomicAdd(dlr + iy.i0 * g.lr + ix.i1, w * iy.l0 * ix.l1);
  atomicAdd(dlr + iy.i1 * g.lr + ix.i0, w * iy.l1 * ix.l0);
  atomicAdd(dlr + iy.i1 * g.lr + ix.i1, w * iy.l1 * ix.l1);
}
__global__ void __launch_bounds__(256)
mask_loss_backward_kernel(const float* __restrict__ low_res, const uint8_t* __restrict__ targets, const float* __restrict__ d_stats,
                          int M, PostGeom g, float* __restrict__ d_low_res) {
  const long mi = blockIdx.x;
  const float a = d_stats[mi * 5 + 0], b = d_stats[mi * 5 + 1];
  if (a == 0.f && b == 0.f) return;   // masks that lost the min over the candidates
  const float* lr = low_res + mi * g.lr * g.lr;
  float* dlr = d_low_res + mi * g.lr * g.lr;
  const uint8_t* tg = targets + (mi / M) * (long)g.out_h * g.out_w;
  for (int y = threadIdx.x >> 5; y < g.out_h; y += 8) {
    for (int x = threadIdx.x & 31; x < g.out_w; x += 32) {
      const float v = full_res(lr, g, y, x);
      const float t = tg[(long)y * g.out_w + x] != 0 ? 1.f : 0.f;
      const float p = 1.0f / (1.0f + __expf(-v));
      const float gv = (a * t + 2.f * b * p) * p * (1.f - p);
      if (g.identity2) {
        stage1_scatter(dlr, g, y, x, gv);
      } else {
        const Interp iy = interp_axis(y, g.s2y, g.in_h), ix = interp_axis(x, g.s2x, g.in_w);
        stage1_scatter(dlr, g, iy.i0, ix.i0, gv * iy.l0 * ix.l0);
        stage1_scatter(dlr, g, iy.i0, ix.i1, gv * iy.l0 * ix.l1);
        stage1_scatter(dlr, g, iy.i1, ix.i0, gv * iy.l1 * ix.l0);
        stage1_scatter(dlr, g, iy.i1, ix.i1, gv * iy.l1 * ix.l1);
      }
    }
  }
}

int post_mask_loss_backward(const float* low_res, const uint8_t* targets, const float* d_stats, int n_obj, int M, int in_h, int in_w,
                            int out_h, int out_w, float* d_low_res, cudaStream_t st) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  if (n_obj <= 0 || M <= 0) return 0;
  prof_begin(st, "mask_loss_backward", 0.0, (double)n_obj * M * 65536.0 * 8 + (double)n_obj * out_h * out_w);
  mask_loss_backward_kernel<<<n_obj * M, 256, 0, st>>>(low_res, targets, d_stats, M, g, d_low_res);
  prof_end(st);
  LAUNCH_CHECK("mask_loss_backward");
  return 0;
}

int post_mask_loss_stats(const float* low_res, const uint8_t* targets, int n_obj, int M, int in_h, int in_w, int out_h, int out_w,
                         float* out, cudaStream_t st) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  if (n_obj <= 0 || M <= 0) return 0;
  prof_begin(st, "mask_loss_stats", 0.0, (double)n_obj * M * 65536.0 * 4 + (double)n_obj * out_h * out_w);
  mask_loss_stats_kernel<<<n_obj * M, 256, 0, st>>>(low_res, targets, M, g, out);
  prof_end(st);
  LAUNCH_CHECK("mask_loss_stats");
  return 0;
}

// =================================================================================================================
// AMG painting without a host round trip: n_sel is read from device memory (the NMS kernel's n_keep) and the
// "descending area, later overwrites" order of mask_data_to_segmentation(merge_exclusively=False) is evaluated per pixel
// as: the covering mask with the smallest (area, -position) wins.  Ids are position + 1 (any unique id works: the
// connected-component pass re-assigns ids in raster order afterwards).
// Survivors are visited in ascending (area, -position) order -- sorted once per block in shared memory (<= PAINT_SORT_MAX
// masks; a block is one row segment of 256 pixels) -- so the FIRST covering mask is the winner and the loop stops there:
// with hundreds of overlapping masks that is ~2 bilinear evaluations per pixel instead of one per mask.
constexpr int PAINT_SORT_MAX = 4096;
__global__ void __launch_bounds__(256)
paint_min_area_kernel(const float* __restrict__ low_res, const int32_t* __restrict__ sel,
                      const int32_t* __restrict__ n_sel_ptr, const int32_t* __restrict__ boxes,
                      const int32_t* __restrict__ area, PostGeom g, float thr, int32_t* __restrict__ label,
                      int ld_label) {
  __shared__ unsigned long long skey[PAINT_SORT_MAX];  // (area << 32) | (0xFFFFFFFF - position): ascending = winner first
  const int n_sel = *n_sel_ptr;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (n_sel <= PAINT_SORT_MAX) {
    int npow2 = 1;
    while (npow2 < n_sel) npow2 <<= 1;
    for (int k = threadIdx.x; k < npow2; k += 256)
      skey[k] = k < n_sel ? (((unsigned long long)(unsigned)area[sel[k]] << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)k)) : ~0ull;
    __syncthreads();
    for (int kk = 2; kk <= npow2; kk <<= 1) {
      for (int j = kk >> 1; j > 0; j >>= 1) {
        for (int i = threadIdx.x; i < npow2; i += 256) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned long long a = skey[i], b = skey[ixj];
            if (((i & kk) == 0) ? (a > b) : (a < b)) { skey[i] = b; skey[ixj] = a; }
          }
        }
        __syncthreads();
      }
    }
    if (x >= g.out_w) return;
    int best_pos = -1;
    for (int k = 0; k < n_sel; ++k) {
      const int pos = (int)(0xFFFFFFFFu - (unsigned)(skey[k] & 0xFFFFFFFFull));
      const int mi = sel[pos];
      const int4 b = *reinterpret_cast<const int4*>(boxes + 4L * mi);
      if (x < b.x || x > b.z || y < b.y || y > b.w) continue;
      if (full_res(low_res + (long)mi * g.lr * g.lr, g, y, x) > thr) { best_pos = pos; break; }
    }
    label[(long)y * ld_label + x] = best_pos + 1;
    return;
  }
  if (x >= g.out_w) return;
  int best_pos = -1, best_area = 0x7fffffff;
  for (int k = 0; k < n_sel; ++k) {
    const int mi = sel[k];
    const int4 b = *reinterpret_cast<const int4*>(boxes + 4L * mi);
    if (x < b.x || x > b.z || y < b.y || y > b.w) continue;
    const int a = area[mi];
    if (a > best_area) continue;  // a later mask only wins with area <= the current winner
    const float v = full_res(low_res + (long)mi * g.lr * g.lr, g, y, x);
    if (v > thr) { best_area = a; best_pos = k; }
  }
  label[(long)y * ld_label + x] = best_pos + 1;
}

// Tile version for the common geometry input_size == original_size == (1024, 1024): one block paints a 32 x 32 pixel region
// for ALL survivors.  The region depends on a 10 x 10 patch of each mask's low-res logits only, which the block stages in
// shared memory (double buffered: the next mask's patch is fetched while the current one is evaluated) -- 0.1 global loads
// per (pixel, mask) instead of 4, which is what bounds a per-pixel kernel with hundreds of overlapping survivors.  Survivors are visited in ascending
// (area, -position) order (block-local bitonic sort), so a pixel is final at its first hit and the block stops as soon as
// all its 1024 pixels are decided.  Same interp_axis / bilerp arithmetic as `stage1`: bit-identical results.
__global__ void __launch_bounds__(256)
paint_min_area_x4_kernel(const float* __restrict__ low_res, const int32_t* __restrict__ sel,
                         const int32_t* __restrict__ n_sel_ptr, const int32_t* __restrict__ boxes,
                         const int32_t* __restrict__ area, PostGeom g, float thr, int32_t* __restrict__ label, int ld_label) {
  __shared__ unsigned long long skey[PAINT_SORT_MAX];
  __shared__ float patch[2][10][12];
  __shared__ unsigned cand_bits[PAINT_SORT_MAX / 32], cand_off[PAINT_SORT_MAX / 32 + 1];
  __shared__ unsigned short cand[PAINT_SORT_MAX];
  const int n_all = *n_sel_ptr;
  const int tid = threadIdx.x;
  const bool sorted = n_all <= PAINT_SORT_MAX;
  const int X0 = blockIdx.x * 32, Y0 = blockIdx.y * 32;
  int n_sel = n_all;
  if (sorted) {
    int npow2 = 1;
    while (npow2 < n_sel) npow2 <<= 1;
    for (int k = tid; k < npow2; k += 256)
      skey[k] = k < n_sel ? (((unsigned long long)(unsigned)area[sel[k]] << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)k)) : ~0ull;
    __syncthreads();
    for (int kk = 2; kk <= npow2; kk <<= 1) {
      for (int j = kk >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < npow2; i += 256) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned long long a = skey[i], b = skey[ixj];
            if (((i & kk) == 0) ? (a > b) : (a < b)) { skey[i] = b; skey[ixj] = a; }
          }
        }
        __syncthreads();
      }
    }
    // Candidates of THIS region, in sorted order: survivors whose box misses the 32 x 32 region are dropped up front (with
    // localised masks a region sees a handful of the survivors instead of all of them).  Order-preserving compaction:
    // ballot words -> exclusive scan of their popcounts by warp 0 -> scatter.
    for (int k0 = 0; k0 < npow2; k0 += 256) {
      const int k = k0 + tid;
      bool hit = false;
      if (k < n_all) {
        const int mi = sel[(int)(0xFFFFFFFFu - (unsigned)(skey[k] & 0xFFFFFFFFull))];
        const int4 b = *reinterpret_cast<const int4*>(boxes + 4L * mi);
        hit = b.x <= X0 + 31 && b.z >= X0 && b.y <= Y0 + 31 && b.w >= Y0;
      }
      const unsigned w = __ballot_sync(0xffffffffu, hit);
      if ((tid & 31) == 0 && k < npow2) cand_bits[k >> 5] = w;
    }
    __syncthreads();
    const int n_words = (npow2 + 31) >> 5;
    if (tid < 32) {
      unsigned run = 0;
      for (int w0 = 0; w0 < n_words; w0 += 32) {
        const int w = w0 + tid;
        const unsigned c = w < n_words ? __popc(cand_bits[w]) : 0u;
        unsigned incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, incl, o); if (tid >= o) incl += t; }
        if (w < n_words) cand_off[w] = run + incl - c;
        run += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (tid == 0) cand_off[n_words] = run;
    }
    __syncthreads();
    for (int k = tid; k < n_all; k += 256) {
      const unsigned w = cand_bits[k >> 5];
      if ((w >> (k & 31)) & 1u) cand[cand_off[k >> 5] + __popc(w & ((1u << (k & 31)) - 1u))] = (unsigned short)k;
    }
    n_sel = (int)cand_off[n_words];
    __syncthreads();
  }
  const int py0 = (Y0 >> 2) - 1, px0 = (X0 >> 2) - 1;          // low-res origin of the patch (may be -1: never referenced)
  const int y = Y0 + (tid >> 3), xb = X0 + (tid & 7) * 4;       // this thread: pixels (y, xb .. xb+3)
  const Interp iy = interp_axis(y, g.s1, g.lr);
  Interp ix[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) ix[q] = interp_axis(xb + q, g.s1, g.lr);
  unsigned long long best[4] = {~0ull, ~0ull, ~0ull, ~0ull};
  const int pr = tid / 10, pc = tid % 10;                        // patch element fetched by threads 0..99
  const int gy = min(max(py0 + pr, 0), g.lr - 1), gx = min(max(px0 + pc, 0), g.lr - 1);
  auto pos_of = [&](int k) -> int { return sorted ? (int)(0xFFFFFFFFu - (unsigned)(skey[cand[k]] & 0xFFFFFFFFull)) : k; };
  float nxt = 0.f;
  if (n_sel > 0 && tid < 100) nxt = __ldg(low_res + (long)sel[pos_of(0)] * g.lr * g.lr + gy * g.lr + gx);
  for (int k = 0; k < n_sel; ++k) {
    const int buf = k & 1;
    if (tid < 100) patch[buf][pr][pc] = nxt;
    const int pos = pos_of(k), mi = sel[pos];
    const unsigned long long key = ((unsigned long long)(unsigned)area[mi] << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)pos);
    if (k + 1 < n_sel && tid < 100) nxt = __ldg(low_res + (long)sel[pos_of(k + 1)] * g.lr * g.lr + gy * g.lr + gx);
    __syncthreads();   // patch[buf] complete; the previous iteration's readers of patch[buf ^ 1] ... are done (they passed this barrier)
    const int4 b = *reinterpret_cast<const int4*>(boxes + 4L * mi);
    bool open = false;
    if (y >= b.y && y <= b.w) {
      const float* r0 = &patch[buf][iy.i0 - py0][0];
      const float* r1 = &patch[buf][iy.i1 - py0][0];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int x = xb + q;
        if (key < best[q] && x >= b.x && x <= b.z) {
          const float v = bilerp(r0[ix[q].i0 - px0], r0[ix[q].i1 - px0], r1[ix[q].i0 - px0], r1[ix[q].i1 - px0], iy, ix[q]);
          if (v > thr) best[q] = key;
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) open = open || best[q] == ~0ull;
    // sorted order: a decided pixel is final -> stop when the whole region is decided (one barrier per mask either way)
    if (sorted && !__syncthreads_or(open)) break;
  }
  int4 o;
  o.x = best[0] == ~0ull ? 0 : (int)(0xFFFFFFFFu - (unsigned)(best[0] & 0xFFFFFFFFull)) + 1;
  o.y = best[1] == ~0ull ? 0 : (int)(0xFFFFFFFFu - (unsigned)(best[1] & 0xFFFFFFFFull)) + 1;
  o.z = best[2] == ~0ull ? 0 : (int)(0xFFFFFFFFu - (unsigned)(best[2] & 0xFFFFFFFFull)) + 1;
  o.w = best[3] == ~0ull ? 0 : (int)(0xFFFFFFFFu - (unsigned)(best[3] & 0xFFFFFFFFull)) + 1;
  *reinterpret_cast<int4*>(label + (long)y * ld_label + xb) = o;
}

int post_paint_min_area(const float* low_res, const int32_t* sel, const int32_t* n_sel, const int32_t* boxes,
                        const int32_t* area, int in_h, int in_w, int out_h, int out_w, float thr, int32_t* label,
                        int ld_label, cudaStream_t st) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  prof_begin(st, "paint_min_area", 0.0, (double)out_h * out_w * 4);
  if (g.identity2 && in_h == 1024 && in_w == 1024 && ld_label % 4 == 0 && (reinterpret_cast<uintptr_t>(label) & 15) == 0) {
    paint_min_area_x4_kernel<<<dim3(32, 32), 256, 0, st>>>(low_res, sel, n_sel, boxes, area, g, thr, label, ld_label);
  } else {
    paint_min_area_kernel<<<dim3((out_w + 255) / 256, out_h), 256, 0, st>>>(low_res, sel, n_sel, boxes, area, g, thr, label,
                                                                          ld_label);
  }
  prof_end(st);
  LAUNCH_CHECK("paint_min_area");
  return 0;
}

// =================================================================================================================
// util.mask_data_to_segmentation tail (util.py:1831-1848) on the device: connected components of equal non-zero labels
// (4-connectivity; union-find with atomicMin roots, so a component's root is its first pixel in raster order), size
// filter, optional removal of the largest segment (`with_background`; the unlabelled area counts as segment 0 exactly
// like np.unique), consecutive relabelling in raster order of the roots.
__device__ __forceinline__ int uf_find(int* parent, int i) {
  int p = parent[i];
  while (p != i) { i = p; p = parent[i]; }
  return i;
}
__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&parent[b], a);
    if (old == b) return;
    b = old;
  }
}
// Initial forest: every pixel points at the first pixel of its horizontal run inside the warp's 32-pixel segment (found with
// one ballot), so the union phase starts from runs instead of single pixels: the chains that uf_find walks are 32x shorter
// and most horizontal unions disappear.  (Roots stay the smallest index of their set, as the relabelling order requires.)
__global__ void cc_init_kernel(const int32_t* __restrict__ seg, int n, int w, int* __restrict__ parent, int* __restrict__ size) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int s = i < n ? seg[i] : 0;
  const int left = __shfl_up_sync(0xffffffffu, s, 1);
  // run boundary: first lane, first pixel of an image row, or a label change
  const bool head = lane == 0 || (i % w) == 0 || left != s;
  const unsigned heads = __ballot_sync(0xffffffffu, head);
  if (i < n) {
    const int start = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));   // nearest head at or below this lane
    parent[i] = s != 0 ? i - (lane - start) : -1;
    size[i] = 0;
  }
}
// Unions: horizontally only across warp-segment boundaries (inside a segment the run already shares a parent); vertically
// only where the link is not implied by the left neighbours (i-1 ~ i and i-1+w ~ i+w by their runs, i-1 ~ i-1+w by the left
// pixel's own link), i.e. at the first column of every vertical contact between two runs.
__global__ void cc_merge_kernel(const int32_t* __restrict__ seg, int h, int w, int* __restrict__ parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= h * w) return;
  const int s = seg[i];
  if (s == 0) return;
  const int x = i % w, y = i / w;
  if ((threadIdx.x & 31) == 0 && x > 0 && seg[i - 1] == s) uf_union(parent, i - 1, i);
  if (y + 1 < h && seg[i + w] == s) {
    const bool implied = x > 0 && seg[i - 1] == s && seg[i + w - 1] == s;
    if (!implied) uf_union(parent, i, i + w);
  }
}
__global__ void cc_flatten_count_kernel(int n, int* __restrict__ parent, int* __restrict__ size, int* __restrict__ bg_count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int bg = 0, r = -1;
  if (i < n) {
    if (parent[i] >= 0) {
      r = uf_find(parent, i);
      parent[i] = r;
    } else {
      bg = 1;
    }
  }
  // one atomic per distinct root per warp (neighbouring pixels mostly share their root; a large component would otherwise
  // take hundreds of thousands of same-address atomics)
  const unsigned same = __match_any_sync(0xffffffffu, r);
  if (r >= 0 && (threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(&size[r], __popc(same));
  const unsigned m = __ballot_sync(0xffffffffu, bg);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(bg_count, __popc(m));
}
// largest component: packed (size << 32 | ~root) maximum -> largest size, smallest root on ties (np.argmax order)
__global__ void cc_largest_kernel(int n, const int* __restrict__ parent, const int* __restrict__ size,
                                  unsigned long long* __restrict__ best) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v = 0;
  if (i < n && parent[i] == i) v = ((unsigned long long)(unsigned)size[i] << 32) | (unsigned)(~(unsigned)i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = v > w ? v : w;
  }
  if ((threadIdx.x & 31) == 0 && v) atomicMax(best, v);
}
// flag[i] = 1 for kept roots; then block-wise inclusive scan in three kernels
__global__ void cc_flag_kernel(int n, const int* __restrict__ parent, const int* __restrict__ size, int min_size,
                               int with_background, const unsigned long long* __restrict__ best,
                               const int* __restrict__ bg_count, int* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int f = 0;
  if (parent[i] == i) {
    f = size[i] >= min_size;
    if (with_background && *best) {
      const int bsize = (int)(*best >> 32), broot = (int)(~(unsigned)(*best & 0xffffffffu));
      // np.unique lists id 0 (unlabelled) first: it is the argmax when its count >= the largest component
      if (*bg_count < bsize && i == broot) f = 0;
    }
  }
  flag[i] = f;
}
__global__ void scan_block_kernel(const int* __restrict__ in, int n, int* __restrict__ out, int* __restrict__ block_sums) {
  __shared__ int s[1024];
  const int i = blockIdx.x * 1024 + threadIdx.x;
  int v = i < n ? in[i] : 0;
  s[threadIdx.x] = v;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
    __syncthreads();
    s[threadIdx.x] += t;
    __syncthreads();
  }
  if (i < n) out[i] = s[threadIdx.x];
  if (threadIdx.x == 1023) block_sums[blockIdx.x] = s[1023];
}
// exclusive scan of the per-block sums in place: single block of 1024 threads, chunks of 1024 sums with a running carry
// (any nb: a 16k x 16k label image has 262144 block sums)
__global__ void scan_sums_kernel(int* __restrict__ block_sums, int nb) {
  __shared__ int s[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < nb ? block_sums[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      const int t = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
      __syncthreads();
      s[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < nb) block_sums[i] = carry + s[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += s[1023];
    __syncthreads();
  }
}
__global__ void cc_relabel_kernel(int n, const int* __restrict__ parent, const int* __restrict__ flag,
                                  const int* __restrict__ scan, const int* __restrict__ block_offs,
                                  uint32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = parent[i];
  uint32_t v = 0;
  if (r >= 0 && flag[r]) v = (uint32_t)(scan[r] + block_offs[r >> 10]);
  out[i] = v;
}

int post_finish_segmentation(const int32_t* seg, int h, int w, int min_size, int with_background, uint32_t* out,
                             int32_t* ws /* 4*h*w + max(4096, ceil(h*w/1024)) + 8 ints */, cudaStream_t st) {
  if ((long)h * w >= (1l << 31) - 1024) return set_error("finish_segmentation: image too large (%d x %d)", h, w);
  const int n = h * w;
  const int nb = (n + 1023) / 1024;
  int* parent = ws;
  int* size = ws + n;
  int* flag = ws + 2 * (size_t)n;
  int* scan = ws + 3 * (size_t)n;
  int* bsums = ws + 4 * (size_t)n;
  int* bg = bsums + (nb > 4096 ? nb : 4096);
  unsigned long long* best = reinterpret_cast<unsigned long long*>(bg + 2);
  cudaMemsetAsync(bg, 0, 6 * sizeof(int), st);
  const unsigned blocks = (unsigned)((n + 255) / 256);
  prof_begin(st, "finish_segmentation (8 kernels)", 0.0, (double)n * 4 * 12);
  cc_init_kernel<<<blocks, 256, 0, st>>>(seg, n, w, parent, size);
  LAUNCH_CHECK("cc_init");
  cc_merge_kernel<<<blocks, 256, 0, st>>>(seg, h, w, parent);
  LAUNCH_CHECK("cc_merge");
  cc_flatten_count_kernel<<<blocks, 256, 0, st>>>(n, parent, size, bg);
  LAUNCH_CHECK("cc_flatten");
  cc_largest_kernel<<<blocks, 256, 0, st>>>(n, parent, size, best);
  LAUNCH_CHECK("cc_largest");
  cc_flag_kernel<<<blocks, 256, 0, st>>>(n, parent, size, min_size, with_background, best, bg, flag);
  LAUNCH_CHECK("cc_flag");
  scan_block_kernel<<<nb, 1024, 0, st>>>(flag, n, scan, bsums);
  LAUNCH_CHECK("scan_block");
  scan_sums_kernel<<<1, 1024, 0, st>>>(bsums, nb);
  LAUNCH_CHECK("scan_sums");
  cc_relabel_kernel<<<blocks, 256, 0, st>>>(n, parent, flag, scan, bsums, out);
  prof_end(st);
  LAUNCH_CHECK("cc_relabel");
  return 0;
}

}  // namespace msam

// =================================================================================================================
// Multi-crop / tiled AMG painting (AutomaticMaskGenerator.generate with several crops, instance_segmentation.py:499-529):
// every crop paints its surviving masks into one global canvas with a packed 64-bit atomicMin
//   key = (area << 32) | (0xFFFFFFFF - global position)   ->  smallest area wins, later position on ties,
// which is the "descending area, later overwrites" order of mask_data_to_segmentation(merge_exclusively=False)
// evaluated per pixel.  canvas_to_label turns the winners into ids (position + 1).
namespace msam {

__global__ void paint_canvas_kernel(const float* __restrict__ low_res, const int32_t* __restrict__ sel,
                                    const int32_t* __restrict__ gpos, int n_sel, const int32_t* __restrict__ boxes,
                                    const int32_t* __restrict__ area, PostGeom g, float thr, int off_x, int off_y,
                                    unsigned long long* __restrict__ canvas, int ld_canvas) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= g.out_w) return;
  unsigned long long best = ~0ull;
  for (int k = 0; k < n_sel; ++k) {
    const int mi = sel[k];
    const int4 b = *reinterpret_cast<const int4*>(boxes + 4L * mi);
    if (x < b.x || x > b.z || y < b.y || y > b.w) continue;
    const unsigned long long key = ((unsigned long long)(unsigned)area[mi] << 32) | (unsigned)(0xFFFFFFFFu - (unsigned)gpos[k]);
    if (key >= best) continue;
    if (full_res(low_res + (long)mi * g.lr * g.lr, g, y, x) > thr) best = key;
  }
  if (best != ~0ull) atomicMin(&canvas[(long)(off_y + y) * ld_canvas + off_x + x], best);
}

__global__ void canvas_to_label_kernel(const unsigned long long* __restrict__ canvas, long n, int32_t* __restrict__ label) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long v = canvas[i];
  label[i] = v == ~0ull ? 0 : (int32_t)(0xFFFFFFFFu - (unsigned)(v & 0xFFFFFFFFull)) + 1;
}

int post_paint_canvas(const float* low_res, const int32_t* sel, const int32_t* gpos, int n_sel, const int32_t* boxes,
                      const int32_t* area, int in_h, int in_w, int out_h, int out_w, float thr, int off_x, int off_y,
                      unsigned long long* canvas, int ld_canvas, cudaStream_t st) {
  PostGeom g;
  if (make_geom(in_h, in_w, out_h, out_w, &g)) return -1;
  if (n_sel <= 0) return 0;
  paint_canvas_kernel<<<dim3((out_w + 255) / 256, out_h), 256, 0, st>>>(low_res, sel, gpos, n_sel, boxes, area, g, thr, off_x,
                                                                        off_y, canvas, ld_canvas);
  LAUNCH_CHECK("paint_canvas");
  return 0;
}

int post_canvas_to_label(const unsigned long long* canvas, long n, int32_t* label, cudaStream_t st) {
  canvas_to_label_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(canvas, n, label);
  LAUNCH_CHECK("canvas_to_label");
  return 0;
}

}  // namespace msam

// =================================================================================================================
// Mask NMS (util._batched_mask_nms / _calculate_ious_between_pred_masks / _calculate_iomin_between_pred_masks,
// util.py:1589-1676) on bit-packed masks: integer popcount intersections (exact), the reference's float32 ratios, box
// pre-filter, greedy suppression that keeps `iou <= thresh`.
namespace msam {

// uint8 masks [n, npix] -> bit-packed [n, words] (npix padded with zeros to 32*words) + areas
__global__ void pack_bits_kernel(const uint8_t* __restrict__ masks, int n, long npix, int words, uint32_t* __restrict__ bits,
                                 int32_t* __restrict__ areas) {
  const int mi = blockIdx.y;
  int cnt = 0;
  for (int wd = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); wd < words; wd += gridDim.x * (blockDim.x >> 5)) {
    const long px = (long)wd * 32 + (threadIdx.x & 31);
    const bool on = px < npix && masks[(long)mi * npix + px] != 0;
    const uint32_t w = __ballot_sync(0xffffffffu, on);
    if ((threadIdx.x & 31) == 0) {
      bits[(long)mi * words + wd] = w;
      cnt += __popc(w);
    }
  }
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&areas[mi], cnt);
}

// one warp per (i, j > i) pair with overlapping boxes: m[i][j] = m[j][i] = ratio
__global__ void mask_overlap_kernel(const uint32_t* __restrict__ bits, const int32_t* __restrict__ areas,
                                    const float* __restrict__ boxes /*xyxy*/, int n, int words, int iomin,
                                    float* __restrict__ m) {
  const long pair = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (pair >= (long)n * n) return;
  const int i = pair / n, j = pair % n, lane = threadIdx.x & 31;
  if (j <= i) {
    if (j == i && lane == 0) m[(long)i * n + i] = 1.0f;
    return;
  }
  const float w = fmaxf(fminf(boxes[4 * i + 2], boxes[4 * j + 2]) - fmaxf(boxes[4 * i], boxes[4 * j]), 0.f);
  const float h = fmaxf(fminf(boxes[4 * i + 3], boxes[4 * j + 3]) - fmaxf(boxes[4 * i + 1], boxes[4 * j + 1]), 0.f);
  float v = 0.f;
  if (w * h > 0.f) {  // warp-uniform
    int inter = 0;
    const uint32_t* a = bits + (long)i * words;
    const uint32_t* b = bits + (long)j * words;
    for (int k = lane; k < words; k += 32) inter += __popc(a[k] & b[k]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) inter += __shfl_xor_sync(0xffffffffu, inter, o);
    if (iomin) v = (float)inter / ((float)min(areas[i], areas[j]) + 1e-6f);
    else v = (float)inter / (float)(areas[i] + areas[j] - inter);
  }
  if (lane == 0) { m[(long)i * n + j] = v; m[(long)j * n + i] = v; }
}

// greedy NMS over a precomputed symmetric overlap matrix: descending score (index ascending on ties), keep <= thresh
__global__ void __launch_bounds__(1024)
matrix_nms_kernel(const float* __restrict__ m, const float* __restrict__ scores, int n, float thresh,
                  int32_t* __restrict__ keep, int32_t* __restrict__ n_keep) {
  extern __shared__ unsigned long long skey[];
  __shared__ int s_cnt;
  int npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  uint8_t* alive = reinterpret_cast<uint8_t*>(skey + npow2);
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int i = tid; i < npow2; i += nt)
    skey[i] = i < n ? (((unsigned long long)orderable(scores[i]) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)i)) : 0ull;
  __syncthreads();
  for (int k = 2; k <= npow2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < npow2; i += nt) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = skey[i], b = skey[ixj];
          if (((i & k) == 0) ? (a < b) : (a > b)) { skey[i] = b; skey[ixj] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = tid; i < n; i += nt) alive[i] = 1;
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  int cur = 0;
  while (true) {
    while (cur < n && !alive[cur]) ++cur;
    if (cur >= n) break;
    const int ci = (int)(0xFFFFFFFFu - (uint32_t)(skey[cur] & 0xFFFFFFFFull));
    if (tid == 0) keep[s_cnt++] = ci;
    __syncthreads();
    for (int j = cur + 1 + tid; j < n; j += nt) {
      if (!alive[j]) continue;
      const int cj = (int)(0xFFFFFFFFu - (uint32_t)(skey[j] & 0xFFFFFFFFull));
      if (m[(long)ci * n + cj] > thresh) alive[j] = 0;
    }
    ++cur;
    __syncthreads();
  }
  if (tid == 0) *n_keep = s_cnt;
}

int post_mask_nms(const uint8_t* masks, int n, int h, int w, const float* boxes_xyxy, const float* scores, float thresh,
                  int iomin, uint32_t* bits_ws, int32_t* areas, float* matrix_ws, int32_t* keep, int32_t* n_keep,
                  cudaStream_t st) {
  if (n <= 0) {
    cudaMemsetAsync(n_keep, 0, 4, st);
    return 0;
  }
  if (n > NMS_MAX) return set_error("mask_nms: n=%d exceeds %d", n, NMS_MAX);
  const long npix = (long)h * w;
  const int words = (int)((npix + 31) / 32);
  cudaMemsetAsync(areas, 0, (size_t)n * 4, st);
  pack_bits_kernel<<<dim3(64, n), 256, 0, st>>>(masks, n, npix, words, bits_ws, areas);
  LAUNCH_CHECK("pack_bits");
  const long pairs = (long)n * n;
  mask_overlap_kernel<<<(unsigned)((pairs + 7) / 8), 256, 0, st>>>(bits_ws, areas, boxes_xyxy, n, words, iomin, matrix_ws);
  LAUNCH_CHECK("mask_overlap");
  int npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(matrix_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    attr = true;
  }
  matrix_nms_kernel<<<1, 1024, (size_t)npow2 * 8 + n + 16, st>>>(matrix_ws, scores, n, thresh, keep, n_keep);
  LAUNCH_CHECK("matrix_nms");
  return 0;
}

}  // namespace msam

// =================================================================================================================
// mask_threshold = "auto" (inference._local_otsu_threshold, inference.py:70-134): per mask, the maximum over all pixels of
// the Otsu threshold of the 31x31 window (zero padded in the normalised domain) of the 64-bin quantised low-res logits.
// One CTA per mask, thread = column; the window histogram slides down the column (31 bins in, 31 out per step) in shared
// memory ([bin][thread] uint16: conflict free).  Arithmetic mirrors the reference run on the CPU: fp32 everywhere, cumsum
// accumulated in double and rounded to fp32 per element (ATen's CPU cumsum), first maximal bin on ties, no FMA contraction.
namespace msam {

__global__ void __launch_bounds__(256)
local_otsu_kernel(const float* __restrict__ low_res, float* __restrict__ thr_out) {
  constexpr int N = 256, WIN = 31, PAD = 15, NB = 64;
  const long mi = blockIdx.x;
  const float* lr = low_res + mi * N * N;
  extern __shared__ uint8_t osm[];
  uint8_t* bins = osm;                                            // [256][256] quantised image
  unsigned short* hist = reinterpret_cast<unsigned short*>(osm + N * N);  // [64][256]
  __shared__ float red[2][8];
  __shared__ int redi[8];
  const int tid = threadIdx.x;
  float mn = INFINITY, mx = -INFINITY;
  for (int i = tid; i < N * N; i += 256) { const float v = lr[i]; mn = fminf(mn, v); mx = fmaxf(mx, v); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
  if ((tid & 31) == 0) { red[0][tid >> 5] = mn; red[1][tid >> 5] = mx; }
  __syncthreads();
  mn = red[0][0]; mx = red[1][0];
  for (int w = 1; w < 8; ++w) { mn = fminf(mn, red[0][w]); mx = fmaxf(mx, red[1][w]); }
  const float range = fmaxf(__fsub_rn(mx, mn), 1e-6f);
  for (int i = tid; i < N * N; i += 256) {
    const float xn = __fdiv_rn(__fsub_rn(lr[i], mn), range);
    long b = (long)__fmul_rn(xn, 63.0f);
    b = b < 0 ? 0 : (b > 63 ? 63 : b);
    bins[i] = (uint8_t)b;
  }
  for (int b = 0; b < NB; ++b) hist[b * 256 + tid] = 0;
  __syncthreads();
  // this thread's column x: window columns [x-15, x+15]; out-of-image pixels are zeros of the normalised image -> bin 0
  const int x = tid;
  const int c0 = x - PAD, c1 = x + PAD;
  auto add_row = [&](int y, int delta) {
    if (y < 0 || y >= N) { hist[tid] = (unsigned short)(hist[tid] + delta * WIN); return; }
    const uint8_t* row = bins + y * N;
    int npad = 0;
    for (int c = c0; c <= c1; ++c) {
      if (c < 0 || c >= N) { ++npad; continue; }
      const int b = row[c];
      hist[b * 256 + tid] = (unsigned short)(hist[b * 256 + tid] + delta);
    }
    if (npad) hist[tid] = (unsigned short)(hist[tid] + delta * npad);
  };
  for (int y = -PAD; y <= PAD; ++y) add_row(y, 1);
  int tmax = 0;
  for (int y = 0; y < N; ++y) {
    // Otsu on the current window (961 samples)
    double om = 0.0, mu = 0.0;
    float muT;
    {
      double m2 = 0.0;
      for (int b = 0; b < NB; ++b) {
        const float p = __fdiv_rn((float)hist[b * 256 + tid], 961.0f);
        m2 += (double)__fmul_rn(p, (float)b);
      }
      muT = (float)m2;
    }
    float best = -1.0f;
    int tb = 0;
    for (int b = 0; b < NB; ++b) {
      const float p = __fdiv_rn((float)hist[b * 256 + tid], 961.0f);
      om += (double)p;
      mu += (double)__fmul_rn(p, (float)b);
      const float omega1 = (float)om, muf = (float)mu;
      const float omega2 = __fsub_rn(1.0f, omega1);
      const float mu1 = __fdiv_rn(muf, fmaxf(omega1, 1e-6f));
      const float mu2 = __fdiv_rn(__fsub_rn(muT, muf), fmaxf(omega2, 1e-6f));
      const float d = __fsub_rn(mu1, mu2);
      const float sig = __fmul_rn(__fmul_rn(omega1, omega2), __fmul_rn(d, d));
      if (sig > best) { best = sig; tb = b; }
    }
    tmax = max(tmax, tb);
    if (y + 1 < N) { add_row(y - PAD, -1); add_row(y + 1 + PAD, 1); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tmax = max(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
  if ((tid & 31) == 0) redi[tid >> 5] = tmax;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) tmax = max(tmax, redi[w]);
    const float tn = __fdiv_rn((float)tmax, 63.0f);
    thr_out[mi] = fmaxf(__fadd_rn(mn, __fmul_rn(tn, range)), 0.0f);
  }
}

int post_local_otsu(const float* low_res, int n, float* thr_out, cudaStream_t st) {
  if (n <= 0) return 0;
  constexpr int SMEM = 256 * 256 + 64 * 256 * 2;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(local_otsu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    attr = true;
  }
  local_otsu_kernel<<<n, 256, SMEM, st>>>(low_res, thr_out);
  LAUNCH_CHECK("local_otsu");
  return 0;
}

}  // namespace msam

// =================================================================================================================
// min_mask_region_area > 0 (AMGBase._postprocess_small_regions, instance_segmentation.py:146-186; the per-mask work is
// segment_anything.utils.amg.remove_small_regions: cv2.connectedComponentsWithStats(8-connectivity) on the mask ("islands")
// or its complement ("holes"), components below `area_thresh` are removed / filled; if every island is small the largest
// one (first in raster order on ties, like np.argmax over cv2's raster-ordered labels) is kept).  Batched over masks
// (blockIdx.y), union-find with atomicMin roots as in the label-image CC above, 8-connectivity.
namespace msam {

__global__ void rsr_init_kernel(const uint8_t* __restrict__ masks, long npix, int holes, int* __restrict__ parent,
                                int* __restrict__ size) {
  const long m = blockIdx.y;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const bool working = (masks[m * npix + i] != 0) != (holes != 0);
  parent[m * npix + i] = working ? (int)i : -1;
  size[m * npix + i] = 0;
}
__global__ void rsr_merge_kernel(int h, int w, int* __restrict__ parent_all) {
  const long m = blockIdx.y;
  const long npix = (long)h * w;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  int* parent = parent_all + m * npix;
  if (parent[i] < 0) return;
  const int x = (int)(i % w), y = (int)(i / w);
  if (x + 1 < w && parent[i + 1] >= 0) uf_union(parent, (int)i, (int)i + 1);
  if (y + 1 < h) {
    if (parent[i + w] >= 0) uf_union(parent, (int)i, (int)(i + w));
    if (x + 1 < w && parent[i + w + 1] >= 0) uf_union(parent, (int)i, (int)(i + w + 1));
    if (x > 0 && parent[i + w - 1] >= 0) uf_union(parent, (int)i, (int)(i + w - 1));
  }
}
__global__ void rsr_flatten_kernel(long npix, int* __restrict__ parent_all, int* __restrict__ size_all) {
  const long m = blockIdx.y;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  int* parent = parent_all + m * npix;
  if (parent[i] < 0) return;
  const int r = uf_find(parent, (int)i);
  parent[i] = r;
  atomicAdd(&size_all[m * npix + r], 1);
}
// per-mask statistics: st[0] = #small components, st[1] = #large components, best = packed (size, ~root) maximum
__global__ void rsr_stats_kernel(long npix, const int* __restrict__ parent_all, const int* __restrict__ size_all, int area_thresh,
                                 int* __restrict__ st, unsigned long long* __restrict__ best) {
  const long m = blockIdx.y;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  if (parent_all[m * npix + i] != (int)i) return;
  const int s = size_all[m * npix + i];
  atomicAdd(&st[2 * m + (s < area_thresh ? 0 : 1)], 1);
  atomicMax(&best[m], ((unsigned long long)(unsigned)s << 32) | (unsigned)(~(unsigned)i));
}
__global__ void rsr_apply_kernel(uint8_t* __restrict__ masks, long npix, int holes, const int* __restrict__ parent_all,
                                 const int* __restrict__ size_all, int area_thresh, const int* __restrict__ st,
                                 const unsigned long long* __restrict__ best, int32_t* __restrict__ changed) {
  const long m = blockIdx.y;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) changed[m] = st[2 * m] > 0;
  if (i >= npix || st[2 * m] == 0) return;  // no small component: the mask is returned unchanged
  const int r = parent_all[m * npix + i];
  if (holes) {
    if (r >= 0 && size_all[m * npix + r] < area_thresh) masks[m * npix + i] = 1;   // fill the small holes
  } else {
    bool keep = false;
    if (r >= 0) {
      if (st[2 * m + 1] > 0) keep = size_all[m * npix + r] >= area_thresh;
      else keep = r == (int)(~(unsigned)(best[m] & 0xffffffffu));                  // every island is small: keep the largest
    }
    masks[m * npix + i] = keep ? 1 : 0;
  }
}

// masks [n, h, w] uint8 (0/1) in place; changed [n]; ws: n * (2*h*w) ints + n * 4 ints
int post_remove_small_regions(uint8_t* masks, int n, int h, int w, int area_thresh, int holes, int32_t* changed, int32_t* ws,
                              cudaStream_t st) {
  if (n <= 0) return 0;
  const long npix = (long)h * w;
  if (npix >= (1l << 31)) return set_error("remove_small_regions: image too large");
  int* parent = ws;
  int* size = ws + (size_t)n * npix;
  int* stats = ws + 2 * (size_t)n * npix;
  unsigned long long* best = reinterpret_cast<unsigned long long*>(stats + 2 * n);  // 2n ints: 8-byte aligned with ws
  cudaMemsetAsync(stats, 0, (size_t)n * 4 * sizeof(int), st);
  const dim3 grid((unsigned)((npix + 255) / 256), n);
  rsr_init_kernel<<<grid, 256, 0, st>>>(masks, npix, holes, parent, size);
  LAUNCH_CHECK("rsr_init");
  rsr_merge_kernel<<<grid, 256, 0, st>>>(h, w, parent);
  LAUNCH_CHECK("rsr_merge");
  rsr_flatten_kernel<<<grid, 256, 0, st>>>(npix, parent, size);
  LAUNCH_CHECK("rsr_flatten");
  rsr_stats_kernel<<<grid, 256, 0, st>>>(npix, parent, size, area_thresh, stats, best);
  LAUNCH_CHECK("rsr_stats");
  rsr_apply_kernel<<<grid, 256, 0, st>>>(masks, npix, holes, parent, size, area_thresh, stats, best, changed);
  LAUNCH_CHECK("rsr_apply");
  return 0;
}

// batched_mask_to_box (_vendored.py:33-85) + area for materialised uint8 masks [n, h, w]: one CTA per mask
__global__ void __launch_bounds__(256)
mask_box_kernel(const uint8_t* __restrict__ masks, int h, int w, int32_t* __restrict__ boxes, int32_t* __restrict__ area) {
  const long m = blockIdx.x;
  const uint8_t* mk = masks + m * (long)h * w;
  int ar = 0, x0 = 1 << 30, y0 = 1 << 30, x1 = -1, y1 = -1;
  for (long i = threadIdx.x; i < (long)h * w; i += 256) {
    if (mk[i]) {
      const int x = (int)(i % w), y = (int)(i / w);
      ++ar; x0 = min(x0, x); x1 = max(x1, x); y0 = min(y0, y); y1 = max(y1, y);
    }
  }
  __shared__ int red[5][8];
  int vals[5] = {ar, x0, y0, x1, y1};
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    int v = vals[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int t = __shfl_xor_sync(0xffffffffu, v, o);
      v = (k == 0) ? v + t : ((k <= 2) ? min(v, t) : max(v, t));
    }
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int r[5];
    for (int k = 0; k < 5; ++k) {
      int v = red[k][0];
      for (int q = 1; q < 8; ++q) v = (k == 0) ? v + red[k][q] : ((k <= 2) ? min(v, red[k][q]) : max(v, red[k][q]));
      r[k] = v;
    }
    area[m] = r[0];
    const bool empty = r[0] == 0;
    boxes[m * 4 + 0] = empty ? 0 : r[1];
    boxes[m * 4 + 1] = empty ? 0 : r[2];
    boxes[m * 4 + 2] = empty ? 0 : r[3];
    boxes[m * 4 + 3] = empty ? 0 : r[4];
  }
}
int post_mask_boxes(const uint8_t* masks, int n, int h, int w, int32_t* boxes, int32_t* area, cudaStream_t st) {
  if (n <= 0) return 0;
  mask_box_kernel<<<n, 256, 0, st>>>(masks, h, w, boxes, area);
  LAUNCH_CHECK("mask_box");
  return 0;
}

}  // namespace msam
