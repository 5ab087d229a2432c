// Training prompts on the GPU (micro_sam/prompt_generators.py, micro_sam/training/util.py:153-265):
//   targets_kernel  : ConvertToSamInputs' one-hot targets (segmentation_to_one_hot), pixel counts and regionprops boxes of
//                     the sampled ids, in one pass over the label image; box_finish_kernel applies _distort_boxes
//   sample_points   : PointAndBoxPromptGenerator._sample_points -- positive points in the object, negative points in the
//                     ring (box widened by dilation_strength minus the dilated object), fill-up from the background
//   iterative       : IterativePromptGenerator.__call__ (2-D) -- one positive point in the false negatives (else the
//                     overlap), one negative point in the false positives (else the box ring, else the background); the
//                     prediction is the best low-res mask evaluated per pixel (postgeom.cuh) or a binary plane
//
// Random numbers: Philox4x32-10 keyed by the 64-bit seed, counter (draw, object, image, stream tag).  Every draw is a pure
// function of the seed and its counter, made by one thread; the per-pixel work only counts and locates pixels in raster
// order.  So the points depend on the seed and the inputs alone, not on the grid or on scheduling.  The only atomics are
// integer sums and min / max in targets_kernel, whose results do not depend on their order.
//
// Sampling a set S: thread 0 draws ranks in [0, |S|) (without replacement: the j-th draw is the r-th of the |S| - j ranks not
// yet taken, so the ordered k-tuple is uniform over distinct tuples, as numpy's choice(replace=False)); one block-wide pass
// over the image then finds the pixel of each rank among the members of S in raster order -- torch.where's order.
#include <algorithm>
#include <climits>

#include "engine.h"
#include "postgeom.cuh"

namespace msam {
namespace {

constexpr int kThreads = 512;         // sampling kernels: one CTA per object
constexpr int kChunk = 16;            // consecutive raster pixels per thread per tile
constexpr int kMaxPts = 64;           // points per object and set
constexpr int kMaxIds = 4096;         // sampled ids per image (targets_kernel keeps them in shared memory)

// stream tags of the Philox counter
enum : uint32_t { kTagBox = 0, kTagPos = 1, kTagNeg = 2, kTagFill = 3, kTagIterPos = 4, kTagIterNeg = 5 };

struct U4 { uint32_t x, y, z, w; };
__device__ __forceinline__ U4 philox4x32_10(U4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = U4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c;
}
// 64 random bits for draw `d` of object `obj` of image `img` in stream `tag`
__device__ __forceinline__ uint64_t draw64(uint64_t seed, uint32_t tag, uint32_t img, uint32_t obj, uint32_t d) {
  const U4 r = philox4x32_10(U4{d, obj, img, tag}, (uint32_t)seed, (uint32_t)(seed >> 32));
  return ((uint64_t)r.x << 32) | r.y;
}
// uniform integer in [0, n): the high word of u * n (bias < n / 2^64)
__device__ __forceinline__ int below(uint64_t u, int n) { return (int)__umul64hi(u, (uint64_t)n); }

// k ranks of a set of n members, kept sorted in rk[] with their draw order in slot[]
struct RankSet {
  int k;
  int rk[kMaxPts], slot[kMaxPts], pix[kMaxPts];
};
__device__ void draw_ranks(RankSet& s, int k, int n, bool replace, uint64_t seed, uint32_t tag, uint32_t img, uint32_t obj) {
  s.k = k;
  for (int j = 0; j < k; ++j) {
    int r = below(draw64(seed, tag, img, obj, j), replace ? n : n - j);
    int pos = j;
    if (replace) {
      for (int i = 0; i < j; ++i)
        if (s.rk[i] > r) { pos = i; break; }
    } else {                      // the r-th rank not taken yet
      for (int i = 0; i < j; ++i) {
        if (s.rk[i] <= r) ++r;
        else { pos = i; break; }
      }
    }
    for (int i = j; i > pos; --i) { s.rk[i] = s.rk[i - 1]; s.slot[i] = s.slot[i - 1]; }
    s.rk[pos] = r; s.slot[pos] = j;
  }
}

// Block-wide exclusive scan of NCH counters per thread; s_scan holds NCH x 32 ints.
template <int NCH>
__device__ __forceinline__ void block_scan(const int (&v)[NCH], int (&excl)[NCH], int (&tot)[NCH], int* s_scan) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int inc[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    int x = v[c];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    inc[c] = x;
  }
  __syncthreads();
  if (lane == 31) {
#pragma unroll
    for (int c = 0; c < NCH; ++c) s_scan[c * 32 + warp] = inc[c];
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    int before = 0, all = 0;
    for (int w = 0; w < nw; ++w) {
      const int t = s_scan[c * 32 + w];
      all += t;
      before += w < warp ? t : 0;
    }
    excl[c] = before + inc[c] - v[c];
    tot[c] = all;
  }
}

// For each channel c, find the pixels whose rank among the pixels with bit c of bits(p) set (raster order) is one of the
// ranks in sets[c]; writes them to sets[c].pix.  bits(p) < 16.  Stops as soon as every rank is found.
template <int NCH, class Bits>
__device__ void select_ranks(const Bits& bits, int npix, RankSet* sets, int* s_scan) {
  int base[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) base[c] = 0;
  for (int t0 = 0; t0 < npix; t0 += kThreads * kChunk) {
    bool done = true;             // block-uniform: base and the rank sets are the same in every thread
#pragma unroll
    for (int c = 0; c < NCH; ++c) done &= sets[c].k == 0 || sets[c].rk[sets[c].k - 1] < base[c];
    if (done) break;
    const int p0 = t0 + threadIdx.x * kChunk;
    uint64_t m = 0;
    int cnt[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) cnt[c] = 0;
#pragma unroll 4
    for (int i = 0; i < kChunk; ++i) {
      const int p = p0 + i;
      if (p < npix) {
        const uint32_t b = bits(p);
        m |= (uint64_t)b << (4 * i);
#pragma unroll
        for (int c = 0; c < NCH; ++c) cnt[c] += (b >> c) & 1;
      }
    }
    int excl[NCH], tot[NCH];
    block_scan<NCH>(cnt, excl, tot, s_scan);
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      RankSet& s = sets[c];
      const int lo = base[c] + excl[c], hi = lo + cnt[c];
      if (cnt[c] > 0 && s.k > 0) {
        int a = 0, e = s.k;       // first rank >= lo
        while (a < e) {
          const int mid = (a + e) >> 1;
          if (s.rk[mid] < lo) a = mid + 1; else e = mid;
        }
        if (a < s.k && s.rk[a] < hi) {
          int r = lo;
          for (int i = 0; i < kChunk && a < s.k; ++i) {
            if ((m >> (4 * i + c)) & 1) {
              while (a < s.k && s.rk[a] == r) { s.pix[a] = p0 + i; ++a; }
              ++r;
            }
          }
        }
      }
      base[c] += tot[c];
    }
  }
  __syncthreads();
}

__device__ __forceinline__ int block_sum(int v, int* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
  return t;
}

// ---------------------------------------------------------------------------------------------------------------------
// 1. targets, counts and boxes
__global__ void targets_init_kernel(int n, int32_t* counts, int32_t* acc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  counts[i] = 0;
  acc[i * 4 + 0] = INT_MAX; acc[i * 4 + 1] = INT_MAX; acc[i * 4 + 2] = -1; acc[i * 4 + 3] = -1;
}

// grid (x: pixel blocks, y: image).  Pixel p gets object o iff labels[p] == ids[o]; each warp combines the lanes of one object
// before the shared-memory atomics, each CTA adds its partial results to the global ones once.
template <typename L>
__global__ void __launch_bounds__(256)
targets_kernel(const L* __restrict__ labels, int H, int W, const int64_t* __restrict__ ids, const int32_t* __restrict__ n_ids,
               int n_obj, uint8_t* __restrict__ targets, int32_t* __restrict__ counts, int32_t* __restrict__ acc) {
  extern __shared__ int64_t s_ids[];                       // [n_obj] ids, then [n_obj][5] int partials
  int* s_acc = reinterpret_cast<int*>(s_ids + n_obj);
  const int b = blockIdx.y, n = min(n_ids[b], n_obj);
  const long HW = (long)H * W;
  for (int o = threadIdx.x; o < n_obj; o += blockDim.x) {
    s_ids[o] = ids[(long)b * n_obj + o];
    s_acc[o * 5 + 0] = 0; s_acc[o * 5 + 1] = INT_MAX; s_acc[o * 5 + 2] = INT_MAX; s_acc[o * 5 + 3] = -1; s_acc[o * 5 + 4] = -1;
  }
  __syncthreads();
  const L* lab = labels + b * HW;
  uint8_t* tg = targets + (long)b * n_obj * HW;
  const int lane = threadIdx.x & 31;
  for (long p0 = (long)blockIdx.x * blockDim.x; p0 < HW; p0 += (long)gridDim.x * blockDim.x) {
    const long p = p0 + threadIdx.x;
    int idx = -1;
    if (p < HW) {
      const int64_t v = (int64_t)lab[p];
      int a = 0, e = n;
      while (a < e) {
        const int mid = (a + e) >> 1;
        if (s_ids[mid] < v) a = mid + 1; else e = mid;
      }
      idx = (a < n && s_ids[a] == v) ? a : -1;
      for (int o = 0; o < n_obj; ++o) tg[(long)o * HW + p] = (uint8_t)(o == idx);
    }
    const unsigned grp = __match_any_sync(0xffffffffu, idx);
    const int y = (int)(p / W), x = (int)(p % W);
    const int cnt = __popc(grp);
    const int ymin = __reduce_min_sync(grp, y), xmin = __reduce_min_sync(grp, x);
    const int ymax = __reduce_max_sync(grp, y), xmax = __reduce_max_sync(grp, x);
    if (idx >= 0 && lane == __ffs(grp) - 1) {
      int* a = s_acc + idx * 5;
      atomicAdd(a + 0, cnt); atomicMin(a + 1, ymin); atomicMin(a + 2, xmin); atomicMax(a + 3, ymax); atomicMax(a + 4, xmax);
    }
  }
  __syncthreads();
  for (int o = threadIdx.x; o < n; o += blockDim.x) {
    const int* a = s_acc + o * 5;
    if (a[0] == 0) continue;
    const long k = (long)b * n_obj + o;
    atomicAdd(counts + k, a[0]);
    atomicMin(acc + k * 4 + 0, a[1]); atomicMin(acc + k * 4 + 1, a[2]); atomicMax(acc + k * 4 + 2, a[3]); atomicMax(acc + k * 4 + 3, a[4]);
  }
}

// regionprops bbox (min_row, min_col, max_row + 1, max_col + 1); empty objects get (0, 0, 0, 0).  With distortion >= 0, then
// ConvertToSamInputs._distort_boxes (training/util.py:174-185) in its float64 arithmetic with numpy's uniform(0, f) = f * U,
// U from draws 0..3 (y0, y1, x0, x1) of the box stream, and Python's round (half to even: rint).
__global__ void box_finish_kernel(int n, int n_per_img, int H, int W, double distortion, uint64_t seed, const int32_t* acc, int32_t* boxes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int y0 = acc[i * 4 + 0], x0 = acc[i * 4 + 1], y1 = acc[i * 4 + 2] + 1, x1 = acc[i * 4 + 3] + 1;
  if (acc[i * 4 + 2] < 0) { y0 = x0 = y1 = x1 = 0; }
  else if (distortion >= 0.0) {
    const uint32_t img = i / n_per_img, obj = i % n_per_img;
    double u[4];
    for (int d = 0; d < 4; ++d) u[d] = distortion * ((double)(draw64(seed, kTagBox, img, obj, d) >> 11) * 0x1.0p-53);
    const double ly = (double)(y1 - y0), lx = (double)(x1 - x0);
    const int ny0 = (int)rint(fmax(0.0, (double)y0 - u[0] * ly));
    const int ny1 = (int)rint(fmin((double)H, (double)y1 + u[1] * ly));
    const int nx0 = (int)rint(fmax(0.0, (double)x0 - u[2] * lx));
    const int nx1 = (int)rint(fmin((double)W, (double)x1 + u[3] * lx));
    y0 = ny0; y1 = ny1; x0 = nx0; x1 = nx1;
  }
  boxes[i * 4 + 0] = y0; boxes[i * 4 + 1] = x0; boxes[i * 4 + 2] = y1; boxes[i * 4 + 3] = x1;
}

// ---------------------------------------------------------------------------------------------------------------------
// 2. point-and-box sampling.  The (2 ds + 1)^2 square dilation (= ds iterations of a 3 x 3 dilation, nothing outside the
// image) is separable: a row pass and a column pass of windowed ORs.
__global__ void dilate_rows_kernel(const uint8_t* __restrict__ in, long total, int W, int ds, uint8_t* __restrict__ out) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const uint8_t* row = in + (i - x);
    const int a = max(x - ds, 0), e = min(x + ds, W - 1);
    uint8_t v = 0;
    for (int j = a; j <= e && !v; ++j) v = row[j] != 0;
    out[i] = v;
  }
}
__global__ void dilate_cols_kernel(const uint8_t* __restrict__ in, long total, int H, int W, int ds, uint8_t* __restrict__ out) {
  const long HW = (long)H * W;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long q = i % HW;
    const int y = (int)(q / W);
    const uint8_t* col = in + (i - (long)y * W);
    const int a = max(y - ds, 0), e = min(y + ds, H - 1);
    uint8_t v = 0;
    for (int j = a; j <= e && !v; ++j) v = col[(long)j * W] != 0;
    out[i] = v;
  }
}

// One CTA per object.  Points: [n_pos positives (the centre first when given)] [negatives from the ring] [fill-up from the
// background], labels 1 / 0 / 0.  An object without pixels (the reference raises) gets coordinates -1.
__global__ void __launch_bounds__(kThreads)
sample_points_kernel(const uint8_t* __restrict__ targets, const uint8_t* __restrict__ dilated, const int32_t* __restrict__ counts,
                     const int32_t* __restrict__ boxes, const int32_t* __restrict__ centers, int n_per_img, int H, int W, int n_pos,
                     int n_neg, int ds, uint64_t seed, int32_t* __restrict__ coords, int32_t* __restrict__ labels) {
  __shared__ RankSet sets[3];
  __shared__ int s_scan[3 * 32];
  __shared__ int s_fail;
  const int n = blockIdx.x, HW = H * W, np = n_pos + n_neg;
  const uint32_t img = n / n_per_img, obj = n % n_per_img;
  const uint8_t* tg = targets + (long)n * HW;
  const uint8_t* dil = dilated ? dilated + (long)n * HW : tg;
  const int* bx = boxes + n * 4;
  const int r0 = max(bx[0] - ds, 0), c0 = max(bx[1] - ds, 0), r1 = min(bx[2] + ds, H), c1 = min(bx[3] + ds, W);
  // _sample_negative_points: |widened box - dilated object|
  auto ring = [&](int p) -> uint32_t {
    const int y = p / W, x = p - y * W;
    const bool inbox = y >= r0 && y < r1 && x >= c0 && x < c1;
    return inbox != (dil[p] != 0);
  };
  int n_ring = 0;
  if (n_neg > 0) {
    int c = 0;
    for (int p = threadIdx.x; p < HW; p += kThreads) c += ring(p);
    n_ring = block_sum(c, s_scan);
  }
  const int cnt = counts[n], has_c = centers != nullptr && n_pos > 0;
  if (threadIdx.x == 0) {
    int fail = 0;
    const int kpos = n_pos - has_c;
    if (kpos > 0 && cnt == 0) fail = 1;
    draw_ranks(sets[0], fail ? 0 : kpos, cnt, kpos > cnt, seed, kTagPos, img, obj);
    const int kneg = min(n_neg, n_ring);
    draw_ranks(sets[1], kneg, n_ring, false, seed, kTagNeg, img, obj);
    const int kfill = n_neg - kneg, n_bg = HW - cnt;
    if (kfill > n_bg) fail = 1;
    draw_ranks(sets[2], fail ? 0 : kfill, n_bg, false, seed, kTagFill, img, obj);
    s_fail = fail;
  }
  __syncthreads();
  if (!s_fail) {
    auto bits = [&](int p) -> uint32_t {
      const uint32_t t = tg[p] != 0;
      return t | (n_neg > 0 ? ring(p) << 1 : 0u) | ((t ^ 1u) << 2);
    };
    select_ranks<3>(bits, HW, sets, s_scan);
  }
  int32_t* out = coords + (long)n * np * 2;
  for (int j = threadIdx.x; j < np; j += kThreads) labels[(long)n * np + j] = j < n_pos ? 1 : 0;
  if (s_fail) {
    for (int j = threadIdx.x; j < np * 2; j += kThreads) out[j] = -1;
    return;
  }
  if (threadIdx.x == 0 && has_c) { out[0] = centers[n * 2 + 1]; out[1] = centers[n * 2 + 0]; }
  const int off[3] = {has_c, n_pos, n_pos + sets[1].k};
  for (int c = 0; c < 3; ++c) {
    const RankSet& s = sets[c];
    for (int j = threadIdx.x; j < s.k; j += kThreads) {
      const int q = off[c] + s.slot[j], p = s.pix[j];
      out[q * 2 + 0] = p % W; out[q * 2 + 1] = p / W;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 3. iterative sampling.  One CTA per object: argmax of the predicted IoUs (first maximum, NaN counts as the maximum as in
// torch), one counting pass (false negatives, false positives, overlap, target pixels and box), the fallback chain, one
// locating pass for the two drawn ranks.  An object without target pixels (the reference raises) gets coordinates -1.
__global__ void __launch_bounds__(kThreads)
iterative_kernel(const uint8_t* __restrict__ targets, const float* __restrict__ low_res, const float* __restrict__ iou, int M,
                 const uint8_t* __restrict__ pred, PostGeom g, int n_per_img, uint64_t seed, int32_t* __restrict__ coords,
                 int32_t* __restrict__ labels) {
  __shared__ RankSet sets[2];
  __shared__ int s_scan[2 * 32];
  __shared__ int s_red[8][32];
  __shared__ int s_best, s_mode[2];
  const int n = blockIdx.x, H = g.out_h, W = g.out_w, HW = H * W;
  const uint32_t img = n / n_per_img, obj = n % n_per_img;
  const uint8_t* tg = targets + (long)n * HW;
  if (threadIdx.x == 0) {
    int best = 0;
    if (iou) {
      float bv = iou[(long)n * M];
      for (int m = 1; m < M; ++m) {
        const float v = iou[(long)n * M + m];
        if (!(bv != bv) && (v > bv || v != v)) { bv = v; best = m; }
      }
    }
    s_best = best;
  }
  __syncthreads();
  const float* lr = low_res ? low_res + ((long)n * M + s_best) * g.lr * g.lr : nullptr;
  const uint8_t* pd = pred ? pred + (long)n * HW : nullptr;
  auto predicted = [&](int p, int y, int x) -> bool { return pd ? pd[p] != 0 : full_res(lr, g, y, x) > 0.f; };

  int fn = 0, fp = 0, ov = 0, nt = 0, ymin = INT_MAX, xmin = INT_MAX, ymax = -1, xmax = -1;
  for (int p = threadIdx.x; p < HW; p += kThreads) {
    const int y = p / W, x = p - y * W;
    const bool t = tg[p] != 0, v = predicted(p, y, x);
    fn += t & !v; fp += v & !t; ov += v & t; nt += t;
    if (t) { ymin = min(ymin, y); xmin = min(xmin, x); ymax = max(ymax, y); xmax = max(xmax, x); }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int r[8] = {__reduce_add_sync(0xffffffffu, fn), __reduce_add_sync(0xffffffffu, fp), __reduce_add_sync(0xffffffffu, ov),
              __reduce_add_sync(0xffffffffu, nt), __reduce_min_sync(0xffffffffu, ymin), __reduce_min_sync(0xffffffffu, xmin),
              __reduce_max_sync(0xffffffffu, ymax), __reduce_max_sync(0xffffffffu, xmax)};
  if (lane == 0)
    for (int i = 0; i < 8; ++i) s_red[i][warp] = r[i];
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 8; ++i) {
      int a = s_red[i][0];
      for (int w = 1; w < kThreads / 32; ++w) a = i < 4 ? a + s_red[i][w] : i < 6 ? min(a, s_red[i][w]) : max(a, s_red[i][w]);
      r[i] = a;
    }
    // _get_positive_points: false negatives, else the overlap
    const int pos_mode = r[0] > 0 ? 0 : 1, n_pos = r[0] > 0 ? r[0] : r[2];
    // _get_negative_points: false positives, else _get_negative_locations_in_obj_bbox (box [min - 3, max + 1 + 3) clipped,
    // minus the target), else the true background
    int neg_mode = 0, n_neg = r[1];
    if (n_neg == 0 && r[3] > 0) {
      const int a = max(r[4] - 3, 0), c = max(r[5] - 3, 0), e = min(r[6] + 4, H), f = min(r[7] + 4, W);
      neg_mode = 1; n_neg = (e - a) * (f - c) - r[3];
    }
    if (n_neg == 0) { neg_mode = 2; n_neg = HW - r[3]; }
    s_red[0][0] = r[4]; s_red[1][0] = r[5]; s_red[2][0] = r[6]; s_red[3][0] = r[7];
    const bool ok = n_pos > 0 && n_neg > 0;
    s_mode[0] = ok ? pos_mode : -1; s_mode[1] = neg_mode;
    sets[0].k = sets[1].k = 0;
    if (ok) {
      draw_ranks(sets[0], 1, n_pos, false, seed, kTagIterPos, img, obj);
      draw_ranks(sets[1], 1, n_neg, false, seed, kTagIterNeg, img, obj);
    }
  }
  __syncthreads();
  const int pos_mode = s_mode[0], neg_mode = s_mode[1];
  int32_t* out = coords + (long)n * 4;
  if (threadIdx.x < 2) labels[(long)n * 2 + threadIdx.x] = threadIdx.x == 0 ? 1 : 0;
  if (pos_mode < 0) {
    if (threadIdx.x < 4) out[threadIdx.x] = -1;
    return;
  }
  const int ra = max(s_red[0][0] - 3, 0), ca = max(s_red[1][0] - 3, 0), re = min(s_red[2][0] + 4, H), ce = min(s_red[3][0] + 4, W);
  auto bits = [&](int p) -> uint32_t {
    const int y = p / W, x = p - y * W;
    const bool t = tg[p] != 0, v = predicted(p, y, x);
    const bool in_pos = pos_mode == 0 ? (t && !v) : (t && v);
    const bool in_neg = neg_mode == 0 ? (v && !t) : neg_mode == 1 ? (!t && y >= ra && y < re && x >= ca && x < ce) : !t;
    return (uint32_t)in_pos | ((uint32_t)in_neg << 1);
  };
  select_ranks<2>(bits, HW, sets, s_scan);
  if (threadIdx.x < 2) {
    const int p = sets[threadIdx.x].pix[0];
    out[threadIdx.x * 2 + 0] = p % W; out[threadIdx.x * 2 + 1] = p / W;
  }
}

}  // namespace

int prompt_targets(const void* labels, int label_dtype, int B, int H, int W, const int64_t* ids, const int32_t* n_ids, int n_obj,
                   double box_distortion, uint64_t seed, uint8_t* targets, int32_t* counts, int32_t* boxes, cudaStream_t st) {
  if (B <= 0 || H <= 0 || W <= 0 || n_obj <= 0 || n_obj > kMaxIds || (label_dtype != 0 && label_dtype != 1))
    return set_error("prompt_targets: bad arguments B=%d H=%d W=%d n_obj=%d (<= %d) dtype=%d", B, H, W, n_obj, kMaxIds, label_dtype);
  const int n = B * n_obj;
  const long HW = (long)H * W;
  // boxes doubles as the min / max accumulator until box_finish_kernel overwrites it with the final boxes
  targets_init_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, counts, boxes);
  LAUNCH_CHECK("prompt_targets_init");
  const size_t smem = (size_t)n_obj * (sizeof(int64_t) + 5 * sizeof(int));
  const int gx = (int)std::min<long>((HW + 255) / 256, 1024);
  prof_begin(st, "prompt_targets", 0.0, (double)B * HW * (label_dtype ? 8 : 4) + (double)n * HW);
  if (label_dtype == 0) {
    cudaFuncSetAttribute(targets_kernel<int32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    targets_kernel<int32_t><<<dim3(gx, B), 256, smem, st>>>((const int32_t*)labels, H, W, ids, n_ids, n_obj, targets, counts, boxes);
  } else {
    cudaFuncSetAttribute(targets_kernel<int64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    targets_kernel<int64_t><<<dim3(gx, B), 256, smem, st>>>((const int64_t*)labels, H, W, ids, n_ids, n_obj, targets, counts, boxes);
  }
  prof_end(st);
  LAUNCH_CHECK("prompt_targets");
  box_finish_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, n_obj, H, W, box_distortion, seed, boxes, boxes);
  LAUNCH_CHECK("prompt_box_finish");
  return 0;
}

int prompt_sample_points(const uint8_t* targets, const int32_t* counts, const int32_t* boxes, const int32_t* centers, int n, int n_per_img,
                         int H, int W, int n_pos, int n_neg, int dilation, uint64_t seed, uint8_t* scratch, int32_t* coords,
                         int32_t* labels, cudaStream_t st) {
  if (n < 0 || n_per_img <= 0 || H <= 0 || W <= 0 || (long)H * W > INT_MAX || n_pos < 0 || n_neg < 0 || dilation < 0 ||
      n_pos + n_neg > kMaxPts || n_pos + n_neg == 0)
    return set_error("prompt_sample_points: bad arguments n=%d H=%d W=%d n_pos=%d n_neg=%d (1..%d points) dilation=%d", n, H, W, n_pos,
                     n_neg, kMaxPts, dilation);
  if (n == 0) return 0;
  const long total = (long)n * H * W;
  const uint8_t* dil = nullptr;
  if (n_neg > 0 && dilation > 0) {
    if (!scratch) return set_error("prompt_sample_points: the dilation needs a scratch buffer of 2 * n * H * W bytes");
    const int blocks = (int)std::min<long>((total + 255) / 256, 4096);
    dilate_rows_kernel<<<blocks, 256, 0, st>>>(targets, total, W, dilation, scratch);
    LAUNCH_CHECK("prompt_dilate_rows");
    dilate_cols_kernel<<<blocks, 256, 0, st>>>(scratch, total, H, W, dilation, scratch + total);
    LAUNCH_CHECK("prompt_dilate_cols");
    dil = scratch + total;
  }
  prof_begin(st, "prompt_sample_points", 0.0, (double)total * (n_neg > 0 ? 3 : 1));
  sample_points_kernel<<<n, kThreads, 0, st>>>(targets, dil, counts, boxes, centers, n_per_img, H, W, n_pos, n_neg, dilation, seed,
                                               coords, labels);
  prof_end(st);
  LAUNCH_CHECK("prompt_sample_points");
  return 0;
}

int prompt_iterative(const uint8_t* targets, const float* low_res, const float* iou, int M, const uint8_t* pred, int n, int n_per_img,
                     int in_h, int in_w, int H, int W, uint64_t seed, int32_t* coords, int32_t* labels, cudaStream_t st) {
  if (n < 0 || n_per_img <= 0 || H <= 0 || W <= 0 || (long)H * W > INT_MAX || (!low_res == !pred) || (low_res && M <= 0) ||
      (low_res && M > 1 && !iou))
    return set_error("prompt_iterative: bad arguments n=%d M=%d H=%d W=%d (exactly one of low_res / pred; iou needed for M > 1)", n, M, H,
                     W);
  PostGeom g{};
  if (low_res) {
    if (make_geom(in_h, in_w, H, W, &g)) return -1;
  } else {
    g.out_h = H; g.out_w = W; M = 1;
  }
  if (n == 0) return 0;
  prof_begin(st, "prompt_iterative", 0.0, (double)n * H * W * 2 + (low_res ? (double)n * 65536.0 * 4 : (double)n * H * W * 2));
  iterative_kernel<<<n, kThreads, 0, st>>>(targets, low_res, iou, M, pred, g, n_per_img, seed, coords, labels);
  prof_end(st);
  LAUNCH_CHECK("prompt_iterative");
  return 0;
}

}  // namespace msam
