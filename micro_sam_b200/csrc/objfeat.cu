// Per-object SAM embedding features of micro-sam's object classification (micro_sam/object_classification.py:20-217) on the
// device, for object_classification.compute_object_features and project_prediction_to_segmentation.
//
// One unit (image, slice or tile) pools a 256 x 64 x 64 embedding E over the objects of a segmentation of h x w, padded to the
// square side S = max(h, w) and resized to the (ry, rx) grid, exactly as skimage's resize computes it:
//   segmentation : nearest source index floor(((o + 0.5) * (S / r) - 0.5) + 0.5), in fp64 (scipy's zoom, order 0, grid mode)
//   embedding    : bilinear taps floor(c), floor(c) + 1 of c = (o + 0.5) * (64 / r) - 0.5, folded at the borders (mode
//                  'mirror'), after a Gaussian prefilter of sigma (64 / r - 1) / 2 on each axis with r < 64 (truncate 4)
// The upsampled ry x rx x 256 tensor is never built.  Upsampling is linear, so the sum of an object's upsampled embedding is
// sum_cell A[cell] * E[:, cell], with A[cell] the sum of the tap weights wy * wx its r-grid pixels put on that cell:
//   reset / axes : per-unit label boxes, and per axis the nearest index, taps and weights of every r-grid row / column
//   transpose    : a cell-major fp32 copy of E, so the contraction reads 1 KB rows (gauss_y / gauss_x: the prefilter,
//                  fp64 sums, written cell-major in fp32 as skimage's float32 filter output is)
//   scan         : r-grid bounding box and pixel count of every label (integer atomics), list of the labels present
//   label        : one CTA of 1024 threads per present label: A over the label's cells, gathered in a fixed order in fp64
//                  (shared memory), then sums[label, c] += sum_cell A[cell] * E[c, cell] in fp64 by four channel groups
// Every floating-point sum runs in a fixed order and the count atomics are integer, so a result is the same bit for bit from
// run to run.  Sums and areas accumulate across units in stream order; finish divides them once.
#include <algorithm>
#include <climits>
#include <cmath>

#include "engine.h"

namespace msam {
namespace {

constexpr int kG = 64;                 // embedding grid side
constexpr int kC = 256;                // embedding channels
constexpr int kCells = kG * kG;
constexpr int kFold = 2 * (kG - 1);    // period of the mirror extension
constexpr int kMaxR = 8192;            // resize grid side
constexpr int kMaxRadius = 4 * 32;     // Gaussian radius int(4 * sigma + 0.5) for r >= 1 (sigma <= 31.5)

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// scipy's 'mirror' extension of an index into [0, 64): ... 2 1 | 0 1 ... 63 | 62 61 ...
__device__ __forceinline__ int fold(int i) {
  i %= kFold;
  if (i < 0) i += kFold;
  return i > kG - 1 ? kFold - i : i;
}

struct Axis {
  int32_t* near;    // [kMaxR] source index of each r-grid index in the padded square, -1 in the padding
  int32_t* tap;     // [kMaxR] floor(c), unfolded
  double* frac;     // [kMaxR] c - floor(c): the weight of tap + 1
  int32_t* range;   // [kG][2] first and last r-grid index whose taps reach each cell
};

// workspace layout, see object_features_workspace
struct Ws {
  float* et;        // [kCells][kC] cell-major embedding after the prefilter
  double* tmp;      // [kCells][kC] after the prefilter's first axis
  Axis ax[2];
  int32_t* box;     // [n_ids][4] oy0, oy1, ox0, ox1 of each label on the r-grid of this unit
  int32_t* list;    // [n_ids] labels present in this unit, then their count
};
Ws carve(void* base, int n_ids) {
  char* p = (char*)base;
  Ws w;
  w.et = (float*)p; p += align256((size_t)4 * kCells * kC);
  w.tmp = (double*)p; p += align256((size_t)8 * kCells * kC);
  for (int a = 0; a < 2; ++a) {
    w.ax[a].near = (int32_t*)p; p += 4 * kMaxR;
    w.ax[a].tap = (int32_t*)p; p += 4 * kMaxR;
    w.ax[a].frac = (double*)p; p += 8 * kMaxR;
    w.ax[a].range = (int32_t*)p; p += 4 * 2 * kG;
  }
  w.box = (int32_t*)p; p += align256((size_t)16 * n_ids);
  w.list = (int32_t*)p;
  return w;
}

__global__ void reset_kernel(int n_ids, int32_t* box, int32_t* list) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n_ids; i += (long)gridDim.x * blockDim.x) {
    box[4 * i] = INT_MAX; box[4 * i + 1] = -1; box[4 * i + 2] = INT_MAX; box[4 * i + 3] = -1;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) list[n_ids] = 0;
}

// block 0: rows (extent h), block 1: columns (extent w), both of the padded square S
__global__ void axes_kernel(int S, int h, int w, int ry, int rx, Axis ay, Axis ax) {
  __shared__ int lo[kG], hi[kG];
  const Axis A = blockIdx.x == 0 ? ay : ax;
  const int r = blockIdx.x == 0 ? ry : rx, extent = blockIdx.x == 0 ? h : w;
  for (int a = threadIdx.x; a < kG; a += blockDim.x) { lo[a] = INT_MAX; hi[a] = -1; }
  __syncthreads();
  const double zs = (double)S / (double)r, ze = (double)kG / (double)r;
  for (int o = threadIdx.x; o < r; o += blockDim.x) {
    // scipy's NI_ZoomShift in grid mode: cc = (o + 0.5) * zoom - 0.5; order 0 takes floor(cc + 0.5).  No FMA contraction.
    const double oc = (double)o + 0.5;
    const int n = (int)floor(__dadd_rn(__dadd_rn(__dmul_rn(oc, zs), -0.5), 0.5));
    A.near[o] = n < extent ? n : -1;
    const double c = __dadd_rn(__dmul_rn(oc, ze), -0.5);
    const double f = floor(c);
    A.tap[o] = (int)f;
    A.frac[o] = c - f;
    atomicMin(&lo[fold((int)f)], o); atomicMax(&hi[fold((int)f)], o);
    atomicMin(&lo[fold((int)f + 1)], o); atomicMax(&hi[fold((int)f + 1)], o);
  }
  __syncthreads();
  for (int a = threadIdx.x; a < kG; a += blockDim.x) { A.range[2 * a] = lo[a]; A.range[2 * a + 1] = hi[a]; }
}

// scipy.ndimage._gaussian_kernel1d(sigma, 0, radius) into shared memory: exp(-0.5 / sigma^2 * k^2), normalised by its sum
__device__ void gauss_weights(double sigma, int radius, double* wt) {
  const double q = -0.5 / (sigma * sigma);
  for (int k = threadIdx.x; k <= 2 * radius; k += blockDim.x) wt[k] = exp(q * (double)((k - radius) * (k - radius)));
  __syncthreads();
  __shared__ double total;
  if (threadIdx.x == 0) {
    double s = 0;
    for (int k = 0; k <= 2 * radius; ++k) s += wt[k];
    total = s;
  }
  __syncthreads();
  for (int k = threadIdx.x; k <= 2 * radius; k += blockDim.x) wt[k] /= total;
  __syncthreads();
}

// tmp[(y, x)][c] = sum_k w[k] E[c][fold(y + k - radius)][x]   (radius 0: a transposed copy)
__global__ void gauss_y_kernel(const float* __restrict__ E, double sigma, int radius, double* __restrict__ tmp) {
  __shared__ double wt[2 * kMaxRadius + 1];
  if (radius > 0) gauss_weights(sigma, radius, wt);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kCells * kC; i += gridDim.x * blockDim.x) {
    const int c = i % kC, cell = i / kC, y = cell / kG, x = cell % kG;
    double s;
    if (radius == 0) {
      s = E[(size_t)c * kCells + cell];
    } else {
      s = 0;
      for (int k = 0; k <= 2 * radius; ++k) s += wt[k] * (double)E[(size_t)c * kCells + fold(y + k - radius) * kG + x];
    }
    tmp[i] = s;
  }
}

// et[(y, x)][c] = sum_k w[k] tmp[(y, fold(x + k - radius))][c]   (radius 0: a copy)
__global__ void gauss_x_kernel(const double* __restrict__ tmp, double sigma, int radius, float* __restrict__ et) {
  __shared__ double wt[2 * kMaxRadius + 1];
  if (radius > 0) gauss_weights(sigma, radius, wt);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kCells * kC; i += gridDim.x * blockDim.x) {
    const int c = i % kC, cell = i / kC, y = cell / kG, x = cell % kG;
    double s;
    if (radius == 0) {
      s = tmp[i];
    } else {
      s = 0;
      for (int k = 0; k <= 2 * radius; ++k) s += wt[k] * tmp[(size_t)(y * kG + fold(x + k - radius)) * kC + c];
    }
    et[i] = (float)s;
  }
}

// et[cell][c] = E[c][cell] through 32 x 32 shared-memory tiles
__global__ void transpose_kernel(const float* __restrict__ E, float* __restrict__ et) {
  __shared__ float t[32][33];
  const int cell0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) t[j][threadIdx.x] = E[(size_t)(c0 + j) * kCells + cell0 + threadIdx.x];
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) et[(size_t)(cell0 + j) * kC + c0 + threadIdx.x] = t[threadIdx.x][j];
}

__device__ __forceinline__ int label_at(const int32_t* __restrict__ seg, int ld, const Axis& ay, const Axis& ax, int oy, int ox) {
  const int sy = ay.near[oy], sx = ax.near[ox];
  return sy < 0 || sx < 0 ? 0 : seg[(size_t)sy * ld + sx];
}

__device__ __forceinline__ void note_label(int L, int y0, int y1, int x0, int x1, unsigned long long n, int n_ids, int32_t* box,
                                           int32_t* list, int64_t* areas) {
  int32_t* b = box + 4 * (size_t)(L - 1);
  if (atomicMin(&b[0], y0) == INT_MAX) list[atomicAdd(&list[n_ids], 1)] = L - 1;
  atomicMax(&b[1], y1); atomicMin(&b[2], x0); atomicMax(&b[3], x1);
  atomicAdd((unsigned long long*)&areas[L - 1], n);
}

// one thread per r-grid pixel; a warp whose pixels all carry one label reduces before its atomics (object interiors)
__global__ void scan_kernel(const int32_t* __restrict__ seg, int ld, int ry, int rx, int n_ids, Axis ay, Axis ax, int32_t* box,
                            int32_t* list, int64_t* areas) {
  const long total = (long)ry * rx;
  const int lane = threadIdx.x & 31;
  for (long base = (blockIdx.x * (long)blockDim.x + threadIdx.x) - lane; base < total; base += (long)gridDim.x * blockDim.x) {
    const long i = base + lane;
    int L = 0, oy = 0, ox = 0;
    if (i < total) {
      oy = (int)(i / rx); ox = (int)(i % rx);
      L = label_at(seg, ld, ay, ax, oy, ox);
      if (L < 1 || L > n_ids) L = 0;
    }
    const int L0 = __shfl_sync(0xffffffffu, L, 0);
    if (__all_sync(0xffffffffu, L == L0)) {
      if (L0 == 0) continue;
      int y0 = oy, y1 = oy, x0 = ox, x1 = ox;
      for (int o = 16; o; o >>= 1) {
        y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o)); y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
        x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o)); x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o));
      }
      if (lane == 0) note_label(L0, y0, y1, x0, x1, 32, n_ids, box, list, areas);
    } else if (L) {
      note_label(L, oy, oy, ox, ox, 1, n_ids, box, list, areas);
    }
  }
}

// weight of cell a in the two taps of r-grid index o
__device__ __forceinline__ double tap_weight(const Axis& A, int o, int a) {
  const int t = A.tap[o];
  const double f = A.frac[o];
  return (fold(t) == a ? 1.0 - f : 0.0) + (fold(t + 1) == a ? f : 0.0);
}

// cells an r-grid range [o0, o1] reaches on one axis: the unfolded taps span [tap(o0), tap(o1) + 1] within [-1, 64]
__device__ __forceinline__ void cell_span(const Axis& A, int o0, int o1, int& lo, int& hi) {
  const int t0 = A.tap[o0], t1 = A.tap[o1] + 1;
  lo = max(t0, 0); hi = min(t1, kG - 1);
  if (t0 < 0) hi = max(hi, fold(t0));
  if (t1 > kG - 1) lo = min(lo, fold(t1));
}

constexpr int kGroups = 4;                       // channel groups of the contraction
constexpr int kLabelThreads = kGroups * kC;

__global__ void __launch_bounds__(kLabelThreads) label_kernel(const int32_t* __restrict__ seg, int ld, int n_ids, Axis ay, Axis ax,
                                                              const int32_t* __restrict__ box, const int32_t* __restrict__ list,
                                                              const float* __restrict__ et, double* __restrict__ sums) {
  __shared__ double A[kCells];
  __shared__ double part[kGroups][kC];
  const int count = list[n_ids];
  for (int k = blockIdx.x; k < count; k += gridDim.x) {
    const int lab = list[k];
    const int32_t* b = box + 4 * (size_t)lab;
    const int oy0 = b[0], oy1 = b[1], ox0 = b[2], ox1 = b[3];
    int cy0, cy1, cx0, cx1;
    cell_span(ay, oy0, oy1, cy0, cy1);
    cell_span(ax, ox0, ox1, cx0, cx1);
    const int ncx = cx1 - cx0 + 1, ncell = (cy1 - cy0 + 1) * ncx;
    // A[cell] = sum over the label's pixels that tap the cell of wy * wx: rows outer, columns inner, ascending
    for (int q = threadIdx.x; q < ncell; q += blockDim.x) {
      const int a = cy0 + q / ncx, b = cx0 + q % ncx;
      const int ya = max(ay.range[2 * a], oy0), yb = min(ay.range[2 * a + 1], oy1);
      const int xa = max(ax.range[2 * b], ox0), xb = min(ax.range[2 * b + 1], ox1);
      double acc = 0;
      for (int oy = ya; oy <= yb; ++oy) {
        const int sy = ay.near[oy];
        if (sy < 0) continue;
        const int32_t* row = seg + (size_t)sy * ld;
        double racc = 0;
        for (int ox = xa; ox <= xb; ++ox) {
          const int sx = ax.near[ox];
          if (sx >= 0 && row[sx] == lab + 1) racc += tap_weight(ax, ox, b);
        }
        if (racc != 0) acc += tap_weight(ay, oy, a) * racc;
      }
      A[q] = acc;
    }
    __syncthreads();
    // sums[lab, c] += sum_cell A[cell] * E[c, cell]: channel c in each of kGroups thread groups, group g taking the cells
    // q = g, g + kGroups, ... with four loads in flight per step; the group partials are added in a fixed order
    const int c = threadIdx.x % kC, g = threadIdx.x / kC;
    double s = 0;
    int q = g;
    for (; q + 3 * kGroups < ncell; q += 4 * kGroups) {
      double w[4];
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int qq = q + j * kGroups;
        w[j] = A[qq];
        v[j] = w[j] != 0 ? et[(size_t)((cy0 + qq / ncx) * kG + cx0 + qq % ncx) * kC + c] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (w[j] != 0) s += w[j] * (double)v[j];
    }
    for (; q < ncell; q += kGroups) {
      const double w = A[q];
      if (w != 0) s += w * (double)et[(size_t)((cy0 + q / ncx) * kG + cx0 + q % ncx) * kC + c];
    }
    part[g][c] = s;
    __syncthreads();
    if (g == 0) sums[(size_t)lab * kC + c] += (part[0][c] + part[1][c]) + (part[2][c] + part[3][c]);
    __syncthreads();
  }
}

__global__ void finish_kernel(const double* __restrict__ sums, const int64_t* __restrict__ areas, int n_ids, int out_f64, void* out) {
  const long total = (long)n_ids * (kC + 1);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / (kC + 1);
    const int col = (int)(i % (kC + 1));
    const int64_t n = areas[row];
    const double v = col == 0 ? (double)n : n > 0 ? sums[row * kC + col - 1] / (double)n : 0.0;
    if (out_f64) ((double*)out)[i] = v;
    else ((float*)out)[i] = (float)v;
  }
}

__global__ void project_kernel(const int64_t* __restrict__ seg, long n, const int64_t* __restrict__ ids,
                               const int64_t* __restrict__ values, int n_ids, int64_t* __restrict__ out) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int64_t v = seg[i];
    int lo = 0, hi = n_ids;   // first id >= v
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ids[mid] < v) lo = mid + 1;
      else hi = mid;
    }
    out[i] = lo < n_ids && ids[lo] == v ? values[lo] : 0;
  }
}

int grid_for(long n, int cap) { return (int)std::max<long>(1, std::min<long>((n + 255) / 256, cap)); }

// skimage's anti-aliasing sigma of an axis resized from 64 to r, and scipy's radius int(truncate * sigma + 0.5); sigmas of at
// most 1e-15 are skipped by gaussian_filter
void prefilter(int r, double& sigma, int& radius) {
  sigma = std::max(0.0, ((double)kG / (double)r - 1.0) / 2.0);
  radius = sigma > 1e-15 ? (int)(4.0 * sigma + 0.5) : 0;
}

}  // namespace

int64_t object_features_workspace(int n_ids) {
  return (int64_t)(align256((size_t)4 * kCells * kC) + align256((size_t)8 * kCells * kC) + 2 * (16 * kMaxR + 8 * kG) +
                   align256((size_t)16 * n_ids) + (size_t)4 * (n_ids + 1));
}

int object_features(const float* emb, const int32_t* seg, int ld, int h, int w, int ry, int rx, int n_ids, void* workspace,
                    int64_t ws_bytes, double* sums, int64_t* areas, cudaStream_t st) {
  const int S = std::max(h, w);
  if (h <= 0 || w <= 0 || ld < w || ry < 1 || rx < 1 || ry > S || rx > S || ry > kMaxR || rx > kMaxR || n_ids < 0)
    return set_error("object_features: bad arguments h=%d w=%d ld=%d ry=%d rx=%d (1 <= r <= min(max(h, w), %d)) n_ids=%d", h, w,
                     ld, ry, rx, kMaxR, n_ids);
  if (ws_bytes < object_features_workspace(n_ids))
    return set_error("object_features: workspace of %lld bytes, need %lld", (long long)ws_bytes,
                     (long long)object_features_workspace(n_ids));
  if (n_ids == 0) return 0;
  const Ws ws = carve(workspace, n_ids);
  reset_kernel<<<grid_for(n_ids, 4096), 256, 0, st>>>(n_ids, ws.box, ws.list);
  LAUNCH_CHECK("objfeat_reset");
  axes_kernel<<<2, 256, 0, st>>>(S, h, w, ry, rx, ws.ax[0], ws.ax[1]);
  LAUNCH_CHECK("objfeat_axes");
  double sy, sx;
  int rdy, rdx;
  prefilter(ry, sy, rdy);
  prefilter(rx, sx, rdx);
  if (rdy == 0 && rdx == 0) {   // no axis is downsampled: skimage does not filter
    transpose_kernel<<<dim3(kCells / 32, kC / 32), dim3(32, 8), 0, st>>>(emb, ws.et);
    LAUNCH_CHECK("objfeat_transpose");
  } else {
    gauss_y_kernel<<<1024, 256, 0, st>>>(emb, sy, rdy, ws.tmp);
    LAUNCH_CHECK("objfeat_gauss_y");
    gauss_x_kernel<<<1024, 256, 0, st>>>(ws.tmp, sx, rdx, ws.et);
    LAUNCH_CHECK("objfeat_gauss_x");
  }
  scan_kernel<<<grid_for((long)ry * rx, 4096), 256, 0, st>>>(seg, ld, ry, rx, n_ids, ws.ax[0], ws.ax[1], ws.box, ws.list, areas);
  LAUNCH_CHECK("objfeat_scan");
  label_kernel<<<std::min(n_ids, 1024), kLabelThreads, 0, st>>>(seg, ld, n_ids, ws.ax[0], ws.ax[1], ws.box, ws.list, ws.et, sums);
  LAUNCH_CHECK("objfeat_label");
  return 0;
}

int object_features_finish(const double* sums, const int64_t* areas, int n_ids, int out_f64, void* out, cudaStream_t st) {
  if (n_ids < 0) return set_error("object_features_finish: bad n_ids=%d", n_ids);
  if (n_ids == 0) return 0;
  finish_kernel<<<grid_for((long)n_ids * (kC + 1), 4096), 256, 0, st>>>(sums, areas, n_ids, out_f64, out);
  LAUNCH_CHECK("objfeat_finish");
  return 0;
}

int project_labels(const int64_t* seg, int64_t n, const int64_t* ids, const int64_t* values, int n_ids, int64_t* out,
                   cudaStream_t st) {
  if (n < 0 || n_ids < 0) return set_error("project_labels: bad arguments n=%lld n_ids=%d", (long long)n, n_ids);
  if (n == 0) return 0;
  project_kernel<<<grid_for(n, 8192), 256, 0, st>>>(seg, n, ids, values, n_ids, out);
  LAUNCH_CHECK("project_labels");
  return 0;
}

}  // namespace msam
