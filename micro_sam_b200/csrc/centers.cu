// Object centres, bounding boxes and one-hot masks of a label image or volume on the device: micro-sam's
// util.get_centers_and_bounding_boxes and util.segmentation_to_one_hot (micro_sam/util.py:1283-1396), for util.py.
//
// Labels are int32 ids in [0, 2^31) (0 is background), 2-D [H, W] or 3-D [Z, H, W], C order.  The objects are the entries of a
// sorted table of the non-zero ids present; pixels map to table indices by binary search.  Mode "v" (DESIGN.md section 2):
//   boundary : the label image padded by one background pixel per side (never materialised: reads outside the image are 0);
//              a pixel of the padded grid is a boundary pixel when it is foreground and a cross / 6-neighbour inside the padded
//              grid carries another label (skimage's find_boundaries(mode="inner"), connectivity 1).  3-D stages
//              shared-memory tiles with a halo of 1.
//   EDT      : exact squared Euclidean distance of every pixel of the padded grid to the nearest boundary pixel, in int32: a
//              1-D distance pass along the first axis, then Meijster's separable lower-envelope pass along every further axis
//              (one line per thread, integer arithmetic only), saturating at INT32_MAX (only pixels with no boundary pixel in
//              reach, never an object pixel: see below).
//   reduce   : one pass over the labels; per object an atomicMax of the key (d2 << 32) | (0xFFFFFFFF - i), i the pixel's linear
//              index in the unpadded image: the largest distance, ties to the first pixel in raster order (np.argmax over the
//              bounding box).  Also min / max per axis (the box), the pixel count and int64 coordinate sums (mode "p").
//              A warp whose 32 pixels share one object reduces before its atomics.
// Key budget: the padded grid has fewer than 2^31 pixels, so i < 2^31 and the low word is > 2^31 - 1 (a set key is never 0).
// An object pixel's nearest boundary pixel lies on its own line along the shortest axis (the object is cut there by the
// padding at the latest), so d <= (n_min - 1) / 2 with n_min^ndim < 2^31: d2 < 2^29 fits the high word.  Distinct integer d2
// below 2^53 keep their order through the reference's fp64 sqrt, so comparing d2 is comparing the reference's distances.
// Every accumulation is an integer atomic: results are bit-identical from run to run.
#include "label_geom.cuh"

namespace msam {
namespace {

// centres ("v": the key's pixel, int32; "p": sums / count in fp64) and boxes (lo..., hi + 1...), ndim columns each
__global__ void finish_kernel(Grid g, int n_ids, int mode_v, Acc a, void* centers, int32_t* boxes) {
  const int nd = g.ndim, d0 = 3 - nd;
  for (long k = blockIdx.x * (long)blockDim.x + threadIdx.x; k < n_ids; k += (long)gridDim.x * blockDim.x) {
    for (int d = 0; d < nd; ++d) {
      boxes[k * 2 * nd + d] = a.lo[3 * k + d0 + d];
      boxes[k * 2 * nd + nd + d] = a.hi[3 * k + d0 + d] + 1;
    }
    if (mode_v) {
      const long i = (long)(0xFFFFFFFFu - (uint32_t)(a.key[k] & 0xFFFFFFFFull));
      const int c[3] = {(int)(i / ((long)g.H * g.W)), (int)(i / g.W % g.H), (int)(i % g.W)};
      for (int d = 0; d < nd; ++d) ((int32_t*)centers)[k * nd + d] = c[d0 + d];
    } else {
      const double n = (double)(long long)a.cnt[k];
      for (int d = 0; d < nd; ++d) ((double*)centers)[k * nd + d] = (double)(long long)a.sum[3 * k + d0 + d] / n;
    }
  }
}

// one-hot planes: each thread takes 4 consecutive pixels, looks their planes up once and writes the 4 floats of every plane
// (16-byte streaming stores when the plane size is a multiple of 4: the pass is bound by the n_planes * n * 4 bytes written)
template <bool kVec>
__global__ void one_hot_kernel(const int32_t* __restrict__ lab, long n, const int32_t* __restrict__ ids, int n_tab, int n_planes,
                               float* __restrict__ out) {
  const long quads = (n + 3) / 4;
  for (long qi = blockIdx.x * (long)blockDim.x + threadIdx.x; qi < quads; qi += (long)gridDim.x * blockDim.x) {
    int p[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long i = 4 * qi + j;
      const int32_t v = i < n ? lab[i] : 0;
      p[j] = v == 0 ? -1 : ids ? find_id(ids, n_tab, v) : (v <= n_planes ? v - 1 : -1);
    }
    for (int pl = 0; pl < n_planes; ++pl) {
      float* o = out + (long)pl * n + 4 * qi;
      if (kVec) {
        __stcs(reinterpret_cast<float4*>(o), make_float4(p[0] == pl, p[1] == pl, p[2] == pl, p[3] == pl));
      } else {
        for (int j = 0; j < 4 && 4 * qi + j < n; ++j) __stcs(o + j, (float)(p[j] == pl));
      }
    }
  }
}

// workspace layout: boundary mask, two int32 distance fields and the two envelope stacks over the padded grid, then the
// per-object accumulators
struct Ws {
  uint8_t* bnd;
  int32_t *da, *db, *sb, *tb;
  Acc acc;
};
Ws carve(void* base, const Grid& g, int n_ids) {
  char* p = (char*)base;
  const size_t pn = (size_t)g.pn();
  Ws w;
  w.bnd = (uint8_t*)p; p += align256(pn);
  w.da = (int32_t*)p; p += align256(4 * pn);
  w.db = (int32_t*)p; p += align256(4 * pn);
  w.sb = (int32_t*)p; p += align256(4 * pn);
  w.tb = (int32_t*)p; p += align256(4 * pn);
  w.acc.key = (unsigned long long*)p; p += align256(8 * (size_t)n_ids);
  w.acc.cnt = (unsigned long long*)p; p += align256(8 * (size_t)n_ids);
  w.acc.sum = (unsigned long long*)p; p += align256(24 * (size_t)n_ids);
  w.acc.lo = (int32_t*)p; p += align256(12 * (size_t)n_ids);
  w.acc.hi = (int32_t*)p;
  return w;
}
int64_t workspace_bytes(const Grid& g, int n_ids) {
  const size_t pn = (size_t)g.pn();
  return (int64_t)(align256(pn) + 4 * align256(4 * pn) + 2 * align256(8 * (size_t)n_ids) + align256(24 * (size_t)n_ids) +
                   align256(12 * (size_t)n_ids) + 12 * (size_t)n_ids);
}

int check_dims(const char* fn, int ndim, const int* dims) {
  if (!dims || (ndim != 2 && ndim != 3)) return set_error("%s: ndim=%d (2 or 3)", fn, ndim);
  long pn = 1;
  for (int d = 0; d < ndim; ++d) {
    if (dims[d] <= 0) return set_error("%s: dimension %d is %d", fn, d, dims[d]);
    pn *= (long)dims[d] + 2;
    if (pn >= (1l << 31)) return set_error("%s: the padded size exceeds the int32 linear index (2^31 - 1 pixels)", fn);
  }
  return 0;
}

}  // namespace
}  // namespace msam

using namespace msam;

extern "C" {

int64_t msam_centers_workspace(int ndim, const int* dims, int n_ids) {
  if (n_ids < 0 || !dims || (ndim != 2 && ndim != 3)) return -1;
  for (int d = 0; d < ndim; ++d)
    if (dims[d] <= 0) return -1;
  return workspace_bytes(make_grid(ndim, dims), n_ids);
}

int msam_centers_boxes(const int32_t* labels, int ndim, const int* dims, int mode, void* ws, int64_t ws_bytes, const int32_t* ids,
                       int n_ids, void* centers, int32_t* boxes, void* stream) {
  if (check_dims("msam_centers_boxes", ndim, dims)) return -1;
  if (mode != 'v' && mode != 'p') return set_error("msam_centers_boxes: mode %d ('v' or 'p')", mode);
  if (n_ids < 0) return set_error("msam_centers_boxes: n_ids=%d", n_ids);
  if (n_ids == 0) return 0;
  if (!labels || !ws || !ids || !centers || !boxes) return set_error("msam_centers_boxes: null argument");
  const Grid g = make_grid(ndim, dims);
  if (ws_bytes < workspace_bytes(g, n_ids))
    return set_error("msam_centers_boxes: workspace of %lld bytes, need %lld", (long long)ws_bytes,
                     (long long)workspace_bytes(g, n_ids));
  if ((uintptr_t)ws & 255) return set_error("msam_centers_boxes: workspace not 256-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const Ws w = carve(ws, g, n_ids);
  reset_kernel<<<blocks_for(n_ids), kThreads, 0, st>>>(n_ids, w.acc);
  LAUNCH_CHECK("centers_reset");
  const long warps = (long)g.Z * g.H * ((g.W + 31) / 32);
  const int rblocks = blocks_for(warps * 32, 1 << 20);
  if (mode == 'v') {
    if (launch_boundary(labels, g, w.bnd, st)) return -1;
    const int e[3] = {g.PZ, g.PH, g.PW};
    const int* ep = ndim == 3 ? e : e + 1;
    const int32_t* d2 = launch_edt(w.bnd, 1, ndim, ep, w.da, w.db, w.sb, w.tb, st);
    if (!d2) return -1;
    reduce_kernel<true><<<rblocks, kThreads, 0, st>>>(labels, g, ids, n_ids, d2, w.acc);
  } else {
    reduce_kernel<false><<<rblocks, kThreads, 0, st>>>(labels, g, ids, n_ids, nullptr, w.acc);
  }
  LAUNCH_CHECK("centers_reduce");
  finish_kernel<<<blocks_for(n_ids), kThreads, 0, st>>>(g, n_ids, mode == 'v', w.acc, centers, boxes);
  LAUNCH_CHECK("centers_finish");
  return 0;
}

int msam_op_label_boundaries(const int32_t* labels, int ndim, const int* dims, uint8_t* out, void* stream) {
  if (check_dims("msam_op_label_boundaries", ndim, dims)) return -1;
  if (!labels || !out) return set_error("msam_op_label_boundaries: null argument");
  return launch_boundary(labels, make_grid(ndim, dims), out, (cudaStream_t)stream);
}

int msam_op_edt_squared(const uint8_t* mask, int ndim, const int* dims, void* ws, int64_t ws_bytes, int32_t* out, void* stream) {
  if (!dims || ndim < 1 || ndim > 3) return set_error("msam_op_edt_squared: ndim=%d (1 to 3)", ndim);
  long n = 1;
  for (int d = 0; d < ndim; ++d) {
    if (dims[d] <= 0) return set_error("msam_op_edt_squared: dimension %d is %d", d, dims[d]);
    n *= dims[d];
    if (n >= (1l << 31)) return set_error("msam_op_edt_squared: more than 2^31 - 1 pixels");
  }
  if (!mask || !ws || !out) return set_error("msam_op_edt_squared: null argument");
  const size_t q = align256(4 * (size_t)n);
  if (ws_bytes < (int64_t)(3 * q)) return set_error("msam_op_edt_squared: workspace of %lld bytes, need %lld", (long long)ws_bytes,
                                                    (long long)(3 * q));
  if ((uintptr_t)ws & 255) return set_error("msam_op_edt_squared: workspace not 256-byte aligned");
  char* p = (char*)ws;
  int32_t* tmp = (int32_t*)p;
  int32_t* sb = (int32_t*)(p + q);
  int32_t* tb = (int32_t*)(p + 2 * q);
  // the passes alternate between out and tmp so that the last one lands in out
  const bool odd = ndim % 2 == 1;
  return launch_edt(mask, 0, ndim, dims, odd ? out : tmp, odd ? tmp : out, sb, tb, (cudaStream_t)stream) ? 0 : -1;
}

int msam_segmentation_one_hot(const int32_t* labels, int64_t n, const int32_t* ids, int n_tab, int n_planes, float* out, void* stream) {
  if (n < 0 || n_planes < 0 || (ids && n_tab < 0)) return set_error("msam_segmentation_one_hot: n=%lld n_planes=%d n_tab=%d",
                                                                     (long long)n, n_planes, n_tab);
  if (n == 0 || n_planes == 0) return 0;
  if (!labels || !out) return set_error("msam_segmentation_one_hot: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const long quads = (n + 3) / 4;
  if (n % 4 == 0 && ((uintptr_t)out & 15) == 0) one_hot_kernel<true><<<blocks_for(quads), kThreads, 0, st>>>(labels, n, ids, n_tab, n_planes, out);
  else one_hot_kernel<false><<<blocks_for(quads), kThreads, 0, st>>>(labels, n, ids, n_tab, n_planes, out);
  LAUNCH_CHECK("segmentation_one_hot");
  return 0;
}

}  // extern "C"
