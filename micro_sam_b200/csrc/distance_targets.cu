// The UNETR decoder's training targets on the device: torch_em's PerObjectDistanceTransform (used by micro-sam's train_sam,
// default_sam_dataset and ResizeLabelTrafo) for a batch of B 2-D label images of one size, for training.py.  The restatement
// and its unpinned points are in DESIGN.md section 2.  Passes:
//   objects  : post_label_objects (postprocess.cu): 8-connected components of equal ids (or the distinct ids), size filter,
//              numbered 1..N over the batch, image by image.  Object k has label k + 1, so no id table is searched.
//   boundary : label_geom.cuh's boundary2d_kernel on the unpadded images (pad 0): an object gets no boundary where it meets
//              the image edge.
//   EDT      : the exact squared distance of every pixel to the nearest boundary pixel of its own image (launch_edt from
//              axis 1).  At the pixels of an object this equals the EDT over the object's bounding box that torch_em computes
//              per object (DESIGN.md section 2 has the proof), so one pass over the batch replaces one EDT per object.
//   reduce   : label_geom.cuh's reduce_kernel<true>: per object the box, the pixel count, int64 coordinate sums and the key
//              (d2 << 32) | (0xFFFFFFFF - i), i the pixel's linear index in the batch: the largest distance, ties to the first
//              pixel in raster order (np.argmax over the crop).
//   finish   : per object the centre rint(sums / count) (fp64, ties to even as np.round); when that pixel is not in the object
//              the key's pixel, or the box's first pixel when every object pixel is a boundary pixel (torch_em's argmax over an
//              all-zero crop).
//   centre   : per object the largest |p - c|^2 over its pixels, warp-aggregated integer atomicMax.
//   write    : the selected channels, 4 pixels per thread with 16-byte streaming stores when H * W is a multiple of 4.
// Key budget: B * H * W < 2^31, so i < 2^31 and the low word is > 2^31 - 1.  Unpadded, an object pixel's nearest boundary
// pixel can lie a whole image side away (a 1 x W strip), so the sides are bounded by 32768: d2 <= 2 * 32767^2 < 2^31 fits
// the high word.  The EDT saturates at INT32_MAX only in an image without any boundary pixel, i.e. one object covering the
// whole image, whose boundary distances are defined as 0.
// Every reduction is an integer atomic and each output value is one correctly rounded fp32 (or fp64 -> fp32) expression of
// integers: the targets are bit-identical from run to run.
#include "engine.h"
#include "label_geom.cuh"

namespace msam {
namespace {

constexpr int kMaxSide = 32768;
constexpr int kChInstances = 1, kChForeground = 2, kChDistances = 4, kChBoundary = 8;

struct Obj {
  int32_t* ctr;    // [N][2] centre (y, x) in image coordinates
  int32_t* bmax;   // [N] largest boundary d2 over the object
  int32_t* cmax;   // [N] largest centre d2 over the object
  int32_t* off;    // [B] objects in the images before b (set only for images with objects)
};

__global__ void to_int32_kernel(const int64_t* __restrict__ in, long n, int32_t* __restrict__ out) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) out[i] = (int32_t)in[i];
}

__global__ void dt_reset_kernel(const int* __restrict__ n_obj, Acc a) {
  const int n = *n_obj;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    a.key[i] = 0; a.cnt[i] = 0;
    for (int d = 0; d < 3; ++d) { a.lo[3 * i + d] = INT_MAX; a.hi[3 * i + d] = -1; a.sum[3 * i + d] = 0; }
  }
}

__device__ __forceinline__ uint32_t unsat(uint32_t d2) { return d2 == (uint32_t)kInf ? 0u : d2; }

__global__ void dt_finish_kernel(const int32_t* __restrict__ lab, Grid g, const int* __restrict__ n_obj, Acc a, Obj o) {
  const int n = *n_obj;
  for (long k = blockIdx.x * (long)blockDim.x + threadIdx.x; k < n; k += (long)gridDim.x * blockDim.x) {
    const int b = a.lo[3 * k], y0 = a.lo[3 * k + 1], x0 = a.lo[3 * k + 2];
    const double cnt = (double)(long long)a.cnt[k];
    int cy = (int)rint((double)(long long)a.sum[3 * k + 1] / cnt);
    int cx = (int)rint((double)(long long)a.sum[3 * k + 2] / cnt);
    const uint32_t d2 = unsat((uint32_t)(a.key[k] >> 32));
    if (lab[((long)b * g.H + cy) * g.W + cx] != k + 1) {
      if (d2 > 0) {
        const long i = (long)(0xFFFFFFFFu - (uint32_t)(a.key[k] & 0xFFFFFFFFull));
        cy = (int)(i / g.W % g.H);
        cx = (int)(i % g.W);
      } else {
        cy = y0;
        cx = x0;
      }
    }
    o.ctr[2 * k] = cy;
    o.ctr[2 * k + 1] = cx;
    o.bmax[k] = (int32_t)d2;
    o.cmax[k] = 0;
    if (k == 0 || a.lo[3 * (k - 1)] != b) o.off[b] = (int32_t)k;
  }
}

// one warp per run of 32 pixels of one row, as reduce_kernel
__global__ void dt_center_max_kernel(const int32_t* __restrict__ lab, Grid g, Obj o) {
  const int lane = threadIdx.x & 31;
  const int runs = (g.W + 31) / 32;
  const long total_warps = (long)g.Z * g.H * runs;
  for (long wi = (blockIdx.x * (long)blockDim.x + threadIdx.x) / 32; wi < total_warps; wi += (long)gridDim.x * blockDim.x / 32) {
    const long row = wi / runs;
    const int x = (int)(wi % runs) * 32 + lane;
    const int y = (int)(row % g.H);
    int k = -1, d = 0;
    if (x < g.W) {
      const int32_t v = lab[row * g.W + x];
      if (v != 0) {
        k = v - 1;
        const int dy = y - o.ctr[2 * k], dx = x - o.ctr[2 * k + 1];
        d = dy * dy + dx * dx;
      }
    }
    const int k0 = __shfl_sync(0xffffffffu, k, 0);
    if (__all_sync(0xffffffffu, k == k0)) {
      if (k0 < 0) continue;
#pragma unroll
      for (int s = 16; s; s >>= 1) d = max(d, __shfl_xor_sync(0xffffffffu, d, s));
      if (lane == 0) atomicMax(&o.cmax[k0], d);
    } else if (k >= 0) {
      atomicMax(&o.cmax[k], d);
    }
  }
}

// torch_em's normalisation v / (max_o v + 1e-7) in fp32; centre distances as np.linalg.norm of the fp32 vector (exact squares
// below 2^24), boundary distances as scipy's fp64 EDT rounded to fp32
__device__ __forceinline__ float center_dist(int32_t d2) { return __fsqrt_rn(__int2float_rn(d2)); }
__device__ __forceinline__ float boundary_dist(uint32_t d2) { return __double2float_rn(__dsqrt_rn((double)d2)); }
__device__ __forceinline__ float normalise(float v, float m) { return __fdiv_rn(v, __fadd_rn(m, 1e-7f)); }

template <bool kVec>
__global__ void dt_write_kernel(const int32_t* __restrict__ lab, const int32_t* __restrict__ d2, Grid g, int channels, float fill,
                                Obj o, float* __restrict__ out) {
  const long plane = (long)g.H * g.W;
  const long qpi = (plane + 3) / 4, quads = g.Z * qpi;
  const int nc = __popc(channels);
  for (long q = blockIdx.x * (long)blockDim.x + threadIdx.x; q < quads; q += (long)gridDim.x * blockDim.x) {
    const int b = (int)(q / qpi);
    const long p0 = (q % qpi) * 4;
    float inst[4], fg[4], cd[4], bd[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long p = p0 + j;
      const long i = b * plane + p;
      const int32_t l = p < plane ? lab[i] : 0;
      inst[j] = l ? (float)(l - o.off[b]) : 0.f;
      fg[j] = l ? 1.f : 0.f;
      cd[j] = bd[j] = fill;
      if (l && (channels & kChDistances)) {
        const int k = l - 1, y = (int)(p / g.W), x = (int)(p % g.W);
        const int dy = y - o.ctr[2 * k], dx = x - o.ctr[2 * k + 1];
        cd[j] = normalise(center_dist(dy * dy + dx * dx), center_dist(o.cmax[k]));
      }
      if (l && (channels & kChBoundary))
        bd[j] = normalise(boundary_dist(unsat((uint32_t)d2[i])), boundary_dist((uint32_t)o.bmax[l - 1]));
    }
    float* dst = out + (long)b * nc * plane + p0;
    auto store = [&](const float (&v)[4]) {
      if (kVec) {
        __stcs(reinterpret_cast<float4*>(dst), make_float4(v[0], v[1], v[2], v[3]));
      } else {
        for (int j = 0; j < 4 && p0 + j < plane; ++j) __stcs(dst + j, v[j]);
      }
      dst += plane;
    };
    if (channels & kChInstances) store(inst);
    if (channels & kChForeground) store(fg);
    if (channels & kChDistances) store(cd);
    if (channels & kChBoundary) store(bd);
  }
}

// workspace: int32 copy of the labels, object labels, the object count, the labelling workspace (its first 16 n bytes are the
// EDT's two fields and two stacks once the objects are numbered), the boundary mask, the accumulators and the per-object
// results, all sized for n objects (the most a batch of n pixels can hold)
struct DtWs {
  int32_t *lab32, *lab;
  int* n_obj;
  void* lws;
  int32_t *da, *db, *sb, *tb;
  uint8_t* bnd;
  Acc acc;
  Obj obj;
};
size_t carve_dt(void* base, int B, int H, int W, int apply_label, DtWs* w) {
  char* p = (char*)base;
  const size_t n = (size_t)B * H * W;
  auto take = [&](size_t bytes) { char* q = p; p += align256(bytes); return (void*)q; };
  w->lab32 = (int32_t*)take(4 * n);
  w->lab = (int32_t*)take(4 * n);
  w->n_obj = (int*)take(sizeof(int));
  w->lws = take((size_t)post_label_objects_ws(B, H, W, apply_label));
  w->da = (int32_t*)w->lws;
  w->db = w->da + n;
  w->sb = w->db + n;
  w->tb = w->sb + n;
  w->bnd = (uint8_t*)take(n);
  w->acc.key = (unsigned long long*)take(8 * n);
  w->acc.cnt = (unsigned long long*)take(8 * n);
  w->acc.sum = (unsigned long long*)take(24 * n);
  w->acc.lo = (int32_t*)take(12 * n);
  w->acc.hi = (int32_t*)take(12 * n);
  w->obj.ctr = (int32_t*)take(8 * n);
  w->obj.bmax = (int32_t*)take(4 * n);
  w->obj.cmax = (int32_t*)take(4 * n);
  w->obj.off = (int32_t*)take(4 * (size_t)B);
  return (size_t)(p - (char*)base);
}

int check_shape(const char* fn, int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return set_error("%s: B=%d, H=%d, W=%d", fn, B, H, W);
  if (H > kMaxSide || W > kMaxSide) return set_error("%s: %d x %d image (sides up to %d)", fn, H, W, kMaxSide);
  if ((long)B * H * W >= (1l << 31) - 1024) return set_error("%s: %d x %d x %d labels (fewer than 2^31 - 1024)", fn, B, H, W);
  return 0;
}

}  // namespace
}  // namespace msam

using namespace msam;

extern "C" {

int64_t msam_distance_targets_workspace(int B, int H, int W, int apply_label) {
  if (B <= 0 || H <= 0 || W <= 0 || H > kMaxSide || W > kMaxSide || (long)B * H * W >= (1l << 31) - 1024) return -1;
  DtWs w;
  return (int64_t)carve_dt(nullptr, B, H, W, apply_label != 0, &w);
}

int msam_distance_targets(const void* labels, int label_dtype, int B, int H, int W, int apply_label, int min_size, int channels,
                          float fill, void* ws, int64_t ws_bytes, float* out, void* stream) {
  const char* fn = "msam_distance_targets";
  if (!labels || !ws || !out) return set_error("%s: null argument", fn);
  if (check_shape(fn, B, H, W)) return -1;
  if (label_dtype != 0 && label_dtype != 1) return set_error("%s: label_dtype %d (0 int32, 1 int64)", fn, label_dtype);
  if (channels <= 0 || (channels & ~(kChInstances | kChForeground | kChDistances | kChBoundary)))
    return set_error("%s: channel flags %d (bits 1 instances, 2 foreground, 4 distances, 8 boundary distances)", fn, channels);
  if (min_size < 0) return set_error("%s: min_size %d", fn, min_size);
  const int64_t need = msam_distance_targets_workspace(B, H, W, apply_label);
  if (ws_bytes < need) return set_error("%s: workspace of %lld bytes, need %lld", fn, (long long)ws_bytes, (long long)need);
  if ((uintptr_t)ws & 255) return set_error("%s: workspace not 256-byte aligned", fn);
  cudaStream_t st = (cudaStream_t)stream;
  DtWs w;
  carve_dt(ws, B, H, W, apply_label != 0, &w);
  const long n = (long)B * H * W;
  const Grid g = make_batch_grid(B, H, W);
  const bool dist = channels & (kChDistances | kChBoundary);

  const int32_t* lab_in = (const int32_t*)labels;
  if (label_dtype == 1) {
    to_int32_kernel<<<blocks_for(n), kThreads, 0, st>>>((const int64_t*)labels, n, w.lab32);
    LAUNCH_CHECK("dt_to_int32");
    lab_in = w.lab32;
  }
  prof_begin(st, "dt_objects", 0.0, 8.0 * n);
  RUN(post_label_objects(lab_in, B, H, W, apply_label != 0, min_size, w.lab, w.n_obj, w.lws, st));
  prof_end(st);
  const int32_t* d2 = nullptr;
  if (dist) {
    prof_begin(st, "dt_boundary", 0.0, 5.0 * n);
    RUN(launch_boundary(w.lab, g, w.bnd, st));
    prof_end(st);
    prof_begin(st, "dt_edt", 0.0, 13.0 * n);
    const int e[3] = {B, H, W};
    d2 = launch_edt(w.bnd, 1, 3, e, w.da, w.db, w.sb, w.tb, st, 1);
    prof_end(st);
    if (!d2) return -1;
  }
  const int oblocks = blocks_for(n);
  dt_reset_kernel<<<oblocks, kThreads, 0, st>>>(w.n_obj, w.acc);
  LAUNCH_CHECK("dt_reset");
  const long warps = (long)B * H * ((W + 31) / 32);
  const int rblocks = blocks_for(warps * 32, 1 << 20);
  prof_begin(st, "dt_reduce", 0.0, 8.0 * n);
  if (dist) reduce_kernel<true><<<rblocks, kThreads, 0, st>>>(w.lab, g, nullptr, 0, d2, w.acc);
  else reduce_kernel<false><<<rblocks, kThreads, 0, st>>>(w.lab, g, nullptr, 0, nullptr, w.acc);
  prof_end(st);
  LAUNCH_CHECK("dt_reduce");
  dt_finish_kernel<<<oblocks, kThreads, 0, st>>>(w.lab, g, w.n_obj, w.acc, w.obj);
  LAUNCH_CHECK("dt_finish");
  if (channels & kChDistances) {
    prof_begin(st, "dt_center_max", 0.0, 4.0 * n);
    dt_center_max_kernel<<<rblocks, kThreads, 0, st>>>(w.lab, g, w.obj);
    prof_end(st);
    LAUNCH_CHECK("dt_center_max");
  }
  const int nc = __builtin_popcount(channels);
  const long quads = (long)B * ((H * (long)W + 3) / 4);
  prof_begin(st, "dt_write", 0.0, (4.0 + (dist ? 4.0 : 0.0) + 4.0 * nc) * n);
  if ((H * (long)W) % 4 == 0 && ((uintptr_t)out & 15) == 0)
    dt_write_kernel<true><<<blocks_for(quads), kThreads, 0, st>>>(w.lab, d2, g, channels, fill, w.obj, out);
  else
    dt_write_kernel<false><<<blocks_for(quads), kThreads, 0, st>>>(w.lab, d2, g, channels, fill, w.obj, out);
  prof_end(st);
  LAUNCH_CHECK("dt_write");
  return 0;
}

}  // extern "C"
