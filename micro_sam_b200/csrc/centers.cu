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
#include <algorithm>
#include <climits>

#include "kernels.h"

namespace msam {
namespace {

constexpr int kThreads = 256;
constexpr int32_t kInf = INT32_MAX;

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

int blocks_for(long n, int cap = 1 << 16) { return (int)std::max<long>(1, std::min<long>((n + kThreads - 1) / kThreads, cap)); }

// padded geometry: a 2-D image is a 3-D volume of depth 1 that is not padded along z
struct Grid {
  int ndim, Z, H, W;   // unpadded (Z = 1 in 2-D)
  int oz, PZ, PH, PW;  // z padding (1 in 3-D, 0 in 2-D) and padded extents
  __host__ __device__ long pn() const { return (long)PZ * PH * PW; }
};

Grid make_grid(int ndim, const int* dims) {
  Grid g;
  g.ndim = ndim;
  g.Z = ndim == 3 ? dims[0] : 1;
  g.H = dims[ndim - 2];
  g.W = dims[ndim - 1];
  g.oz = ndim == 3 ? 1 : 0;
  g.PZ = g.Z + 2 * g.oz;
  g.PH = g.H + 2;
  g.PW = g.W + 2;
  return g;
}

// label at padded coordinates; 0 outside the image
__device__ __forceinline__ int32_t padded_label(const int32_t* __restrict__ lab, const Grid& g, int z, int y, int x) {
  z -= g.oz; y -= 1; x -= 1;
  return (unsigned)z < (unsigned)g.Z && (unsigned)y < (unsigned)g.H && (unsigned)x < (unsigned)g.W
             ? lab[((long)z * g.H + y) * g.W + x] : 0;
}

// 2-D: one thread per padded pixel, the four neighbours through L1
__global__ void boundary2d_kernel(const int32_t* __restrict__ lab, Grid g, uint8_t* __restrict__ out) {
  const long total = g.pn();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int y = (int)(i / g.PW), x = (int)(i % g.PW);
    const int32_t c = padded_label(lab, g, 0, y, x);
    bool b = false;
    if (c != 0) {
      b = (y > 0 && padded_label(lab, g, 0, y - 1, x) != c) || (y + 1 < g.PH && padded_label(lab, g, 0, y + 1, x) != c) ||
          (x > 0 && padded_label(lab, g, 0, y, x - 1) != c) || (x + 1 < g.PW && padded_label(lab, g, 0, y, x + 1) != c);
    }
    out[i] = b;
  }
}

// 3-D: a (kTZ, kTY, kTX) tile of the padded grid per block, staged with a halo of 1 (halo cells outside the padded grid are
// marked -1 and never compared)
constexpr int kTX = 32, kTY = 8, kTZ = 4;
__global__ void __launch_bounds__(kTX * kTY) boundary3d_kernel(const int32_t* __restrict__ lab, Grid g, uint8_t* __restrict__ out) {
  __shared__ int32_t t[kTZ + 2][kTY + 2][kTX + 2];
  const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY, z0 = blockIdx.z * kTZ;
  const int tid = threadIdx.y * kTX + threadIdx.x;
  constexpr int kCells = (kTZ + 2) * (kTY + 2) * (kTX + 2);
  for (int q = tid; q < kCells; q += kTX * kTY) {
    const int lx = q % (kTX + 2), ly = (q / (kTX + 2)) % (kTY + 2), lz = q / ((kTX + 2) * (kTY + 2));
    const int x = x0 + lx - 1, y = y0 + ly - 1, z = z0 + lz - 1;
    const bool in = (unsigned)x < (unsigned)g.PW && (unsigned)y < (unsigned)g.PH && (unsigned)z < (unsigned)g.PZ;
    t[lz][ly][lx] = in ? padded_label(lab, g, z, y, x) : -1;
  }
  __syncthreads();
  const int lx = threadIdx.x + 1, ly = threadIdx.y + 1, x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= g.PW || y >= g.PH) return;
  for (int dz = 0; dz < kTZ; ++dz) {
    const int z = z0 + dz, lz = dz + 1;
    if (z >= g.PZ) break;
    const int32_t c = t[lz][ly][lx];
    bool b = false;
    if (c != 0) {
      const int32_t nb[6] = {t[lz - 1][ly][lx], t[lz + 1][ly][lx], t[lz][ly - 1][lx], t[lz][ly + 1][lx], t[lz][ly][lx - 1],
                             t[lz][ly][lx + 1]};
#pragma unroll
      for (int k = 0; k < 6; ++k) b |= nb[k] >= 0 && nb[k] != c;
    }
    out[((long)z * g.PH + y) * g.PW + x] = b;
  }
}

// Lines along one axis of a C-order array: n elements at stride s; line L starts at (L / s) * s * n + L % s.
struct Lines {
  long count;
  int n;
  long s;
  __device__ __forceinline__ long base(long L) const { return (L / s) * s * n + L % s; }
};

__device__ __forceinline__ int32_t sat(long long v) { return v >= kInf ? kInf : (int32_t)v; }

// first axis: squared 1-D distance to the nearest feature pixel (m == feat) on the line; kInf when the line has none.
// Lines are adjacent in memory across threads (coalesced).
__global__ void edt_first_kernel(const uint8_t* __restrict__ m, int feat, Lines ln, int32_t* __restrict__ out) {
  for (long L = blockIdx.x * (long)blockDim.x + threadIdx.x; L < ln.count; L += (long)gridDim.x * blockDim.x) {
    const long b = ln.base(L);
    long d = kInf;
    for (int q = 0; q < ln.n; ++q) {   // distance to the nearest feature at or before q
      const long i = b + q * ln.s;
      d = ((m[i] != 0) == (feat != 0)) ? 0 : (d == kInf ? kInf : d + 1);
      out[i] = (int32_t)d;
    }
    for (int q = ln.n - 1; q >= 0; --q) {   // ... or after q; then squared
      const long i = b + q * ln.s;
      const long f = out[i];
      d = f == 0 ? 0 : (d == kInf ? f : std::min<long>(f, d + 1));
      out[i] = d == kInf ? kInf : sat(d * d);
    }
  }
}

// further axes: Meijster's lower envelope of the parabolas (u - q)^2 + f(q), exact in int64, out = min_q (u - q)^2 + f(q)
// saturated at kInf.  kInf input values are treated as the finite value kInf: saturation commutes with the minimum, so
// every result below kInf is exact.  s_buf / t_buf: [n][lines] per-line stacks (line-interleaved, so a warp's stack accesses
// at equal depth are adjacent).
__device__ __forceinline__ long long sep(long long i, long long u, long long fi, long long fu) {
  // the first coordinate from which parabola u is below parabola i (i < u): floor((u^2 - i^2 + f(u) - f(i)) / (2 (u - i)))
  const long long num = u * u - i * i + fu - fi, den = 2 * (u - i);
  return num >= 0 ? num / den : -((-num + den - 1) / den);
}
__global__ void edt_envelope_kernel(const int32_t* __restrict__ f, Lines ln, int32_t* __restrict__ s_buf, int32_t* __restrict__ t_buf,
                                    int32_t* __restrict__ out) {
  for (long L = blockIdx.x * (long)blockDim.x + threadIdx.x; L < ln.count; L += (long)gridDim.x * blockDim.x) {
    const long b = ln.base(L);
    const long ls = ln.count;
    auto F = [&](long q) -> long long { return f[b + q * ln.s]; };
    auto S = [&](int k) -> int32_t& { return s_buf[(long)k * ls + L]; };
    auto T = [&](int k) -> int32_t& { return t_buf[(long)k * ls + L]; };
    const int n = ln.n;
    int k = 0;
    S(0) = 0; T(0) = 0;
    long long fs = F(0);   // f at the top of the stack
    for (int u = 1; u < n; ++u) {
      const long long fu = F(u);
      // pop while parabola u is below the top at the top's start: (t - s)^2 + f(s) > (t - u)^2 + f(u)
      while (k >= 0) {
        const long long tk = T(k), sk = S(k);
        if ((tk - sk) * (tk - sk) + fs <= (tk - u) * (tk - u) + fu) break;
        --k;
        if (k >= 0) fs = F(S(k));
      }
      if (k < 0) {
        k = 0; S(0) = u; T(0) = 0; fs = fu;
      } else {
        const long long w = 1 + sep(S(k), u, fs, fu);
        if (w < n) { ++k; S(k) = u; T(k) = (int32_t)w; fs = fu; }
      }
    }
    for (int u = n - 1; u >= 0; --u) {
      const long long sk = S(k);
      out[b + u * ln.s] = sat((u - sk) * (u - sk) + F(sk));
      if (u == T(k)) --k;
    }
  }
}

// lower-bound search of v in the sorted table; -1 when absent
__device__ __forceinline__ int find_id(const int32_t* __restrict__ ids, int n, int32_t v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && ids[lo] == v ? lo : -1;
}

struct Acc {
  unsigned long long* key;   // [n_ids]
  int32_t* lo;               // [n_ids][3] (z, y, x) minima
  int32_t* hi;               // [n_ids][3] maxima
  unsigned long long* cnt;   // [n_ids]
  unsigned long long* sum;   // [n_ids][3] coordinate sums (int64)
};

__global__ void reset_kernel(int n_ids, Acc a) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n_ids; i += (long)gridDim.x * blockDim.x) {
    a.key[i] = 0; a.cnt[i] = 0;
    for (int d = 0; d < 3; ++d) { a.lo[3 * i + d] = INT_MAX; a.hi[3 * i + d] = -1; a.sum[3 * i + d] = 0; }
  }
}

// one warp per run of 32 pixels of one row (rows of W are split into ceil(W / 32) runs)
template <bool kDist>
__global__ void reduce_kernel(const int32_t* __restrict__ lab, Grid g, const int32_t* __restrict__ ids, int n_ids,
                              const int32_t* __restrict__ d2, Acc a) {
  const int lane = threadIdx.x & 31;
  const int runs = (g.W + 31) / 32;
  const long total_warps = (long)g.Z * g.H * runs;
  for (long wi = (blockIdx.x * (long)blockDim.x + threadIdx.x) / 32; wi < total_warps; wi += (long)gridDim.x * blockDim.x / 32) {
    const long row = wi / runs;
    const int x = (int)(wi % runs) * 32 + lane;
    const int z = (int)(row / g.H), y = (int)(row % g.H);
    int k = -1;
    unsigned long long key = 0;
    if (x < g.W) {
      const long i = row * g.W + x;
      const int32_t v = lab[i];
      if (v != 0) {
        k = find_id(ids, n_ids, v);
        if (kDist && k >= 0) {
          const int32_t d = d2[((long)(z + g.oz) * g.PH + y + 1) * g.PW + x + 1];
          key = ((unsigned long long)(uint32_t)d << 32) | (0xFFFFFFFFu - (uint32_t)i);
        }
      }
    }
    const int k0 = __shfl_sync(0xffffffffu, k, 0);
    if (__all_sync(0xffffffffu, k == k0)) {   // the whole run is one object (or background)
      if (k0 < 0) continue;
      if (kDist) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          const unsigned long long w = __shfl_xor_sync(0xffffffffu, key, o);
          key = key > w ? key : w;
        }
      }
      if (lane == 0) {
        if (kDist) atomicMax(&a.key[k0], key);
        atomicMin(&a.lo[3 * k0], z); atomicMax(&a.hi[3 * k0], z);
        atomicMin(&a.lo[3 * k0 + 1], y); atomicMax(&a.hi[3 * k0 + 1], y);
        atomicMin(&a.lo[3 * k0 + 2], x); atomicMax(&a.hi[3 * k0 + 2], x + 31);
        atomicAdd(&a.cnt[k0], 32ull);
        atomicAdd(&a.sum[3 * k0], 32ull * z); atomicAdd(&a.sum[3 * k0 + 1], 32ull * y);
        atomicAdd(&a.sum[3 * k0 + 2], 32ull * x + 496ull);
      }
    } else if (k >= 0) {
      if (kDist) atomicMax(&a.key[k], key);
      atomicMin(&a.lo[3 * k], z); atomicMax(&a.hi[3 * k], z);
      atomicMin(&a.lo[3 * k + 1], y); atomicMax(&a.hi[3 * k + 1], y);
      atomicMin(&a.lo[3 * k + 2], x); atomicMax(&a.hi[3 * k + 2], x);
      atomicAdd(&a.cnt[k], 1ull);
      atomicAdd(&a.sum[3 * k], (unsigned long long)z); atomicAdd(&a.sum[3 * k + 1], (unsigned long long)y);
      atomicAdd(&a.sum[3 * k + 2], (unsigned long long)x);
    }
  }
}

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

int launch_boundary(const int32_t* lab, const Grid& g, uint8_t* out, cudaStream_t st) {
  if (g.ndim == 2) {
    boundary2d_kernel<<<blocks_for(g.pn()), kThreads, 0, st>>>(lab, g, out);
  } else {
    const dim3 grid((g.PW + kTX - 1) / kTX, (g.PH + kTY - 1) / kTY, (g.PZ + kTZ - 1) / kTZ);
    boundary3d_kernel<<<grid, dim3(kTX, kTY), 0, st>>>(lab, g, out);
  }
  LAUNCH_CHECK("centers_boundary");
  return 0;
}

// squared EDT of the C-order array m of extents e[0..nd) (feature pixels: (m != 0) == feat): the first pass writes buf0 and
// every further pass the other buffer; returns the buffer holding the result (buf0 for odd nd, buf1 for even), null on error
int32_t* launch_edt(const uint8_t* m, int feat, int nd, const int* e, int32_t* buf0, int32_t* buf1, int32_t* sb, int32_t* tb,
                    cudaStream_t st) {
  long total = 1;
  for (int d = 0; d < nd; ++d) total *= e[d];
  auto lines = [&](int axis) {
    long s = 1;
    for (int d = axis + 1; d < nd; ++d) s *= e[d];
    return Lines{total / e[axis], e[axis], s};
  };
  const Lines l0 = lines(0);
  edt_first_kernel<<<blocks_for(l0.count), kThreads, 0, st>>>(m, feat, l0, buf0);
  if (launch_check("centers_edt_first")) return nullptr;
  int32_t* cur = buf0;
  for (int axis = 1; axis < nd; ++axis) {
    int32_t* nxt = cur == buf0 ? buf1 : buf0;
    const Lines l = lines(axis);
    edt_envelope_kernel<<<blocks_for(l.count), kThreads, 0, st>>>(cur, l, sb, tb, nxt);
    if (launch_check("centers_edt_envelope")) return nullptr;
    cur = nxt;
  }
  return cur;
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
