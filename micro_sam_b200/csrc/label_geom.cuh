// Label-image geometry shared by the object-centre op (centers.cu) and the distance targets (distance_targets.cu): inner
// boundaries, the exact squared EDT and the per-object reduction.  Everything lives in an anonymous namespace, so each
// translation unit that includes this compiles its own copy of the kernels.
#pragma once
#include <algorithm>
#include <climits>

#include "kernels.h"

namespace msam {
namespace {

constexpr int kThreads = 256;
constexpr int32_t kInf = INT32_MAX;

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

int blocks_for(long n, int cap = 1 << 16) { return (int)std::max<long>(1, std::min<long>((n + kThreads - 1) / kThreads, cap)); }

// padded geometry: a 2-D image is a 3-D volume of depth 1 that is not padded along z.  A batch of B 2-D images is a volume
// of depth B, not padded along z, whose slices never see each other (the 2-D boundary kernel and an EDT from axis 1 on).
struct Grid {
  int ndim, Z, H, W;   // unpadded (Z = 1 in 2-D, B for a batch)
  int oz, PZ, PH, PW;  // z padding (1 in 3-D, 0 in 2-D) and padded extents
  int pad;             // y and x padding: 1 (centres), 0 (distance targets)
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
  g.pad = 1;
  return g;
}

// B unpadded 2-D images of one size
Grid make_batch_grid(int B, int H, int W) {
  Grid g;
  g.ndim = 2;
  g.Z = g.PZ = B;
  g.H = g.PH = H;
  g.W = g.PW = W;
  g.oz = g.pad = 0;
  return g;
}

// label at padded coordinates; 0 outside the image
__device__ __forceinline__ int32_t padded_label(const int32_t* __restrict__ lab, const Grid& g, int z, int y, int x) {
  z -= g.oz; y -= g.pad; x -= g.pad;
  return (unsigned)z < (unsigned)g.Z && (unsigned)y < (unsigned)g.H && (unsigned)x < (unsigned)g.W
             ? lab[((long)z * g.H + y) * g.W + x] : 0;
}

// 2-D: one thread per padded pixel, the four neighbours of its own slice through L1 (neighbours outside the padded grid
// are ignored: skimage's reflect border at radius 1)
__global__ void boundary2d_kernel(const int32_t* __restrict__ lab, Grid g, uint8_t* __restrict__ out) {
  const long total = g.pn();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long zy = i / g.PW;
    const int z = (int)(zy / g.PH), y = (int)(zy % g.PH), x = (int)(i % g.PW);
    const int32_t c = padded_label(lab, g, z, y, x);
    bool b = false;
    if (c != 0) {
      b = (y > 0 && padded_label(lab, g, z, y - 1, x) != c) || (y + 1 < g.PH && padded_label(lab, g, z, y + 1, x) != c) ||
          (x > 0 && padded_label(lab, g, z, y, x - 1) != c) || (x + 1 < g.PW && padded_label(lab, g, z, y, x + 1) != c);
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
        k = ids ? find_id(ids, n_ids, v) : v - 1;
        if (kDist && k >= 0) {
          const int32_t d = d2[((long)(z + g.oz) * g.PH + y + g.pad) * g.PW + x + g.pad];
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

// squared EDT of the C-order array m of extents e[0..nd) (feature pixels: (m != 0) == feat) along the axes a0..nd-1 (a0 = 1:
// each slice of the first axis on its own, as for a batch of images): the first pass writes buf0 and every further pass the
// other buffer; returns the buffer holding the result (buf0 for an odd number of axes, buf1 for even), null on error
int32_t* launch_edt(const uint8_t* m, int feat, int nd, const int* e, int32_t* buf0, int32_t* buf1, int32_t* sb, int32_t* tb,
                    cudaStream_t st, int a0 = 0) {
  long total = 1;
  for (int d = 0; d < nd; ++d) total *= e[d];
  auto lines = [&](int axis) {
    long s = 1;
    for (int d = axis + 1; d < nd; ++d) s *= e[d];
    return Lines{total / e[axis], e[axis], s};
  };
  const Lines l0 = lines(a0);
  edt_first_kernel<<<blocks_for(l0.count), kThreads, 0, st>>>(m, feat, l0, buf0);
  if (launch_check("centers_edt_first")) return nullptr;
  int32_t* cur = buf0;
  for (int axis = a0 + 1; axis < nd; ++axis) {
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
