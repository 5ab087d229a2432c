// Windowed ViT attention (head_dim 64 / 80, 14x14 windows, 196 keys incl. the zero-pad tokens), second generation.
// Restates segment_anything's Attention.forward + add_decomposed_rel_pos (oracle/sam_ref.py:Attention) like attention.cu,
// with everything except max / exp on the tensor core (a CUDA-core bias costs ~10 instructions per logit and 28 bias values per
// thread):
//   * rel-pos bias inside the S MMA: T = Q R^T (as before) is shifted per query row, scaled by 1/scale and written as 28
//     extra bf16 K-columns next to Q (box 1, columns 16..43) plus their bf16 rounding residuals (a second tile over the dead
//     R table: hi + lo carries 16 mantissa bits, the bias stays at fp32-accumulator accuracy); the key tile gets the matching
//     one-hot columns E[k, kh(k)] = E[k, 14 + kw(k)] = 1, so S = Q K^T + (T/scale) E^T comes out of ONE accumulation chain
//     (9 k-steps instead of 5) and softmax(scale * S) needs no per-element bias arithmetic;
//   * row sums from the tensor core: V gets a ones column (box 1, column 16), O[:, 80] = sum_k P[:, k] of the bf16-rounded
//     probabilities (the same values the P V product sees);
//   * keys 192..195 (P covers 3 boxes = 192 keys) as a 13th k-step whose A tile lives in unused columns of the V tile
//     (box 1, columns 32..47), instead of 320 CUDA-core FMAs per row in the epilogue;
//   * row max, exp pass = fma + ex2 + half a pack, straight from the wgmma accumulator fragments (row
//     reductions across the quad of lanes that shares a row).
// Layout: [box A0 16 KB | box A1 16 KB | R 16 KB | box B0 26 KB | box B1 26 KB]; P (keys 0..191, 3 boxes) goes over A0 | A1 | R
// once S is complete, V is loaded over K (B0 / B1).  head_dim 80: A0 | A1 = Q (80 of 128 columns), the bias columns sit in A1
// columns 16..47, the one-hot columns in B1 (= K box 1) columns 16..47, the ones column in V box 1 column 16.  head_dim 64:
// A0 = Q, A1 = the bias tile (columns 0..31), B0 = K / V, B1 = the one-hot tile (columns 0..31; column 0 becomes the ones
// column once S is complete): the same byte offsets, only the column offset inside box 1 differs.
// Warp roles: warps 0-3 / 4-7 = two warpgroups that each issue the wgmma chains (T, S, O) for 64 of the 128 query rows and
// run their softmax / epilogue; warp 8 TMA.
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace {

constexpr int W8_THREADS = 288;
constexpr int W8_QBOX = 128 * 128;   // 128 rows x 64 bf16
constexpr int W8_NK = 208;           // keys padded to a multiple of 16
constexpr int W8_KBOX = W8_NK * 128;
constexpr int W8_RTBOX = 64 * 128;
constexpr int W8_OFF_RT = 2 * W8_QBOX;
constexpr int W8_OFF_K = W8_OFF_RT + 2 * W8_RTBOX;
constexpr int W8_OFF_BAR = W8_OFF_K + 2 * W8_KBOX;
constexpr int W8_SMEM = W8_OFF_BAR + 128 + 1024;
static_assert(W8_OFF_K % 1024 == 0 && W8_KBOX % 1024 == 0, "SW128 tiles must be 1024-byte aligned");

struct W8Params {
  __nv_bfloat16* out;
  int d_model, grid;
  float sl2;        // scale * log2(e)
  float inv_scale;  // 1 / scale
  unsigned long long* trace;
};

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(a, fmaxf(b, c)); }
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_shared_u16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// byte address of bf16 element `col` (0..63) of row `r` in a K-major SWIZZLE_128B tile at `base`
__device__ __forceinline__ uint32_t sw128_addr(uint32_t base, int r, int col) {
  return base + (uint32_t)r * 128u + ((uint32_t)((col >> 3) ^ (r & 7)) << 4) + (uint32_t)(col & 7) * 2u;
}

#define W8_TRACE(slot) do { if (tr) tr[slot] = gtimer(); } while (0)

template <int D>
__global__ void __launch_bounds__(W8_THREADS, 1)
attn_window2_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                     const __grid_constant__ CUtensorMap tmRT, const W8Params p) {
  constexpr int S = 14, G = 196;
  constexpr int NB = (D + 63) / 64;          // TMA boxes per operand
  constexpr int KS = D / 16;                 // k-steps of Q K^T
  constexpr int AUGC = (D == 80) ? 2 : 0;    // first 16-byte chunk of the bias / one-hot columns inside box 1
  constexpr int NO = D + 16;                 // P V columns: values + the ones column (+ 15 unused)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sRT = smem + W8_OFF_RT;
  uint8_t* sK = smem + W8_OFF_K;   // V later
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + W8_OFF_BAR);
  uint64_t *ld_full = bars, *v_full = bars + 1, *s_done = bars + 2, *q_full = bars + 3;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, group = blockIdx.z;
  unsigned long long* tr = nullptr;
  if (p.trace && threadIdx.x == 0 && qt == 0 && head == 0 && group < 64) tr = p.trace + group * 16;
  W8_TRACE(0);

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmKV);
    prefetch_tmap(&tmRT);
    mbar_init(ld_full, 1);
    mbar_init(q_full, 1);
    mbar_init(v_full, 1);
    mbar_init(s_done, 8);
    fence_barrier_init();
  }
  __syncthreads();
  const int row0 = group * G;
  pdl_wait();
  pdl_trigger();
  W8_TRACE(1);

  if (warp == 8) {
    if (lane == 0) {
      const int qcol = head * D, kcol = p.d_model + head * D, vcol = 2 * p.d_model + head * D;
      mbar_expect_tx(q_full, NB * (W8_QBOX + W8_RTBOX));   // T = Q R^T can start before K has landed
      for (int b = 0; b < NB; ++b) {
        tma_load_2d(sQ + b * W8_QBOX, &tmQ, q_full, qcol + b * 64, row0 + qt * 128);
        tma_load_2d(sRT + b * W8_RTBOX, &tmRT, q_full, b * 64, 0);
      }
      mbar_expect_tx(ld_full, NB * W8_KBOX);
      for (int b = 0; b < NB; ++b) tma_load_2d(sK + b * W8_KBOX, &tmKV, ld_full, kcol + b * 64, row0);
      mbar_wait(s_done, 0, 44);  // both S chains have completed: V goes over the dead K tile
      mbar_expect_tx(v_full, NB * W8_KBOX);
      for (int b = 0; b < NB; ++b) tma_load_2d(sK + b * W8_KBOX, &tmKV, v_full, vcol + b * 64, row0);
    }
    return;
  }

  // ---- two warpgroups; warpgroup g owns query rows [64 g, 64 g + 64) of the tile.  Fragment element i of a thread holds
  // row 64 g + 16 wq + qr + 8 ((i >> 1) & 1), column 8 (i >> 2) + qc + (i & 1).
  const int g = warp >> 2, wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
  const int rbase = 64 * g + 16 * wq + qr;   // + 8 rs
  const uint32_t aQ = smem_u32(sQ), aK = smem_u32(sK), aRT = smem_u32(sRT);
  const uint32_t own = (uint32_t)(64 * g) * 128u;   // byte offset of this warpgroup's rows in a 128-row K-major tile
  auto kdesc = [](uint32_t base, uint32_t box_bytes, int ks) {
    return make_desc_sw128(base + (uint32_t)(ks >> 2) * box_bytes + (uint32_t)(ks & 3) * 32u, 0, 1024);
  };

  // T = Q R^T (64 columns: rel_h over [0, 27), rel_w over [32, 59))
  mbar_wait(q_full, 0, 40);
  W8_TRACE(2);
  {
    float t[32];
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) wgmma<64>(t, kdesc(aQ + own, W8_QBOX, ks), kdesc(aRT, W8_RTBOX, ks), ks > 0);
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(t);
    named_bar_sync(1, 256);   // both warpgroups have read R: its tile takes the bias residuals now
    // bias columns of row q: e = kh in [0, 14) <- T[q, 13 + qh - kh], e = 14 + kw <- T[q, 32 + 13 + qw - kw], e in [28, 32) = 0;
    // hi = bf16(T / scale) next to Q (box 1), lo = bf16(T / scale - hi) in its own tile over the dead R table
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      const int r = rbase + 8 * rs;
      const int qi = qt * 128 + r;
      int qh = qi / S;
      const int qw = qi - qh * S;
      if (qh > S - 1) qh = S - 1;
      const uint32_t qrow = aQ + W8_QBOX, lrow = aRT;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (((i >> 1) & 1) != rs) continue;
        const int c = 8 * (i >> 2) + qc + (i & 1);
        const int e = c < 32 ? 13 + qh - c : 14 + 13 + qw - (c - 32);
        if (c < 32 ? (e < 0 || e > 13) : (e < 14 || e > 27)) continue;
        const float y = t[i] * p.inv_scale;
        const __nv_bfloat16 hi = __float2bfloat16_rn(y);
        const __nv_bfloat16 lo = __float2bfloat16_rn(y - __bfloat162float(hi));
        st_shared_u16(sw128_addr(qrow, r, AUGC * 8 + e), __bfloat16_as_ushort(hi));
        st_shared_u16(sw128_addr(lrow, r, e), __bfloat16_as_ushort(lo));
      }
      if ((lane & 3) == 0) {   // e = 28..31: the second half of chunk 3 of the bias columns
        asm volatile("st.shared.v2.b32 [%0], {%1, %1};" ::"r"(sw128_addr(qrow, r, AUGC * 8 + 28)), "r"(0u) : "memory");
        asm volatile("st.shared.v2.b32 [%0], {%1, %1};" ::"r"(sw128_addr(lrow, r, 28)), "r"(0u) : "memory");
      }
    }
  }
  // one-hot key columns: rows k of box B1.  head_dim 80: B1 is K box 1 -- wait until the K tile has landed (its TMA box
  // covers these columns with the next head's data); head_dim 64: B1 is a tile of its own
  mbar_wait(ld_full, 0, 54);
  for (int k = threadIdx.x; k < W8_NK; k += 256) {
    unsigned long long bits = 0ull;
    if (k < G) {
      const int kh = k / S, kw = k - kh * S;
      bits = (1ull << kh) | (1ull << (S + kw));
    }
    const uint32_t krow = aK + W8_KBOX + (uint32_t)k * 128u;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      uint32_t e[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = 2 * (4 * c + j);
        e[j] = (((bits >> col) & 1ull) ? 0x3F80u : 0u) | (((bits >> (col + 1)) & 1ull) ? 0x3F800000u : 0u);
      }
      st_shared_v4(krow + ((uint32_t)((c + AUGC) ^ (k & 7)) << 4), make_uint4(e[0], e[1], e[2], e[3]));
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 256);
  W8_TRACE(3);

  // S = Q K^T + (T / scale) E^T : KS k-steps, then bias hi and lo against the one-hot columns
  float sacc[W8_NK / 2];
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) wgmma<W8_NK>(sacc, kdesc(aQ + own, W8_QBOX, ks), kdesc(aK, W8_KBOX, ks), ks > 0);
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    const uint64_t de = make_desc_sw128(aK + W8_KBOX + (uint32_t)(AUGC * 16 + ks * 32), 0, 1024);
    wgmma<W8_NK>(sacc, make_desc_sw128(aQ + W8_QBOX + own + (uint32_t)(AUGC * 16 + ks * 32), 0, 1024), de, 1);
    wgmma<W8_NK>(sacc, make_desc_sw128(aRT + own + (uint32_t)ks * 32u, 0, 1024), de, 1);
  }
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(sacc);
  __syncwarp();
  if (lane == 0) mbar_arrive(s_done);
  W8_TRACE(4);

  // softmax over keys 0..195: P (keys 0..191) over this warpgroup's rows of A0 | A1 | R, keys 192..207 parked in V box 1
  // columns 32..47 once V has landed (zero beyond 195)
  const float sl2 = p.sl2;
  uint32_t ptail[2][2] = {{0u, 0u}, {0u, 0u}};
#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    const int r = rbase + 8 * rs;
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < W8_NK / 8; ++j) {
      const int c = 8 * j + qc;
      const float a0 = sacc[4 * j + 2 * rs], a1 = sacc[4 * j + 2 * rs + 1];
      if (c < G) m = fmax3(m, a0, a1);   // G % 2 == 0: the pair is entirely inside or outside
    }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    const float nmsl2 = -m * sl2;
#pragma unroll
    for (int j = 0; j < W8_NK / 8; ++j) {
      const int c = 8 * j + qc;
      const uint32_t pk = pack_bf16(ex2_approx(fmaf(sacc[4 * j + 2 * rs], sl2, nmsl2)), ex2_approx(fmaf(sacc[4 * j + 2 * rs + 1], sl2, nmsl2)));
      if (c < 192) st_shared_u32(sw128_addr(aQ + (uint32_t)(c >> 6) * W8_QBOX, r, c & 63), pk);
      else if (c < G) ptail[rs][(c - 192) >> 1] = pk;
    }
  }
  W8_TRACE(5);
  // V has landed: ones column (box 1, column 8 AUGC) for all key rows, and this warpgroup's tail probabilities
  mbar_wait(v_full, 0, 53);
  for (int k = threadIdx.x; k < W8_NK; k += 256) st_shared_u16(sw128_addr(aK + W8_KBOX, k, AUGC * 8), (uint16_t)0x3F80);
#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    const int r = rbase + 8 * rs;
#pragma unroll
    for (int j = 24; j < 26; ++j) {
      const int c = 8 * j + qc;
      st_shared_u32(sw128_addr(aK + W8_KBOX, r, 32 + c - 192), c < G ? ptail[rs][(c - 192) >> 1] : 0u);
    }
  }
  fence_proxy_async_smem();
  named_bar_sync(1, 256);   // the ones column is written by both warpgroups
  W8_TRACE(6);

  // O = P V (+ the row sums in column D): 12 k-steps over keys 0..191, a 13th over keys 192..207
  float oacc[NO / 2];
  wg_fence();
#pragma unroll
  for (int ks = 0; ks < 12; ++ks) {
    const uint64_t da = make_desc_sw128(aQ + own + (uint32_t)(ks >> 2) * W8_QBOX + (uint32_t)(ks & 3) * 32u, 0, 1024);
    const uint64_t db = make_desc_sw128(aK + (uint32_t)ks * 2048u, W8_KBOX, 1024);
    wgmma<NO, 0, 1>(oacc, da, db, ks > 0);
  }
  wgmma<NO, 0, 1>(oacc, make_desc_sw128(aK + W8_KBOX + own + 64u, 0, 1024), make_desc_sw128(aK + 12u * 2048u, W8_KBOX, 1024), 1);
  wg_commit();
  wg_wait<0>();
  wg_fence_acc(oacc);
  W8_TRACE(8);

  const int wpr = (p.grid + S - 1) / S;
  const int b = group / (wpr * wpr), wy = (group / wpr) % wpr, wx = group % wpr;
#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    const int qi = qt * 128 + rbase + 8 * rs;
    // row sum = column D, held by the lane with qc == 0 of the quad
    const float sum = __shfl_sync(0xffffffffu, oacc[4 * (D / 8) + 2 * rs], lane & ~3);
    const int y = wy * S + qi / S, x = wx * S + qi % S;
    if (qi >= G || y >= p.grid || x >= p.grid) continue;
    const float inv = 1.0f / sum;
    __nv_bfloat16* orow = p.out + ((long)b * p.grid * p.grid + y * p.grid + x) * p.d_model + head * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<uint32_t*>(orow + 8 * j + qc) = pack_bf16(oacc[4 * j + 2 * rs] * inv, oacc[4 * j + 2 * rs + 1] * inv);
  }
  W8_TRACE(9);
}

unsigned long long* g_attn_trace = nullptr;

}  // namespace

void set_attn_trace(unsigned long long* dev_buf) { g_attn_trace = dev_buf; }
unsigned long long* get_attn_trace() { return g_attn_trace; }

template <int D>
static int launch_attn_window2_t(const AttnArgs& a, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_window2_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, W8_SMEM);
    if (e != cudaSuccess) return set_error("attention: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  constexpr int NB = (D + 63) / 64;
  const int d_model = a.heads * D, S = 14;
  const int wpr = (a.grid + S - 1) / S;
  const int groups = a.batch * wpr * wpr;
  const long rows = (long)groups * 196;
  CUtensorMap tmQ, tmKV, tmRT;
  if (make_tmap_bf16_2d(&tmQ, a.qkv, rows, 3 * d_model, 3 * d_model, 128)) return -1;
  if (make_tmap_bf16_2d(&tmKV, a.qkv, rows, 3 * d_model, 3 * d_model, W8_NK)) return -1;
  if (make_tmap_bf16_2d(&tmRT, a.rel_table, 64, NB * 64, NB * 64, 64)) return -1;
  W8Params p;
  p.out = a.out; p.d_model = d_model; p.grid = a.grid; p.sl2 = a.scale * 1.4426950408889634f; p.inv_scale = 1.0f / a.scale;
  p.trace = g_attn_trace;
  prof_begin(stream, D == 64 ? "attn_window<64>" : "attn_window<80>",
             (double)groups * a.heads * (4.0 * 196 * 196 * D + 4.0 * 196 * S * D), (double)groups * 196 * a.heads * D * 2 * 4);
  launch_pdl(attn_window2_kernel<D>, dim3(2, a.heads, groups), dim3(W8_THREADS), W8_SMEM, stream, tmQ, tmKV, tmRT, p);
  prof_end(stream);
  LAUNCH_CHECK("window attention");
  return 0;
}

int launch_attn_window2(const AttnArgs& a, cudaStream_t stream) {
  return a.head_dim == 64 ? launch_attn_window2_t<64>(a, stream) : launch_attn_window2_t<80>(a, stream);
}

}  // namespace msam
