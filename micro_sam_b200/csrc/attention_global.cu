// Global (64x64 = 4096 token) ViT-encoder attention for sm_90a, one CTA per (128-query tile, head, image):
//   softmax(scale * Q K^T + rel_h[q, kh] + rel_w[q, kw]) V      (segment_anything Attention.forward + add_decomposed_rel_pos,
//                                                                restated in oracle/sam_ref.py:Attention)
//   * two warpgroups, each owning 64 query rows (= one query grid row) over all 32 key tiles of 128 keys: S = Q K^T with
//     wgmma m64n128k16 (fp32 accumulators in registers), online softmax straight from the accumulator fragments (row
//     reductions across the quad of lanes that shares a row), P packed to bf16 in registers and fed back as the A operand
//     of O += P V (wgmma with A from registers, V consumed MN-major);
//   * rel-pos bias: T_w = Q RelW^T (128 columns) and T_h = Q RelH[qh0 .. qh0+80)^T (80 columns) are computed once, dumped to
//     shared memory (over the K / V stages, before the first key tile is loaded) and gathered: 32 rel_w values per thread
//     in registers, two rel_h values per row and key tile re-read from shared memory;
//   * one TMA warp: Q and the rel-pos tables, then K / V tiles through 2-4 stage rings shared by both warpgroups.
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace {

constexpr int BOX = 128 * 128;  // [128 rows x 64 bf16] SWIZZLE_128B box

template <int D>
struct GCfg {
  static constexpr int NB = (D + 63) / 64;
  static constexpr int KSTEPS = D / 16;
  static constexpr int TILE = NB * BOX;
  static constexpr int KST = 2;
  static constexpr int VST = (D == 64) ? 4 : 2;
  static constexpr int RTH_ROWS = 80, RTH_BOX = RTH_ROWS * 128, RTW_BOX = 128 * 128;
  static constexpr int TH_PITCH = 82, TW_PITCH = 130;  // fp32 scratch rows of T_h / T_w (padded against bank conflicts)
  static constexpr int T_BYTES = 128 * (TH_PITCH + TW_PITCH) * 4;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + TILE;          // the T scratch aliases the K / V stages until the first K tile
  static constexpr int OFF_V = OFF_K + KST * TILE;    // the rel-pos table tiles alias the V stages until T has been computed
  static constexpr int KV_END = OFF_V + VST * TILE;
  static constexpr int OFF_BAR = (KV_END > OFF_K + T_BYTES ? KV_END : OFF_K + T_BYTES + 1023) & ~1023;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
  static_assert(NB * (RTH_BOX + RTW_BOX) <= VST * TILE, "rel-pos tiles must fit in the V stages");
};

struct GParams {
  __nv_bfloat16* out;
  int d_model;
  float scale_log2;
};

template <int D>
__global__ void __launch_bounds__(288, 1)
attn_global_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmRTh,
                   const __grid_constant__ CUtensorMap tmRTw, const GParams p) {
  using C = GCfg<D>;
  constexpr int NKT = 32;
  constexpr float LOG2E = 1.4426950408889634f;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* t_done = bars + 1;
  uint64_t* kfull = bars + 2;     // [2]
  uint64_t* kempty = bars + 4;    // [2]
  uint64_t* vfull = bars + 6;     // [4]
  uint64_t* vempty = bars + 10;   // [4]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, img = blockIdx.z;
  const int row0 = img * 4096;
  const int qh0 = 2 * qt;  // first query grid row of this tile (128 queries = 2 grid rows)

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmQKV); prefetch_tmap(&tmRTh); prefetch_tmap(&tmRTw);
    mbar_init(q_full, 1); mbar_init(t_done, 8);
    for (int i = 0; i < C::KST; ++i) { mbar_init(&kfull[i], 1); mbar_init(&kempty[i], 8); }
    for (int i = 0; i < C::VST; ++i) { mbar_init(&vfull[i], 1); mbar_init(&vempty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  uint8_t* sQ = smem + C::OFF_Q;
  uint8_t* sK = smem + C::OFF_K;
  uint8_t* sV = smem + C::OFF_V;

  if (warp == 8) {
    // =========================================================== TMA producer
    if (lane == 0) {
      const int qcol = head * D, kcol = p.d_model + head * D, vcol = 2 * p.d_model + head * D;
      mbar_expect_tx(q_full, C::TILE + C::NB * (C::RTH_BOX + C::RTW_BOX));
      for (int b = 0; b < C::NB; ++b) tma_load_2d(sQ + b * BOX, &tmQKV, q_full, qcol + b * 64, row0 + qt * 128);
      for (int b = 0; b < C::NB; ++b) tma_load_2d(sV + b * C::RTH_BOX, &tmRTh, q_full, b * 64, qh0);
      for (int b = 0; b < C::NB; ++b) tma_load_2d(sV + C::NB * C::RTH_BOX + b * C::RTW_BOX, &tmRTw, q_full, b * 64, 128);
      mbar_wait(t_done, 0, 42);  // T has been computed and gathered: the K / V stages are free
      for (int j = 0; j < NKT; ++j) {
        const int ks = j % C::KST, vs = j % C::VST;
        mbar_wait(&kempty[ks], ((j / C::KST) & 1) ^ 1, 40);
        mbar_expect_tx(&kfull[ks], C::TILE);
        for (int b = 0; b < C::NB; ++b) tma_load_2d(sK + ks * C::TILE + b * BOX, &tmQKV, &kfull[ks], kcol + b * 64, row0 + j * 128);
        mbar_wait(&vempty[vs], ((j / C::VST) & 1) ^ 1, 41);
        mbar_expect_tx(&vfull[vs], C::TILE);
        for (int b = 0; b < C::NB; ++b) tma_load_2d(sV + vs * C::TILE + b * BOX, &tmQKV, &vfull[vs], vcol + b * 64, row0 + j * 128);
      }
    }
    return;
  }

  // =========================================================== warpgroup g: query rows [64 g, 64 g + 64) = grid row qh0 + g.
  // Fragment element i of a thread: row 64 g + 16 wq + qr + 8 ((i >> 1) & 1), column 8 (i >> 2) + qc + (i & 1).
  const int g = warp >> 2, wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
  const int rbase = 64 * g + 16 * wq + qr;
  const uint32_t aQ = smem_u32(sQ) + (uint32_t)g * 8192u, aK = smem_u32(sK), aV = smem_u32(sV);
  auto kdesc = [](uint32_t base, uint32_t box_bytes, int ks) {  // K-major operand, K step ks: box ks/4, +32 B per step
    return make_desc_sw128(base + (uint32_t)(ks >> 2) * box_bytes + (uint32_t)(ks & 3) * 32u, 0, 1024);
  };
  float* th = reinterpret_cast<float*>(sK);                         // [128][TH_PITCH]
  float* tw = th + 128 * C::TH_PITCH;                               // [128][TW_PITCH]

  mbar_wait(q_full, 0, 50);
  {
    float t_h[C::RTH_ROWS / 2], t_w[64];
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < C::KSTEPS; ++ks) wgmma<C::RTH_ROWS>(t_h, kdesc(aQ, BOX, ks), kdesc(aV, C::RTH_BOX, ks), ks > 0);
#pragma unroll
    for (int ks = 0; ks < C::KSTEPS; ++ks)
      wgmma<128>(t_w, kdesc(aQ, BOX, ks), kdesc(aV + C::NB * C::RTH_BOX, C::RTW_BOX, ks), ks > 0);
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(t_h);
    wg_fence_acc(t_w);
    named_bar_sync(1, 256);   // both warpgroups have read the rel-pos tables: the scratch may overwrite them
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      const int r = rbase + 8 * rs;
#pragma unroll
      for (int j = 0; j < C::RTH_ROWS / 8; ++j)
        *reinterpret_cast<float2*>(th + r * C::TH_PITCH + 8 * j + qc) = make_float2(t_h[4 * j + 2 * rs], t_h[4 * j + 2 * rs + 1]);
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<float2*>(tw + r * C::TW_PITCH + 8 * j + qc) = make_float2(t_w[4 * j + 2 * rs], t_w[4 * j + 2 * rs + 1]);
    }
  }
  named_bar_sync(1, 256);
  // rel_w[q, kw] * log2e = T_w[q][qw - kw + 63] for this thread's key columns kw = 8 jj + qc + e (the same in both key grid
  // rows of a tile); rel_h[q, kh] * log2e = T_h[q][g + 63 - kh], kh = 2 j + (column >> 6)
  float yw[2][16];
#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    const int r = rbase + 8 * rs, qw = (qt * 128 + r) & 63;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) yw[rs][2 * jj + e] = tw[r * C::TW_PITCH + qw + 63 - (8 * jj + qc + e)] * LOG2E;
  }
  float rhv[2][64 / 4];   // rel_h of this thread's rows for kh = 4 t + (lane & 3): the lane of the quad that holds it
#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    const int r = rbase + 8 * rs;
#pragma unroll
    for (int t = 0; t < 16; ++t) rhv[rs][t] = th[r * C::TH_PITCH + g + 63 - (4 * t + (lane & 3))] * LOG2E;
  }
  named_bar_sync(1, 256);   // everyone has gathered: K / V may overwrite the scratch
  __syncwarp();
  if (lane == 0) mbar_arrive(t_done);

  const float sl2 = p.scale_log2;
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll 1
  for (int j = 0; j < NKT; ++j) {
    const int ks_ = j % C::KST, vs = j % C::VST;
    float sacc[64];
    mbar_wait(&kfull[ks_], (j / C::KST) & 1, 61);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < C::KSTEPS; ++ks) wgmma<128>(sacc, kdesc(aQ, BOX, ks), kdesc(aK + ks_ * C::TILE, BOX, ks), ks > 0);
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(sacc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kempty[ks_]);

    uint32_t pk[32];
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      // kh = 2 j + h for the two key grid rows of the tile: rel_h from the quad lane that holds kh = 4 t + (lane & 3)
      float rh[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int kh = 2 * j + h;
        float v = 0.f;
#pragma unroll
        for (int t = 0; t < 16; ++t) v = (t == (kh >> 2)) ? rhv[rs][t] : v;
        rh[h] = __shfl_sync(0xffffffffu, v, (lane & ~3) | (kh & 3));
      }
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const float b = rh[jj >> 3];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& x = sacc[4 * jj + 2 * rs + e];
          x = fmaf(x, sl2, yw[rs][2 * (jj & 7) + e] + b);
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[rs], mx);
      const float f = ex2_approx(m_run[rs] - m_new);
      m_run[rs] = m_new;
      float ls = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const float p0 = ex2_approx(sacc[4 * jj + 2 * rs] - m_new), p1 = ex2_approx(sacc[4 * jj + 2 * rs + 1] - m_new);
        ls += p0 + p1;
        pk[2 * jj + rs] = pack_bf16(p0, p1);
      }
      l_run[rs] = l_run[rs] * f + ls;
#pragma unroll
      for (int jd = 0; jd < D / 8; ++jd) { o[4 * jd + 2 * rs] *= f; o[4 * jd + 2 * rs + 1] *= f; }
    }
    // O += P V: A fragment of keys [16 ks, 16 ks + 16) = (row, cols 16 ks + qc), (row + 8, ...), (row, + 8), (row + 8, + 8)
    mbar_wait(&vfull[vs], (j / C::VST) & 1, 62);
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t a[4] = {pk[4 * ks], pk[4 * ks + 1], pk[4 * ks + 2], pk[4 * ks + 3]};
      // V tile: rows = keys (K), 128-B rows of 64 head-dim elements (MN); 16 keys = 2048 B; next 64-col block = one box
      wgmma_rs<D, 1>(o, a, make_desc_sw128(aV + vs * C::TILE + (uint32_t)ks * 2048u, BOX, 1024), 1);
    }
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&vempty[vs]);
  }

#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    float l = l_run[rs];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int qi = qt * 128 + rbase + 8 * rs;
    __nv_bfloat16* orow = p.out + ((size_t)row0 + qi) * p.d_model + head * D;
#pragma unroll
    for (int jd = 0; jd < D / 8; ++jd)
      *reinterpret_cast<uint32_t*>(orow + 8 * jd + qc) = pack_bf16(o[4 * jd + 2 * rs] * inv, o[4 * jd + 2 * rs + 1] * inv);
  }
}

template <int D>
int launch_global_t(const AttnArgs& a, cudaStream_t stream) {
  using C = GCfg<D>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_global_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return set_error("attention: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  const int d_model = a.heads * D;
  const long rows = (long)a.batch * 4096;
  CUtensorMap tmQKV, tmRTh, tmRTw;
  if (make_tmap_bf16_2d(&tmQKV, a.qkv, rows, 3 * d_model, 3 * d_model, 128)) return -1;
  if (make_tmap_bf16_2d(&tmRTh, a.rel_table, 256, C::NB * 64, C::NB * 64, C::RTH_ROWS)) return -1;
  if (make_tmap_bf16_2d(&tmRTw, a.rel_table, 256, C::NB * 64, C::NB * 64, 128)) return -1;
  GParams p;
  p.out = a.out; p.d_model = d_model; p.scale_log2 = a.scale * 1.4426950408889634f;
  prof_begin(stream, D == 64 ? "attn_global<64>" : "attn_global<80>", (double)a.batch * a.heads * (4.0 * 4096 * 4096 * D + 4.0 * 4096 * 64 * D),
             (double)a.batch * 4096 * a.heads * D * 2 * 4);
  launch_pdl(attn_global_kernel<D>, dim3(32, a.heads, a.batch), dim3(288), C::SMEM_BYTES, stream, tmQKV, tmRTh, tmRTw, p);
  prof_end(stream);
  LAUNCH_CHECK("global attention");
  return 0;
}

}  // namespace

int launch_attention_global(const AttnArgs& a, cudaStream_t stream) {
  if (a.grid != 64 || a.window != 0) return set_error("global attention: 64x64 token grid only");
  if (a.head_dim == 64) return launch_global_t<64>(a, stream);
  if (a.head_dim == 80) return launch_global_t<80>(a, stream);
  return set_error("global attention: unsupported head_dim=%d", a.head_dim);
}

}  // namespace msam
