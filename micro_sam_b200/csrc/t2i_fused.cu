// Fused token -> image cross-attention of the two-way transformer (Attention(q = tokens + pe, k = keys + pe, v = keys),
// restated in oracle/sam_ref.py) without materialising the projected keys / values:
//   scores[(h,t), j] = q_h[t] . Wk_h (x_j + pe_j)  =  Q'[(h,t)] . (x_j + pe_j),   Q'[(h,t)] = 0.25 * Wk_h^T q_h[t]   ([rows, 256])
//   out_h[t]         = Wv_h (sum_j p[(h,t), j] x_j) + bv_h                                   (k bias: softmax invariant)
// i.e. a flash attention with "head dim" 256 in which the image tokens x ([4096, 256] bf16, read ONCE: 2 MB per prompt
// instead of the 4 MB written + 4 MB read by the k/v projection GEMM and the attention core) are both K and V:
//   S = Q' X^T (+ Q' PE^T)   wgmma m64n64k16, K-major operands                  (X tile [64 keys x 256] via TMA, SW128)
//   U += P X                 wgmma m64n256k16, P from registers, X consumed MN-major from the same shared-memory tile
// with the online softmax on the accumulator fragments; one warpgroup per 64 rows (head, token).  The tiny per-head value
// projection runs afterwards (t2i_head_proj_kernel).
//
// One work item = 128 Q' rows against 4096 image tokens: mode 1 -> one prompt (rows h*16 + t, own keys); mode 0 (layer 0:
// the image tokens are shared by all prompts) -> rows of one prompt (T > 8) or of two prompts (T <= 8, rows pl*64 + h*8 + t).
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace t2i {
constexpr int PESLOTS = 4;
constexpr int XT = 64;                              // image tokens per tile
constexpr int SUBX = XT * 128;                      // [64 tokens x 64 channels] sub-tile, 8 KB
constexpr int XSTAGE_BYTES = 4 * SUBX;              // 32 KB
// ROWS = Q' rows per work item: 128 (two warpgroups), or 64 for one prompt with T <= 8 tokens (one warpgroup; the A tiles
// and their shared-memory reads halve, and the space buys a 4th image-token stage).
template <int ROWS>
struct Cfg {
  static constexpr int NWG = ROWS / 64;
  static constexpr int THREADS = NWG * 128 + 128;   // consumer warpgroups, then a warpgroup whose first two warps load
  static constexpr int XSTAGES = ROWS == 64 ? 4 : 3;
  static constexpr int QSUB = ROWS * 128;           // one 64-channel slice of Q'
  static constexpr int OFF_PE = XSTAGES * XSTAGE_BYTES;
  static constexpr int OFF_Q = OFF_PE + PESLOTS * SUBX;
  static constexpr int OFF_BAR = OFF_Q + 4 * QSUB;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};
constexpr int NTILES = 4096 / XT;
}  // namespace t2i

struct T2iParams {
  int n_items;
  float* out;  // [n_items * 128, 256] fp32: softmax-weighted mean of the image tokens per row
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int ROWS, int MODE>
__global__ void __launch_bounds__(t2i::Cfg<ROWS>::THREADS, 1)
t2i_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmXS,
                 const __grid_constant__ CUtensorMap tmQ, const T2iParams p) {
  using namespace t2i;
  using C = Cfg<ROWS>;
  constexpr int NWG = C::NWG, XSTAGES = C::XSTAGES, QSUB = C::QSUB, OFF_PE = C::OFF_PE, OFF_Q = C::OFF_Q, OFF_BAR = C::OFF_BAR;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* xfull = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* xempty = xfull + XSTAGES;
  uint64_t* pefull = xempty + XSTAGES;
  uint64_t* peempty = pefull + PESLOTS;
  uint64_t* q_full = peempty + PESLOTS;
  uint64_t* q_empty = q_full + 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == NWG * 4 && lane == 0) {
    prefetch_tmap(&tmX); prefetch_tmap(&tmXS); prefetch_tmap(&tmQ);
    for (int i = 0; i < XSTAGES; ++i) { mbar_init(&xfull[i], 1); mbar_init(&xempty[i], NWG * 4); }
    for (int i = 0; i < PESLOTS; ++i) { mbar_init(&pefull[i], 1); mbar_init(&peempty[i], NWG * 4); }
    mbar_init(q_full, 1); mbar_init(q_empty, NWG * 4);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // The U accumulator alone takes 128 registers: the loading warpgroup hands its registers to the consumer warpgroups
    // (2 x 128 x 232 + 128 x 40 <= 64 K registers, the per-sub-partition split included).
    if constexpr (NWG == 2) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == NWG * 4) {
    // ------------------------------------------------------------ TMA producer: Q' per item, image-token tiles (K = V)
    if (lane == 0) {
      int stage = 0, ni = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x, ++ni) {
        mbar_wait(q_empty, (ni & 1) ^ 1, 20);
        mbar_expect_tx(q_full, 4 * QSUB);
#pragma unroll
        for (int j = 0; j < 4; ++j) tma_load_2d(smem + OFF_Q + j * QSUB, &tmQ, q_full, 64 * j, item * ROWS);
        const int row0 = MODE ? item * 4096 : 0;
        for (int kt = 0; kt < NTILES; ++kt) {
          if (MODE && kt + 8 < NTILES) {  // own keys: a tile 8 steps ahead -> L2
#pragma unroll
            for (int j = 0; j < 4; ++j) tma_prefetch_2d(&tmX, 64 * j, row0 + (kt + 8) * XT);
          }
          mbar_wait(&xempty[stage], phase ^ 1, 21);
          uint8_t* sx = smem + stage * XSTAGE_BYTES;
          mbar_expect_tx(&xfull[stage], XSTAGE_BYTES);
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_load_2d(sx + j * SUBX, &tmX, &xfull[stage], 64 * j, row0 + kt * XT);
          if (++stage == XSTAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    } else if (warp == NWG * 4 + 1) {
    // ------------------------------------------------------------ TMA producer: second score operand (pe, or src + pe)
    if (lane == 0) {
      int slot = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        for (int kt = 0; kt < NTILES; ++kt) {
          for (int j = 0; j < 4; ++j) {
            mbar_wait(&peempty[slot], phase ^ 1, 22);
            mbar_expect_tx(&pefull[slot], SUBX);
            tma_load_2d(smem + OFF_PE + slot * SUBX, &tmXS, &pefull[slot], 64 * j, kt * XT);
            if (++slot == PESLOTS) { slot = 0; phase ^= 1; }
          }
        }
      }
    }
    }
    return;
  }
  if constexpr (NWG == 2) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");

  // ------------------------------------------------------------ warpgroup g: rows [64 g, 64 g + 64) of the item.
  // Fragment element i of a thread: row 64 g + 16 wq + qr + 8 ((i >> 1) & 1), column 8 (i >> 2) + qc + (i & 1).
  const int g = warp >> 2, wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
  const uint32_t aQ = smem_u32(smem + OFF_Q) + (uint32_t)g * 8192u;
  int stage = 0, slot = 0, ni = 0;
  uint32_t phase = 0, pephase = 0;
  for (int item = blockIdx.x; item < p.n_items; item += gridDim.x, ++ni) {
    mbar_wait(q_full, ni & 1, 26);
    float u[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) u[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll 1
    for (int kt = 0; kt < NTILES; ++kt) {
      const uint32_t xb = smem_u32(smem + stage * XSTAGE_BYTES);
      float s[32];
      int slots[4];
      // every operand of the S chain has landed before the first wgmma: no spin loop between the MMAs of one group
      if constexpr (MODE) mbar_wait(&xfull[stage], phase, 28);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mbar_wait(&pefull[slot], pephase, 29);
        slots[j] = slot;
        if (++slot == PESLOTS) { slot = 0; pephase ^= 1; }
      }
      wg_fence();
      if constexpr (MODE) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma<64>(s, make_desc_sw128(aQ + j * QSUB + k * 32, 0, 1024), make_desc_sw128(xb + j * SUBX + k * 32, 0, 1024), (j | k) != 0);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t pb = smem_u32(smem + OFF_PE + slots[j] * SUBX);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma<64>(s, make_desc_sw128(aQ + j * QSUB + k * 32, 0, 1024), make_desc_sw128(pb + k * 32, 0, 1024), (MODE | j | k) != 0);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(s);
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) mbar_arrive(&peempty[slots[j]]);
        if (kt == NTILES - 1) mbar_arrive(q_empty);   // every read of Q' by this item has completed
      }
      // online softmax (log2 units)
      uint32_t pk[16];
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        float mt = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s[4 * j + 2 * rs] *= 1.4426950408889634f;
          s[4 * j + 2 * rs + 1] *= 1.4426950408889634f;
          mt = fmaxf(mt, fmaxf(s[4 * j + 2 * rs], s[4 * j + 2 * rs + 1]));
        }
        mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
        mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
        const float m_new = fmaxf(m_run[rs], mt);
        const float f = ex2f(m_run[rs] - m_new);
        m_run[rs] = m_new;
        float ls = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float p0 = ex2f(s[4 * j + 2 * rs] - m_new), p1 = ex2f(s[4 * j + 2 * rs + 1] - m_new);
          ls += p0 + p1;
          pk[2 * j + rs] = pack_bf16(p0, p1);
        }
        l_run[rs] = l_run[rs] * f + ls;
#pragma unroll
        for (int j = 0; j < 32; ++j) { u[4 * j + 2 * rs] *= f; u[4 * j + 2 * rs + 1] *= f; }
      }
      // U += P X (X consumed MN-major: 16 tokens = 2048 B; next 64 channels = 8 KB)
      if constexpr (!MODE) mbar_wait(&xfull[stage], phase, 24);
      wg_fence();
#pragma unroll
      for (int kk = 0; kk < XT / 16; ++kk) {
        const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
        wgmma_rs<256, 1>(u, a, make_desc_sw128(xb + kk * 2048, SUBX, 1024), 1);
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(u);
      __syncwarp();
      if (lane == 0) mbar_arrive(&xempty[stage]);
      if (++stage == XSTAGES) { stage = 0; phase ^= 1; }
    }
    // ---- item epilogue: U / l -> global
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      float l = l_run[rs];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv = 1.0f / l;
      float* dst = p.out + ((size_t)item * ROWS + 64 * g + 16 * wq + qr + 8 * rs) * 256;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        *reinterpret_cast<float2*>(dst + 8 * j + qc) = make_float2(u[4 * j + 2 * rs] * inv, u[4 * j + 2 * rs + 1] * inv);
    }
  }
}

template <int ROWS, int MODE>
static int launch_t2i_fused_t(const T2iFusedArgs& a, int num_sms, cudaStream_t stream) {
  using namespace t2i;
  using C = Cfg<ROWS>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(t2i_fused_kernel<ROWS, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return set_error("t2i_fused: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap tmX, tmXS, tmQ;
  const uint64_t xrows = a.mode ? (uint64_t)a.n_items * 4096 : 4096;
  if (make_tmap_bf16_2d(&tmX, a.x, xrows, 256, 256, XT)) return -1;
  if (make_tmap_bf16_2d(&tmXS, a.xs, 4096, 256, 256, XT)) return -1;
  if (make_tmap_bf16_2d(&tmQ, a.qp, (uint64_t)a.n_items * ROWS, 256, 256, ROWS)) return -1;
  T2iParams p;
  p.n_items = a.n_items; p.out = a.out;
  const int grid = a.n_items < num_sms ? a.n_items : num_sms;
  prof_begin(stream, ROWS == 64 ? "t2i_fused<64>" : "t2i_fused<128>", (double)a.n_items * 4096 * ROWS * 256 * 2.0 * 3,
             (double)a.n_items * (ROWS * 256.0 * 2 + ROWS * 256.0 * 4) + (a.mode ? (double)a.n_items * 4096 * 512 : 0.0));
  t2i_fused_kernel<ROWS, MODE><<<grid, C::THREADS, C::SMEM_BYTES, stream>>>(tmX, tmXS, tmQ, p);
  prof_end(stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("t2i_fused launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

int launch_t2i_fused(const T2iFusedArgs& a, int num_sms, cudaStream_t stream) {
  if (a.n_items <= 0) return set_error("t2i_fused: empty problem");
  if (a.rows == 64) return a.mode ? launch_t2i_fused_t<64, 1>(a, num_sms, stream) : launch_t2i_fused_t<64, 0>(a, num_sms, stream);
  if (a.rows == 128) return a.mode ? launch_t2i_fused_t<128, 1>(a, num_sms, stream) : launch_t2i_fused_t<128, 0>(a, num_sms, stream);
  return set_error("t2i_fused: rows per item must be 64 or 128 (%d)", a.rows);
}

// Row of prompt pp, head h, token t inside the Q' / U tensors.
__device__ __forceinline__ size_t t2i_row(int pp, int h, int t, int paired) {
  return paired ? (size_t)(pp >> 1) * 128 + (pp & 1) * 64 + h * 8 + t : (size_t)pp * 128 + h * 16 + t;
}

// qexp[(item row), 128]: row of (prompt, head h, token t) = 0.25 * q[p, t] restricted to head h's 16 channels, zero elsewhere
// (and zero for the unused rows), so that the plain GEMM  Q' = qexp . WkT^T  yields the per-head products.
__global__ void t2i_prep_kernel(const __nv_bfloat16* __restrict__ q, int P, int T, int paired, __nv_bfloat16* __restrict__ qexp) {
  const int item = blockIdx.x;
  for (int i = threadIdx.x; i < 128 * 128; i += blockDim.x) {
    const int row = i >> 7, c = i & 127;
    int pp, h, t;
    if (paired) { pp = item * 2 + (row >> 6); h = (row >> 3) & 7; t = row & 7; }
    else { pp = item; h = row >> 4; t = row & 15; }
    float v = 0.f;
    if (pp < P && t < T && (c >> 4) == h) v = 0.25f * __bfloat162float(q[((size_t)pp * T + t) * 128 + c]);
    qexp[(size_t)item * 128 * 128 + i] = __float2bfloat16(v);
  }
}

// out[p, t, o = h*16 + d] = bv[o] + Wv[o, :] . U[row(p, h, t), :]     grid = P, block = 128 (thread = output channel o);
// WvT = Wv transposed [256, 128] so that the weight reads are coalesced.  All T (<= 16) tokens of the prompt are staged in
// shared memory (T x 8 heads x 256 fp32 <= 128 KB) so that every weight is loaded once per prompt.
template <int TT>
__global__ void __launch_bounds__(128)
t2i_head_proj_kernel(const float* __restrict__ U, const __nv_bfloat16* __restrict__ WvT, const float* __restrict__ bv, int T,
                     int paired, __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(16) float su[];  // [T][8][256]
  const int pp = blockIdx.x, o = threadIdx.x, h = o >> 4;
  for (int i = threadIdx.x; i < T * 8 * 64; i += 128) {
    const int t = i / 512, hh = (i >> 6) & 7, c4 = i & 63;
    reinterpret_cast<float4*>(su)[i] = __ldg(reinterpret_cast<const float4*>(U + t2i_row(pp, hh, t, paired) * 256) + c4);
  }
  __syncthreads();
  float acc[TT];
#pragma unroll
  for (int t = 0; t < TT; ++t) acc[t] = 0.f;
  const float* uh = su + h * 256;
#pragma unroll 4
  for (int c = 0; c < 256; c += 4) {
    const float w0 = __bfloat162float(WvT[(c + 0) * 128 + o]), w1 = __bfloat162float(WvT[(c + 1) * 128 + o]);
    const float w2 = __bfloat162float(WvT[(c + 2) * 128 + o]), w3 = __bfloat162float(WvT[(c + 3) * 128 + o]);
#pragma unroll
    for (int t = 0; t < TT; ++t) {
      if (t < T) {
        const float4 u = *reinterpret_cast<const float4*>(uh + t * 2048 + c);
        acc[t] = fmaf(w0, u.x, fmaf(w1, u.y, fmaf(w2, u.z, fmaf(w3, u.w, acc[t]))));
      }
    }
  }
  const float b = bv[o];
#pragma unroll
  for (int t = 0; t < TT; ++t)
    if (t < T) out[((size_t)pp * T + t) * 128 + o] = __float2bfloat16(b + acc[t]);
}

int launch_t2i_prep(const __nv_bfloat16* q, int P, int T, int paired, int n_items, __nv_bfloat16* qexp, cudaStream_t stream) {
  t2i_prep_kernel<<<n_items, 256, 0, stream>>>(q, P, T, paired, qexp);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("t2i_prep launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}
int launch_t2i_head_proj(const float* U, const __nv_bfloat16* WvT, const float* bv, int P, int T, int paired,
                         __nv_bfloat16* out, cudaStream_t stream) {
  const int smem = T * 8 * 256 * 4;
  cudaError_t e = cudaSuccess;
  if (T <= 8) {
    static bool attr8 = false;
    if (!attr8) { e = cudaFuncSetAttribute(t2i_head_proj_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 8192); attr8 = true; }
    if (e == cudaSuccess) t2i_head_proj_kernel<8><<<P, 128, smem, stream>>>(U, WvT, bv, T, paired, out);
  } else {
    static bool attr16 = false;
    if (!attr16) { e = cudaFuncSetAttribute(t2i_head_proj_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16 * 8192); attr16 = true; }
    if (e == cudaSuccess) t2i_head_proj_kernel<16><<<P, 128, smem, stream>>>(U, WvT, bv, T, paired, out);
  }
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("t2i_head_proj launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

}  // namespace msam
