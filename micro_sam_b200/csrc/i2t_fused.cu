// Fused image -> token cross-attention block of the two-way transformer (TwoWayAttentionBlock step 4, restated in
// oracle/sam_ref.py):        keys <- LayerNorm(keys + out_proj(softmax((keys + pe) Wq^T . k_tok^T / 4) v_tok))
// for P prompts x 4096 image tokens x T <= 8 prompt tokens, as ONE pass over `keys` (read 2 MB + write 2 MB per prompt;
// the unfused chain -- q projection GEMM, attention core, out-projection GEMM + LN -- moved ~3.5x those bytes).
//
// Algebra (exact up to bf16 rounding of the small per-prompt operands):
//   scores[r, (h,t)] = (x_r + pe_r) . Mq[(h,t)] + c[(h,t)],  Mq[(h,t)] = 0.25 * Wq_h^T k_tok[t,h]   ([64, 256] per prompt)
//   attn_out . Wo^T  = P[r, (h,t)] . V'[(h,t)],              V'[(h,t)] = Wo_h v_tok[t,h]            ([64, 256] per prompt)
// so per 64-row item the tensor core runs  S = X Mq^T (+ PE Mq^T)  and  O = X + P V'  (the residual X is read from the
// ring stage into registers, in fragment order, while the score MMAs run; it seeds the O accumulator, bf16 -> fp32 exactly,
// before P V' accumulates onto it) and the CUDA cores only do the 8-head x T softmax and the LayerNorm.  Mq / V'^T come
// from two small plain GEMMs (decoder.cu).
//
// Work item = (prompt, 64-row tile).  CTA = 2 consumer warpgroups (wgmma chains, softmax and LayerNorm straight from the
// accumulator fragments, P fed back from registers) + 1 warpgroup of which warps 8 / 9 issue the TMA loads and warps
// 10 / 11 the TMA stores of consumer warpgroup 0 / 1; persistent over a contiguous range of items, which the two consumers
// take alternately, so Mq / V' stay resident while the prompt does not change.  Each consumer has its own keys ring and
// output staging tiles, so the two drift apart: one warpgroup's softmax, LayerNorm and staging writes run while the other's
// MMAs keep the tensor core busy.
//   ring per warpgroup (3 stages x 16 KB; 3 stages + 2 staging tiles per warpgroup measured faster than 4 stages + 1):
//     [a0_j | a1_j], j = 64-column slice, [64 x 64] each
//     mode 1 (per-prompt keys): a0 = keys tile, a1 = pe tile:       S += a0 Mq_j^T + a1 Mq_j^T ; O[:, 64j..] = a0
//     mode 0 (layer 0, shared): a0 = (src+pe) tile, a1 = src tile: S += a0 Mq_j^T             ; O[:, 64j..] = a1
//   output: each warpgroup writes its normalised rows slice by slice into two [64 x 64] SW128 staging tiles (full / empty
//   mbarriers with its store warp), which stores them with TMA, so the stores leave as whole 128-B rows.
// Mode 1 writes `keys` in place.  That is safe because every item reads (TMA-loads) only its own 64 rows, all four slices
// of them before its store warp writes them, and no other item reads those rows.  The keys are not prefetched into L2
// ahead of their loads: at P = 1024 a prefetch of the warpgroup's next items made the own-keys launch 1.4x slower.
//
// Mq / V' handover.  The 64 KB of a prompt's operands are single-buffered and shared by both consumers.  Warp 8 loads them
// for the prompts p_first, p_first + 1, ... of the CTA's range in order; its n-th load completes phase n of mv_full, and
// before it issues load n > 0 it waits for phase n - 1 of mv_empty.  Each consumer warpgroup walks the same prompts in the
// same order: it waits for phase n of mv_full, then each of its 4 warps arrives on mv_empty exactly once for prompt n --
// after the warpgroup's last P V' MMA of the prompt, or at once when it has no item of the prompt (a range holding one
// item of a prompt; at P = 1 warpgroup 1 has no item at all).  So every phase of mv_empty collects exactly its 8 arrivals.
// They cannot complete an earlier phase: a warpgroup arrives for prompt n only after it observed load n, which warp 8
// issued after phase n - 1 of mv_empty had completed.  Hence Mq / V' are overwritten only once both warpgroups are done
// with them.  And mv_full is never more than one phase ahead of a waiting warpgroup (load n + 1 needs that warpgroup's
// arrival for prompt n), so its parity wait cannot be satisfied by the wrong phase.
#include "kernels.h"
#include "ptx.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace msam {

namespace i2t {
constexpr int STAGES = 3;                      // keys ring stages per warpgroup
constexpr int SUB = 64 * 128;                  // [64 rows x 64 bf16] SWIZZLE_128B sub-tile
constexpr int STAGE_BYTES = 2 * SUB;
constexpr int OFF_M = 2 * STAGES * STAGE_BYTES;  // Mq[p]: 4 K-slices of [64 x 64]
constexpr int OFF_V = OFF_M + 32768;           // V'^T[p]: [256 x 64]
constexpr int OBUF = 2;                        // output staging buffers per warpgroup
constexpr int OFF_O = OFF_V + 32768;           // output staging: 2 warpgroups x OBUF x [64 x 64] bf16 SW128
constexpr int OFF_BAR = OFF_O + 2 * OBUF * 8192;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
constexpr int THREADS = 256 + 128;             // 2 warpgroups, then a warpgroup: warps 8 / 9 issue the TMA loads, 10 / 11 the stores
constexpr int TILES = 64;                      // 4096 image tokens / 64 rows = items per prompt
static_assert(SMEM_BYTES + 768 * 4 <= 227 * 1024, "rings + operands + staging + rowp exceed the shared memory of an SM");

// first item of warpgroup g (items it_begin + g, + 2, ...) in prompt pp of the range
__device__ __forceinline__ int first_item(int pp, int it_begin, int g) {
  const int lo = max(it_begin, pp * TILES);
  return lo + ((lo - it_begin - g) & 1);
}
}  // namespace i2t

struct I2tParams {
  int P, T, mode;
  const float* sbias;  // [P, 64] score bias c
  const float *bias, *gamma, *beta;
  float eps;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(i2t::THREADS, 1)
i2t_fused_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmM, const __grid_constant__ CUtensorMap tmV,
                 const __grid_constant__ CUtensorMap tmO, const I2tParams p) {
  using namespace i2t;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);  // [g * STAGES + s]
  uint64_t* empty_bar = full_bar + 2 * STAGES;  // [g * STAGES + s]: the 4 warps of warpgroup g arrive
  uint64_t* mv_full = empty_bar + 2 * STAGES;
  uint64_t* mv_empty = mv_full + 1;     // the 8 consumer warps arrive once per prompt of the range
  uint64_t* ofull = mv_empty + 1;       // [g * OBUF + b]: staging tile b of warpgroup g written (4 warps arrive)
  uint64_t* oempty = ofull + 2 * OBUF;  // [g * OBUF + b]: its TMA store has read it
  __shared__ __align__(16) float rowp[768];  // out-proj bias | gamma | beta

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long total = (long)p.P * TILES;
  const int it_begin = (int)(total * blockIdx.x / gridDim.x), it_end = (int)(total * (blockIdx.x + 1) / gridDim.x);
  const int p_first = it_begin / TILES, p_last = (it_end - 1) / TILES;  // the launch keeps every range non-empty

  if (warp == 8 && lane == 0) {
    prefetch_tmap(&tmA0); prefetch_tmap(&tmA1); prefetch_tmap(&tmM); prefetch_tmap(&tmV); prefetch_tmap(&tmO);
    for (int i = 0; i < 2 * STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    mbar_init(mv_full, 1); mbar_init(mv_empty, 8);
    for (int i = 0; i < 2 * OBUF; ++i) { mbar_init(&ofull[i], 4); mbar_init(&oempty[i], 1); }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 256; i += THREADS) { rowp[i] = p.bias[i]; rowp[256 + i] = p.gamma[i]; rowp[512 + i] = p.beta[i]; }
  __syncthreads();

  if (warp >= 8) {
    // O (128 registers) + S (32): the loading warpgroup hands its registers to the two consumer warpgroups
    // (2 x 128 x 232 + 128 x 40 <= 64 K registers, the per-sub-partition split included)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp < 10 && lane == 0) {
      // ---------------------------------------------------------- TMA loads of consumer warpgroup g = warp - 8; warp 8
      // also loads Mq / V' of every prompt of the range (handover protocol in the header comment)
      const int g = warp - 8;
      int stage = 0;
      uint32_t phase = 0;
      for (int pp = p_first; pp <= p_last; ++pp) {
        if (g == 0) {
          if (pp > p_first) mbar_wait(mv_empty, (pp - p_first - 1) & 1, 10);  // both warpgroups are done with Mq / V'
          mbar_expect_tx(mv_full, 65536);
#pragma unroll
          for (int j = 0; j < 4; ++j) tma_load_2d(smem + OFF_M + j * 8192, &tmM, mv_full, 64 * j, pp * 64);
          tma_load_2d(smem + OFF_V, &tmV, mv_full, pp * 64, 0);
        }
        const int hi = min(it_end, (pp + 1) * TILES);
        for (int item = first_item(pp, it_begin, g); item < hi; item += 2) {
          const int rt = item - pp * TILES;
          const int row0 = p.mode ? item * 64 : rt * 64, row1 = rt * 64;
          for (int j = 0; j < 4; ++j) {
            mbar_wait(&empty_bar[g * STAGES + stage], phase ^ 1, 11);
            uint8_t* sa = smem + (g * STAGES + stage) * STAGE_BYTES;
            mbar_expect_tx(&full_bar[g * STAGES + stage], STAGE_BYTES);
            tma_load_2d(sa, &tmA0, &full_bar[g * STAGES + stage], 64 * j, row0);
            tma_load_2d(sa + SUB, &tmA1, &full_bar[g * STAGES + stage], 64 * j, row1);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else if (lane == 0) {
      // ---------------------------------------------------------- TMA stores of consumer warpgroup g = warp - 10 (kept out
      // of the consumers' code, where the store instructions cost ptxas the registers of the wgmma pipeline)
      const int g = warp - 10;
      int ob = 0;
      uint32_t ophase = 0;
      for (int item = it_begin + g; item < it_end; item += 2) {
        for (int j = 0; j < 4; ++j) {
          mbar_wait(&ofull[g * OBUF + ob], ophase, 14);
          tma_store_2d(&tmO, smem + OFF_O + (g * OBUF + ob) * 8192, 64 * j, item * 64);
          tma_store_commit();
          tma_store_wait_read<0>();
          mbar_arrive(&oempty[g * OBUF + ob]);
          if (++ob == OBUF) { ob = 0; ophase ^= 1; }
        }
      }
      tma_store_wait_all();
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");

  // ------------------------------------------------------------ consumer warpgroup g: items it_begin + g, + 2, ...
  // Fragment element i of a thread: row 16 wq + qr + 8 ((i >> 1) & 1) of the item, column 8 (i >> 2) + qc + (i & 1).
  // In a [64 x 64] SW128 tile (the ring's residual half, the output staging) the bf16 pair (row r, columns 8 jj + qc, +1)
  // sits at byte r * 128 + ((jj ^ (r & 7)) << 4) + 2 qc, and r & 7 = qr: the 8 rows of a warp hit 8 distinct 16-B chunks.
  const int g = warp >> 2, wq = warp & 3, qr = lane >> 2, qc = 2 * (lane & 3);
  const uint32_t ring = smem_u32(smem) + (uint32_t)(g * STAGES * STAGE_BYTES);
  const uint32_t frag = (uint32_t)(16 * wq + qr) * 128u + (uint32_t)qc * 2u;  // byte offset of rows rs = 0 (+1024: rs = 1)
  const uint32_t aV = smem_u32(smem + OFF_V), ostage = smem_u32(smem + OFF_O) + (uint32_t)g * (OBUF * 8192u);
  const int T = p.T;
  int stage = 0, ob = 0;
  uint32_t phase = 0, ophase = 0;
  for (int pp = p_first; pp <= p_last; ++pp) {
    mbar_wait(mv_full, (pp - p_first) & 1, 12);
    const int hi = min(it_end, (pp + 1) * TILES);
    int item = first_item(pp, it_begin, g);
    if (item >= hi) {  // no item of this prompt: release Mq / V' at once
      __syncwarp();
      if (lane == 0) mbar_arrive(mv_empty);
    }
    for (; item < hi; item += 2) {
      float sacc[32], o[128];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mbar_wait(&full_bar[g * STAGES + stage], phase, 13);
        const uint32_t sa = ring + (uint32_t)(stage * STAGE_BYTES);
        const uint64_t d0 = make_desc_sw128(sa, 0, 1024), d1 = make_desc_sw128(sa + SUB, 0, 1024);
        const uint64_t dm = make_desc_sw128(smem_u32(smem + OFF_M + j * 8192), 0, 1024);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma<64>(sacc, d0 + 2 * k, dm + 2 * k, (j | k) != 0);
        if (p.mode) {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma<64>(sacc, d1 + 2 * k, dm + 2 * k, 1);
        }
        wg_commit();
        // residual columns [64 j, 64 j + 64), read while the score MMAs run
        const uint32_t res = (p.mode ? sa : sa + SUB) + frag;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            uint32_t v;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(res + rs * 1024u + ((uint32_t)(jj ^ qr) << 4)));
            o[32 * j + 4 * jj + 2 * rs] = __uint_as_float(v << 16);  // bf16 -> fp32 is exact
            o[32 * j + 4 * jj + 2 * rs + 1] = __uint_as_float(v & 0xFFFF0000u);
          }
        }
        wg_wait<0>();
        wg_fence_acc(sacc);
        wg_fence_acc(*reinterpret_cast<float(*)[32]>(&o[32 * j]));
        // The stage was read by the wgmma (async proxy, complete after the wait) and by the ld.shared above (generic proxy).
        // Those loads have returned their values before the arrive, whose release semantics order them before the producer's
        // acquire of the empty barrier and hence before the TMA that overwrites the stage.
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[g * STAGES + stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      // softmax over the T tokens of each head h (columns 8 h + t): this thread holds t = qc, qc + 1
      const float* cb = p.sbias + (size_t)pp * 64;
      uint32_t pk[16];
#pragma unroll
      for (int h = 0; h < 8; ++h) {
        const float2 c = __ldg(reinterpret_cast<const float2*>(cb + 8 * h + qc));
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
          const float s0 = (qc < T) ? (sacc[4 * h + 2 * rs] + c.x) * 1.4426950408889634f : -1e30f;
          const float s1 = (qc + 1 < T) ? (sacc[4 * h + 2 * rs + 1] + c.y) * 1.4426950408889634f : -1e30f;
          float m = fmaxf(s0, s1);
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
          const float e0 = ex2_approx(s0 - m), e1 = ex2_approx(s1 - m);
          float l = e0 + e1;
          l += __shfl_xor_sync(0xffffffffu, l, 1);
          l += __shfl_xor_sync(0xffffffffu, l, 2);
          const float inv = __fdividef(1.0f, l);
          pk[2 * h + rs] = pack_bf16(e0 * inv, e1 * inv);
        }
      }
      // O += P V', per 64-column slice j (V'^T rows [64 j, 64 j + 64))
      wg_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float(&oj)[32] = *reinterpret_cast<float(*)[32]>(&o[32 * j]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t a[4] = {pk[4 * k], pk[4 * k + 1], pk[4 * k + 2], pk[4 * k + 3]};
          wgmma_rs<64>(oj, a, make_desc_sw128(aV + 8192 * j + 32 * k, 0, 1024), 1);
        }
      }
      wg_commit();
      wg_wait<0>();
      wg_fence_acc(o);
      if (item + 2 >= hi) {  // this warpgroup's last MMA on Mq / V' of the prompt has completed
        __syncwarp();
        if (lane == 0) mbar_arrive(mv_empty);
      }
      // + out-proj bias, LayerNorm over the 256 channels of each row (this thread: 64 of them, the quad: all)
      float sums[2] = {0.f, 0.f}, rstd[2], shift[2];
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) {
        const float2 b = *reinterpret_cast<const float2*>(&rowp[8 * jj + qc]);
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
          o[4 * jj + 2 * rs] += b.x;
          o[4 * jj + 2 * rs + 1] += b.y;
          sums[rs] += o[4 * jj + 2 * rs] + o[4 * jj + 2 * rs + 1];
        }
      }
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        float sum = sums[rs];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float mean = sum * (1.0f / 256);
        float q = 0.f;
#pragma unroll
        for (int jj = 0; jj < 32; ++jj) {
          const float d0 = o[4 * jj + 2 * rs] - mean, d1 = o[4 * jj + 2 * rs + 1] - mean;
          q = fmaf(d0, d0, fmaf(d1, d1, q));
        }
        q += __shfl_xor_sync(0xffffffffu, q, 1);
        q += __shfl_xor_sync(0xffffffffu, q, 2);
        rstd[rs] = rsqrtf(q * (1.0f / 256) + p.eps);
        shift[rs] = -mean * rstd[rs];
      }
      // normalised rows of slice j -> staging tile ob, stored by this warpgroup's store warp as the [64 x 64] block at
      // (column 64 j, rows of the item)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mbar_wait(&oempty[g * OBUF + ob], ophase ^ 1, 15);
        const uint32_t buf = ostage + (uint32_t)ob * 8192u;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int col = 64 * j + 8 * jj + qc;
          const float2 ga = *reinterpret_cast<const float2*>(&rowp[256 + col]);
          const float2 be = *reinterpret_cast<const float2*>(&rowp[512 + col]);
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            const float y0 = fmaf(fmaf(o[32 * j + 4 * jj + 2 * rs], rstd[rs], shift[rs]), ga.x, be.x);
            const float y1 = fmaf(fmaf(o[32 * j + 4 * jj + 2 * rs + 1], rstd[rs], shift[rs]), ga.y, be.y);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(buf + frag + rs * 1024u + ((uint32_t)(jj ^ qr) << 4)), "r"(pack_bf16(y0, y1))
                         : "memory");
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&ofull[g * OBUF + ob]);
        if (++ob == OBUF) { ob = 0; ophase ^= 1; }
      }
    }
  }
}

int launch_i2t_fused(const I2tFusedArgs& a, int num_sms, cudaStream_t stream) {
  using namespace i2t;
  if (a.P <= 0 || a.T < 1 || a.T > 8) return set_error("i2t_fused: needs 1 <= T <= 8 (T=%d)", a.T);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(i2t_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return set_error("i2t_fused: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  CUtensorMap tmA0, tmA1, tmM, tmV, tmO;
  const uint64_t xrows = a.mode ? (uint64_t)a.P * 4096 : 4096;
  if (make_tmap_bf16_2d(&tmA0, a.a0, xrows, 256, 256, 64)) return -1;
  if (make_tmap_bf16_2d(&tmA1, a.a1, 4096, 256, 256, 64)) return -1;
  if (make_tmap_bf16_2d(&tmM, a.mq, (uint64_t)a.P * 64, 256, 256, 64)) return -1;
  if (make_tmap_bf16_2d(&tmV, a.vt, 256, (uint64_t)a.P * 64, (uint64_t)a.P * 64, 256)) return -1;
  if (make_tmap_bf16_2d(&tmO, a.out, (uint64_t)a.P * 4096, 256, 256, 64)) return -1;
  I2tParams p;
  p.P = a.P; p.T = a.T; p.mode = a.mode; p.sbias = a.sbias; p.bias = a.bias; p.gamma = a.gamma; p.beta = a.beta; p.eps = a.eps;
  const long total = (long)a.P * TILES;
  const int grid = total < num_sms ? (int)total : num_sms;
  const double bytes = (double)a.P * 4096 * 256 * 2 * (a.mode ? 2 : 1) + (double)a.P * 64 * 256 * 2 * 2;
  prof_begin(stream, a.mode ? "i2t_fused (own keys)" : "i2t_fused (shared image)", (double)a.P * 4096 * (2.0 * 256 * 64 * (a.mode ? 2 : 1) + 2.0 * 64 * 256), bytes);
  i2t_fused_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(tmA0, tmA1, tmM, tmV, tmO, p);
  prof_end(stream);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("i2t_fused launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

// Per-prompt operands of the fused block.  kexp/vexp [(p, h, t), 128]: row (p*64 + h*8 + t) holds 0.25 * k_tok[p,t] /
// v_tok[p,t] restricted to head h's 16 channels (zero elsewhere, zero rows for t >= T), so that the plain GEMMs
//   Mq = kexp . WqT^T  ([P*64, 256])    and    V'^T = Wo . vexp^T  ([256, P*64])
// produce the block-diagonal products; sbias[(p,h,t)] = 0.25 * bq_h . k_tok[p,t,h].
__global__ void i2t_prep_kernel(const __nv_bfloat16* __restrict__ ktok, const __nv_bfloat16* __restrict__ vtok,
                                const float* __restrict__ bq, int T, __nv_bfloat16* __restrict__ kexp,
                                __nv_bfloat16* __restrict__ vexp, float* __restrict__ sbias) {
  const int pp = blockIdx.x;
  for (int i = threadIdx.x; i < 64 * 128; i += blockDim.x) {
    const int row = i >> 7, c = i & 127, h = row >> 3, t = row & 7;
    float kv = 0.f, vv = 0.f;
    if (t < T && (c >> 4) == h) {
      kv = 0.25f * __bfloat162float(ktok[((size_t)pp * T + t) * 128 + c]);
      vv = __bfloat162float(vtok[((size_t)pp * T + t) * 128 + c]);
    }
    kexp[(size_t)pp * 64 * 128 + i] = __float2bfloat16(kv);
    vexp[(size_t)pp * 64 * 128 + i] = __float2bfloat16(vv);
  }
  if (threadIdx.x < 64) {
    const int h = threadIdx.x >> 3, t = threadIdx.x & 7;
    float s = 0.f;
    if (t < T)
      for (int d = 0; d < 16; ++d) s += bq[h * 16 + d] * __bfloat162float(ktok[((size_t)pp * T + t) * 128 + h * 16 + d]);
    sbias[(size_t)pp * 64 + threadIdx.x] = 0.25f * s;
  }
}

int launch_i2t_prep(const __nv_bfloat16* ktok, const __nv_bfloat16* vtok, const float* bq, int P, int T,
                    __nv_bfloat16* kexp, __nv_bfloat16* vexp, float* sbias, cudaStream_t stream) {
  i2t_prep_kernel<<<P, 256, 0, stream>>>(ktok, vtok, bq, T, kexp, vexp, sbias);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("i2t_prep launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return 0;
}

}  // namespace msam
