// HBM-bound kernels of the ViT-encoder backward pass (BASELINE.json configs[4]: "encoder fwd/bwd"; micro_sam/training/
// sam_trainer.py:393 _train_epoch_impl -> loss.backward()).  Reference arithmetic = torch autograd over oracle/sam_ref.py
// (ImageEncoderViT), checked tensor by tensor in tests/gpu_diag.py (section "bwd") and tests/test_gpu_backward.py.
// The contractions (dgrad / wgrad of the linear layers, the five products of the attention backward) run on the tensor cores
// (gemm*.cu, gemm_tn.cu, bgemm.cu); what is here are the row-wise / element-wise pieces between them.
#include "kernels.h"
#include "ptx.cuh"

namespace msam {

namespace {

__device__ __forceinline__ uint32_t bpk2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float blo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bhi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

#define BWD_CHECK(what)                                                                              \
  do {                                                                                               \
    cudaError_t e_ = cudaGetLastError();                                                             \
    if (e_ != cudaSuccess) return set_error(what " launch failed: %s", cudaGetErrorString(e_));      \
    count_launch();                                                                                  \
  } while (0)

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm backward, one warp per row (rows strided over the grid), row held in registers as in the forward kernel:
//   xhat = (x - mean) rstd,  g = dy gamma,  dx = rstd (g - mean(g) - xhat mean(g xhat)),  dgamma += dy xhat,  dbeta += dy.
// dgamma / dbeta: per-lane register partials over the warp's rows -> shared-memory reduction over the block's warps -> one
// atomicAdd per column and block.
constexpr int LNB_V4 = 10;   // D <= 1280
constexpr int LNB_WARPS = 8;

__global__ void __launch_bounds__(LNB_WARPS * 32)
layernorm_bwd_kernel(const float* __restrict__ x, int rows, int D, const float* __restrict__ gamma, float eps,
                     const float* __restrict__ dy, int window_mode, int grid, int ws, int accumulate, float* __restrict__ dx,
                     float* __restrict__ dgamma, float* __restrict__ dbeta) {
  extern __shared__ float red[];   // [2][D]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nv = D >> 2;
  for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
  float4 pg[LNB_V4], pb[LNB_V4];
#pragma unroll
  for (int i = 0; i < LNB_V4; ++i) { pg[i] = make_float4(0, 0, 0, 0); pb[i] = make_float4(0, 0, 0, 0); }
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  for (long row = (long)blockIdx.x * LNB_WARPS + warp; row < rows; row += (long)gridDim.x * LNB_WARPS) {
    long drow = row;
    if (window_mode) {
      const int gg = grid * grid;
      const int b = row / gg, t = row % gg, y = t / grid, xx = t % grid;
      const int wpr = (grid + ws - 1) / ws;
      drow = ((long)(b * wpr + y / ws) * wpr + xx / ws) * (ws * ws) + (y % ws) * ws + (xx % ws);
    }
    const float4* xs = reinterpret_cast<const float4*>(x + row * D);
    const float4* ds = reinterpret_cast<const float4*>(dy + drow * D);
    float4 v[LNB_V4], d[LNB_V4];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < LNB_V4; ++i) {
      const int k = lane + 32 * i;
      if (k < nv) { v[i] = xs[k]; d[i] = ds[k]; sum += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
    }
    const float mean = warp_sum(sum) / (float)D;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < LNB_V4; ++i) {
      const int k = lane + 32 * i;
      if (k < nv) {
        v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
        sq += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) / (float)D + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < LNB_V4; ++i) {
      const int k = lane + 32 * i;
      if (k < nv) {
        const float4 g = __ldg(g4 + k);
        v[i].x *= rstd; v[i].y *= rstd; v[i].z *= rstd; v[i].w *= rstd;      // xhat
        pg[i].x += d[i].x * v[i].x; pg[i].y += d[i].y * v[i].y; pg[i].z += d[i].z * v[i].z; pg[i].w += d[i].w * v[i].w;
        pb[i].x += d[i].x; pb[i].y += d[i].y; pb[i].z += d[i].z; pb[i].w += d[i].w;
        d[i].x *= g.x; d[i].y *= g.y; d[i].z *= g.z; d[i].w *= g.w;          // g = dy * gamma
        sg += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        sgx += (d[i].x * v[i].x + d[i].y * v[i].y) + (d[i].z * v[i].z + d[i].w * v[i].w);
      }
    }
    const float mg = warp_sum(sg) / (float)D, mgx = warp_sum(sgx) / (float)D;
    float4* out = reinterpret_cast<float4*>(dx + row * D);
#pragma unroll
    for (int i = 0; i < LNB_V4; ++i) {
      const int k = lane + 32 * i;
      if (k < nv) {
        float4 r;
        r.x = rstd * (d[i].x - mg - v[i].x * mgx); r.y = rstd * (d[i].y - mg - v[i].y * mgx);
        r.z = rstd * (d[i].z - mg - v[i].z * mgx); r.w = rstd * (d[i].w - mg - v[i].w * mgx);
        if (accumulate) { const float4 o = out[k]; r.x += o.x; r.y += o.y; r.z += o.z; r.w += o.w; }
        out[k] = r;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < LNB_V4; ++i) {
    const int k = lane + 32 * i;
    if (k < nv) {
      atomicAdd(&red[4 * k], pg[i].x); atomicAdd(&red[4 * k + 1], pg[i].y); atomicAdd(&red[4 * k + 2], pg[i].z); atomicAdd(&red[4 * k + 3], pg[i].w);
      atomicAdd(&red[D + 4 * k], pb[i].x); atomicAdd(&red[D + 4 * k + 1], pb[i].y); atomicAdd(&red[D + 4 * k + 2], pb[i].z); atomicAdd(&red[D + 4 * k + 3], pb[i].w);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    atomicAdd(dgamma + i, red[i]);
    atomicAdd(dbeta + i, red[D + i]);
  }
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void gelu_fwd_kernel(const uint4* __restrict__ pre, long n8, uint4* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint4 u = pre[i];
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float a = blo(w[j]), b = bhi(w[j]);
    o[j] = bpk2(0.5f * a * (1.0f + erff(a * 0.70710678118654752440f)), 0.5f * b * (1.0f + erff(b * 0.70710678118654752440f)));
  }
  out[i] = make_uint4(o[0], o[1], o[2], o[3]);
}
// d/dx [x Phi(x)] = Phi(x) + x phi(x)
__device__ __forceinline__ float gelu_grad(float x) {
  return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}
__global__ void gelu_bwd_kernel(const uint4* __restrict__ dh, const uint4* __restrict__ pre, long n8, uint4* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint4 u = pre[i], g = dh[i];
  const uint32_t w[4] = {u.x, u.y, u.z, u.w}, gw[4] = {g.x, g.y, g.z, g.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) o[j] = bpk2(blo(gw[j]) * gelu_grad(blo(w[j])), bhi(gw[j]) * gelu_grad(bhi(w[j])));
  out[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

// out[N] += column sums of bf16 x [rows, N]: block = 64 columns x 4 row lanes, 256 rows per block
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ x, long rows, int N, float* __restrict__ out) {
  __shared__ float part[4][64];
  const int c = blockIdx.x * 64 + (threadIdx.x & 63), rl = threadIdx.x >> 6;
  const long r0 = (long)blockIdx.y * 256, r1 = (r0 + 256 < rows) ? r0 + 256 : rows;
  float s = 0.f;
  if (c < N)
    for (long r = r0 + rl; r < r1; r += 4) s += __bfloat162float(x[r * N + c]);
  part[rl][threadIdx.x & 63] = s;
  __syncthreads();
  if (rl == 0 && c < N) atomicAdd(out + c, part[0][threadIdx.x] + part[1][threadIdx.x] + part[2][threadIdx.x] + part[3][threadIdx.x]);
}

// image-order bf16 [B*g*g, D] -> window-partitioned bf16 [B*wpr*wpr*ws*ws, D], zeros at the pad rows.  One thread = 8 channels.
__global__ void window_gather_kernel(const __nv_bfloat16* __restrict__ x, int B, int grid, int ws, int D,
                                     __nv_bfloat16* __restrict__ out) {
  const int wpr = (grid + ws - 1) / ws, c8 = D / 8;
  const long total = (long)B * wpr * wpr * ws * ws * c8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = idx % c8;
  const long row = idx / c8;
  const int t = row % (ws * ws);
  const long win = row / (ws * ws);
  const int wx = win % wpr, wy = (win / wpr) % wpr;
  const long b = win / ((long)wpr * wpr);
  const int y = wy * ws + t / ws, xx = wx * ws + t % ws;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (y < grid && xx < grid) v = *reinterpret_cast<const uint4*>(x + ((b * grid + y) * grid + xx) * D + cc * 8);
  *reinterpret_cast<uint4*>(out + row * D + cc * 8) = v;
}

// ---------------------------------------------------------------------------------------------------------------
// Attention backward, element-wise stages.  One warp per query row of one batch entry (window | image, head).
// Geometry: keys k = kh * side + kw (kh, kw < side), queries likewise; bias[q, k] = T[q, qh - kh + side - 1] + T[q, woff + qw - kw + side - 1]
// with T = Q RelTable^T (rows [0, 2 side - 1) = rel_pos_h, rows [woff, woff + 2 side - 1) = rel_pos_w), exactly the forward kernels.
// P = softmax_k(scale * S + bias)  (bf16 out, the operand of dV = P^T dO)
// Three passes over the row (max, sum, write): the 0.8 .. 16 KB row stays in L1 / L2 between them.  (A register-resident variant --
// 128 logits per lane for the 4096-key rows -- needs 255 registers and runs one block per SM.)
__global__ void attn_probs_kernel(const float* __restrict__ S, const float* __restrict__ T, long n_rows, AttnBwdGeom g, int pitch_s,
                                  int pitch_p, float scale, __nv_bfloat16* __restrict__ P) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int q = row % g.n_tok;
  const int qh = q / g.side, qw = q % g.side;
  const float* s = S + row * pitch_s;
  const float* t = T + row * g.nt;
  __nv_bfloat16* p = P + row * pitch_p;
  const int oh = qh + g.side - 1, ow = g.woff + qw + g.side - 1;
  // flat key loop, all 32 lanes busy for every geometry (a (kh, kw) double loop without the integer divisions leaves lanes idle for
  // the 14-wide windows and doubles the loop overhead for the 64-wide rows).
  float m = -INFINITY;
  for (int k = lane; k < g.n_tok; k += 32) m = fmaxf(m, fmaf(s[k], scale, t[oh - k / g.side] + t[ow - k % g.side]));
  m = warp_max(m);
  float l = 0.f;
  for (int k = lane; k < g.n_tok; k += 32) l += __expf(fmaf(s[k], scale, t[oh - k / g.side] + t[ow - k % g.side]) - m);
  const float inv = 1.0f / warp_sum(l);
  for (int k = lane; k < pitch_p; k += 32)
    p[k] = __float2bfloat16(k < g.n_tok ? __expf(fmaf(s[k], scale, t[oh - k / g.side] + t[ow - k % g.side]) - m) * inv : 0.f);
}

// dS = P o (dP - delta), delta = sum_k P dP;  dT[q, j] = the bias gradients scattered to the table-row index j (zero elsewhere)
__global__ void attn_ds_kernel(const __nv_bfloat16* __restrict__ P, const float* __restrict__ dP, long n_rows, AttnBwdGeom g,
                               int pitch_s, int pitch_p, __nv_bfloat16* __restrict__ dS, __nv_bfloat16* __restrict__ dT) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int q = row % g.n_tok;
  const int qh = q / g.side, qw = q % g.side;
  const __nv_bfloat16* p = P + row * pitch_p;
  const float* dp = dP + row * pitch_s;
  __nv_bfloat16* ds = dS + row * pitch_p;
  __nv_bfloat16* dt = dT + row * g.nt;
  float del = 0.f;
  for (int k = lane; k < g.n_tok; k += 32) del += __bfloat162float(p[k]) * dp[k];   // second use below hits L1 / L2 (8 .. 24 KB per row)
  del = warp_sum(del);
  for (int j = lane; j < g.nt; j += 32) dt[j] = __float2bfloat16(0.f);
  __syncwarp();
  float accw[2] = {0.f, 0.f};   // dTw[kw] for kw = lane, lane + 32
  for (int kh = 0; kh < g.side; ++kh) {
    float rowsum = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int kw = lane + 32 * i;
      if (kw < g.side) {
        const int k = kh * g.side + kw;
        const float v = __bfloat162float(p[k]) * (dp[k] - del);
        ds[k] = __float2bfloat16(v);
        rowsum += v;
        accw[i] += v;
      }
    }
    rowsum = warp_sum(rowsum);
    if (lane == 0) dt[qh - kh + g.side - 1] = __float2bfloat16(rowsum);
  }
  for (int k = g.n_tok + lane; k < pitch_p; k += 32) ds[k] = __float2bfloat16(0.f);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int kw = lane + 32 * i;
    if (kw < g.side) dt[g.woff + qw - kw + g.side - 1] = __float2bfloat16(accw[i]);
  }
}

// dq / dk / dv fp32 [outer, heads, T, d] -> dqkv bf16 [outer * T, 3 * heads * d]
__global__ void pack_dqkv_kernel(const float* __restrict__ dq, const float* __restrict__ dk, const float* __restrict__ dv, int outer,
                                 int heads, int T, int d, __nv_bfloat16* __restrict__ dqkv) {
  const int d4 = d / 4;
  const long total = (long)outer * heads * T * d4 * 3;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = idx % d4;
  long r = idx / d4;
  const int t = r % T; r /= T;
  const int h = r % heads; r /= heads;
  const int w = r % outer;
  const int which = r / outer;
  const float* src = (which == 0 ? dq : (which == 1 ? dk : dv)) + (((long)w * heads + h) * T + t) * d + c4 * 4;
  const float4 v = *reinterpret_cast<const float4*>(src);
  const int D = heads * d;
  __nv_bfloat16* dst = dqkv + ((long)w * T + t) * (3 * D) + which * D + h * d + c4 * 4;
  *reinterpret_cast<uint2*>(dst) = make_uint2(bpk2(v.x, v.y), bpk2(v.z, v.w));
}

__global__ void sum_batch_kernel(const float* __restrict__ x, long n_batch, long n, float* __restrict__ out, int accumulate) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = accumulate ? out[i] : 0.f;
  for (long b = 0; b < n_batch; ++b) s += x[b * n + i];
  out[i] = s;
}

// fp32 NCHW [B, C, T] -> token-major [B*T, C] through a 32 x 32 shared-memory tile
__global__ void nchw_to_tok_kernel(const float* __restrict__ in, int C, int T, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) tile[i][threadIdx.x] = in[((long)b * C + c0 + i) * T + t0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) out[((long)b * T + t0 + i) * C + c0 + threadIdx.x] = tile[threadIdx.x][i];
}

// col2im of the 3x3 / pad 1 im2col layout [tok][(ky*3+kx)*C + c] (elementwise.cu:im2col3x3): out[tok, c] = sum_k dcol[tok - off_k, k*C + c]
__global__ void col2im3x3_kernel(const __nv_bfloat16* __restrict__ dcol, int B, int g, int C, float* __restrict__ out) {
  const int c8 = C / 8;
  const long total = (long)B * g * g * c8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = idx % c8;
  const long tok = idx / c8;
  const int xx = tok % g, y = (tok / g) % g;
  const long b = tok / ((long)g * g);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    // output token (oy, ox) read input (oy + k/3 - 1, ox + k%3 - 1) = (y, xx)  ->  oy = y - k/3 + 1, ox = xx - k%3 + 1
    const int oy = y - k / 3 + 1, ox = xx - k % 3 + 1;
    if (oy < 0 || oy >= g || ox < 0 || ox >= g) continue;
    const uint4 u = *reinterpret_cast<const uint4*>(dcol + (((b * g + oy) * g + ox) * 9 + k) * (long)C + cc * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[2 * j] += blo(w[j]); acc[2 * j + 1] += bhi(w[j]); }
  }
  float4* o = reinterpret_cast<float4*>(out + tok * C + cc * 8);
  o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

__global__ void cast_f32_kernel(const uint2* __restrict__ x, long n4, float4* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const uint2 u = x[i];
  out[i] = make_float4(blo(u.x), bhi(u.x), blo(u.y), bhi(u.y));
}

}  // namespace

int launch_layernorm_bwd(const float* x, int rows, int D, const float* gamma, float eps, const float* dy, int window_mode, int grid,
                         int ws, int accumulate, float* dx, float* dgamma, float* dbeta, cudaStream_t stream) {
  if (D % 4 != 0 || D > LNB_V4 * 128) return set_error("layernorm_bwd: unsupported D=%d", D);
  if (rows <= 0) return 0;
  int blocks = (rows + LNB_WARPS - 1) / LNB_WARPS;
  if (blocks > 528) blocks = 528;   // 4 x 132 SMs: bounds the number of global atomics per column
  prof_begin(stream, "layernorm_bwd", 0.0, (double)rows * D * 12);
  layernorm_bwd_kernel<<<blocks, LNB_WARPS * 32, 2 * D * sizeof(float), stream>>>(x, rows, D, gamma, eps, dy, window_mode, grid, ws,
                                                                                 accumulate, dx, dgamma, dbeta);
  prof_end(stream);
  BWD_CHECK("layernorm_bwd");
  return 0;
}
int launch_gelu_fwd(const __nv_bfloat16* pre, long n, __nv_bfloat16* out, cudaStream_t stream) {
  if (n % 8) return set_error("gelu: n must be a multiple of 8");
  gelu_fwd_kernel<<<(unsigned)((n / 8 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(pre), n / 8, reinterpret_cast<uint4*>(out));
  BWD_CHECK("gelu_fwd");
  return 0;
}
int launch_gelu_bwd(const __nv_bfloat16* dh, const __nv_bfloat16* pre, long n, __nv_bfloat16* dpre, cudaStream_t stream) {
  if (n % 8) return set_error("gelu: n must be a multiple of 8");
  gelu_bwd_kernel<<<(unsigned)((n / 8 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(dh), reinterpret_cast<const uint4*>(pre),
                                                                      n / 8, reinterpret_cast<uint4*>(dpre));
  BWD_CHECK("gelu_bwd");
  return 0;
}
int launch_colsum(const __nv_bfloat16* x, long rows, int N, float* out, cudaStream_t stream) {
  if (rows <= 0) return 0;
  colsum_kernel<<<dim3((N + 63) / 64, (unsigned)((rows + 255) / 256)), 256, 0, stream>>>(x, rows, N, out);
  BWD_CHECK("colsum");
  return 0;
}
int launch_window_gather(const __nv_bfloat16* x, int B, int grid, int ws, int D, __nv_bfloat16* out_win, cudaStream_t stream) {
  const int wpr = (grid + ws - 1) / ws;
  const long total = (long)B * wpr * wpr * ws * ws * (D / 8);
  window_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, B, grid, ws, D, out_win);
  BWD_CHECK("window_gather");
  return 0;
}
int launch_attn_probs(const float* S, const float* T, long n_batch, AttnBwdGeom g, int pitch_s, int pitch_p, float scale,
                      __nv_bfloat16* P, cudaStream_t stream) {
  const long rows = n_batch * g.n_tok;
  prof_begin(stream, "attn_bwd softmax", 0.0, (double)rows * (pitch_s * 4.0 + pitch_p * 2.0));
  attn_probs_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(S, T, rows, g, pitch_s, pitch_p, scale, P);
  prof_end(stream);
  BWD_CHECK("attn_probs");
  return 0;
}
int launch_attn_ds(const __nv_bfloat16* P, const float* dP, long n_batch, AttnBwdGeom g, int pitch_s, int pitch_p,
                   __nv_bfloat16* dS, __nv_bfloat16* dT, cudaStream_t stream) {
  if (g.side > 64) return set_error("attn_ds: side %d > 64", g.side);
  const long rows = n_batch * g.n_tok;
  prof_begin(stream, "attn_bwd dS", 0.0, (double)rows * (pitch_s * 4.0 + pitch_p * 4.0));
  attn_ds_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(P, dP, rows, g, pitch_s, pitch_p, dS, dT);
  prof_end(stream);
  BWD_CHECK("attn_ds");
  return 0;
}
int launch_pack_dqkv(const float* dq, const float* dk, const float* dv, int outer, int heads, int T, int d, __nv_bfloat16* dqkv,
                     cudaStream_t stream) {
  const long total = (long)outer * heads * T * (d / 4) * 3;
  pack_dqkv_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dq, dk, dv, outer, heads, T, d, dqkv);
  BWD_CHECK("pack_dqkv");
  return 0;
}
int launch_sum_batch(const float* x, long n_batch, long n, float* out, int accumulate, cudaStream_t stream) {
  sum_batch_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(x, n_batch, n, out, accumulate);
  BWD_CHECK("sum_batch");
  return 0;
}
int launch_nchw_to_tok(const float* nchw, int B, int C, int T, float* tok, cudaStream_t stream) {
  if (C % 32 || T % 32) return set_error("nchw_to_tok: C and T must be multiples of 32");
  nchw_to_tok_kernel<<<dim3(T / 32, C / 32, B), dim3(32, 8), 0, stream>>>(nchw, C, T, tok);
  BWD_CHECK("nchw_to_tok");
  return 0;
}
int launch_col2im3x3(const __nv_bfloat16* dcol, int B, int g, int C, float* out, cudaStream_t stream) {
  const long total = (long)B * g * g * (C / 8);
  col2im3x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dcol, B, g, C, out);
  BWD_CHECK("col2im");
  return 0;
}
int launch_cast_f32(const __nv_bfloat16* x, long n, float* out, cudaStream_t stream) {
  if (n % 4) return set_error("cast: n must be a multiple of 4");
  cast_f32_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const uint2*>(x), n / 4, reinterpret_cast<float4*>(out));
  BWD_CHECK("cast_f32");
  return 0;
}

}  // namespace msam
