// Mask decoder in training mode (BASELINE.json configs[4]; micro_sam/training/trainable_sam.py:62-114 + sam_trainer.py:131-172):
// MaskDecoder.forward on the prompts of ONE image, keeping the activations, and its backward pass -- gradients of every mask-decoder
// and prompt-encoder parameter plus dL/d(image embedding), which is what the encoder backward pass (encoder_train.cu) consumes.
// Restates oracle/sam_ref.py:MaskDecoder / TwoWayTransformer / DecAttention (the inference kernels t2i_fused / i2t_fused /
// upscale_fused fold projections into each other and keep nothing, so they cannot be differentiated through); checked against torch
// autograd in tests/test_gpu_backward.py.
//
// Structure: a tape.  Every forward op (linear, LayerNorm, add+cast, attention, GELU, ...) runs on the existing kernels -- wgmma
// GEMMs (gemm.cu), the batched attention GEMM (bgemm.cu), LayerNorm -- allocates its output from a per-slot arena
// and pushes its backward closure; backward() replays the closures in reverse.  Tensors carry an fp32 value, an fp32 gradient
// (accumulated: every consumer ADDS) and a bf16 copy (the GEMM operand).  Parameter gradients accumulate across calls (images,
// sub-iterations) until msam_decoder_zero_grads.  Supported prompts: points and / or boxes (dense prompt = no_mask_embed).
#include "engine.h"

#include <algorithm>
#include <cmath>
#include <functional>

namespace msam {

#define CHK(p) do { if (!(p)) return -1; } while (0)
#define RUN(x) do { if (x) return -1; } while (0)
#define KCHECK(what)                                                                                 \
  do {                                                                                               \
    cudaError_t e_ = cudaGetLastError();                                                             \
    if (e_ != cudaSuccess) return set_error(what " launch failed: %s", cudaGetErrorString(e_));      \
    count_launch();                                                                                  \
  } while (0)

namespace {

__device__ __forceinline__ uint32_t dpk2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float dwarp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float dwarp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// out_bf16[r, c] = bf16(a[r, c] + b[r % b_rows, c]); b may be null.  n4 = rows * cols / 4
__global__ void add_cast_kernel(const float4* __restrict__ a, const float4* __restrict__ b, long n4, long b_n4, uint2* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = a[i];
  if (b) { const float4 w = b[i % b_n4]; v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
  out[i] = make_uint2(dpk2(v.x, v.y), dpk2(v.z, v.w));
}
// dst += src (fp32)
__global__ void add_inplace_kernel(float4* __restrict__ dst, const float4* __restrict__ src, long n4) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 d = dst[i];
  const float4 s = src[i];
  d.x += s.x; d.y += s.y; d.z += s.z; d.w += s.w;
  dst[i] = d;
}
// dy_bf16 = bf16(g) [masked by y > 0 when relu_y != null]
__global__ void grad_cast_kernel(const float4* __restrict__ g, const uint2* __restrict__ relu_y, long n4, uint2* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = g[i];
  if (relu_y) {
    const uint2 y = relu_y[i];
    if (!(__uint_as_float(y.x << 16) > 0.f)) v.x = 0.f;
    if (!(__uint_as_float(y.x & 0xffff0000u) > 0.f)) v.y = 0.f;
    if (!(__uint_as_float(y.y << 16) > 0.f)) v.z = 0.f;
    if (!(__uint_as_float(y.y & 0xffff0000u) > 0.f)) v.w = 0.f;
  }
  out[i] = make_uint2(dpk2(v.x, v.y), dpk2(v.z, v.w));
}
// strided row copy / accumulate: dst[r * dp + c] (+)= src[r * sp + c], c < cols
__global__ void copy_rows_kernel(const float* __restrict__ src, long sp, float* __restrict__ dst, long dp, long rows, int cols, int accumulate) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const long r = i / cols;
  const int c = i % cols;
  const float v = src[r * sp + c];
  if (accumulate) dst[r * dp + c] += v; else dst[r * dp + c] = v;
}
// softmax over the first n_valid entries of fp32 rows (pitch entries each) -> bf16 probabilities (zero beyond n_valid)
__global__ void softmax_rows_kernel(const float* __restrict__ S, long rows, int n_valid, int pitch, __nv_bfloat16* __restrict__ P) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + row * pitch;
  __nv_bfloat16* p = P + row * pitch;
  float m = -INFINITY;
  for (int k = lane; k < n_valid; k += 32) m = fmaxf(m, s[k]);
  m = dwarp_max(m);
  float l = 0.f;
  for (int k = lane; k < n_valid; k += 32) l += __expf(s[k] - m);
  const float inv = 1.0f / dwarp_sum(l);
  for (int k = lane; k < pitch; k += 32) p[k] = __float2bfloat16(k < n_valid ? __expf(s[k] - m) * inv : 0.f);
}
// dS = P o (dP - sum_k P dP)
__global__ void ds_rows_kernel(const __nv_bfloat16* __restrict__ P, const float* __restrict__ dP, long rows, int n_valid, int pitch,
                               __nv_bfloat16* __restrict__ dS) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const __nv_bfloat16* p = P + row * pitch;
  const float* dp = dP + row * pitch;
  __nv_bfloat16* ds = dS + row * pitch;
  float del = 0.f;
  for (int k = lane; k < n_valid; k += 32) del += __bfloat162float(p[k]) * dp[k];
  del = dwarp_sum(del);
  for (int k = lane; k < pitch; k += 32) ds[k] = __float2bfloat16(k < n_valid ? __bfloat162float(p[k]) * (dp[k] - del) : 0.f);
}
// tokens [P, T, 256]: rows 0..4 = output tokens (iou token, 4 mask tokens), rows 5.. = sparse prompt embeddings [P, Ts, 256]
__global__ void assemble_tokens_kernel(const float* __restrict__ out_tokens, const float* __restrict__ sparse, int P, int T, int Ts,
                                       float* __restrict__ tok) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * T * 256) return;
  const int c = i % 256, t = (i / 256) % T;
  const long p = i / (256L * T);
  tok[i] = t < 5 ? out_tokens[t * 256 + c] : sparse[(p * Ts + (t - 5)) * 256 + c];
}
// gradients of the embedding tables behind the tokens: output tokens (rows 0..4) and, per sparse token, the table row emb_index
// selects (0..3 = point_embeddings, 4 = not_a_point_embed; the positional part has no parameters)
__global__ void token_grads_kernel(const float* __restrict__ g_tok, const int* __restrict__ emb_index, int P, int T, int Ts,
                                   float* __restrict__ g_out_tokens, float* __restrict__ g_point_emb, float* __restrict__ g_nap) {
  const int c = threadIdx.x, t = blockIdx.x;   // 256 threads, T blocks
  float s = 0.f;
  if (t < 5) {
    for (int p = 0; p < P; ++p) s += g_tok[((long)p * T + t) * 256 + c];
    g_out_tokens[t * 256 + c] += s;
  } else {
    for (int p = 0; p < P; ++p) {
      const int e = emb_index[p * Ts + (t - 5)];
      const float v = g_tok[((long)p * T + t) * 256 + c];
      if (e >= 0 && e < 4) atomicAdd(g_point_emb + e * 256 + c, v);
      else if (e == 4) atomicAdd(g_nap + c, v);
    }
  }
}
// keys0[p, pix, c] = emb_nchw[c, pix] + no_mask[c]
__global__ void src_broadcast_kernel(const float* __restrict__ emb_nchw, const float* __restrict__ no_mask, int P, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int pix0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) tile[i][threadIdx.x] = emb_nchw[(long)(c0 + i) * 4096 + pix0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const float v = tile[threadIdx.x][i] + no_mask[c0 + threadIdx.x];
    for (int p = 0; p < P; ++p) out[((long)p * 4096 + pix0 + i) * 256 + c0 + threadIdx.x] = v;
  }
}
// d_emb_nchw[c, pix] = sum_p g[p, pix, c];  g_no_mask[c] += sum_{p, pix} g[p, pix, c]
__global__ void src_grad_kernel(const float* __restrict__ g, int P, float* __restrict__ d_emb_nchw, float* __restrict__ g_no_mask) {
  __shared__ float tile[32][33];
  const int pix0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += g[((long)p * 4096 + pix0 + i) * 256 + c0 + threadIdx.x];
    tile[i][threadIdx.x] = s;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) d_emb_nchw[(long)(c0 + i) * 4096 + pix0 + threadIdx.x] = tile[threadIdx.x][i];
  if (threadIdx.y == 0) {
    float s = 0.f;
    for (int i = 0; i < 32; ++i) s += tile[i][threadIdx.x];
    atomicAdd(g_no_mask + c0 + threadIdx.x, s);
  }
}
// hyper product output [P, 65536 (pixel order ((i*64+j)*4+s1)*4+s2), 4] <-> low-res masks [P, nm, 256, 256] (masks m0 .. m0 + nm - 1)
__device__ __forceinline__ long up_row(int Y, int X) {
  return ((((long)(Y >> 2) * 64 + (X >> 2)) * 4 + (((Y >> 1) & 1) * 2 + ((X >> 1) & 1))) * 4 + ((Y & 1) * 2 + (X & 1)));
}
__global__ void masks_out_kernel(const float* __restrict__ o4, int P, int nm, int m0, float* __restrict__ low_res) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * nm * 65536) return;
  const int X = i % 256, Y = (i / 256) % 256, m = (i / 65536) % nm;
  const long p = i / (65536L * nm);
  low_res[i] = o4[(p * 65536 + up_row(Y, X)) * 4 + m0 + m];
}
// d_low_res [P, nm, 256, 256] -> bf16 [P, 65536, 8] in pixel order (columns m0 .. m0+nm-1, zero elsewhere)
__global__ void masks_grad_kernel(const float* __restrict__ d_low, int P, int nm, int m0, __nv_bfloat16* __restrict__ out8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)P * 65536) return;
  const int X = i % 256, Y = (i / 256) % 256;
  const long p = i / 65536;
  float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int m = 0; m < nm; ++m) v[m0 + m] = d_low[((p * nm + m) * 256 + Y) * 256 + X];
  *reinterpret_cast<uint4*>(out8 + (p * 65536 + up_row(Y, X)) * 8) = make_uint4(dpk2(v[0], v[1]), dpk2(v[2], v[3]), dpk2(v[4], v[5]), dpk2(v[6], v[7]));
}
__global__ void transpose_bf16_dk(const __nv_bfloat16* __restrict__ in, int rows, int cols, __nv_bfloat16* __restrict__ out) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    if (r0 + i < rows && c0 + threadIdx.x < cols) tile[i][threadIdx.x] = in[(long)(r0 + i) * cols + c0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    if (c0 + i < cols && r0 + threadIdx.x < rows) out[(long)(c0 + i) * rows + r0 + threadIdx.x] = tile[threadIdx.x][i];
}

inline unsigned nblk(long n, int per = 256) { return (unsigned)((n + per - 1) / per); }

}  // namespace

// ------------------------------------------------------------------------------------------------ data structures
struct Ten {
  float* v = nullptr;            // fp32 value
  float* g = nullptr;            // fp32 gradient (accumulated by the consumers' backward closures)
  __nv_bfloat16* b = nullptr;    // bf16 copy (GEMM operand)
  long rows = 0;
  int cols = 0;
  long n() const { return rows * cols; }
};
struct DLin { int out = 0, in = 0; __nv_bfloat16 *w = nullptr, *wT = nullptr; float *bias = nullptr, *gw = nullptr, *gb = nullptr; };
struct DLn { int D = 0; float eps = 1e-5f; float *g = nullptr, *b = nullptr, *gg = nullptr, *gb = nullptr; };
struct DAttn { DLin q, k, v, o; int inner = 0; };
struct DLayer { DAttn self, t2i, i2t; DLn n1, n2, n3, n4; DLin mlp1, mlp2; };

struct DecSlot {
  uint8_t* arena = nullptr;
  size_t cap = 0, used = 0;
  std::vector<std::function<int(cudaStream_t)>> tape;
  int P = 0, T = 0, Ts = 0, nm = 0, m0 = 0;
  Ten low4, iou32, keys0, tok;
  int* emb_index = nullptr;
  __nv_bfloat16* dmask8 = nullptr;
  bool live = false;
};

struct DecTrain {
  DLayer layer[2];
  DAttn fin;
  DLn nfin, upln;
  DLin ct1, ct2, hyper[4][3], iou[3];
  float *point_emb = nullptr, *not_a_point = nullptr, *no_mask = nullptr, *out_tokens = nullptr;
  float *g_point_emb = nullptr, *g_nap = nullptr, *g_no_mask = nullptr, *g_out_tokens = nullptr;
  std::unordered_map<std::string, std::pair<float*, int64_t>> grads;
  DecSlot slot[8];
};

namespace {

struct Ctx {
  Engine& e;
  DecTrain& d;
  DecSlot& s;
  cudaStream_t st;
  int err = 0;

  void* take(size_t bytes) {
    const size_t off = (s.used + 255) & ~size_t(255);
    if (off + bytes > s.cap) { err = set_error("decoder training: arena of %zu bytes exhausted (need %zu more)", s.cap, off + bytes - s.cap); return nullptr; }
    s.used = off + bytes;
    return s.arena + off;
  }
  Ten ten(long rows, int cols, bool v, bool g, bool b) {
    Ten t; t.rows = rows; t.cols = cols;
    if (v) t.v = (float*)take((size_t)rows * cols * 4);
    if (g) { t.g = (float*)take((size_t)rows * cols * 4); if (t.g) cudaMemsetAsync(t.g, 0, (size_t)rows * cols * 4, st); }
    if (b) t.b = (__nv_bfloat16*)take((size_t)rows * cols * 2);
    return t;
  }
};

int cast_grad(const float* g, const __nv_bfloat16* relu_y, long n, __nv_bfloat16* out, cudaStream_t st) {
  grad_cast_kernel<<<nblk(n / 4), 256, 0, st>>>((const float4*)g, (const uint2*)relu_y, n / 4, (uint2*)out);
  KCHECK("grad_cast");
  return 0;
}
int add_inplace(float* dst, const float* src, long n, cudaStream_t st) {
  add_inplace_kernel<<<nblk(n / 4), 256, 0, st>>>((float4*)dst, (const float4*)src, n / 4);
  KCHECK("add_inplace");
  return 0;
}

// y = act(x W^T + b) (+ residual).  bf16_out: y.b only (consumed by GEMMs / attention), else y.v fp32.
// backward: dy = y.g [o relu mask]; gW += dy^T x, gb += colsum(dy), x.g += dy W, residual.g += y.g
int op_linear(Ctx& c, const Ten& x, DLin& L, Ten& y, int act, const Ten* residual, bool bf16_out) {
  if (c.err) return -1;
  y = c.ten(x.rows, L.out, !bf16_out, true, bf16_out);
  if (c.err) return -1;
  GemmArgs a;
  a.A = x.b; a.W = L.w; a.M = (int)x.rows; a.N = L.out; a.K = L.in; a.lda = L.in; a.ldw = L.in; a.bias = L.bias; a.act = act;
  if (residual) { a.residual = residual->v; }
  a.out = bf16_out ? (void*)y.b : (void*)y.v; a.out_fp32 = bf16_out ? 0 : 1;
  RUN(launch_gemm(a, c.e.num_sms, c.st));
  Engine* e = &c.e;
  DLin* Lp = &L;
  const Ten xin = x, yout = y;
  const Ten res = residual ? *residual : Ten();
  const bool relu = act == 2;
  __nv_bfloat16* scratch = (__nv_bfloat16*)c.take((size_t)y.rows * L.out * 2);
  if (c.err) return -1;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(cast_grad(yout.g, relu ? yout.b : nullptr, yout.n(), scratch, st));
    RUN(launch_gemm_tn(scratch, xin.b, Lp->out, Lp->in, (int)xin.rows, Lp->out, Lp->in, Lp->gw, Lp->in, st, 1));
    RUN(launch_colsum(scratch, xin.rows, Lp->out, Lp->gb, st));
    if (xin.g) {
      GemmArgs a;
      a.A = scratch; a.W = Lp->wT; a.M = (int)xin.rows; a.N = Lp->in; a.K = Lp->out; a.lda = Lp->out; a.ldw = Lp->out;
      a.residual = xin.g; a.out = xin.g; a.out_fp32 = 1;
      RUN(launch_gemm(a, e->num_sms, st));
    }
    if (res.g) RUN(add_inplace(res.g, yout.g, yout.n(), st));
    return 0;
  });
  return 0;
}

int op_layernorm(Ctx& c, const Ten& x, DLn& L, Ten& y, bool want_v = true) {
  if (c.err) return -1;
  y = c.ten(x.rows, x.cols, want_v, true, true);
  if (c.err) return -1;
  LnArgs l;
  l.x = x.v; l.rows = (int)x.rows; l.D = x.cols; l.gamma = L.g; l.beta = L.b; l.eps = L.eps; l.out = y.b; l.out_f32 = y.v;
  RUN(launch_layernorm(l, c.st));
  const Ten xin = x, yout = y;
  DLn* Lp = &L;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    return launch_layernorm_bwd(xin.v, (int)xin.rows, xin.cols, Lp->g, Lp->eps, yout.g, 0, 64, 14, 1, xin.g, Lp->gg, Lp->gb, st);
  });
  return 0;
}

// y.b = bf16(a.v + b_v[row % b_rows]) ; backward: a.g += y.g ; b_g += y.g (same row count only)
int op_add_cast(Ctx& c, const Ten& a, const float* b_v, long b_rows, float* b_g, Ten& y) {
  if (c.err) return -1;
  y = c.ten(a.rows, a.cols, false, true, true);
  if (c.err) return -1;
  add_cast_kernel<<<nblk(a.n() / 4), 256, 0, c.st>>>((const float4*)a.v, (const float4*)b_v, a.n() / 4, b_rows * a.cols / 4, (uint2*)y.b);
  KCHECK("add_cast");
  const Ten ain = a, yout = y;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(add_inplace(ain.g, yout.g, yout.n(), st));
    if (b_g) RUN(add_inplace(b_g, yout.g, yout.n(), st));
    return 0;
  });
  return 0;
}

// softmax(q k^T / sqrt(hd)) v per (prompt, head); q [P*Tq, inner], k / v [P*Tk, inner] (bf16 + fp32 gradients) -> o (fp32 + bf16)
int op_attention(Ctx& c, const Ten& q, const Ten& k, const Ten& v, int P, int Tq, int Tk, int inner, int heads, Ten& o) {
  if (c.err) return -1;
  const int hd = inner / heads, pitch = (Tk + 7) & ~7;
  const float scale = 1.0f / sqrtf((float)hd);
  const long nb = (long)P * heads;
  o = c.ten((long)P * Tq, inner, true, true, true);
  float* S = (float*)c.take((size_t)nb * Tq * pitch * 4);
  __nv_bfloat16* Pm = (__nv_bfloat16*)c.take((size_t)nb * Tq * pitch * 2);
  __nv_bfloat16* dS = (__nv_bfloat16*)c.take((size_t)nb * Tq * pitch * 2);
  __nv_bfloat16* dOb = (__nv_bfloat16*)c.take((size_t)P * Tq * inner * 2);
  if (c.err) return -1;
  const long s_h = (long)Tq * pitch, s_w = (long)heads * Tq * pitch;
  BGemmArgs a;
  a.A = q.b; a.B = k.b; a.M = Tq; a.N = pitch; a.K = hd; a.lda = a.ldb = inner; a.a_hstride = a.b_hstride = hd;
  a.a_wstride = (long)Tq * inner; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk;
  a.heads = heads; a.outer = P; a.out = S; a.ldc = pitch; a.o_hstride = s_h; a.o_wstride = s_w; a.alpha = scale;
  RUN(launch_bgemm(a, c.st));
  softmax_rows_kernel<<<nblk(nb * Tq, 8), 256, 0, c.st>>>(S, nb * Tq, Tk, pitch, Pm);
  KCHECK("softmax_rows");
  // O = P V, written head-interleaved [P*Tq, inner]
  a = BGemmArgs();
  a.A = Pm; a.B = v.b; a.b_mn = 1; a.M = Tq; a.N = hd; a.K = pitch; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
  a.b_hstride = hd; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk; a.heads = heads; a.outer = P;
  a.out = o.v; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tq * inner;
  RUN(launch_bgemm(a, c.st));
  RUN(launch_cast_bf16(o.v, o.n(), o.b, c.st));
  const Ten qq = q, kk = k, vv = v, oo = o;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(cast_grad(oo.g, nullptr, oo.n(), dOb, st));
    BGemmArgs a;
    // dV += P^T dO
    a.A = Pm; a.B = dOb; a.a_mn = a.b_mn = 1; a.M = Tk; a.N = hd; a.K = Tq; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
    a.b_hstride = hd; a.b_wstride = (long)Tq * inner; a.heads = heads; a.outer = P;
    a.out = vv.g; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tk * inner; a.accumulate = 1;
    RUN(launch_bgemm(a, st));
    // dP = dO V^T (over S)
    a = BGemmArgs();
    a.A = dOb; a.B = vv.b; a.M = Tq; a.N = pitch; a.K = hd; a.lda = a.ldb = inner; a.a_hstride = a.b_hstride = hd;
    a.a_wstride = (long)Tq * inner; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk;
    a.heads = heads; a.outer = P; a.out = S; a.ldc = pitch; a.o_hstride = s_h; a.o_wstride = s_w;
    RUN(launch_bgemm(a, st));
    ds_rows_kernel<<<nblk(nb * Tq, 8), 256, 0, st>>>(Pm, S, nb * Tq, Tk, pitch, dS);
    KCHECK("ds_rows");
    // dQ += scale dS K
    a = BGemmArgs();
    a.A = dS; a.B = kk.b; a.b_mn = 1; a.M = Tq; a.N = hd; a.K = pitch; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
    a.b_hstride = hd; a.b_wstride = (long)Tk * inner; a.b_rows_valid = Tk; a.heads = heads; a.outer = P;
    a.out = qq.g; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tq * inner; a.alpha = scale; a.accumulate = 1;
    RUN(launch_bgemm(a, st));
    // dK += scale dS^T Q
    a = BGemmArgs();
    a.A = dS; a.B = qq.b; a.a_mn = a.b_mn = 1; a.M = Tk; a.N = hd; a.K = Tq; a.lda = pitch; a.ldb = inner; a.a_hstride = s_h; a.a_wstride = s_w;
    a.b_hstride = hd; a.b_wstride = (long)Tq * inner; a.heads = heads; a.outer = P;
    a.out = kk.g; a.ldc = inner; a.o_hstride = hd; a.o_wstride = (long)Tk * inner; a.alpha = scale; a.accumulate = 1;
    RUN(launch_bgemm(a, st));
    return 0;
  });
  return 0;
}

// y.b = gelu(x.b); backward: x.g += y.g o gelu'(x)
int op_gelu(Ctx& c, const Ten& x, Ten& y) {
  if (c.err) return -1;
  y = c.ten(x.rows, x.cols, false, true, true);
  __nv_bfloat16* t1 = (__nv_bfloat16*)c.take((size_t)x.n() * 2);
  float* t2 = (float*)c.take((size_t)x.n() * 4);
  if (c.err) return -1;
  RUN(launch_gelu_fwd(x.b, x.n(), y.b, c.st));
  const Ten xin = x, yout = y;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    RUN(cast_grad(yout.g, nullptr, yout.n(), t1, st));
    RUN(launch_gelu_bwd(t1, xin.b, xin.n(), t1, st));
    RUN(launch_cast_f32(t1, xin.n(), t2, st));
    return add_inplace(xin.g, t2, xin.n(), st);
  });
  return 0;
}

// rows of a [P, pitch] view <-> compact [P, cols] tensor (token slices)
int op_slice_rows(Ctx& c, const Ten& x, long offset, long pitch, long rows, int cols, Ten& y) {
  if (c.err) return -1;
  y = c.ten(rows, cols, true, true, true);
  if (c.err) return -1;
  copy_rows_kernel<<<nblk(rows * cols), 256, 0, c.st>>>(x.v + offset, pitch, y.v, cols, rows, cols, 0);
  KCHECK("slice_rows");
  RUN(launch_cast_bf16(y.v, y.n(), y.b, c.st));
  const Ten xin = x, yout = y;
  c.s.tape.push_back([=](cudaStream_t st) -> int {
    copy_rows_kernel<<<nblk(rows * cols), 256, 0, st>>>(yout.g, cols, xin.g + offset, pitch, rows, cols, 1);
    KCHECK("slice_rows_bwd");
    return 0;
  });
  return 0;
}

int attn_module(Ctx& c, DAttn& A, const Ten& q_in, const Ten& k_in, const Ten& v_in, int P, int Tq, int Tk, const Ten* residual, Ten& out) {
  Ten q, k, v, o;
  RUN(op_linear(c, q_in, A.q, q, 0, nullptr, true));
  RUN(op_linear(c, k_in, A.k, k, 0, nullptr, true));
  RUN(op_linear(c, v_in, A.v, v, 0, nullptr, true));
  RUN(op_attention(c, q, k, v, P, Tq, Tk, A.inner, 8, o));
  return op_linear(c, o, A.o, out, 0, residual, false);
}

}  // namespace

// ------------------------------------------------------------------------------------------------ setup
static int dt_lin(Engine& e, DecTrain& d, const std::string& key, int out, int in, DLin* L, int out_pad = 0) {
  const auto* w = e.host(key + ".weight", {out, in});
  const auto* b = e.host(key + ".bias", {out});
  if (!w || !b) return -1;
  const int op = out_pad > out ? out_pad : out;
  std::vector<float> wp((size_t)op * in, 0.f), bp(op, 0.f);
  std::copy(w->begin(), w->end(), wp.begin());
  std::copy(b->begin(), b->end(), bp.begin());
  L->out = op; L->in = in;
  CHK(L->w = e.upload_bf16(wp.data(), wp.size()));
  CHK(L->wT = (__nv_bfloat16*)e.dalloc((size_t)op * in * 2));
  transpose_bf16_dk<<<dim3((in + 31) / 32, (op + 31) / 32), dim3(32, 8)>>>(L->w, op, in, L->wT);
  CHK(L->bias = e.upload_f32(bp.data(), bp.size()));
  CHK(L->gw = (float*)e.dalloc((size_t)op * in * 4, true));
  CHK(L->gb = (float*)e.dalloc((size_t)op * 4, true));
  d.grads[key + ".weight"] = {L->gw, (int64_t)op * in};
  d.grads[key + ".bias"] = {L->gb, op};
  OptParam pw, pb;
  pw.key = key + ".weight"; CHK(pw.w = e.upload_f32(wp.data(), wp.size())); pw.g = L->gw; pw.n = (int64_t)op * in;
  pw.refresh = 2; pw.dst = L->w; pw.dstT = L->wT; pw.rows = op; pw.cols = in;
  pb.key = key + ".bias"; pb.w = L->bias; pb.g = L->gb; pb.n = op;
  e.opt_add(pw); e.opt_add(pb);
  return 0;
}
static int dt_ln(Engine& e, DecTrain& d, const std::string& key, int D, float eps, DLn* L) {
  L->D = D; L->eps = eps;
  CHK(L->g = e.up_f32(key + ".weight", {D}));
  CHK(L->b = e.up_f32(key + ".bias", {D}));
  CHK(L->gg = (float*)e.dalloc((size_t)D * 4, true));
  CHK(L->gb = (float*)e.dalloc((size_t)D * 4, true));
  d.grads[key + ".weight"] = {L->gg, D};
  d.grads[key + ".bias"] = {L->gb, D};
  OptParam pg, pb;
  pg.key = key + ".weight"; pg.w = L->g; pg.g = L->gg; pg.n = D;
  pb.key = key + ".bias"; pb.w = L->b; pb.g = L->gb; pb.n = D;
  e.opt_add(pg); e.opt_add(pb);
  return 0;
}
static int dt_attn(Engine& e, DecTrain& d, const std::string& key, int inner, DAttn* A) {
  A->inner = inner;
  RUN(dt_lin(e, d, key + ".q_proj", inner, 256, &A->q));
  RUN(dt_lin(e, d, key + ".k_proj", inner, 256, &A->k));
  RUN(dt_lin(e, d, key + ".v_proj", inner, 256, &A->v));
  return dt_lin(e, d, key + ".out_proj", 256, inner, &A->o);
}
// ConvTranspose2d(k = 2, s = 2) weight [ci, co, 2, 2] as the GEMM operand [(dy*2+dx)*co_n + co][ci]; gradients are exposed in this
// layout under "<key>.weight@gemm" / "<key>.bias@gemm" (bias tiled over the 4 sub-pixels): micro_sam_b200/sam.py folds them back
static int dt_convT(Engine& e, DecTrain& d, const std::string& key, int ci, int co, DLin* L) {
  const auto* w = e.host(key + ".weight", {ci, co, 2, 2});
  const auto* b = e.host(key + ".bias", {co});
  if (!w || !b) return -1;
  std::vector<float> wg((size_t)4 * co * ci), bg((size_t)4 * co);
  for (int i = 0; i < ci; ++i)
    for (int o = 0; o < co; ++o)
      for (int s = 0; s < 4; ++s) wg[((size_t)s * co + o) * ci + i] = (*w)[((size_t)i * co + o) * 4 + s];
  for (int s = 0; s < 4; ++s)
    for (int o = 0; o < co; ++o) bg[s * co + o] = (*b)[o];
  L->out = 4 * co; L->in = ci;
  CHK(L->w = e.upload_bf16(wg.data(), wg.size()));
  CHK(L->wT = (__nv_bfloat16*)e.dalloc(wg.size() * 2));
  transpose_bf16_dk<<<dim3((ci + 31) / 32, (4 * co + 31) / 32), dim3(32, 8)>>>(L->w, 4 * co, ci, L->wT);
  CHK(L->bias = e.upload_f32(bg.data(), bg.size()));
  CHK(L->gw = (float*)e.dalloc(wg.size() * 4, true));
  CHK(L->gb = (float*)e.dalloc(bg.size() * 4, true));
  d.grads[key + ".weight@gemm"] = {L->gw, (int64_t)wg.size()};
  d.grads[key + ".bias@gemm"] = {L->gb, (int64_t)bg.size()};
  OptParam pw, pb;
  pw.key = key + ".weight@gemm"; CHK(pw.w = e.upload_f32(wg.data(), wg.size())); pw.g = L->gw; pw.n = (int64_t)wg.size();
  pw.refresh = 2; pw.dst = L->w; pw.dstT = L->wT; pw.rows = 4 * co; pw.cols = ci;
  pb.key = key + ".bias@gemm"; pb.w = L->bias; pb.g = L->gb; pb.n = (int64_t)bg.size(); pb.refresh = 6;
  e.opt_add(pw); e.opt_add(pb);
  return 0;
}

int Engine::dec_train_setup() {
  if (dtrain) return 0;
  if (!finalized || !dec) return set_error("decoder training: weights not loaded");
  if (dec_host.empty()) return set_error("decoder training: host copies of the decoder weights are gone");
  host_weights.swap(dec_host);   // host()/up_f32() read host_weights
  dtrain = new DecTrain();
  DecTrain& d = *dtrain;
  int rc = 0;
  auto go = [&]() -> int {
    const std::string m = "mask_decoder.", tr = m + "transformer.";
    for (int l = 0; l < 2; ++l) {
      const std::string p = tr + "layers." + std::to_string(l) + ".";
      DLayer& L = d.layer[l];
      RUN(dt_attn(*this, d, p + "self_attn", 256, &L.self));
      RUN(dt_attn(*this, d, p + "cross_attn_token_to_image", 128, &L.t2i));
      RUN(dt_attn(*this, d, p + "cross_attn_image_to_token", 128, &L.i2t));
      RUN(dt_ln(*this, d, p + "norm1", 256, 1e-5f, &L.n1));
      RUN(dt_ln(*this, d, p + "norm2", 256, 1e-5f, &L.n2));
      RUN(dt_ln(*this, d, p + "norm3", 256, 1e-5f, &L.n3));
      RUN(dt_ln(*this, d, p + "norm4", 256, 1e-5f, &L.n4));
      RUN(dt_lin(*this, d, p + "mlp.lin1", 2048, 256, &L.mlp1));
      RUN(dt_lin(*this, d, p + "mlp.lin2", 256, 2048, &L.mlp2));
    }
    RUN(dt_attn(*this, d, tr + "final_attn_token_to_image", 128, &d.fin));
    RUN(dt_ln(*this, d, tr + "norm_final_attn", 256, 1e-5f, &d.nfin));
    RUN(dt_convT(*this, d, m + "output_upscaling.0", 256, 64, &d.ct1));
    RUN(dt_ln(*this, d, m + "output_upscaling.1", 64, 1e-6f, &d.upln));
    RUN(dt_convT(*this, d, m + "output_upscaling.3", 64, 32, &d.ct2));
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 3; ++j)
        RUN(dt_lin(*this, d, m + "output_hypernetworks_mlps." + std::to_string(i) + ".layers." + std::to_string(j), j == 2 ? 32 : 256, 256, &d.hyper[i][j]));
    for (int j = 0; j < 3; ++j)
      RUN(dt_lin(*this, d, m + "iou_prediction_head.layers." + std::to_string(j), j == 2 ? 4 : 256, 256, &d.iou[j], 32));
    // embedding tables
    std::vector<float> pe(4 * 256), ot(5 * 256);
    for (int i = 0; i < 4; ++i) {
      const auto* w = host("prompt_encoder.point_embeddings." + std::to_string(i) + ".weight", {1, 256});
      CHK(w);
      std::copy(w->begin(), w->end(), pe.begin() + i * 256);
    }
    const auto* it = host(m + "iou_token.weight", {1, 256});
    const auto* mt = host(m + "mask_tokens.weight", {4, 256});
    CHK(it && mt);
    std::copy(it->begin(), it->end(), ot.begin());
    std::copy(mt->begin(), mt->end(), ot.begin() + 256);
    CHK(d.point_emb = upload_f32(pe.data(), pe.size()));
    CHK(d.out_tokens = upload_f32(ot.data(), ot.size()));
    CHK(d.not_a_point = up_f32("prompt_encoder.not_a_point_embed.weight", {1, 256}));
    CHK(d.no_mask = up_f32("prompt_encoder.no_mask_embed.weight", {1, 256}));
    CHK(d.g_point_emb = (float*)dalloc(4 * 256 * 4, true));
    CHK(d.g_out_tokens = (float*)dalloc(5 * 256 * 4, true));
    CHK(d.g_nap = (float*)dalloc(256 * 4, true));
    CHK(d.g_no_mask = (float*)dalloc(256 * 4, true));
    d.grads["prompt_encoder.point_embeddings@stack"] = {d.g_point_emb, 4 * 256};
    d.grads["mask_decoder.output_tokens@stack"] = {d.g_out_tokens, 5 * 256};
    d.grads["prompt_encoder.not_a_point_embed.weight"] = {d.g_nap, 256};
    d.grads["prompt_encoder.no_mask_embed.weight"] = {d.g_no_mask, 256};
    OptParam p;
    p.key = "prompt_encoder.point_embeddings@stack"; p.w = d.point_emb; p.g = d.g_point_emb; p.n = 4 * 256; p.refresh = 5; opt_add(p);
    p.key = "prompt_encoder.not_a_point_embed.weight"; p.w = d.not_a_point; p.g = d.g_nap; p.n = 256; p.refresh = 5; opt_add(p);
    p.key = "mask_decoder.output_tokens@stack"; p.w = d.out_tokens; p.g = d.g_out_tokens; p.n = 5 * 256; p.refresh = 0; opt_add(p);
    p.key = "prompt_encoder.no_mask_embed.weight"; p.w = d.no_mask; p.g = d.g_no_mask; p.n = 256; p.refresh = 0; opt_add(p);
    return 0;
  };
  rc = go();
  host_weights.swap(dec_host);
  if (rc == 0 && cudaDeviceSynchronize() != cudaSuccess) rc = set_error("decoder training setup: %s", cudaGetErrorString(cudaGetLastError()));
  if (rc) { delete dtrain; dtrain = nullptr; }
  return rc;
}

// ------------------------------------------------------------------------------------------------ forward
int Engine::decoder_train_forward(int slot, const float* emb_nchw, const float* sparse, const int* emb_index, int Ts, int P, int multimask,
                                  float* low_res, float* iou, cudaStream_t st) {
  if (slot < 0 || slot >= 8) return set_error("decoder training: slot %d outside [0, 8)", slot);
  if (P <= 0 || Ts <= 0 || !sparse || !emb_index) return set_error("decoder training: needs sparse prompt embeddings (points and / or boxes)");
  RUN(dec_train_setup());
  DecTrain& d = *dtrain;
  DecSlot& s = d.slot[slot];
  const int T = 5 + Ts;
  const long Rt = (long)P * T, Ri = (long)P * 4096;
  {   // arena: ~ 110 fp32-equivalents of [P*4096, 256] cover the image-side tensors of both layers + the upscaling path
    const size_t need = (size_t)Ri * 256 * 4 * 64 + ((size_t)64 << 20);
    if (s.cap < need) {
      if (s.arena) cudaFree(s.arena);
      s.arena = nullptr; s.cap = 0;
      if (cudaMalloc(&s.arena, need) != cudaSuccess) return set_error("decoder training: cudaMalloc of %zu bytes failed", need);
      s.cap = need;
    }
  }
  s.used = 0; s.tape.clear(); s.live = false;
  s.P = P; s.T = T; s.Ts = Ts; s.nm = multimask ? 3 : 1; s.m0 = multimask ? 1 : 0;
  Ctx c{*this, d, s, st};
  s.emb_index = (int*)c.take((size_t)P * Ts * 4);
  if (c.err) return -1;
  if (cudaMemcpyAsync(s.emb_index, emb_index, (size_t)P * Ts * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("decoder training: copy failed");
  // tokens and image-side source
  Ten tok = c.ten(Rt, 256, true, true, true);
  Ten keys0 = c.ten(Ri, 256, true, true, true);
  if (c.err) return -1;
  assemble_tokens_kernel<<<nblk(Rt * 256), 256, 0, st>>>(d.out_tokens, sparse, P, T, Ts, tok.v);
  KCHECK("assemble_tokens");
  RUN(launch_cast_bf16(tok.v, tok.n(), tok.b, st));
  src_broadcast_kernel<<<dim3(128, 8), dim3(32, 8), 0, st>>>(emb_nchw, d.no_mask, P, keys0.v);
  KCHECK("src_broadcast");
  RUN(launch_cast_bf16(keys0.v, keys0.n(), keys0.b, st));
  s.tok = tok; s.keys0 = keys0;
  const float* pos = dec_pos();     // dense positional encoding, token-major [4096, 256] (no parameters)
  Ten Q = tok, K = keys0;
  for (int l = 0; l < 2; ++l) {
    DLayer& L = d.layer[l];
    Ten a, Q1, Q2, Q3, qin, kin, h;
    // self attention
    if (l == 0) {
      RUN(attn_module(c, L.self, Q, Q, Q, P, T, T, nullptr, a));
    } else {
      RUN(op_add_cast(c, Q, tok.v, Rt, tok.g, qin));
      RUN(attn_module(c, L.self, qin, qin, Q, P, T, T, &Q, a));
    }
    RUN(op_layernorm(c, a, L.n1, Q1));
    // token -> image
    RUN(op_add_cast(c, Q1, tok.v, Rt, tok.g, qin));
    RUN(op_add_cast(c, K, pos, 4096, nullptr, kin));
    RUN(attn_module(c, L.t2i, qin, kin, K, P, T, 4096, &Q1, a));
    RUN(op_layernorm(c, a, L.n2, Q2));
    // MLP
    RUN(op_linear(c, Q2, L.mlp1, h, 2, nullptr, true));
    RUN(op_linear(c, h, L.mlp2, a, 0, &Q2, false));
    RUN(op_layernorm(c, a, L.n3, Q3));
    // image -> token
    RUN(op_add_cast(c, Q3, tok.v, Rt, tok.g, qin));
    RUN(attn_module(c, L.i2t, kin, qin, Q3, P, 4096, T, &K, a));
    Ten K1;
    RUN(op_layernorm(c, a, L.n4, K1));
    Q = Q3; K = K1;
  }
  Ten qin, kin, a, hs;
  RUN(op_add_cast(c, Q, tok.v, Rt, tok.g, qin));
  RUN(op_add_cast(c, K, pos, 4096, nullptr, kin));
  RUN(attn_module(c, d.fin, qin, kin, K, P, T, 4096, &Q, a));
  RUN(op_layernorm(c, a, d.nfin, hs));
  // upscaling: convT1 -> LayerNorm2d -> GELU -> convT2 -> GELU, all as row-wise ops on [pixel, sub-pixel] rows
  Ten u1, y1, a1, u2, up;
  RUN(op_linear(c, K, d.ct1, u1, 0, nullptr, false));                  // [Ri, 4 * 64]
  Ten u1r = u1; u1r.rows = Ri * 4; u1r.cols = 64;
  RUN(op_layernorm(c, u1r, d.upln, y1, false));                         // [Ri * 4, 64]
  RUN(op_gelu(c, y1, a1));
  RUN(op_linear(c, a1, d.ct2, u2, 0, nullptr, true));                  // [Ri * 4, 4 * 32]
  RUN(op_gelu(c, u2, up));                                              // rows of 32 channels: [Ri * 16, 32]
  // hyper-network MLPs on the mask tokens, IoU head on the IoU token
  Ten hyper = c.ten((long)P * 8, 32, true, true, true);                 // [P, 8 (4 used), 32]
  if (c.err) return -1;
  if (cudaMemsetAsync(hyper.v, 0, (size_t)hyper.n() * 4, st) != cudaSuccess) return set_error("decoder training: memset failed");
  for (int i = 0; i < 4; ++i) {
    Ten x, h1, h2, h3;
    RUN(op_slice_rows(c, hs, (long)(1 + i) * 256, (long)T * 256, P, 256, x));
    RUN(op_linear(c, x, d.hyper[i][0], h1, 2, nullptr, true));
    RUN(op_linear(c, h1, d.hyper[i][1], h2, 2, nullptr, true));
    RUN(op_linear(c, h2, d.hyper[i][2], h3, 0, nullptr, false));       // [P, 32]
    copy_rows_kernel<<<nblk((long)P * 32), 256, 0, st>>>(h3.v, 32, hyper.v + i * 32, 8 * 32, P, 32, 0);
    KCHECK("hyper_gather");
    const Ten h3c = h3, hyc = hyper;
    const int ii = i, PP = P;
    s.tape.push_back([=](cudaStream_t st2) -> int {
      copy_rows_kernel<<<nblk((long)PP * 32), 256, 0, st2>>>(hyc.g + ii * 32, 8 * 32, h3c.g, 32, PP, 32, 1);
      KCHECK("hyper_scatter");
      return 0;
    });
  }
  RUN(launch_cast_bf16(hyper.v, hyper.n(), hyper.b, st));
  {
    Ten x, h1, h2;
    RUN(op_slice_rows(c, hs, 0, (long)T * 256, P, 256, x));
    RUN(op_linear(c, x, d.iou[0], h1, 2, nullptr, true));
    RUN(op_linear(c, h1, d.iou[1], h2, 2, nullptr, true));
    RUN(op_linear(c, h2, d.iou[2], s.iou32, 0, nullptr, false));       // [P, 32], columns 0..3 real
    copy_rows_kernel<<<nblk((long)P * s.nm), 256, 0, st>>>(s.iou32.v + s.m0, 32, iou, s.nm, P, s.nm, 0);
    KCHECK("iou_out");
  }
  // masks = hyper @ upscaled: per prompt [65536 x 32] x [32 x 4]
  s.low4 = c.ten((long)P * 65536, 4, true, false, false);
  s.dmask8 = (__nv_bfloat16*)c.take((size_t)P * 65536 * 8 * 2);
  if (c.err) return -1;
  {
    BGemmArgs g;
    g.A = up.b; g.B = hyper.b; g.M = 65536; g.N = 4; g.K = 32; g.lda = 32; g.ldb = 32; g.a_wstride = 65536L * 32; g.b_wstride = 8 * 32;
    g.b_rows_valid = 4; g.heads = 1; g.outer = P; g.out = s.low4.v; g.ldc = 4; g.o_wstride = 65536L * 4;
    RUN(launch_bgemm(g, st));
    masks_out_kernel<<<nblk((long)P * s.nm * 65536), 256, 0, st>>>(s.low4.v, P, s.nm, s.m0, low_res);
    KCHECK("masks_out");
    const Ten upc = up, hyc = hyper;
    __nv_bfloat16* dm = s.dmask8;
    const int PP = P;
    s.tape.push_back([=](cudaStream_t st2) -> int {   // dmask8 was filled by decoder_train_backward
      BGemmArgs g;
      // d up += dmask hyper
      g.A = dm; g.B = hyc.b; g.b_mn = 1; g.M = 65536; g.N = 32; g.K = 8; g.lda = 8; g.ldb = 32; g.a_wstride = 65536L * 8; g.b_wstride = 8 * 32;
      g.heads = 1; g.outer = PP; g.out = upc.g; g.ldc = 32; g.o_wstride = 65536L * 32; g.accumulate = 1;
      RUN(launch_bgemm(g, st2));
      // d hyper += dmask^T up
      g = BGemmArgs();
      g.A = dm; g.B = upc.b; g.a_mn = g.b_mn = 1; g.M = 8; g.N = 32; g.K = 65536; g.lda = 8; g.ldb = 32; g.a_wstride = 65536L * 8;
      g.b_wstride = 65536L * 32; g.heads = 1; g.outer = PP; g.out = hyc.g; g.ldc = 32; g.o_wstride = 8 * 32; g.accumulate = 1;
      return launch_bgemm(g, st2);
    });
  }
  if (c.err) return -1;
  s.live = true;
  return 0;
}

// ------------------------------------------------------------------------------------------------ backward
int Engine::decoder_train_backward(int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, cudaStream_t st) {
  if (!dtrain || slot < 0 || slot >= 8 || !dtrain->slot[slot].live) return set_error("decoder training: no saved forward pass in slot %d", slot);
  DecTrain& d = *dtrain;
  DecSlot& s = d.slot[slot];
  const int P = s.P;
  if (d_low_res) {
    masks_grad_kernel<<<nblk((long)P * 65536), 256, 0, st>>>(d_low_res, P, s.nm, s.m0, s.dmask8);
    KCHECK("masks_grad");
  } else if (cudaMemsetAsync(s.dmask8, 0, (size_t)P * 65536 * 16, st) != cudaSuccess) {
    return set_error("decoder training: memset failed");
  }
  if (d_iou) {
    copy_rows_kernel<<<nblk((long)P * s.nm), 256, 0, st>>>(d_iou, s.nm, s.iou32.g + s.m0, 32, P, s.nm, 1);
    KCHECK("iou_grad");
  }
  for (auto it = s.tape.rbegin(); it != s.tape.rend(); ++it) RUN((*it)(st));
  token_grads_kernel<<<s.T, 256, 0, st>>>(s.tok.g, s.emb_index, P, s.T, s.Ts, d.g_out_tokens, d.g_point_emb, d.g_nap);
  KCHECK("token_grads");
  src_grad_kernel<<<dim3(128, 8), dim3(32, 8), 0, st>>>(s.keys0.g, P, d_emb_nchw, d.g_no_mask);
  KCHECK("src_grad");
  s.live = false;   // gradients of the activations are consumed: one backward per forward
  return 0;
}

int Engine::decoder_grad(const char* name, float* dst, int64_t n, cudaStream_t st) {
  if (!dtrain) return set_error("msam_decoder_grad: decoder training mode was never entered");
  auto it = dtrain->grads.find(name);
  if (it == dtrain->grads.end()) return set_error("msam_decoder_grad: no gradient named '%s'", name);
  if (it->second.second != n) return set_error("msam_decoder_grad: '%s' has %lld elements, caller expects %lld", name, (long long)it->second.second, (long long)n);
  if (cudaMemcpyAsync(dst, it->second.first, (size_t)n * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("msam_decoder_grad: copy failed");
  return 0;
}

void Engine::dec_train_free() {
  if (!dtrain) return;
  for (DecSlot& s : dtrain->slot)
    if (s.arena) cudaFree(s.arena);
  delete dtrain;
  dtrain = nullptr;
}

int Engine::decoder_zero_grads(cudaStream_t st) {
  if (!dtrain) return 0;
  for (auto& kv : dtrain->grads)
    if (cudaMemsetAsync(kv.second.first, 0, (size_t)kv.second.second * 4, st) != cudaSuccess) return set_error("decoder training: memset failed");
  return 0;
}

}  // namespace msam
