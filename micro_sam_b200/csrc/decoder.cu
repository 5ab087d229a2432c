// Prompt encoder + two-way-transformer mask decoder (segment_anything PromptEncoder / MaskDecoder / TwoWayTransformer,
// restated in oracle/sam_ref.py) batched over P prompts of one image embedding.
//
// Layout: image tokens are rows (token-major [4096, 256]); per-prompt image-side tensors are [P*4096, C].  All dense
// projections run on the wgmma GEMM (gemm.cu); this file adds the small fused CUDA-core kernels around them
// (prompt PE, 7-token self attention, token->image and image->token attention cores, hyper-network mask product).
// Exact algebraic hoist: in layer 0 the image-side projections (k/v of token->image, q of image->token) act on
// `image_embedding + dense (+ pe)`, identical for every prompt when no mask prompt is given -> computed once per
// image in set_image_embedding (SURVEY.md 8d).
#include "engine.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace msam {

constexpr int DC = 256;     // transformer dim
constexpr int DI = 128;     // cross-attention internal dim
constexpr int NHEAD = 8;
constexpr int TMAX = 16;    // max tokens per prompt (5 output tokens + sparse prompt tokens)
constexpr int TMAX_TRAIN = 64;   // max tokens per prompt of the prompt encoder feeding the training decoder (decoder_train.cu)

struct AttnW {  // one SamAttention: q,k,v [inner, 256], out [256, inner]
  __nv_bfloat16 *q = nullptr, *k = nullptr, *v = nullptr, *o = nullptr, *qk = nullptr, *qkv = nullptr;
  float *qb = nullptr, *kb = nullptr, *vb = nullptr, *ob = nullptr, *qkb = nullptr, *qkvb = nullptr;
  __nv_bfloat16 *kT = nullptr, *vT = nullptr;  // cross attention: k_proj / v_proj weights transposed [256, inner] (t2i_fused.cu)
};
struct DecLayer {
  AttnW self_attn, t2i, i2t;
  __nv_bfloat16* i2t_qT = nullptr;  // image->token q_proj weight transposed [256, 128] (operand of the Mq GEMM, i2t_fused.cu)
  float *n1g, *n1b, *n2g, *n2b, *n3g, *n3b, *n4g, *n4b;
  __nv_bfloat16 *mlp1, *mlp2;
  float *mlp1b, *mlp2b;
};
struct Mlp3 {
  __nv_bfloat16* w[3];
  float* b[3];
};

struct DecoderState {
  // prompt encoder
  float *gauss = nullptr, *point_emb = nullptr /*[4,256]*/, *not_a_point = nullptr, *no_mask = nullptr;
  float* pos = nullptr;  // dense PE, token-major [4096, 256]
  __nv_bfloat16* pos_bf = nullptr;
  // mask decoder
  float* out_tokens = nullptr;  // [5, 256] = iou_token ; mask_tokens
  DecLayer layers[2];
  AttnW final_t2i;
  float *nfg, *nfb;
  __nv_bfloat16* ct1 = nullptr;                   // conv-transpose 1 weight as GEMM operand
  __half* ct2_f16 = nullptr;                      // conv-transpose 2 in fp16 (upscale_fused.cu)
  float *ct1b = nullptr, *ct2b = nullptr, *upln_g = nullptr, *upln_b = nullptr;
  Mlp3 hyper[4], iou_head;
  // per-image state (set_image_embedding)
  bool image_set = false;
  float* src = nullptr;               // [4096,256] image embedding + no_mask_embed (fp32, residual of layer 0)
  __nv_bfloat16 *src_bf = nullptr, *src_pe_bf = nullptr;
  float* emb = nullptr;               // [4096,256] image embedding without no_mask_embed (mask prompts add their own dense term)
  __nv_bfloat16* q0 = nullptr;        // hoisted layer-0 image->token q projection [4096,128] (unfused path, T > 8)
  // (keys + pe) Wq^T = keys Wq^T + pe Wq^T for the unfused image->token path (T > 8): the prompt-independent second term is
  // precomputed per layer ([4096, 128] fp32) and added through the GEMM's row-modulus residual.
  float* q_res[2] = {nullptr, nullptr};
  // PromptEncoder.mask_downscaling (mask prompts): conv 1->4 k2s2, LN2d, GELU, conv 4->16 k2s2, LN2d, GELU, conv 16->256 k1
  float *md_w1 = nullptr, *md_b1 = nullptr, *md_g1 = nullptr, *md_be1 = nullptr, *md_w2 = nullptr, *md_b2 = nullptr,
        *md_g2 = nullptr, *md_be2 = nullptr, *md_w3 = nullptr, *md_b3 = nullptr;
  // per-chunk workspace (P = max_prompts)
  float *tok0 = nullptr, *queries = nullptr, *tok_f32 = nullptr;
  __nv_bfloat16 *tok0_bf = nullptr, *q_bf = nullptr, *qpe_bf = nullptr, *t_qkv = nullptr, *t_att = nullptr, *t_mlp = nullptr;
  __nv_bfloat16 *t_q128 = nullptr, *t_k128 = nullptr, *t_v128 = nullptr, *t_att128 = nullptr;
  __nv_bfloat16 *keys = nullptr, *img_kvq = nullptr, *img_att = nullptr;
  __nv_bfloat16 *kexp = nullptr, *vexp = nullptr, *mq = nullptr, *vt = nullptr;  // fused i2t operands (i2t_fused.cu)
  float* sbias = nullptr;
  __nv_bfloat16 *qexp = nullptr, *qp = nullptr;  // fused t2i operands (t2i_fused.cu)
  float* un = nullptr;
  __nv_bfloat16 *h1 = nullptr, *h2 = nullptr;
  float *hyper_in = nullptr, *iou_out = nullptr;
};

// ================================================================================================ kernels
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pk2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Dense PE of the 64x64 pixel-centre grid (PositionEmbeddingRandom.forward) -> token-major [g*g, 256].
__global__ void dense_pe_kernel(const float* __restrict__ G, int g, float* __restrict__ pos) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= g * g * 128) return;
  const int f = idx % 128, t = idx / 128, y = t / g, x = t % g;
  const float cx = 2.f * (((float)x + 0.5f) / (float)g) - 1.f, cy = 2.f * (((float)y + 0.5f) / (float)g) - 1.f;
  const float v = 6.283185307179586f * (cx * G[f] + cy * G[128 + f]);
  pos[(long)t * 256 + f] = sinf(v);
  pos[(long)t * 256 + 128 + f] = cosf(v);
}

// NCHW fp32 image embedding [256, T] -> token-major src = emb + no_mask_embed (fp32, bf16) and src + pos (bf16).
__global__ void set_image_kernel(const float* __restrict__ feat, const float* __restrict__ no_mask,
                                 const float* __restrict__ pos, int T, float* __restrict__ src,
                                 __nv_bfloat16* __restrict__ src_bf, __nv_bfloat16* __restrict__ src_pe_bf,
                                 float* __restrict__ emb) {
  __shared__ float tile[32][33];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) tile[i][tx] = feat[(long)(c0 + i) * T + t0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, c = c0 + tx;
    emb[(long)t * 256 + c] = tile[tx][i];
    const float v = tile[tx][i] + no_mask[c];
    src[(long)t * 256 + c] = v;
    src_bf[(long)t * 256 + c] = __float2bfloat16(v);
    src_pe_bf[(long)t * 256 + c] = __float2bfloat16(v + pos[(long)t * 256 + c]);
  }
}

// Mask prompts (PromptEncoder._embed_masks): keys0[p, token, :] = image_embedding[token, :] + mask_downscaling(mask[p])[:, token]
// grid = (4096 / 16, P), block = 256 (thread = output channel; 16 tokens per block).  LayerNorm2d: eps 1e-6, biased variance.
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__global__ void __launch_bounds__(256)
mask_dense_kernel(const float* __restrict__ mask, const float* __restrict__ w1, const float* __restrict__ b1,
                  const float* __restrict__ g1, const float* __restrict__ be1, const float* __restrict__ w2,
                  const float* __restrict__ b2, const float* __restrict__ g2, const float* __restrict__ be2,
                  const float* __restrict__ w3, const float* __restrict__ b3, const float* __restrict__ emb,
                  __nv_bfloat16* __restrict__ keys, float* __restrict__ dense_out) {
  const int p = blockIdx.y, t0 = blockIdx.x * 16, tid = threadIdx.x;
  __shared__ float sa[16][16];  // [token][c*4 + sy*2 + sx] after stage 1
  __shared__ float sg[16][16];  // [token][o] after stage 2
  const float* m = mask + (size_t)p * 65536;
  if (tid < 64) {  // stage 1: thread = (token, sub-position): 4 channels
    const int tk = tid >> 2, sy = (tid >> 1) & 1, sx = tid & 1, t = t0 + tk, ty = t >> 6, tx = t & 63;
    const float* mp = m + (size_t)(4 * ty + 2 * sy) * 256 + 4 * tx + 2 * sx;
    const float m00 = mp[0], m01 = mp[1], m10 = mp[256], m11 = mp[257];
    float y[4], mean = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      y[c] = b1[c] + w1[c * 4 + 0] * m00 + w1[c * 4 + 1] * m01 + w1[c * 4 + 2] * m10 + w1[c * 4 + 3] * m11;
      mean += y[c];
    }
    mean *= 0.25f;
    float var = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) var += (y[c] - mean) * (y[c] - mean);
    const float rstd = rsqrtf(var * 0.25f + 1e-6f);
#pragma unroll
    for (int c = 0; c < 4; ++c) sa[tk][c * 4 + sy * 2 + sx] = gelu_exact((y[c] - mean) * rstd * g1[c] + be1[c]);
  }
  __syncthreads();
  if (tid < 16) {  // stage 2: thread = token: 16 channels (w2[o][c][sy][sx] contiguous = [o][16])
    float z[16], mean = 0.f;
#pragma unroll
    for (int o = 0; o < 16; ++o) {
      float acc = b2[o];
#pragma unroll
      for (int k = 0; k < 16; ++k) acc += w2[o * 16 + k] * sa[tid][k];
      z[o] = acc;
      mean += acc;
    }
    mean *= (1.0f / 16);
    float var = 0.f;
#pragma unroll
    for (int o = 0; o < 16; ++o) var += (z[o] - mean) * (z[o] - mean);
    const float rstd = rsqrtf(var * (1.0f / 16) + 1e-6f);
#pragma unroll
    for (int o = 0; o < 16; ++o) sg[tid][o] = gelu_exact((z[o] - mean) * rstd * g2[o] + be2[o]);
  }
  __syncthreads();
  float w[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) w[o] = w3[tid * 16 + o];
  const float bb = b3[tid];
#pragma unroll 4
  for (int tk = 0; tk < 16; ++tk) {
    float acc = bb;
#pragma unroll
    for (int o = 0; o < 16; ++o) acc += w[o] * sg[tk][o];
    const size_t tok = (size_t)(t0 + tk);
    if (dense_out) dense_out[((size_t)p * 256 + tid) * 4096 + tok] = acc;   // PromptEncoder output (NCHW fp32)
    else keys[((size_t)p * 4096 + tok) * 256 + tid] = __float2bfloat16(acc + emb[tok * 256 + tid]);
  }
}

// Tokens from GIVEN sparse prompt embeddings (the `mask_decoder(sparse_prompt_embeddings=...)` call of
// training/trainable_sam.py:88-106): tok[p, 0..4] = output tokens, tok[p, 5 + s] = sparse[p, s].  grid = (T, P), block = 128.
__global__ void tokens_from_sparse_kernel(const float* __restrict__ sparse, int n_sparse, int T,
                                          const float* __restrict__ out_tokens, float* __restrict__ tok,
                                          __nv_bfloat16* __restrict__ tok_bf) {
  const int p = blockIdx.y, t = blockIdx.x, f = threadIdx.x;
  const float* src = t < 5 ? out_tokens + t * 256 : sparse + ((long)p * n_sparse + (t - 5)) * 256;
  const long o = ((long)p * T + t) * 256;
  const float a = src[f], b = src[128 + f];
  tok[o + f] = a; tok[o + 128 + f] = b;
  tok_bf[o + f] = __float2bfloat16(a); tok_bf[o + 128 + f] = __float2bfloat16(b);
}

// keys0[p, token, c] = image_embedding[token, c] + dense[p, c, token]  for GIVEN dense prompt embeddings (NCHW fp32
// [P, 256, 4096]).  grid = (4096/32, 256/32, P), block = (32, 8): transposed through shared memory.
__global__ void dense_to_keys_kernel(const float* __restrict__ dense, const float* __restrict__ emb,
                                     __nv_bfloat16* __restrict__ keys) {
  __shared__ float tile[32][33];
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32, p = blockIdx.z, tx = threadIdx.x, ty = threadIdx.y;
  const float* d = dense + (size_t)p * 256 * 4096;
  for (int i = ty; i < 32; i += 8) tile[i][tx] = d[(size_t)(c0 + i) * 4096 + t0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const size_t tok = (size_t)(t0 + i);
    keys[((size_t)p * 4096 + tok) * 256 + c0 + tx] = __float2bfloat16(tile[tx][i] + emb[tok * 256 + c0 + tx]);
  }
}

// Tokens [P, T, 256] = [iou_token, mask_tokens(4), sparse prompt embeddings].  Sparse = points (+ pad point when no
// box) then box corners (PromptEncoder._embed_points/_embed_boxes; SURVEY A.8-7).  grid = (T-5, P), block = 128.
__global__ void prompt_tokens_kernel(const float* __restrict__ points, const float* __restrict__ labels, int np,
                                     const float* __restrict__ boxes, int T, int n_sparse, float img_size,
                                     const float* __restrict__ G, const float* __restrict__ point_emb,
                                     const float* __restrict__ not_a_point, const float* __restrict__ out_tokens,
                                     float* __restrict__ tok, __nv_bfloat16* __restrict__ tok_bf) {
  const int p = blockIdx.y, s = blockIdx.x, f = threadIdx.x;
  if (s == 0) {  // the 5 output tokens of this prompt
    float* d0 = tok + (long)p * T * 256;
    __nv_bfloat16* d0b = tok_bf + (long)p * T * 256;
    for (int i = f; i < 5 * 256; i += 128) {
      d0[i] = out_tokens[i];
      d0b[i] = __float2bfloat16(out_tokens[i]);
    }
  }
  if (s >= n_sparse) return;  // mask-only prompts have no sparse tokens
  const int n_pts = points ? np + (boxes ? 0 : 1) : 0;
  float* dst = tok + ((long)p * T + 5 + s) * 256;
  __nv_bfloat16* dstb = tok_bf + ((long)p * T + 5 + s) * 256;
  float x, y;
  int kind;  // -1 not-a-point, 0/1 point labels, 2/3 box corners
  if (s < n_pts) {
    if (s < np) {
      x = points[((long)p * np + s) * 2];
      y = points[((long)p * np + s) * 2 + 1];
      const int lb = (int)labels[(long)p * np + s];
      kind = (lb == -1) ? -1 : ((lb == 0 || lb == 1) ? lb : 4);  // other labels: plain PE (upstream adds nothing)
    } else {
      x = 0.f; y = 0.f; kind = -1;
    }
  } else {
    const int c = s - n_pts;
    x = boxes[(long)p * 4 + 2 * c];
    y = boxes[(long)p * 4 + 2 * c + 1];
    kind = 2 + c;
  }
  const float cx = 2.f * ((x + 0.5f) / img_size) - 1.f, cy = 2.f * ((y + 0.5f) / img_size) - 1.f;
  const float v = 6.283185307179586f * (cx * G[f] + cy * G[128 + f]);
  float e0 = sinf(v), e1 = cosf(v);
  if (kind < 0) {
    e0 = not_a_point[f];
    e1 = not_a_point[128 + f];
  } else if (kind < 4) {
    e0 += point_emb[kind * 256 + f];
    e1 += point_emb[kind * 256 + 128 + f];
  }
  dst[f] = e0; dst[128 + f] = e1;
  dstb[f] = __float2bfloat16(e0); dstb[128 + f] = __float2bfloat16(e1);
}

// Token self attention: T x T per (prompt, head), 8 heads x 32 dims.  One warp per (prompt, head); lane t = query t.
__global__ void token_self_attn_kernel(const __nv_bfloat16* __restrict__ q, int ldq, const __nv_bfloat16* __restrict__ k,
                                       int ldk, const __nv_bfloat16* __restrict__ v, int ldv, int P, int T,
                                       __nv_bfloat16* __restrict__ out) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= P * NHEAD) return;
  const int p = w / NHEAD, h = w % NHEAD;
  __shared__ float sk[4][TMAX][33], sv[4][TMAX][33];
  const int wib = threadIdx.x >> 5;
  for (int i = lane; i < T * 32; i += 32) {
    const int t = i / 32, d = i % 32;
    sk[wib][t][d] = __bfloat162float(k[((long)p * T + t) * ldk + h * 32 + d]);
    sv[wib][t][d] = __bfloat162float(v[((long)p * T + t) * ldv + h * 32 + d]);
  }
  __syncwarp();
  if (lane < T) {
    float qv[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) qv[d] = __bfloat162float(q[((long)p * T + lane) * ldq + h * 32 + d]);
    float s[TMAX], m = -INFINITY;
#pragma unroll
    for (int j = 0; j < TMAX; ++j) {
      s[j] = -INFINITY;
      if (j < T) {
        float a = 0.f;
#pragma unroll
        for (int d = 0; d < 32; ++d) a += qv[d] * sk[wib][j][d];
        s[j] = a * 0.17677669529663687f;  // 1/sqrt(32)
        m = fmaxf(m, s[j]);
      }
    }
    float l = 0.f, o[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) o[d] = 0.f;
#pragma unroll
    for (int j = 0; j < TMAX; ++j) {
      if (j < T) {
        const float pj = expf(s[j] - m);
        l += pj;
#pragma unroll
        for (int d = 0; d < 32; ++d) o[d] += pj * sv[wib][j][d];
      }
    }
    const float inv = 1.f / l;
    __nv_bfloat16* dst = out + ((long)p * T + lane) * 256 + h * 32;
#pragma unroll
    for (int d = 0; d < 32; d += 2) *reinterpret_cast<uint32_t*>(dst + d) = pk2(o[d] * inv, o[d + 1] * inv);
  }
}

// image -> token attention core.  q_img [*, ldq] (q_stride_rows = 0 when shared), k_tok / v_tok [P*T,128].
// grid = (NI/64, P), block = 256: thread = (head = tid%8, two image tokens n0 = blockIdx.x*64 + tid/8 and n0 + 32);
// token keys/values live in shared memory as 16-byte vectors (LDS.128, conflict-free with the 20-float pitch).
__global__ void __launch_bounds__(256)
i2t_attn_kernel(const __nv_bfloat16* __restrict__ qimg, int ldq, long q_stride_rows, const __nv_bfloat16* __restrict__ ktok,
                const __nv_bfloat16* __restrict__ vtok, int T, int NI, __nv_bfloat16* __restrict__ out) {
  const int p = blockIdx.y;
  __shared__ __align__(16) float sk[TMAX][NHEAD][20], sv[TMAX][NHEAD][20];
  for (int i = threadIdx.x; i < T * DI; i += 256) {
    const int t = i / DI, c = i % DI;
    sk[t][c / 16][c % 16] = __bfloat162float(ktok[((long)p * T + t) * DI + c]) * 0.25f;
    sv[t][c / 16][c % 16] = __bfloat162float(vtok[((long)p * T + t) * DI + c]);
  }
  __syncthreads();
  const int h = threadIdx.x & 7;
  float qf[2][16];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int n = blockIdx.x * 64 + (threadIdx.x >> 3) + 32 * r;
    const __nv_bfloat16* qp = qimg + ((long)p * q_stride_rows + n) * ldq + h * 16;
    const uint4 qa = *reinterpret_cast<const uint4*>(qp), qb = *reinterpret_cast<const uint4*>(qp + 8);
    const uint32_t qw[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) { qf[r][2 * i] = bf_lo(qw[i]); qf[r][2 * i + 1] = bf_hi(qw[i]); }
  }
  float s[2][TMAX], m[2] = {-1e30f, -1e30f};
#pragma unroll
  for (int t = 0; t < TMAX; ++t) {
    s[0][t] = s[1][t] = -1e30f;
    if (t < T) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int d = 0; d < 16; d += 4) {
        const float4 kk = *reinterpret_cast<const float4*>(&sk[t][h][d]);
        a0 += qf[0][d] * kk.x + qf[0][d + 1] * kk.y + qf[0][d + 2] * kk.z + qf[0][d + 3] * kk.w;
        a1 += qf[1][d] * kk.x + qf[1][d + 1] * kk.y + qf[1][d + 2] * kk.z + qf[1][d + 3] * kk.w;
      }
      s[0][t] = a0; s[1][t] = a1;
      m[0] = fmaxf(m[0], a0); m[1] = fmaxf(m[1], a1);
    }
  }
  float l[2] = {0.f, 0.f}, o[2][16];
#pragma unroll
  for (int d = 0; d < 16; ++d) o[0][d] = o[1][d] = 0.f;
#pragma unroll
  for (int t = 0; t < TMAX; ++t) {
    if (t < T) {
      const float p0 = __expf(s[0][t] - m[0]), p1 = __expf(s[1][t] - m[1]);
      l[0] += p0; l[1] += p1;
#pragma unroll
      for (int d = 0; d < 16; d += 4) {
        const float4 vv = *reinterpret_cast<const float4*>(&sv[t][h][d]);
        o[0][d] += p0 * vv.x; o[0][d + 1] += p0 * vv.y; o[0][d + 2] += p0 * vv.z; o[0][d + 3] += p0 * vv.w;
        o[1][d] += p1 * vv.x; o[1][d + 1] += p1 * vv.y; o[1][d + 2] += p1 * vv.z; o[1][d + 3] += p1 * vv.w;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float inv = 1.f / l[r];
    const int n = blockIdx.x * 64 + (threadIdx.x >> 3) + 32 * r;
    uint4 o0, o1;
    o0.x = pk2(o[r][0] * inv, o[r][1] * inv); o0.y = pk2(o[r][2] * inv, o[r][3] * inv);
    o0.z = pk2(o[r][4] * inv, o[r][5] * inv); o0.w = pk2(o[r][6] * inv, o[r][7] * inv);
    o1.x = pk2(o[r][8] * inv, o[r][9] * inv); o1.y = pk2(o[r][10] * inv, o[r][11] * inv);
    o1.z = pk2(o[r][12] * inv, o[r][13] * inv); o1.w = pk2(o[r][14] * inv, o[r][15] * inv);
    __nv_bfloat16* dst = out + ((long)p * NI + n) * DI + h * 16;
    *reinterpret_cast<uint4*>(dst) = o0;
    *reinterpret_cast<uint4*>(dst + 8) = o1;
  }
}

__global__ void gather_iou_kernel(const float* __restrict__ iou32, int P, int m0, int nm, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P * nm) out[i] = iou32[(long)(i / nm) * 32 + m0 + i % nm];
}

#define LAUNCH_CHECK(name)                                                                        \
  do {                                                                                            \
    cudaError_t e_ = cudaGetLastError();                                                          \
    if (e_ != cudaSuccess) return set_error(name " launch failed: %s", cudaGetErrorString(e_)); \
    count_launch();                                                                               \
  } while (0)
#define CHK(p) do { if (!(p)) return -1; } while (0)

// ================================================================================================ weights
static int load_attn(Engine& E, const std::string& p, int inner, AttnW& w, bool fuse_qkv) {
  CHK(w.q = E.up_bf16(p + "q_proj.weight", {inner, DC}));
  CHK(w.k = E.up_bf16(p + "k_proj.weight", {inner, DC}));
  CHK(w.v = E.up_bf16(p + "v_proj.weight", {inner, DC}));
  CHK(w.o = E.up_bf16(p + "out_proj.weight", {DC, inner}));
  CHK(w.qb = E.up_f32(p + "q_proj.bias", {inner}));
  CHK(w.kb = E.up_f32(p + "k_proj.bias", {inner}));
  CHK(w.vb = E.up_f32(p + "v_proj.bias", {inner}));
  CHK(w.ob = E.up_f32(p + "out_proj.bias", {DC}));
  if (inner == DI) {
    for (int which = 0; which < 2; ++which) {
      const auto* hw = E.host(p + (which ? "v_proj.weight" : "k_proj.weight"), {inner, DC});
      CHK(hw);
      std::vector<float> wt((size_t)DC * inner);
      for (int o = 0; o < inner; ++o)
        for (int c = 0; c < DC; ++c) wt[(size_t)c * inner + o] = (*hw)[(size_t)o * DC + c];
      CHK((which ? w.vT : w.kT) = E.upload_bf16(wt.data(), wt.size()));
    }
  }
  if (fuse_qkv) {  // [q;k;v] and [q;k] stacked along the output dim for single-GEMM projections
    const auto *hq = E.host(p + "q_proj.weight", {inner, DC}), *hk = E.host(p + "k_proj.weight", {inner, DC}),
               *hv = E.host(p + "v_proj.weight", {inner, DC});
    const auto *bq = E.host(p + "q_proj.bias", {inner}), *bk = E.host(p + "k_proj.bias", {inner}),
               *bv = E.host(p + "v_proj.bias", {inner});
    std::vector<float> cat, catb;
    cat.insert(cat.end(), hq->begin(), hq->end());
    cat.insert(cat.end(), hk->begin(), hk->end());
    catb.insert(catb.end(), bq->begin(), bq->end());
    catb.insert(catb.end(), bk->begin(), bk->end());
    CHK(w.qk = E.upload_bf16(cat.data(), cat.size()));
    CHK(w.qkb = E.upload_f32(catb.data(), catb.size()));
    cat.insert(cat.end(), hv->begin(), hv->end());
    catb.insert(catb.end(), bv->begin(), bv->end());
    CHK(w.qkv = E.upload_bf16(cat.data(), cat.size()));
    CHK(w.qkvb = E.upload_f32(catb.data(), catb.size()));
  }
  return 0;
}

static int load_mlp3(Engine& E, const std::string& p, int out_dim, Mlp3& m) {
  CHK(m.w[0] = E.up_bf16(p + "layers.0.weight", {DC, DC}));
  CHK(m.b[0] = E.up_f32(p + "layers.0.bias", {DC}));
  CHK(m.w[1] = E.up_bf16(p + "layers.1.weight", {DC, DC}));
  CHK(m.b[1] = E.up_f32(p + "layers.1.bias", {DC}));
  const auto* w2 = E.host(p + "layers.2.weight", {out_dim, DC});
  const auto* b2 = E.host(p + "layers.2.bias", {out_dim});
  CHK(w2 && b2);
  std::vector<float> wp((size_t)32 * DC, 0.f), bp(32, 0.f);  // pad the output dim to 32 (GEMM N granularity)
  std::copy(w2->begin(), w2->end(), wp.begin());
  std::copy(b2->begin(), b2->end(), bp.begin());
  CHK(m.w[2] = E.upload_bf16(wp.data(), wp.size()));
  CHK(m.b[2] = E.upload_f32(bp.data(), bp.size()));
  return 0;
}

int Engine::finalize_decoder() {
  if (host_weights.find("mask_decoder.iou_token.weight") == host_weights.end()) return 0;  // encoder-only model
  dec = new DecoderState();
  DecoderState& d = *dec;
  const int g = cfg.image_size / cfg.patch_size, NI = g * g;
  const std::string pe = "prompt_encoder.", md = "mask_decoder.";
  CHK(d.gauss = up_f32(pe + "pe_layer.positional_encoding_gaussian_matrix", {2, 128}));
  {
    std::vector<float> pts;
    for (int i = 0; i < 4; ++i) {
      const auto* h = host(pe + "point_embeddings." + std::to_string(i) + ".weight", {1, DC});
      CHK(h);
      pts.insert(pts.end(), h->begin(), h->end());
    }
    CHK(d.point_emb = upload_f32(pts.data(), pts.size()));
  }
  CHK(d.not_a_point = up_f32(pe + "not_a_point_embed.weight", {1, DC}));
  CHK(d.no_mask = up_f32(pe + "no_mask_embed.weight", {1, DC}));
  {
    const auto *it = host(md + "iou_token.weight", {1, DC}), *mt = host(md + "mask_tokens.weight", {4, DC});
    CHK(it && mt);
    std::vector<float> t(it->begin(), it->end());
    t.insert(t.end(), mt->begin(), mt->end());
    CHK(d.out_tokens = upload_f32(t.data(), t.size()));
  }
  for (int l = 0; l < 2; ++l) {
    DecLayer& L = d.layers[l];
    const std::string p = md + "transformer.layers." + std::to_string(l) + ".";
    if (load_attn(*this, p + "self_attn.", DC, L.self_attn, true)) return -1;
    if (load_attn(*this, p + "cross_attn_token_to_image.", DI, L.t2i, false)) return -1;
    if (load_attn(*this, p + "cross_attn_image_to_token.", DI, L.i2t, false)) return -1;
    CHK(L.n1g = up_f32(p + "norm1.weight", {DC})); CHK(L.n1b = up_f32(p + "norm1.bias", {DC}));
    CHK(L.n2g = up_f32(p + "norm2.weight", {DC})); CHK(L.n2b = up_f32(p + "norm2.bias", {DC}));
    CHK(L.n3g = up_f32(p + "norm3.weight", {DC})); CHK(L.n3b = up_f32(p + "norm3.bias", {DC}));
    CHK(L.n4g = up_f32(p + "norm4.weight", {DC})); CHK(L.n4b = up_f32(p + "norm4.bias", {DC}));
    CHK(L.mlp1 = up_bf16(p + "mlp.lin1.weight", {2048, DC})); CHK(L.mlp1b = up_f32(p + "mlp.lin1.bias", {2048}));
    CHK(L.mlp2 = up_bf16(p + "mlp.lin2.weight", {DC, 2048})); CHK(L.mlp2b = up_f32(p + "mlp.lin2.bias", {DC}));
    {
      const auto* wq = host(p + "cross_attn_image_to_token.q_proj.weight", {DI, DC});
      CHK(wq);
      std::vector<float> wt((size_t)DC * DI);
      for (int o = 0; o < DI; ++o)
        for (int c = 0; c < DC; ++c) wt[(size_t)c * DI + o] = (*wq)[(size_t)o * DC + c];
      CHK(L.i2t_qT = upload_bf16(wt.data(), wt.size()));
    }
  }
  if (load_attn(*this, md + "transformer.final_attn_token_to_image.", DI, d.final_t2i, false)) return -1;
  CHK(d.nfg = up_f32(md + "transformer.norm_final_attn.weight", {DC}));
  CHK(d.nfb = up_f32(md + "transformer.norm_final_attn.bias", {DC}));
  {  // ConvTranspose2d(256->64,k2,s2): W[c,o,dy,dx] -> GEMM weight [(dy*2+dx)*64 + o][c], bias[(.)*64 + o] = b[o]
    const auto *w = host(md + "output_upscaling.0.weight", {DC, 64, 2, 2}), *b = host(md + "output_upscaling.0.bias", {64});
    CHK(w && b);
    std::vector<float> W((size_t)256 * DC), B(256);
    for (int c = 0; c < DC; ++c)
      for (int o = 0; o < 64; ++o)
        for (int s = 0; s < 4; ++s) W[((size_t)s * 64 + o) * DC + c] = (*w)[((size_t)c * 64 + o) * 4 + s];
    for (int s = 0; s < 4; ++s)
      for (int o = 0; o < 64; ++o) B[s * 64 + o] = (*b)[o];
    CHK(d.ct1 = upload_bf16(W.data(), W.size()));
    CHK(d.ct1b = upload_f32(B.data(), B.size()));
  }
  CHK(d.upln_g = up_f32(md + "output_upscaling.1.weight", {64}));
  CHK(d.upln_b = up_f32(md + "output_upscaling.1.bias", {64}));
  {  // ConvTranspose2d(64->32,k2,s2) -> GEMM weight [(ey*2+ex)*32 + o][c]
    const auto *w = host(md + "output_upscaling.3.weight", {64, 32, 2, 2}), *b = host(md + "output_upscaling.3.bias", {32});
    CHK(w && b);
    std::vector<float> W((size_t)128 * 64), B(128);
    for (int c = 0; c < 64; ++c)
      for (int o = 0; o < 32; ++o)
        for (int s = 0; s < 4; ++s) W[((size_t)s * 32 + o) * 64 + c] = (*w)[((size_t)c * 32 + o) * 4 + s];
    for (int s = 0; s < 4; ++s)
      for (int o = 0; o < 32; ++o) B[s * 32 + o] = (*b)[o];
    CHK(d.ct2_f16 = upload_f16(W.data(), W.size()));
    CHK(d.ct2b = upload_f32(B.data(), B.size()));
  }
  for (int i = 0; i < 4; ++i)
    if (load_mlp3(*this, md + "output_hypernetworks_mlps." + std::to_string(i) + ".", 32, d.hyper[i])) return -1;
  if (load_mlp3(*this, md + "iou_prediction_head.", 4, d.iou_head)) return -1;

  // dense PE + per-image buffers
  CHK(d.pos = (float*)dalloc((size_t)NI * DC * 4));
  dense_pe_kernel<<<(NI * 128 + 255) / 256, 256>>>(d.gauss, g, d.pos);
  LAUNCH_CHECK("dense_pe");
  {
    // positional-encoding terms of the (unfused) image->token q projections
    __nv_bfloat16* pos_bf = d.pos_bf = (__nv_bfloat16*)dalloc((size_t)NI * DC * 2);
    CHK(pos_bf);
    if (launch_cast_bf16(d.pos, (long)NI * DC, pos_bf, 0)) return -1;
    for (int l = 0; l < 2; ++l) {
      CHK(d.q_res[l] = (float*)dalloc((size_t)NI * DI * 4, true));
      GemmArgs a;
      a.A = pos_bf; a.W = d.layers[l].i2t.q; a.M = NI; a.N = DI; a.K = DC; a.lda = DC; a.ldw = DC; a.out = d.q_res[l];
      a.ldc = DI; a.out_fp32 = 1;
      if (launch_gemm(a, num_sms, 0)) return -1;
    }
  }
  {
    const std::string mk = pe + "mask_downscaling.";
    CHK(d.md_w1 = up_f32(mk + "0.weight", {4, 1, 2, 2})); CHK(d.md_b1 = up_f32(mk + "0.bias", {4}));
    CHK(d.md_g1 = up_f32(mk + "1.weight", {4}));          CHK(d.md_be1 = up_f32(mk + "1.bias", {4}));
    CHK(d.md_w2 = up_f32(mk + "3.weight", {16, 4, 2, 2})); CHK(d.md_b2 = up_f32(mk + "3.bias", {16}));
    CHK(d.md_g2 = up_f32(mk + "4.weight", {16}));         CHK(d.md_be2 = up_f32(mk + "4.bias", {16}));
    CHK(d.md_w3 = up_f32(mk + "6.weight", {DC, 16, 1, 1})); CHK(d.md_b3 = up_f32(mk + "6.bias", {DC}));
  }
  CHK(d.src = (float*)dalloc((size_t)NI * DC * 4));
  CHK(d.src_bf = (__nv_bfloat16*)dalloc((size_t)NI * DC * 2));
  CHK(d.src_pe_bf = (__nv_bfloat16*)dalloc((size_t)NI * DC * 2));
  CHK(d.emb = (float*)dalloc((size_t)NI * DC * 4));
  CHK(d.q0 = (__nv_bfloat16*)dalloc((size_t)NI * DI * 2));
  // per-chunk workspace
  const size_t P = cfg.max_prompts, PT = P * TMAX, PN = P * NI;
  CHK(d.tok0 = (float*)dalloc(PT * DC * 4));
  CHK(d.tok0_bf = (__nv_bfloat16*)dalloc(PT * DC * 2));
  CHK(d.queries = (float*)dalloc(PT * DC * 4));
  CHK(d.tok_f32 = (float*)dalloc(PT * DC * 4));
  CHK(d.q_bf = (__nv_bfloat16*)dalloc(PT * DC * 2));
  CHK(d.qpe_bf = (__nv_bfloat16*)dalloc(PT * DC * 2));
  CHK(d.t_qkv = (__nv_bfloat16*)dalloc(PT * 3 * DC * 2));
  CHK(d.t_att = (__nv_bfloat16*)dalloc(PT * DC * 2));
  CHK(d.t_mlp = (__nv_bfloat16*)dalloc(PT * 2048 * 2));
  CHK(d.t_q128 = (__nv_bfloat16*)dalloc(PT * DI * 2));
  CHK(d.t_k128 = (__nv_bfloat16*)dalloc(PT * DI * 2));
  CHK(d.t_v128 = (__nv_bfloat16*)dalloc(PT * DI * 2));
  CHK(d.t_att128 = (__nv_bfloat16*)dalloc(PT * DI * 2));
  CHK(d.keys = (__nv_bfloat16*)dalloc(PN * DC * 2));
  CHK(d.img_kvq = (__nv_bfloat16*)dalloc(PN * 3 * DI * 2));
  CHK(d.img_att = (__nv_bfloat16*)dalloc(PN * DI * 2));
  CHK(d.kexp = (__nv_bfloat16*)dalloc(P * 64 * DI * 2));
  CHK(d.vexp = (__nv_bfloat16*)dalloc(P * 64 * DI * 2));
  CHK(d.mq = (__nv_bfloat16*)dalloc(P * 64 * DC * 2));
  CHK(d.vt = (__nv_bfloat16*)dalloc(P * 64 * DC * 2));
  CHK(d.sbias = (float*)dalloc(P * 64 * 4));
  CHK(d.qexp = (__nv_bfloat16*)dalloc(P * 128 * DI * 2));
  CHK(d.qp = (__nv_bfloat16*)dalloc(P * 128 * DC * 2));
  CHK(d.un = (float*)dalloc(P * 128 * DC * 4));
  CHK(d.h1 = (__nv_bfloat16*)dalloc(P * DC * 2));
  CHK(d.h2 = (__nv_bfloat16*)dalloc(P * DC * 2));
  CHK(d.hyper_in = (float*)dalloc(P * 4 * 32 * 4));
  CHK(d.iou_out = (float*)dalloc(P * 32 * 4));
  return 0;
}

// ================================================================================================ forward
static int gemm(Engine& E, cudaStream_t st, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int M, int N, int K,
                const float* bias, void* out, int ldc, int out_fp32, int act = 0, const void* residual = nullptr,
                int res_rows = 0, int res_bf16 = 0, int epi = 0, const float* ln_g = nullptr, const float* ln_b = nullptr,
                float ln_eps = 1e-5f, int ldr = 0) {
  GemmArgs a;
  a.A = A; a.W = W; a.M = M; a.N = N; a.K = K; a.lda = lda; a.ldw = K; a.bias = bias; a.out = out; a.ldc = ldc;
  a.out_fp32 = out_fp32; a.act = act; a.residual = residual; a.res_rows = res_rows; a.res_bf16 = res_bf16;
  a.epi = epi; a.ln_gamma = ln_g; a.ln_beta = ln_b; a.ln_eps = ln_eps; a.ldr = ldr;
  return launch_gemm(a, E.num_sms, st);
}
static int ln(cudaStream_t st, const float* x, int rows, int D, const float* g, const float* b, float eps,
              __nv_bfloat16* out, float* out_f32 = nullptr, const float* add = nullptr, int add_rows = 1,
              __nv_bfloat16* out2 = nullptr, int act = 0) {
  LnArgs l;
  l.x = x; l.rows = rows; l.D = D; l.gamma = g; l.beta = b; l.eps = eps; l.out = out; l.out_f32 = out_f32;
  l.add = add; l.add_rows = add_rows; l.out2 = out2; l.act = act;
  return launch_layernorm(l, st);
}

int Engine::set_image_embedding(const float* feat, cudaStream_t st) {
  if (!finalized || !dec) return set_error("set_image_embedding: decoder weights not loaded");
  DecoderState& d = *dec;
  const int g = cfg.image_size / cfg.patch_size, NI = g * g;
  set_image_kernel<<<dim3(NI / 32, DC / 32), dim3(32, 8), 0, st>>>(feat, d.no_mask, d.pos, NI, d.src, d.src_bf, d.src_pe_bf, d.emb);
  LAUNCH_CHECK("set_image");
  const DecLayer& L0 = d.layers[0];
  if (gemm(*this, st, d.src_pe_bf, DC, L0.i2t.q, NI, DI, DC, L0.i2t.qb, d.q0, DI, 0)) return -1;
  d.image_set = true;
  return 0;
}

// ---- The three blocks that do most of a decode.  decode_chunk and the op-level entry points (msam_op_dec_*) both call these
// functions, so the tests exercise the production launch sequence.

// Token -> image attention of instance A: qpe = queries + query_pe [P*T, 256] -> per-head output before out_proj
// [P*T, 128] (t2i_fused.cu).  keys [P*4096, 256], or nullptr: the bound image, shared by every prompt.
static int t2i_block(Engine& E, cudaStream_t st, const AttnW& A, int P, int T, const __nv_bfloat16* qpe,
                     const __nv_bfloat16* keys, __nv_bfloat16* out) {
  DecoderState& d = *E.dec;
  const int mode = keys ? 1 : 0;
  if (gemm(E, st, qpe, DC, A.q, P * T, DI, DC, A.qb, d.t_q128, DI, 0)) return -1;
  // T <= 8: 64 rows per prompt (row pp*64 + h*8 + t).  Shared image tokens (mode 0): two prompts per 128-row item;
  // own keys (mode 1): one 64-row item per prompt (one warpgroup).  T > 8: 128 rows per prompt (h*16 + t).
  const int small = T <= 8 ? 1 : 0;
  const int prep_items = small ? (P + 1) / 2 : P;   // 128-row blocks of the Q' operand
  if (launch_t2i_prep(d.t_q128, P, T, small, prep_items, d.qexp, st)) return -1;
  if (gemm(E, st, d.qexp, DI, A.kT, prep_items * 128, DC, DI, nullptr, d.qp, DC, 0)) return -1;
  T2iFusedArgs ta;
  ta.mode = mode;
  ta.rows = (small && mode) ? 64 : 128;
  ta.n_items = (small && mode) ? P : prep_items;
  ta.x = mode ? keys : d.src_bf;
  ta.xs = mode ? d.pos_bf : d.src_pe_bf;
  ta.qp = d.qp; ta.out = d.un;
  if (launch_t2i_fused(ta, E.num_sms, st)) return -1;
  return launch_t2i_head_proj(d.un, A.vT, A.vb, P, T, small, out, st);
}

// Image -> token attention block of layer l (TwoWayAttentionBlock step 4): keys <- norm4(keys + attn(q = keys + pe,
// k = qpe, v = q)) for P prompts, q / qpe = queries / queries + query_pe [P*T, 256].  Own keys are updated in place;
// shared (layer 0 without per-prompt keys) reads the bound image and only writes keys.
static int i2t_block(Engine& E, cudaStream_t st, int l, int P, int T, const __nv_bfloat16* q, const __nv_bfloat16* qpe,
                     bool shared, __nv_bfloat16* keys) {
  DecoderState& d = *E.dec;
  const DecLayer& L = d.layers[l];
  const int NI = 4096, PN = P * NI;
  const bool fused = T <= 8;
  if (!shared && !fused) {  // q of the (unfused) image -> token attention: (keys + pe) Wq^T, pe term through the residual
    if (gemm(E, st, keys, DC, L.i2t.q, PN, DI, DC, L.i2t.qb, d.img_kvq, DI, 0, 0, d.q_res[l], NI)) return -1;
  }
  if (gemm(E, st, qpe, DC, L.i2t.k, P * T, DI, DC, L.i2t.kb, d.t_k128, DI, 0)) return -1;
  if (gemm(E, st, q, DC, L.i2t.v, P * T, DI, DC, L.i2t.vb, d.t_v128, DI, 0)) return -1;
  if (fused) {
    // keys = norm4(keys + out_proj(attn)) in one pass over the image tokens (i2t_fused.cu)
    if (launch_i2t_prep(d.t_k128, d.t_v128, L.i2t.qb, P, T, d.kexp, d.vexp, d.sbias, st)) return -1;
    if (gemm(E, st, d.kexp, DI, L.i2t_qT, P * 64, DC, DI, nullptr, d.mq, DC, 0)) return -1;
    if (gemm(E, st, L.i2t.o, DI, d.vexp, DC, P * 64, DI, nullptr, d.vt, P * 64, 0)) return -1;
    I2tFusedArgs fa;
    fa.P = P; fa.T = T; fa.mode = shared ? 0 : 1;
    fa.a0 = shared ? d.src_pe_bf : keys;
    fa.a1 = shared ? d.src_bf : d.pos_bf;
    fa.mq = d.mq; fa.vt = d.vt; fa.sbias = d.sbias;
    fa.bias = L.i2t.ob; fa.gamma = L.n4g; fa.beta = L.n4b; fa.eps = 1e-5f;
    fa.out = keys;
    return launch_i2t_fused(fa, E.num_sms, st);
  }
  if (shared) {
    i2t_attn_kernel<<<dim3(NI / 64, P), 256, 0, st>>>(d.q0, DI, 0, d.t_k128, d.t_v128, T, NI, d.img_att);
  } else {
    i2t_attn_kernel<<<dim3(NI / 64, P), 256, 0, st>>>(d.img_kvq, DI, NI, d.t_k128, d.t_v128, T, NI, d.img_att);
  }
  LAUNCH_CHECK("i2t_attn");
  // LayerNorm fused into the out-projection GEMM epilogue (in place for own keys: every thread reads the residual of
  // exactly the row segment it later overwrites)
  if (shared) return gemm(E, st, d.img_att, DI, L.i2t.o, PN, DC, DI, L.i2t.ob, keys, DC, 0, 0, d.src_bf, NI, 1, 1, L.n4g, L.n4b, 1e-5f);
  return gemm(E, st, d.img_att, DI, L.i2t.o, PN, DC, DI, L.i2t.ob, keys, DC, 0, 0, keys, PN, 1, 1, L.n4g, L.n4b, 1e-5f);
}

// Output upscaling + hyper product: convT(256->64) -> LN2d(64) -> GELU -> convT(64->32) -> GELU, dotted with hyper_in
// [P, 4, 32]: one fused kernel (upscale_fused.cu); neither up-scaled embedding ever reaches HBM.
static int upscale_block(Engine& E, cudaStream_t st, int P, int multimask, const __nv_bfloat16* keys, const float* hyper,
                         float* low_res) {
  DecoderState& d = *E.dec;
  UpscaleFusedArgs ua;
  ua.P = P; ua.nm = multimask ? 3 : 1; ua.m0 = multimask ? 1 : 0; ua.keys = keys; ua.w1 = d.ct1; ua.w2_f16 = d.ct2_f16;
  ua.b1 = d.ct1b; ua.gamma = d.upln_g; ua.beta = d.upln_b; ua.eps = 1e-6f; ua.b2 = d.ct2b; ua.hyper = hyper; ua.out = low_res;
  return launch_upscale_fused(ua, E.num_sms, st);
}

// One chunk of P <= max_prompts prompts.
static int decode_chunk(Engine& E, cudaStream_t st, const float* points, const float* labels, int np, const float* boxes,
                        const float* mask_in, int P, int multimask, float* low_res, float* iou,
                        const float* sparse = nullptr, int n_sparse_given = 0, const float* dense = nullptr) {
  DecoderState& d = *E.dec;
  const int NI = 4096;
  const int n_sparse = sparse ? n_sparse_given : (points ? np + (boxes ? 0 : 1) : 0) + (boxes ? 2 : 0);
  const int T = 5 + n_sparse, PT = P * T;
  // Given embeddings with n_sparse = 0 and the no-mask dense embedding are what PromptEncoder returns for an empty prompt:
  // upstream decodes the 5 output tokens alone (T = 5, shared image-side operands), and so does this path.
  if (n_sparse <= 0 && !mask_in && !dense && n_sparse_given >= 0) return set_error("decode: need points, boxes and/or mask prompts");
  if (T > TMAX) return set_error("decode: %d tokens per prompt exceeds the supported %d", T, TMAX);

  if (sparse || n_sparse_given < 0) {  // given sparse embeddings (model-level mask_decoder call)
    tokens_from_sparse_kernel<<<dim3(T, P), 128, 0, st>>>(sparse, n_sparse, T, d.out_tokens, d.tok0, d.tok0_bf);
    LAUNCH_CHECK("tokens_from_sparse");
  } else {
    prompt_tokens_kernel<<<dim3(n_sparse > 0 ? n_sparse : 1, P), 128, 0, st>>>(points, labels, np, boxes, T, n_sparse, (float)E.cfg.image_size, d.gauss,
                                                            d.point_emb, d.not_a_point, d.out_tokens, d.tok0, d.tok0_bf);
    LAUNCH_CHECK("prompt_tokens");
  }

  // Mask prompts / given dense embeddings: the dense prompt embedding differs per prompt, so layer 0 cannot share its
  // image-side operands; the per-prompt keys are materialised up front and layer 0 runs exactly like layer 1 on the image side.
  if (mask_in) {
    mask_dense_kernel<<<dim3(NI / 16, P), 256, 0, st>>>(mask_in, d.md_w1, d.md_b1, d.md_g1, d.md_be1, d.md_w2, d.md_b2, d.md_g2,
                                                         d.md_be2, d.md_w3, d.md_b3, d.emb, d.keys, nullptr);
    LAUNCH_CHECK("mask_dense");
  } else if (dense) {
    dense_to_keys_kernel<<<dim3(NI / 32, DC / 32, P), dim3(32, 8), 0, st>>>(dense, d.emb, d.keys);
    LAUNCH_CHECK("dense_to_keys");
  }
  const bool own_keys = mask_in || dense;

  for (int l = 0; l < 2; ++l) {
    const DecLayer& L = d.layers[l];
    const bool shared = (l == 0) && !own_keys;  // image-side operands identical for every prompt
    // ---- (1) token self attention
    if (l == 0) {
      if (gemm(E, st, d.tok0_bf, DC, L.self_attn.qkv, PT, 3 * DC, DC, L.self_attn.qkvb, d.t_qkv, 3 * DC, 0)) return -1;
      token_self_attn_kernel<<<(P * NHEAD + 3) / 4, 128, 0, st>>>(d.t_qkv, 3 * DC, d.t_qkv + DC, 3 * DC, d.t_qkv + 2 * DC,
                                                                    3 * DC, P, T, d.t_att);
      LAUNCH_CHECK("token_self_attn");
      // skip_first_layer_pe: the attention output REPLACES the tokens (no residual)
      if (gemm(E, st, d.t_att, DC, L.self_attn.o, PT, DC, DC, L.self_attn.ob, d.tok_f32, DC, 1)) return -1;
    } else {
      if (gemm(E, st, d.qpe_bf, DC, L.self_attn.qk, PT, 2 * DC, DC, L.self_attn.qkb, d.t_qkv, 2 * DC, 0)) return -1;
      if (gemm(E, st, d.q_bf, DC, L.self_attn.v, PT, DC, DC, L.self_attn.vb, d.t_mlp, DC, 0)) return -1;
      token_self_attn_kernel<<<(P * NHEAD + 3) / 4, 128, 0, st>>>(d.t_qkv, 2 * DC, d.t_qkv + DC, 2 * DC, d.t_mlp, DC, P, T,
                                                                    d.t_att);
      LAUNCH_CHECK("token_self_attn");
      if (gemm(E, st, d.t_att, DC, L.self_attn.o, PT, DC, DC, L.self_attn.ob, d.tok_f32, DC, 1, 0, d.queries, PT)) return -1;
    }
    if (ln(st, d.tok_f32, PT, DC, L.n1g, L.n1b, 1e-5f, d.q_bf, d.queries, d.tok0, PT, d.qpe_bf)) return -1;
    // ---- (2) token -> image cross attention
    if (t2i_block(E, st, L.t2i, P, T, d.qpe_bf, shared ? nullptr : d.keys, d.t_att128)) return -1;
    if (gemm(E, st, d.t_att128, DI, L.t2i.o, PT, DC, DI, L.t2i.ob, d.tok_f32, DC, 1, 0, d.queries, PT)) return -1;
    if (ln(st, d.tok_f32, PT, DC, L.n2g, L.n2b, 1e-5f, d.q_bf, d.queries)) return -1;
    // ---- (3) MLP (ReLU)
    if (gemm(E, st, d.q_bf, DC, L.mlp1, PT, 2048, DC, L.mlp1b, d.t_mlp, 2048, 0, 2)) return -1;
    if (gemm(E, st, d.t_mlp, 2048, L.mlp2, PT, DC, 2048, L.mlp2b, d.tok_f32, DC, 1, 0, d.queries, PT)) return -1;
    if (ln(st, d.tok_f32, PT, DC, L.n3g, L.n3b, 1e-5f, d.q_bf, d.queries, d.tok0, PT, d.qpe_bf)) return -1;
    // ---- (4) image -> token cross attention (updates all image tokens of every prompt)
    if (i2t_block(E, st, l, P, T, d.q_bf, d.qpe_bf, shared, d.keys)) return -1;
  }
  // ---- final token -> image attention
  {
    const AttnW& A = d.final_t2i;
    if (t2i_block(E, st, A, P, T, d.qpe_bf, d.keys, d.t_att128)) return -1;
    if (gemm(E, st, d.t_att128, DI, A.o, PT, DC, DI, A.ob, d.tok_f32, DC, 1, 0, d.queries, PT)) return -1;
    if (ln(st, d.tok_f32, PT, DC, d.nfg, d.nfb, 1e-5f, d.q_bf)) return -1;
  }
  // ---- heads: IoU MLP on token 0, hyper-network MLPs on tokens 1..4 (rows p*T + i, lda = T*256)
  {
    const Mlp3& m = d.iou_head;
    if (gemm(E, st, d.q_bf, T * DC, m.w[0], P, DC, DC, m.b[0], d.h1, DC, 0, 2)) return -1;
    if (gemm(E, st, d.h1, DC, m.w[1], P, DC, DC, m.b[1], d.h2, DC, 0, 2)) return -1;
    if (gemm(E, st, d.h2, DC, m.w[2], P, 32, DC, m.b[2], d.iou_out, 32, 1)) return -1;
    for (int i = 0; i < 4; ++i) {
      const Mlp3& hm = d.hyper[i];
      if (gemm(E, st, d.q_bf + (1 + i) * DC, T * DC, hm.w[0], P, DC, DC, hm.b[0], d.h1, DC, 0, 2)) return -1;
      if (gemm(E, st, d.h1, DC, hm.w[1], P, DC, DC, hm.b[1], d.h2, DC, 0, 2)) return -1;
      if (gemm(E, st, d.h2, DC, hm.w[2], P, 32, DC, hm.b[2], d.hyper_in + i * 32, 128, 1)) return -1;
    }
  }
  // ---- output upscaling + hyper product
  const int m0 = multimask ? 1 : 0, nm = multimask ? 3 : 1;
  if (upscale_block(E, st, P, multimask, d.keys, d.hyper_in, low_res)) return -1;
  gather_iou_kernel<<<(P * nm + 127) / 128, 128, 0, st>>>(d.iou_out, P, m0, nm, iou);
  LAUNCH_CHECK("gather_iou");
  return 0;
}

int Engine::decode(const float* points, const float* labels, int np, const float* boxes, const float* mask_in, int P,
                   int multimask, float* low_res, float* iou, cudaStream_t st) {
  if (!finalized || !dec) return set_error("decode: decoder weights not loaded");
  if (!dec->image_set) return set_error("decode: no image embedding set (call msam_set_image_embedding first)");
  if (P <= 0) return set_error("decode: empty prompt batch");
  const int nm = multimask ? 3 : 1;
  for (int p0 = 0; p0 < P; p0 += cfg.max_prompts) {
    const int n = (P - p0 < cfg.max_prompts) ? (P - p0) : cfg.max_prompts;
    if (decode_chunk(*this, st, points ? points + (size_t)p0 * np * 2 : nullptr, labels ? labels + (size_t)p0 * np : nullptr,
                     np, boxes ? boxes + (size_t)p0 * 4 : nullptr, mask_in ? mask_in + (size_t)p0 * 65536 : nullptr, n, multimask,
                     low_res + (size_t)p0 * nm * 65536,
                     iou + (size_t)p0 * nm))
      return -1;
  }
  return 0;
}

// PromptEncoder.forward as a stand-alone call: sparse [P, n_sparse, 256] (points incl. the padding point when no box is
// given, then the two box corners) and, for mask prompts, the dense embedding [P, 256, 64, 64] (NCHW fp32).
const float* Engine::dec_pos() { return dec ? dec->pos : nullptr; }
int Engine::dec_set_prompt_tables(const float* point_emb, const float* not_a_point, cudaStream_t st) {
  if (!dec) return set_error("decoder weights not loaded");
  if ((point_emb && cudaMemcpyAsync(dec->point_emb, point_emb, 4 * 256 * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) ||
      (not_a_point && cudaMemcpyAsync(dec->not_a_point, not_a_point, 256 * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess))
    return set_error("prompt tables: copy failed");
  return 0;
}

int Engine::prompt_encode(const float* points, const float* labels, int np, const float* boxes, const float* mask_in, int P,
                          float* sparse_out, float* dense_out, cudaStream_t st) {
  if (!finalized || !dec) return set_error("prompt_encode: decoder weights not loaded");
  DecoderState& d = *dec;
  const int n_sparse = (points ? np + (boxes ? 0 : 1) : 0) + (boxes ? 2 : 0), T = 5 + n_sparse;
  // The encoder itself has no token limit: prompts with more than TMAX tokens (the limit of the inference decoder; the training
  // decoder takes up to TMAX_TRAIN) are encoded in chunks of fewer prompts so that chunk * T tokens fit the max_prompts * TMAX
  // token workspace.
  if (T > TMAX_TRAIN || T > cfg.max_prompts * TMAX)
    return set_error("prompt_encode: %d tokens per prompt exceeds the supported %d", T, std::min(TMAX_TRAIN, cfg.max_prompts * TMAX));
  const int chunk = T <= TMAX ? cfg.max_prompts : cfg.max_prompts * TMAX / T;
  for (int p0 = 0; p0 < P; p0 += chunk) {
    const int n = (P - p0 < chunk) ? (P - p0) : chunk;
    if (n_sparse > 0) {
      if (!sparse_out) return set_error("prompt_encode: sparse_out is null");
      prompt_tokens_kernel<<<dim3(n_sparse, n), 128, 0, st>>>(points ? points + (size_t)p0 * np * 2 : nullptr,
                                                             labels ? labels + (size_t)p0 * np : nullptr, np,
                                                             boxes ? boxes + (size_t)p0 * 4 : nullptr, T, n_sparse,
                                                             (float)cfg.image_size, d.gauss, d.point_emb, d.not_a_point,
                                                             d.out_tokens, d.tok0, d.tok0_bf);
      LAUNCH_CHECK("prompt_tokens");
      if (cudaMemcpy2DAsync(sparse_out + (size_t)p0 * n_sparse * 256, (size_t)n_sparse * 1024, d.tok0 + 5 * 256, (size_t)T * 1024,
                            (size_t)n_sparse * 1024, n, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return set_error("prompt_encode: copy failed");
    }
    if (mask_in) {
      if (!dense_out) return set_error("prompt_encode: dense_out is null");
      mask_dense_kernel<<<dim3(4096 / 16, n), 256, 0, st>>>(mask_in + (size_t)p0 * 65536, d.md_w1, d.md_b1, d.md_g1, d.md_be1,
                                                           d.md_w2, d.md_b2, d.md_g2, d.md_be2, d.md_w3, d.md_b3, d.emb, nullptr,
                                                           dense_out + (size_t)p0 * 256 * 4096);
      LAUNCH_CHECK("mask_dense");
    }
  }
  return 0;
}

// MaskDecoder.forward on given prompt embeddings (training/trainable_sam.py:88-106): sparse [P, n_sparse, 256]; dense
// [P, 256, 64, 64] or NULL = the no-mask embedding (shared fast path).  The image embedding must have been bound.
int Engine::mask_decode(const float* sparse, int n_sparse, const float* dense, int P, int multimask, float* low_res,
                        float* iou, cudaStream_t st) {
  if (!finalized || !dec) return set_error("mask_decode: decoder weights not loaded");
  if (!dec->image_set) return set_error("mask_decode: no image embedding set");
  if (P <= 0) return set_error("mask_decode: empty prompt batch");
  if (n_sparse < 0 || (n_sparse > 0 && !sparse)) return set_error("mask_decode: bad sparse embeddings");
  const int nm = multimask ? 3 : 1;
  for (int p0 = 0; p0 < P; p0 += cfg.max_prompts) {
    const int n = (P - p0 < cfg.max_prompts) ? (P - p0) : cfg.max_prompts;
    if (decode_chunk(*this, st, nullptr, nullptr, 0, nullptr, nullptr, n, multimask, low_res + (size_t)p0 * nm * 65536,
                     iou + (size_t)p0 * nm, n_sparse > 0 ? sparse + (size_t)p0 * n_sparse * 256 : nullptr,
                     n_sparse > 0 ? n_sparse : -1, dense ? dense + (size_t)p0 * 256 * 4096 : nullptr))
      return -1;
  }
  return 0;
}

// ---- op-level entry points of the three blocks (msam_op_dec_*): the functions decode_chunk calls, on explicit inputs.
// The persistent kernels split their work items over min(items, num_sms) CTAs; num_sms > 0 overrides the device's count for
// this call so that tests can vary the launch geometry.
namespace {
struct SmsOverride {
  Engine& E;
  int saved;
  SmsOverride(Engine& e, int n) : E(e), saved(e.num_sms) { if (n > 0) e.num_sms = n; }
  ~SmsOverride() { E.num_sms = saved; }
};
}  // namespace

static int check_block(Engine& E, const char* name, int P, int T, int num_sms) {
  if (!E.finalized || !E.dec) return set_error("%s: decoder weights not loaded", name);
  if (P < 1 || P > E.cfg.max_prompts) return set_error("%s: P = %d outside [1, max_prompts = %d]", name, P, E.cfg.max_prompts);
  if (T < 5 || T > TMAX) return set_error("%s: T = %d tokens per prompt outside [5, %d]", name, T, TMAX);
  if (num_sms < 0) return set_error("%s: num_sms = %d < 0", name, num_sms);
  return 0;
}

int Engine::op_dec_t2i(int which, const __nv_bfloat16* qpe, const __nv_bfloat16* keys, int P, int T, __nv_bfloat16* out,
                       int sms, cudaStream_t st) {
  if (check_block(*this, "op_dec_t2i", P, T, sms)) return -1;
  if (!qpe || !out) return set_error("op_dec_t2i: null argument");
  if (which < 0 || which > 2) return set_error("op_dec_t2i: attention instance %d (0, 1 = layers, 2 = final)", which);
  if (!keys && !dec->image_set) return set_error("op_dec_t2i: the shared mode needs a bound image embedding");
  SmsOverride o(*this, sms);
  return t2i_block(*this, st, which == 2 ? dec->final_t2i : dec->layers[which].t2i, P, T, qpe, keys, out);
}

int Engine::op_dec_i2t(int layer, const __nv_bfloat16* q, const __nv_bfloat16* qpe, int shared, __nv_bfloat16* keys, int P,
                       int T, int sms, cudaStream_t st) {
  if (check_block(*this, "op_dec_i2t", P, T, sms)) return -1;
  if (!q || !qpe || !keys) return set_error("op_dec_i2t: null argument");
  if (layer < 0 || layer > 1) return set_error("op_dec_i2t: layer %d (0 or 1)", layer);
  if (shared && (layer != 0 || !dec->image_set)) return set_error("op_dec_i2t: the shared mode is layer 0 on a bound image");
  SmsOverride o(*this, sms);
  return i2t_block(*this, st, layer, P, T, q, qpe, shared != 0, keys);
}

int Engine::op_dec_upscale(const __nv_bfloat16* keys, const float* hyper, int P, int multimask, float* low_res, int sms,
                           cudaStream_t st) {
  if (check_block(*this, "op_dec_upscale", P, 5, sms)) return -1;
  if (!keys || !hyper || !low_res) return set_error("op_dec_upscale: null argument");
  SmsOverride o(*this, sms);
  return upscale_block(*this, st, P, multimask, keys, hyper, low_res);
}

int Engine::dense_pe(float* out_tokmajor, cudaStream_t st) {
  if (!finalized || !dec) return set_error("dense_pe: decoder weights not loaded");
  if (cudaMemcpyAsync(out_tokmajor, dec->pos, (size_t)4096 * 256 * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return set_error("dense_pe: copy failed");
  return 0;
}

}  // namespace msam
