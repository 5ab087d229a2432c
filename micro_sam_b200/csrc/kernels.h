// Internal kernel launch interface (host side).  All pointers are device pointers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

namespace msam {

// Launch with programmatic dependent launch allowed (see ptx.cuh:pdl_wait).  ONLY for kernels in which every thread executes
// pdl_wait() before touching global memory.  The attribute is only set when MSAM_PDL=1 (see engine.cu).
bool pdl_enabled();   // engine.cu
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

int set_error(const char* fmt, ...);  // records msam_last_error(); returns -1
// After a launch: records "<name> launch failed: ..." and returns -1 if it failed, else counts it (msam_launch_count), returns 0
int launch_check(const char* name);
#define LAUNCH_CHECK(name) do { if (launch_check(name)) return -1; } while (0)

// Optional per-kernel timing (bench.py roofline / per-stage table): CUDA events recorded on the launching stream around a
// launch, aggregated by `name` (a string literal) in msam_profile_report; flops / bytes = ALGORITHMIC work of the launch.
void prof_begin(cudaStream_t st, const char* name, double flops, double bytes);
void prof_end(cudaStream_t st);

// Launch arithmetic: blocks of `per` threads covering n items; 16-byte alignment of a vectorised operand; workspace slices
// rounded up to 256 bytes
inline unsigned nblk(long n, int per = 256) { return (unsigned)((n + per - 1) / per); }
inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }
inline size_t up256(size_t b) { return (b + 255) & ~size_t(255); }

// ---- gemm.cu :  out[M,N] = act(A[M,K] * W[N,K]^T + bias) (+ residual[row % res_rows])
struct GemmArgs {
  const __nv_bfloat16* A = nullptr;  // [M, lda]
  const __nv_bfloat16* W = nullptr;  // [N, ldw]
  int M = 0, N = 0, K = 0, lda = 0, ldw = 0;
  const float* bias = nullptr;
  const void* residual = nullptr;   // fp32, or bf16 when res_bf16
  int res_rows = 0, ldr = 0, res_bf16 = 0;
  void* out = nullptr;
  int ldc = 0;
  int out_fp32 = 0;
  int act = 0;  // 0 none, 1 GELU(erf), 2 ReLU
  int act_after_res = 0;  // apply `act` after the residual add (MBConv: act3(conv3(x) + shortcut)); bf16 / strided-residual path only
  // fused row epilogue (gemm.cu): 0 plain, 1 LayerNorm over N=256
  int epi = 0;
  const float* ln_gamma = nullptr;
  const float* ln_beta = nullptr;
  float ln_eps = 1e-5f;
  int path = 0;  // GEMM_PATH_*: which kernel runs a plain-epilogue product
};
enum {
  GEMM_PATH_AUTO = 0,   // the wide-tile kernel when N % 256 == 0 and the product has a 128 x 256 tile for every SM, else the tiled one
  GEMM_PATH_TILED = 1,  // gemm_bf16_kernel<BN, EPI> (BN = 256 / 128 / 64)
  GEMM_PATH_WIDE = 2,   // gemm_wide_kernel (needs N % 256 == 0 and the plain epilogue)
};
int launch_gemm(const GemmArgs& a, int num_sms, cudaStream_t stream);

// ---- gemm_tn.cu : out[M,N] fp32 = A[K,M]^T B[K,N]  (weight gradient dW = dY^T X; both operands MN-major)
int launch_gemm_tn(const __nv_bfloat16* A, const __nv_bfloat16* B, int M, int N, int K, int lda, int ldb, float* out, int ldc,
                   cudaStream_t stream, int accumulate = 0);
// out[M,N] fp32 = A[M,K] B[K,N]  (input gradient dX = dY W; A K-major, B = the forward weight [out, in] consumed MN-major)
int launch_gemm_nn(const __nv_bfloat16* A, const __nv_bfloat16* B, int M, int N, int K, int lda, int ldb, float* out, int ldc,
                   cudaStream_t stream);

// ---- bgemm.cu : batched GEMM over (outer = window | image, head) pairs, fp32 out: C[w,h] (+)= alpha * op(A[w,h]) op(B[w,h])
struct BGemmArgs {
  const __nv_bfloat16* A = nullptr;
  const __nv_bfloat16* B = nullptr;
  int a_mn = 0, b_mn = 0;       // 0: K-major (contraction along the contiguous features), 1: MN-major (contraction along the rows)
  int M = 0, N = 0, K = 0;
  int lda = 0, ldb = 0;         // row pitch of A / B (elements)
  long a_hstride = 0, a_wstride = 0, b_hstride = 0, b_wstride = 0;   // element offsets per head / per outer index; 0 = shared
  int heads = 1, outer = 1;
  float* out = nullptr;         // [outer, heads, M, ldc] through o_wstride / o_hstride
  int ldc = 0;
  long o_hstride = 0, o_wstride = 0;
  float alpha = 1.f;
  int accumulate = 0;
  int a_rows_valid = 0, b_rows_valid = 0;   // row extent of an operand if smaller than its tile extent (rows beyond are read as zeros)
};
int launch_bgemm(const BGemmArgs& a, cudaStream_t stream);

// ---- backward.cu : HBM-bound pieces of the encoder backward pass (cfg 5)
// LayerNorm backward over rows: dx (+)= d LN(x) ; dgamma / dbeta += (atomics into zero-initialised fp32 [D]).
// window_mode: dy is indexed in the window-partitioned row order of the forward LayerNorm (pad rows are skipped).
int launch_layernorm_bwd(const float* x, int rows, int D, const float* gamma, float eps, const float* dy, int window_mode, int grid,
                         int ws, int accumulate, float* dx, float* dgamma, float* dbeta, cudaStream_t stream);
int launch_gelu_fwd(const __nv_bfloat16* pre, long n, __nv_bfloat16* out, cudaStream_t stream);
int launch_gelu_bwd(const __nv_bfloat16* dh, const __nv_bfloat16* pre, long n, __nv_bfloat16* dpre, cudaStream_t stream);
int launch_colsum(const __nv_bfloat16* x, long rows, int N, float* out, cudaStream_t stream);   // out[N] += column sums
int launch_window_gather(const __nv_bfloat16* x, int B, int grid, int ws, int D, __nv_bfloat16* out_win, cudaStream_t stream);
struct AttnBwdGeom { int side = 14, n_tok = 196, nt = 64, woff = 32; };   // window: 14 / 196 / 64 / 32; global: 64 / 4096 / 256 / 128
// Packed rel-pos table of one encoder block, bf16 [nt, rel_table_cols(head_dim)]: rows [0, 2 side - 1) = rel_pos_h, rows
// [woff, woff + 2 side - 1) = rel_pos_w, zero elsewhere.  The attention kernels (forward and backward) read this layout.
inline AttnBwdGeom rel_table_geom(bool global, int window, int grid) {
  AttnBwdGeom g;
  g.side = global ? grid : window;
  g.n_tok = g.side * g.side;
  g.nt = global ? 256 : 64;
  g.woff = global ? 128 : 32;
  return g;
}
inline int rel_table_cols(int head_dim) { return ((head_dim + 63) / 64) * 64; }
int launch_attn_probs(const float* S, const float* T, long n_batch, AttnBwdGeom g, int pitch_s, int pitch_p, float scale,
                      __nv_bfloat16* P, cudaStream_t stream);
int launch_attn_ds(const __nv_bfloat16* P, const float* dP, long n_batch, AttnBwdGeom g, int pitch_s, int pitch_p,
                   __nv_bfloat16* dS, __nv_bfloat16* dT, cudaStream_t stream);
int launch_pack_dqkv(const float* dq, const float* dk, const float* dv, int outer, int heads, int T, int d, __nv_bfloat16* dqkv,
                     cudaStream_t stream);
int launch_sum_batch(const float* x, long n_batch, long n, float* out, int accumulate, cudaStream_t stream);   // out[n] (+)= sum_b x[b, n]
int launch_nchw_to_tok(const float* nchw, int B, int C, int T, float* tok, cudaStream_t stream);
int launch_col2im3x3(const __nv_bfloat16* dcol, int B, int g, int C, float* out, cudaStream_t stream);
int launch_cast_f32(const __nv_bfloat16* x, long n, float* out, cudaStream_t stream);
// out [cols, rows] = in [rows, cols]^T (the W^T operands of the dgrad GEMMs)
int launch_transpose_bf16(const __nv_bfloat16* in, int rows, int cols, __nv_bfloat16* out, cudaStream_t stream);

// ---- upscale_fused.cu : conv-transpose 1 + LayerNorm2d + GELU + conv-transpose 2 + GELU + hyper-network product in one pass
struct UpscaleFusedArgs {
  int P = 0, nm = 3, m0 = 1;          // prompts; masks written per prompt = hyper rows [m0, m0 + nm)
  const __nv_bfloat16* keys = nullptr;  // [P*4096, 256] image tokens after the transformer
  const __nv_bfloat16* w1 = nullptr;    // conv-transpose-1 weight as GEMM operand [(sub-pixel, out-ch) = 256, 256]
  const void* w2_f16 = nullptr;         // conv-transpose-2 weight, fp16 [(sub-sub-pixel, out-ch) = 128, 64]
  const float* b1 = nullptr;            // [256]
  const float* gamma = nullptr;         // LayerNorm2d(64)
  const float* beta = nullptr;
  float eps = 1e-6f;
  const float* b2 = nullptr;            // [128]
  const float* hyper = nullptr;         // [P, 4, 32]
  float* out = nullptr;                 // [P, nm, 256, 256] low-res mask logits
};
int launch_upscale_fused(const UpscaleFusedArgs& a, int num_sms, cudaStream_t stream);

// ---- i2t_fused.cu : fused image -> token cross-attention block (q projection + attention + out projection + residual +
// LayerNorm in one pass over the per-prompt image tokens); T <= 8 prompt tokens
struct I2tFusedArgs {
  int P = 0, T = 0;
  int mode = 0;                       // 0: layer 0 (a0 = src + pe, a1 = src, shared by all prompts); 1: a0 = keys [P*4096,256], a1 = pe
  const __nv_bfloat16* a0 = nullptr;
  const __nv_bfloat16* a1 = nullptr;
  const __nv_bfloat16* mq = nullptr;  // [P*64, 256]
  const __nv_bfloat16* vt = nullptr;  // [256, P*64]
  const float* sbias = nullptr;       // [P*64]
  const float* bias = nullptr;        // out-proj bias [256]
  const float* gamma = nullptr;
  const float* beta = nullptr;
  float eps = 1e-5f;
  __nv_bfloat16* out = nullptr;       // keys [P*4096, 256] (may alias a0)
};
int launch_i2t_fused(const I2tFusedArgs& a, int num_sms, cudaStream_t stream);
int launch_i2t_prep(const __nv_bfloat16* ktok, const __nv_bfloat16* vtok, const float* bq, int P, int T,
                    __nv_bfloat16* kexp, __nv_bfloat16* vexp, float* sbias, cudaStream_t stream);

// ---- t2i_fused.cu : fused token -> image cross-attention (k / v projections folded into the query / output side; the image
// tokens are read once and used as both K and V)
struct T2iFusedArgs {
  int P = 0;                          // prompts
  int paired = 0;                     // 128-row items of Q' / out: 1 = two prompts (pl*64 + h*8 + t, T <= 8), 0 = one (h*16 + t)
  int mode = 0;                       // 1: x = keys [P*4096, 256], xs = pe;  0: x = src (shared), xs = src + pe
  const __nv_bfloat16* x = nullptr;
  const __nv_bfloat16* xs = nullptr;
  const __nv_bfloat16* qp = nullptr;  // Q' [items*128, 256]
  float* out = nullptr;               // [items*128, 256]
};
int launch_t2i_fused(const T2iFusedArgs& a, int num_sms, cudaStream_t stream);
int launch_t2i_prep(const __nv_bfloat16* q, int P, int T, int paired, int n_items, __nv_bfloat16* qexp, cudaStream_t stream);
int launch_t2i_head_proj(const float* U, const __nv_bfloat16* WvT, const float* bv, int P, int T, int paired,
                         __nv_bfloat16* out, cudaStream_t stream);

// ---- attention.cu : ViT encoder attention with decomposed relative-position bias
struct AttnArgs {
  const __nv_bfloat16* qkv = nullptr;  // [groups*G, 3*D] rows = tokens (window-partitioned incl. pad tokens, or global)
  const __nv_bfloat16* rel_table = nullptr;  // [NT, hd_pad] : rows [0,2S-1) rel_pos_h, rows [S_off, S_off+2S-1) rel_pos_w
  __nv_bfloat16* out = nullptr;        // [B*grid*grid, D] in image token order
  int batch = 0;      // images
  int heads = 0;
  int head_dim = 0;   // 64 or 80
  int grid = 0;       // tokens per image side (64)
  int window = 0;     // 0 = global attention, else window size (14)
  float scale = 0.f;
};
int launch_attention(const AttnArgs& a, cudaStream_t stream);
int launch_attention_global(const AttnArgs& a, cudaStream_t stream);  // attention_global.cu (window == 0)
int launch_attn_window2(const AttnArgs& a, cudaStream_t stream);      // attention_win2.cu (window 14, head_dim 64 / 80)
// debug: per-CTA phase timestamps (%globaltimer, 16 slots x 64 windows) of the window-attention kernels; nullptr = off
void set_attn_trace(unsigned long long* dev_buf);
unsigned long long* get_attn_trace();

// ---- elementwise.cu
int launch_patchify(const uint8_t* u8, const float* f32, int B, int h, int w, int img, const float* mean,
                    const float* stdv, __nv_bfloat16* out, cudaStream_t stream);
struct LnArgs {
  const float* x = nullptr;  // [rows, D] fp32
  int rows = 0, D = 0;
  const float* gamma = nullptr;
  const float* beta = nullptr;
  float eps = 1e-6f;
  __nv_bfloat16* out = nullptr;  // bf16 [rows(or window-partitioned rows), D] (optional)
  float* out_f32 = nullptr;      // fp32 copy of the normalised rows (optional)
  int window_mode = 0, grid = 64, ws = 14;
  int act = 0;                   // 1: exact GELU after the affine
  const float* add = nullptr;    // [add_rows, D] fp32 added after the affine for out2 (optional)
  int add_rows = 1;
  __nv_bfloat16* out2 = nullptr;
};
int launch_layernorm(const LnArgs& a, cudaStream_t stream);
int launch_layernorm2d_nchw(const float* x, int B, int T, const float* gamma, const float* beta, float eps, float* out,
                            cudaStream_t stream);
int launch_cast_bf16(const float* x, long n, __nv_bfloat16* out, cudaStream_t stream);
int launch_im2col3x3(const __nv_bfloat16* x, int B, int g, int C, __nv_bfloat16* out, cudaStream_t stream);

// ---- tinyvit.cu : the CUDA-core kernels of the TinyViT (vit_t) encoder.  No argument checks here (the msam_op_tv_* entry
// points of engine.cu make them); each helper is the launch Engine::encode_tinyvit makes.
// Stem conv 1: Sam.preprocess of uint8 HWC [B, h, w, 3] (or preprocessed fp32 NCHW [B, 3, img, img] when f32 is set) + conv3x3/2
// (w [27][32], tap-major (ky*3+kx)*3 + c) + folded BN + GELU -> bf16 NHWC [B, img/2, img/2, 32].
int launch_tv_stem1(const uint8_t* u8, const float* f32, int B, int h, int w, int img, const float* wt, const float* bias,
                    __nv_bfloat16* out, cudaStream_t stream);
// im2col of a 3x3 / pad 1 conv with stride on bf16 NHWC [B, Hin, Hin, C] -> [B * Ho * Ho, 9 * C], Ho = Hin / stride.
int launch_tv_im2col(const __nv_bfloat16* x, int B, int Hin, int C, int stride, __nv_bfloat16* out, cudaStream_t stream);
// Depth-wise conv3x3 pad 1 + folded BN (w [9][C], b [C]) (+ GELU when act) on NHWC: bf16 with stride 1 / 2, fp32 with stride 1.
int launch_tv_dwconv_bf16(const __nv_bfloat16* x, int B, int Hin, int C, int stride, const float* w, const float* b, int act,
                          __nv_bfloat16* out, cudaStream_t stream);
int launch_tv_dwconv_f32(const float* x, int B, int Hin, int C, const float* w, const float* b, float* out, cudaStream_t stream);
// LayerNorm of fp32 [B, H, H, D] scattered into the window-partitioned bf16 rows of ws x ws windows; pad rows = bf16(beta).
int launch_tv_ln_window(const float* x, int B, int H, int D, int ws, const float* gamma, const float* beta, float eps,
                        __nv_bfloat16* out, cudaStream_t stream);
// Window attention (head_dim 32, scale 32^-0.5, bias_tab [heads][ws*ws] indexed by |dy|*ws + |dx|) on window-partitioned qkv
// [windows * ws*ws, heads * 96] -> bf16 [B*H*H, heads * 32] in image token order.  ws = 7 or 14.
int launch_tv_attention(const __nv_bfloat16* qkv, const float* bias_tab, int B, int H, int ws, int heads, __nv_bfloat16* out,
                        cudaStream_t stream);

}  // namespace msam
