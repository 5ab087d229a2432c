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
void count_launch();                  // per-thread launch counter (msam_launch_count)

// Optional per-kernel timing (bench.py roofline / per-stage table): CUDA events recorded on the launching stream around a
// launch, aggregated by `name` (a string literal) in msam_profile_report; flops / bytes = ALGORITHMIC work of the launch.
void prof_begin(cudaStream_t st, const char* name, double flops, double bytes);
void prof_end(cudaStream_t st);

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
  int n_items = 0;                    // work items of `rows` Q' rows
  int rows = 128;                     // 128: one prompt (h*16 + t) or two prompts (pl*64 + h*8 + t); 64: one prompt, T <= 8
  int mode = 0;                       // 1: x = keys [n_items*4096, 256], xs = pe;  0: x = src (shared), xs = src + pe
  const __nv_bfloat16* x = nullptr;
  const __nv_bfloat16* xs = nullptr;
  const __nv_bfloat16* qp = nullptr;  // Q' [n_items*128, 256]
  float* out = nullptr;               // [n_items*128, 256]
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

}  // namespace msam
