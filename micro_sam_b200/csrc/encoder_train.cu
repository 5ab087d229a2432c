// ViT image encoder, training mode (BASELINE.json configs[4] "vit_b fine-tuning step: encoder fwd/bwd"): a forward pass that keeps
// what the backward pass needs, and the backward pass itself.  Reference: torch autograd over ImageEncoderViT (oracle/sam_ref.py)
// as driven by micro_sam/training/sam_trainer.py:393 (loss.backward()); gradients are checked tensor by tensor against it in
// tests/test_gpu_backward.py.
//
// Saved per block (bf16 unless noted): x_in (fp32), qkv, attention output, x_mid (fp32), fc1 pre-activation.  LayerNorm outputs and
// GELU(fc1) are recomputed (HBM-bound, cheaper than keeping them).  Per block, in reverse:
//   MLP    dW2 = dy^T h | dh = dy W2 | dpre = dh o gelu'(pre) | dW1 = dpre^T LN2(x_mid) | dxn = dpre W1 | dx += LN2'(dxn)
//   attn   dWp = dy^T a | da = dy Wp | (dq, dk, dv, drel) = attention'(qkv, da) | dWqkv = dqkv^T LN1(x_in) | dxn = dqkv Wqkv | dx += LN1'(dxn)
// dgrad products use the forward wgmma GEMMs on weights transposed once per weight update (W^T as the K-major operand: the
// GEMM of gemm.cu and its epilogues apply), wgrad products the MN-major GEMM of gemm_tn.cu, the five attention products the batched
// GEMM of bgemm.cu (one launch per product for all windows / images and heads), with S / P / dS materialised in HBM per block
// (window blocks: 0.1 GB, global blocks: 0.07 GB per image and head).  Gradients are fp32, operands bf16.
#include "engine.h"

#include <algorithm>
#include <cmath>

namespace msam {

#define CHK(p) do { if (!(p)) return -1; } while (0)
#define RUN(x) do { if (x) return -1; } while (0)

namespace {

__global__ void transpose_bf16_kernel(const __nv_bfloat16* __restrict__ in, int rows, int cols, __nv_bfloat16* __restrict__ out) {
  __shared__ __nv_bfloat16 tile[32][34];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    if (r0 + i < rows && c0 + threadIdx.x < cols) tile[i][threadIdx.x] = in[(long)(r0 + i) * cols + c0 + threadIdx.x];
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y)
    if (c0 + i < cols && r0 + threadIdx.x < rows) out[(long)(c0 + i) * rows + r0 + threadIdx.x] = tile[threadIdx.x][i];
}

int transpose_bf16(const __nv_bfloat16* in, int rows, int cols, __nv_bfloat16* out, cudaStream_t st) {
  transpose_bf16_kernel<<<dim3((cols + 31) / 32, (rows + 31) / 32), dim3(32, 8), 0, st>>>(in, rows, cols, out);
  if (cudaGetLastError() != cudaSuccess) return set_error("transpose launch failed");
  count_launch();
  return 0;
}

// [o][k][c] (GEMM operand of the 3x3 neck conv) gradient -> upstream [o][c][k]
__global__ void neck2_grad_relayout_kernel(const float* __restrict__ g, int C, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)C * C * 9) return;
  const int c = i % C, k = (i / C) % 9, o = i / (9 * C);
  out[((long)o * C + c) * 9 + k] = g[i];
}

}  // namespace

struct TrainSave {
  float *x_in = nullptr, *x_mid = nullptr;
  __nv_bfloat16 *qkv = nullptr, *attn = nullptr, *pre = nullptr;
  __nv_bfloat16 *qkv_wT = nullptr, *proj_wT = nullptr, *fc1_wT = nullptr, *fc2_wT = nullptr;
  float *g_ln1_g = nullptr, *g_ln1_b = nullptr, *g_ln2_g = nullptr, *g_ln2_b = nullptr, *g_qkv_w = nullptr, *g_qkv_b = nullptr,
        *g_proj_w = nullptr, *g_proj_b = nullptr, *g_fc1_w = nullptr, *g_fc1_b = nullptr, *g_fc2_w = nullptr, *g_fc2_b = nullptr,
        *g_rel_h = nullptr, *g_rel_w = nullptr;
};

struct TrainState {
  int B = 0;                 // batch of the saved forward pass (0 = none)
  bool transposed = false;
  std::vector<TrainSave> blk;
  __nv_bfloat16 *neck1_wT = nullptr, *neck2_wT = nullptr;
  float *g_patch_w = nullptr, *g_patch_b = nullptr, *g_pos = nullptr, *g_neck1_w = nullptr, *g_neck_ln1_g = nullptr, *g_neck_ln1_b = nullptr,
        *g_neck2_w = nullptr, *g_neck2_w_up = nullptr, *g_neck_ln2_g = nullptr, *g_neck_ln2_b = nullptr;
  // scratch
  float *dx = nullptr, *dxn = nullptr, *dtok = nullptr;
  __nv_bfloat16 *gb = nullptr, *hid = nullptr, *dhid = nullptr, *xn = nullptr, *xn_win = nullptr, *dqkv = nullptr, *do_win = nullptr,
                *dcol = nullptr;
  float *S = nullptr, *T = nullptr, *dq = nullptr, *dk = nullptr, *dv = nullptr, *drt = nullptr;
  __nv_bfloat16 *P = nullptr, *dS = nullptr, *dT = nullptr;
  std::unordered_map<std::string, std::pair<float*, int64_t>> grads;   // upstream key -> (device fp32 buffer, elements)
};

static float* galloc(Engine& e, TrainState& t, const std::string& name, int64_t n) {
  float* p = (float*)e.dalloc((size_t)n * 4, true);
  if (p && !name.empty()) t.grads[name] = {p, n};
  return p;
}

int Engine::train_setup() {
  if (train) return 0;
  if (is_tinyvit()) return set_error("training mode: the TinyViT encoder has no backward pass");
  train = new TrainState();
  TrainState& t = *train;
  const int D = cfg.embed_dim, hd = D / cfg.num_heads, g = cfg.image_size / cfg.patch_size, T = g * g, B = cfg.max_batch, C = cfg.out_chans;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const size_t Tw = (size_t)wpr * wpr * cfg.window_size * cfg.window_size, M = (size_t)B * T, Mq = (size_t)B * Tw;
  const std::string e = "image_encoder.";
  t.blk.resize(cfg.depth);
  for (int i = 0; i < cfg.depth; ++i) {
    TrainSave& s = t.blk[i];
    const bool glob = enc.blocks[i].global;
    const int S = glob ? g : cfg.window_size;
    const std::string p = e + "blocks." + std::to_string(i) + ".";
    CHK(s.x_in = (float*)dalloc(M * D * 4));
    CHK(s.x_mid = (float*)dalloc(M * D * 4));
    CHK(s.qkv = (__nv_bfloat16*)dalloc((glob ? M : Mq) * 3 * D * 2));
    CHK(s.attn = (__nv_bfloat16*)dalloc(M * D * 2));
    CHK(s.pre = (__nv_bfloat16*)dalloc(M * 4 * D * 2));
    CHK(s.qkv_wT = (__nv_bfloat16*)dalloc((size_t)3 * D * D * 2));
    CHK(s.proj_wT = (__nv_bfloat16*)dalloc((size_t)D * D * 2));
    CHK(s.fc1_wT = (__nv_bfloat16*)dalloc((size_t)4 * D * D * 2));
    CHK(s.fc2_wT = (__nv_bfloat16*)dalloc((size_t)4 * D * D * 2));
    CHK(s.g_ln1_g = galloc(*this, t, p + "norm1.weight", D));
    CHK(s.g_ln1_b = galloc(*this, t, p + "norm1.bias", D));
    CHK(s.g_ln2_g = galloc(*this, t, p + "norm2.weight", D));
    CHK(s.g_ln2_b = galloc(*this, t, p + "norm2.bias", D));
    CHK(s.g_qkv_w = galloc(*this, t, p + "attn.qkv.weight", (int64_t)3 * D * D));
    CHK(s.g_qkv_b = galloc(*this, t, p + "attn.qkv.bias", 3 * D));
    CHK(s.g_proj_w = galloc(*this, t, p + "attn.proj.weight", (int64_t)D * D));
    CHK(s.g_proj_b = galloc(*this, t, p + "attn.proj.bias", D));
    CHK(s.g_fc1_w = galloc(*this, t, p + "mlp.lin1.weight", (int64_t)4 * D * D));
    CHK(s.g_fc1_b = galloc(*this, t, p + "mlp.lin1.bias", 4 * D));
    CHK(s.g_fc2_w = galloc(*this, t, p + "mlp.lin2.weight", (int64_t)4 * D * D));
    CHK(s.g_fc2_b = galloc(*this, t, p + "mlp.lin2.bias", D));
    CHK(s.g_rel_h = galloc(*this, t, p + "attn.rel_pos_h", (int64_t)(2 * S - 1) * hd));
    CHK(s.g_rel_w = galloc(*this, t, p + "attn.rel_pos_w", (int64_t)(2 * S - 1) * hd));
    // optimizer registry (train_opt.cu): fp32 parameters are updated in place, bf16 operands from fp32 masters
    EncBlock& b = enc.blocks[i];
    auto inplace = [&](const std::string& k, float* w, float* g, int64_t n) { OptParam q; q.key = k; q.w = w; q.g = g; q.n = n; opt_add(q); };
    auto casted = [&](const std::string& k, float* g, int64_t n, __nv_bfloat16* dst) -> int {
      OptParam q; q.key = k; q.g = g; q.n = n; q.refresh = 1; q.dst = dst;
      CHK(q.w = opt_master_from_host(k, n));
      opt_add(q);
      return 0;
    };
    inplace(p + "norm1.weight", b.ln1_g, s.g_ln1_g, D); inplace(p + "norm1.bias", b.ln1_b, s.g_ln1_b, D);
    inplace(p + "norm2.weight", b.ln2_g, s.g_ln2_g, D); inplace(p + "norm2.bias", b.ln2_b, s.g_ln2_b, D);
    RUN(casted(p + "attn.qkv.weight", s.g_qkv_w, (int64_t)3 * D * D, b.qkv_w)); inplace(p + "attn.qkv.bias", b.qkv_b, s.g_qkv_b, 3 * D);
    RUN(casted(p + "attn.proj.weight", s.g_proj_w, (int64_t)D * D, b.proj_w)); inplace(p + "attn.proj.bias", b.proj_b, s.g_proj_b, D);
    RUN(casted(p + "mlp.lin1.weight", s.g_fc1_w, (int64_t)4 * D * D, b.fc1_w)); inplace(p + "mlp.lin1.bias", b.fc1_b, s.g_fc1_b, 4 * D);
    RUN(casted(p + "mlp.lin2.weight", s.g_fc2_w, (int64_t)4 * D * D, b.fc2_w)); inplace(p + "mlp.lin2.bias", b.fc2_b, s.g_fc2_b, D);
    for (int hw = 0; hw < 2; ++hw) {
      OptParam q;
      q.key = p + (hw ? "attn.rel_pos_w" : "attn.rel_pos_h"); q.g = hw ? s.g_rel_w : s.g_rel_h; q.n = (int64_t)(2 * S - 1) * hd;
      q.refresh = 3; q.dst = b.rel_table; q.rows = 2 * S - 1; q.cols = hd; q.cols_pad = ((hd + 63) / 64) * 64; q.row_off = hw ? (glob ? 128 : 32) : 0;
      CHK(q.w = opt_master_from_host(q.key, q.n));
      opt_add(q);
    }
  }
  CHK(t.neck1_wT = (__nv_bfloat16*)dalloc((size_t)C * D * 2));
  CHK(t.neck2_wT = (__nv_bfloat16*)dalloc((size_t)9 * C * C * 2));
  CHK(t.g_patch_w = galloc(*this, t, e + "patch_embed.proj.weight", (int64_t)D * 768));
  CHK(t.g_patch_b = galloc(*this, t, e + "patch_embed.proj.bias", D));
  CHK(t.g_pos = galloc(*this, t, e + "pos_embed", (int64_t)T * D));
  CHK(t.g_neck1_w = galloc(*this, t, e + "neck.0.weight", (int64_t)C * D));
  CHK(t.g_neck_ln1_g = galloc(*this, t, e + "neck.1.weight", C));
  CHK(t.g_neck_ln1_b = galloc(*this, t, e + "neck.1.bias", C));
  CHK(t.g_neck2_w = galloc(*this, t, "", (int64_t)9 * C * C));
  CHK(t.g_neck2_w_up = galloc(*this, t, e + "neck.2.weight", (int64_t)9 * C * C));
  CHK(t.g_neck_ln2_g = galloc(*this, t, e + "neck.3.weight", C));
  CHK(t.g_neck_ln2_b = galloc(*this, t, e + "neck.3.bias", C));
  {
    auto inplace = [&](const std::string& k, float* w, float* g, int64_t n) { OptParam q; q.key = k; q.w = w; q.g = g; q.n = n; opt_add(q); };
    OptParam q;
    q.key = e + "patch_embed.proj.weight"; q.g = t.g_patch_w; q.n = (int64_t)D * 768; q.refresh = 1; q.dst = enc.patch_w;
    CHK(q.w = opt_master_from_host(q.key, q.n)); opt_add(q);
    inplace(e + "patch_embed.proj.bias", enc.patch_b, t.g_patch_b, D);
    inplace(e + "pos_embed", enc.pos_embed, t.g_pos, (int64_t)T * D);
    q = OptParam(); q.key = e + "neck.0.weight"; q.g = t.g_neck1_w; q.n = (int64_t)C * D; q.refresh = 1; q.dst = enc.neck_conv1;
    CHK(q.w = opt_master_from_host(q.key, q.n)); opt_add(q);
    inplace(e + "neck.1.weight", enc.neck_ln1_g, t.g_neck_ln1_g, C); inplace(e + "neck.1.bias", enc.neck_ln1_b, t.g_neck_ln1_b, C);
    q = OptParam(); q.key = e + "neck.2.weight"; q.g = t.g_neck2_w_up; q.n = (int64_t)9 * C * C; q.refresh = 4; q.dst = enc.neck_conv2; q.rows = C;
    CHK(q.w = opt_master_from_host(q.key, q.n)); opt_add(q);
    inplace(e + "neck.3.weight", enc.neck_ln2_g, t.g_neck_ln2_g, C); inplace(e + "neck.3.bias", enc.neck_ln2_b, t.g_neck_ln2_b, C);
  }
  // scratch
  const size_t Dm = D > C ? D : C;
  CHK(t.dx = (float*)dalloc(M * Dm * 4));
  CHK(t.dxn = (float*)dalloc(Mq * Dm * 4));
  CHK(t.dtok = (float*)dalloc(M * C * 4));
  CHK(t.gb = (__nv_bfloat16*)dalloc(M * Dm * 2));
  CHK(t.hid = (__nv_bfloat16*)dalloc(M * 4 * D * 2));
  CHK(t.dhid = (__nv_bfloat16*)dalloc(M * 4 * D * 2));
  CHK(t.xn = (__nv_bfloat16*)dalloc(M * D * 2));
  CHK(t.xn_win = (__nv_bfloat16*)dalloc(Mq * D * 2, true));     // pad rows stay zero
  CHK(t.dqkv = (__nv_bfloat16*)dalloc(Mq * 3 * D * 2));
  CHK(t.do_win = (__nv_bfloat16*)dalloc(Mq * D * 2));
  CHK(t.dcol = (__nv_bfloat16*)dalloc(M * 9 * C * 2));
  // attention backward: the global blocks set the sizes (batch entries = B * heads, 4096 x 4096 each)
  const size_t nbg = (size_t)B * cfg.num_heads, nbw = (size_t)B * wpr * wpr * cfg.num_heads;
  const size_t s_el = std::max(nbg * T * T, nbw * 196 * 200), t_el = std::max(nbg * T * 256, nbw * 196 * 64);
  const size_t q_el = std::max(nbg * T * hd, nbw * 196 * hd), r_el = std::max(nbg * 256 * hd, nbw * 64 * hd);
  CHK(t.S = (float*)dalloc(s_el * 4));
  CHK(t.P = (__nv_bfloat16*)dalloc(s_el * 2));
  CHK(t.dS = (__nv_bfloat16*)dalloc(s_el * 2));
  CHK(t.T = (float*)dalloc(t_el * 4));
  CHK(t.dT = (__nv_bfloat16*)dalloc(t_el * 2));
  CHK(t.dq = (float*)dalloc(q_el * 4));
  CHK(t.dk = (float*)dalloc(q_el * 4));
  CHK(t.dv = (float*)dalloc(q_el * 4));
  CHK(t.drt = (float*)dalloc(r_el * 4));
  return 0;
}

// ------------------------------------------------------------------------------------------------ forward, keeping activations
int Engine::encode_train(const float* f32, int B, float* out, cudaStream_t st) {
  if (!finalized) return set_error("msam_encode_train: weights not finalized");
  if (B <= 0 || B > cfg.max_batch) return set_error("msam_encode_train: batch %d outside [1, max_batch = %d]", B, cfg.max_batch);
  RUN(train_setup());
  TrainState& t = *train;
  const int D = cfg.embed_dim, hd = D / cfg.num_heads, g = cfg.image_size / cfg.patch_size, T = g * g, C = cfg.out_chans;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const int Tw = wpr * wpr * cfg.window_size * cfg.window_size;
  const int M = B * T;
  static const float mean[3] = {123.675f, 116.28f, 103.53f}, stdv[3] = {58.395f, 57.12f, 57.375f};
  if (!t.transposed) {   // W^T operands of the dgrad GEMMs (again after every weight update: msam_finalize_weights resets this)
    for (int i = 0; i < cfg.depth; ++i) {
      const EncBlock& b = enc.blocks[i];
      TrainSave& s = t.blk[i];
      RUN(transpose_bf16(b.qkv_w, 3 * D, D, s.qkv_wT, st));
      RUN(transpose_bf16(b.proj_w, D, D, s.proj_wT, st));
      RUN(transpose_bf16(b.fc1_w, 4 * D, D, s.fc1_wT, st));
      RUN(transpose_bf16(b.fc2_w, D, 4 * D, s.fc2_wT, st));
    }
    RUN(transpose_bf16(enc.neck_conv1, C, D, t.neck1_wT, st));
    RUN(transpose_bf16(enc.neck_conv2, C, 9 * C, t.neck2_wT, st));
    t.transposed = true;
  }
  RUN(launch_patchify(nullptr, f32, B, cfg.image_size, cfg.image_size, cfg.image_size, mean, stdv, ws.patches, st));
  {
    GemmArgs a;
    a.A = ws.patches; a.W = enc.patch_w; a.M = M; a.N = D; a.K = 768; a.lda = 768; a.ldw = 768;
    a.bias = enc.patch_b; a.residual = enc.pos_embed; a.res_rows = T; a.out = ws.x; a.out_fp32 = 1;
    RUN(launch_gemm(a, num_sms, st));
  }
  for (int i = 0; i < cfg.depth; ++i) {
    const EncBlock& b = enc.blocks[i];
    TrainSave& s = t.blk[i];
    if (cudaMemcpyAsync(s.x_in, ws.x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("encode_train: copy failed");
    LnArgs l;
    l.x = ws.x; l.rows = M; l.D = D; l.gamma = b.ln1_g; l.beta = b.ln1_b; l.eps = 1e-6f; l.grid = g; l.ws = cfg.window_size;
    if (b.global) { l.out = ws.xn; } else { l.out = ws.xn_win; l.window_mode = 1; }
    RUN(launch_layernorm(l, st));
    const int Mq = b.global ? M : B * Tw;
    {
      GemmArgs a;
      a.A = b.global ? ws.xn : ws.xn_win; a.W = b.qkv_w; a.M = Mq; a.N = 3 * D; a.K = D; a.lda = D; a.ldw = D;
      a.bias = b.qkv_b; a.out = s.qkv;
      RUN(launch_gemm(a, num_sms, st));
    }
    {
      AttnArgs a;
      a.qkv = s.qkv; a.rel_table = b.rel_table; a.out = s.attn; a.batch = B; a.heads = cfg.num_heads;
      a.head_dim = hd; a.grid = g; a.window = b.global ? 0 : cfg.window_size; a.scale = 1.0f / sqrtf((float)hd);
      RUN(launch_attention(a, st));
    }
    {
      GemmArgs a;
      a.A = s.attn; a.W = b.proj_w; a.M = M; a.N = D; a.K = D; a.lda = D; a.ldw = D;
      a.bias = b.proj_b; a.residual = ws.x; a.out = ws.x; a.out_fp32 = 1;
      RUN(launch_gemm(a, num_sms, st));
    }
    if (cudaMemcpyAsync(s.x_mid, ws.x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("encode_train: copy failed");
    l = LnArgs();
    l.x = ws.x; l.rows = M; l.D = D; l.gamma = b.ln2_g; l.beta = b.ln2_b; l.eps = 1e-6f; l.out = ws.xn;
    RUN(launch_layernorm(l, st));
    {
      GemmArgs a;   // pre-activation kept; GELU as its own pass
      a.A = ws.xn; a.W = b.fc1_w; a.M = M; a.N = 4 * D; a.K = D; a.lda = D; a.ldw = D; a.bias = b.fc1_b; a.out = s.pre;
      RUN(launch_gemm(a, num_sms, st));
    }
    RUN(launch_gelu_fwd(s.pre, (long)M * 4 * D, ws.hidden, st));
    {
      GemmArgs a;
      a.A = ws.hidden; a.W = b.fc2_w; a.M = M; a.N = D; a.K = 4 * D; a.lda = 4 * D; a.ldw = 4 * D;
      a.bias = b.fc2_b; a.residual = ws.x; a.out = ws.x; a.out_fp32 = 1;
      RUN(launch_gemm(a, num_sms, st));
    }
  }
  // neck (every intermediate stays in the workspace for the backward pass)
  RUN(launch_cast_bf16(ws.x, (long)M * D, ws.xn, st));
  {
    GemmArgs a;
    a.A = ws.xn; a.W = enc.neck_conv1; a.M = M; a.N = C; a.K = D; a.lda = D; a.ldw = D; a.out = ws.neck1; a.out_fp32 = 1;
    RUN(launch_gemm(a, num_sms, st));
  }
  {
    LnArgs l;
    l.x = ws.neck1; l.rows = M; l.D = C; l.gamma = enc.neck_ln1_g; l.beta = enc.neck_ln1_b; l.eps = 1e-6f; l.out = ws.neck1b;
    RUN(launch_layernorm(l, st));
  }
  RUN(launch_im2col3x3(ws.neck1b, B, g, C, ws.neck_col, st));
  {
    GemmArgs a;
    a.A = ws.neck_col; a.W = enc.neck_conv2; a.M = M; a.N = C; a.K = 9 * C; a.lda = 9 * C; a.ldw = 9 * C; a.out = ws.neck2; a.out_fp32 = 1;
    RUN(launch_gemm(a, num_sms, st));
  }
  RUN(launch_layernorm2d_nchw(ws.neck2, B, T, enc.neck_ln2_g, enc.neck_ln2_b, 1e-6f, out, st));
  t.B = B;
  return 0;
}

// ------------------------------------------------------------------------------------------------ backward
// y = x W^T + b with x [M, K] bf16 and dy [M, N] bf16:  dW [N, K] = dy^T x,  db = column sums of dy
static int linear_wgrad(const __nv_bfloat16* dy, const __nv_bfloat16* x, int M, int N, int K, float* dW, float* db, cudaStream_t st) {
  RUN(launch_gemm_tn(dy, x, N, K, M, N, K, dW, K, st));
  if (db) {
    if (cudaMemsetAsync(db, 0, (size_t)N * 4, st) != cudaSuccess) return set_error("backward: memset failed");
    RUN(launch_colsum(dy, M, N, db, st));
  }
  return 0;
}
// dx [M, K] = dy [M, N] W [N, K], as the forward GEMM on W^T [K, N]
static int linear_dgrad(Engine& e, const __nv_bfloat16* dy, const __nv_bfloat16* wT, int M, int N, int K, void* dx, int out_fp32,
                        cudaStream_t st) {
  GemmArgs a;
  a.A = dy; a.W = wT; a.M = M; a.N = K; a.K = N; a.lda = N; a.ldw = N; a.out = dx; a.out_fp32 = out_fp32;
  return launch_gemm(a, e.num_sms, st);
}

// (dq, dk, dv) and the rel-pos table gradients of one block; qkv / do in the block's row order (window-partitioned or image)
static int attention_backward(Engine& e, TrainState& t, const EncBlock& b, TrainSave& s, const __nv_bfloat16* d_out, int B, cudaStream_t st) {
  const msam_config& cfg = e.cfg;
  const int D = cfg.embed_dim, H = cfg.num_heads, hd = D / H, g = cfg.image_size / cfg.patch_size;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  AttnBwdGeom geo;
  int outer;
  if (b.global) { geo.side = g; geo.n_tok = g * g; geo.nt = 256; geo.woff = 128; outer = B; }
  else { geo.side = cfg.window_size; geo.n_tok = geo.side * geo.side; geo.nt = 64; geo.woff = 32; outer = B * wpr * wpr; }
  const int Tk = geo.n_tok, pitch = (Tk + 7) & ~7, rt_cols = ((hd + 63) / 64) * 64;
  const long nb = (long)outer * H;
  const float scale = 1.0f / sqrtf((float)hd);
  const __nv_bfloat16 *Q = s.qkv, *K = s.qkv + D, *V = s.qkv + 2 * D;
  const long row_w = (long)Tk * 3 * D;     // elements between consecutive outer entries of qkv
  BGemmArgs a;
  // S = Q K^T
  a = BGemmArgs();
  a.A = Q; a.B = K; a.M = Tk; a.N = Tk; a.K = hd; a.lda = a.ldb = 3 * D; a.a_hstride = a.b_hstride = hd; a.a_wstride = a.b_wstride = row_w;
  a.heads = H; a.outer = outer; a.out = t.S; a.ldc = pitch; a.o_hstride = (long)Tk * pitch; a.o_wstride = (long)H * Tk * pitch;
  RUN(launch_bgemm(a, st));
  // T = Q R^T  (rel-pos projections, unscaled q as in the forward pass)
  a = BGemmArgs();
  a.A = Q; a.B = b.rel_table; a.M = Tk; a.N = geo.nt; a.K = hd; a.lda = 3 * D; a.ldb = rt_cols; a.a_hstride = hd; a.a_wstride = row_w;
  a.heads = H; a.outer = outer; a.out = t.T; a.ldc = geo.nt; a.o_hstride = (long)Tk * geo.nt; a.o_wstride = (long)H * Tk * geo.nt;
  RUN(launch_bgemm(a, st));
  RUN(launch_attn_probs(t.S, t.T, nb, geo, pitch, pitch, scale, t.P, st));
  // dP = dO V^T (over the S buffer)
  a = BGemmArgs();
  a.A = d_out; a.B = V; a.M = Tk; a.N = Tk; a.K = hd; a.lda = D; a.ldb = 3 * D; a.a_hstride = hd; a.b_hstride = hd;
  a.a_wstride = (long)Tk * D; a.b_wstride = row_w;
  a.heads = H; a.outer = outer; a.out = t.S; a.ldc = pitch; a.o_hstride = (long)Tk * pitch; a.o_wstride = (long)H * Tk * pitch;
  RUN(launch_bgemm(a, st));
  RUN(launch_attn_ds(t.P, t.S, nb, geo, pitch, pitch, t.dS, t.dT, st));
  const long sp_h = (long)Tk * pitch, sp_w = (long)H * Tk * pitch, tt_h = (long)Tk * geo.nt, tt_w = (long)H * Tk * geo.nt;
  const long o_h = (long)Tk * hd, o_w = (long)H * Tk * hd;
  // dV = P^T dO
  a = BGemmArgs();
  a.A = t.P; a.B = d_out; a.a_mn = a.b_mn = 1; a.M = Tk; a.N = hd; a.K = Tk; a.lda = pitch; a.ldb = D; a.a_hstride = sp_h; a.a_wstride = sp_w;
  a.b_hstride = hd; a.b_wstride = (long)Tk * D; a.heads = H; a.outer = outer; a.out = t.dv; a.ldc = hd; a.o_hstride = o_h; a.o_wstride = o_w;
  RUN(launch_bgemm(a, st));
  // dK = scale dS^T Q
  a.A = t.dS; a.B = Q; a.ldb = 3 * D; a.b_wstride = row_w; a.out = t.dk; a.alpha = scale;
  RUN(launch_bgemm(a, st));
  // dQ = scale dS K + dT R
  a = BGemmArgs();
  a.A = t.dS; a.B = K; a.b_mn = 1; a.M = Tk; a.N = hd; a.K = Tk; a.lda = pitch; a.ldb = 3 * D; a.a_hstride = sp_h; a.a_wstride = sp_w;
  a.b_hstride = hd; a.b_wstride = row_w; a.heads = H; a.outer = outer; a.out = t.dq; a.ldc = hd; a.o_hstride = o_h; a.o_wstride = o_w; a.alpha = scale;
  RUN(launch_bgemm(a, st));
  a = BGemmArgs();
  a.A = t.dT; a.B = b.rel_table; a.b_mn = 1; a.M = Tk; a.N = hd; a.K = geo.nt; a.lda = geo.nt; a.ldb = rt_cols; a.a_hstride = tt_h; a.a_wstride = tt_w;
  a.heads = H; a.outer = outer; a.out = t.dq; a.ldc = hd; a.o_hstride = o_h; a.o_wstride = o_w; a.accumulate = 1;
  RUN(launch_bgemm(a, st));
  // dR = sum over (window | image, head) of dT^T Q
  a = BGemmArgs();
  a.A = t.dT; a.B = Q; a.a_mn = a.b_mn = 1; a.M = geo.nt; a.N = hd; a.K = Tk; a.lda = geo.nt; a.ldb = 3 * D; a.a_hstride = tt_h; a.a_wstride = tt_w;
  a.b_hstride = hd; a.b_wstride = row_w; a.heads = H; a.outer = outer; a.out = t.drt; a.ldc = hd; a.o_hstride = (long)geo.nt * hd;
  a.o_wstride = (long)H * geo.nt * hd;
  RUN(launch_bgemm(a, st));
  const int nrel = 2 * geo.side - 1;
  RUN(launch_sum_batch(t.drt, nb, (long)geo.nt * hd, t.dxn, 0, st));   // dxn is free here: [nt, hd] fp32
  if (cudaMemcpyAsync(s.g_rel_h, t.dxn, (size_t)nrel * hd * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(s.g_rel_w, t.dxn + (size_t)geo.woff * hd, (size_t)nrel * hd * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return set_error("backward: copy failed");
  return launch_pack_dqkv(t.dq, t.dk, t.dv, outer, H, Tk, hd, t.dqkv, st);
}

int Engine::encode_backward(const float* d_out, cudaStream_t st) {
  if (!train || train->B == 0) return set_error("msam_encode_backward: no saved forward pass (call msam_encode_train first)");
  TrainState& t = *train;
  const int B = t.B, D = cfg.embed_dim, g = cfg.image_size / cfg.patch_size, T = g * g, C = cfg.out_chans;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const int Tw = wpr * wpr * cfg.window_size * cfg.window_size;
  const int M = B * T;
  auto zero = [&](float* p, size_t n) { return cudaMemsetAsync(p, 0, n * 4, st) == cudaSuccess ? 0 : set_error("backward: memset failed"); };
  // ---- neck: out = LN2d(conv3x3(LN2d(conv1x1(x))))
  RUN(launch_nchw_to_tok(d_out, B, C, T, t.dtok, st));
  RUN(zero(t.g_neck_ln2_g, C)); RUN(zero(t.g_neck_ln2_b, C));
  RUN(launch_layernorm_bwd(ws.neck2, M, C, enc.neck_ln2_g, 1e-6f, t.dtok, 0, g, cfg.window_size, 0, t.dx, t.g_neck_ln2_g, t.g_neck_ln2_b, st));
  RUN(launch_cast_bf16(t.dx, (long)M * C, t.gb, st));
  RUN(linear_wgrad(t.gb, ws.neck_col, M, C, 9 * C, t.g_neck2_w, nullptr, st));
  {
    const long n = (long)C * C * 9;
    neck2_grad_relayout_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t.g_neck2_w, C, t.g_neck2_w_up);
    count_launch();
  }
  RUN(linear_dgrad(*this, t.gb, t.neck2_wT, M, C, 9 * C, t.dcol, 0, st));
  RUN(launch_col2im3x3(t.dcol, B, g, C, t.dtok, st));
  RUN(zero(t.g_neck_ln1_g, C)); RUN(zero(t.g_neck_ln1_b, C));
  RUN(launch_layernorm_bwd(ws.neck1, M, C, enc.neck_ln1_g, 1e-6f, t.dtok, 0, g, cfg.window_size, 0, t.dxn, t.g_neck_ln1_g, t.g_neck_ln1_b, st));
  RUN(launch_cast_bf16(t.dxn, (long)M * C, t.gb, st));
  RUN(linear_wgrad(t.gb, ws.xn, M, C, D, t.g_neck1_w, nullptr, st));
  RUN(linear_dgrad(*this, t.gb, t.neck1_wT, M, C, D, t.dx, 1, st));      // dx = gradient of the last block's output
  // ---- blocks, in reverse
  for (int i = cfg.depth - 1; i >= 0; --i) {
    const EncBlock& b = enc.blocks[i];
    TrainSave& s = t.blk[i];
    const int Mq = b.global ? M : B * Tw;
    // MLP
    RUN(launch_cast_bf16(t.dx, (long)M * D, t.gb, st));
    RUN(launch_gelu_fwd(s.pre, (long)M * 4 * D, t.hid, st));
    RUN(linear_wgrad(t.gb, t.hid, M, D, 4 * D, s.g_fc2_w, s.g_fc2_b, st));
    RUN(linear_dgrad(*this, t.gb, s.fc2_wT, M, D, 4 * D, t.dhid, 0, st));
    RUN(launch_gelu_bwd(t.dhid, s.pre, (long)M * 4 * D, t.dhid, st));
    {
      LnArgs l;
      l.x = s.x_mid; l.rows = M; l.D = D; l.gamma = b.ln2_g; l.beta = b.ln2_b; l.eps = 1e-6f; l.out = t.xn;
      RUN(launch_layernorm(l, st));
    }
    RUN(linear_wgrad(t.dhid, t.xn, M, 4 * D, D, s.g_fc1_w, s.g_fc1_b, st));
    RUN(linear_dgrad(*this, t.dhid, s.fc1_wT, M, 4 * D, D, t.dxn, 1, st));
    RUN(zero(s.g_ln2_g, D)); RUN(zero(s.g_ln2_b, D));
    RUN(launch_layernorm_bwd(s.x_mid, M, D, b.ln2_g, 1e-6f, t.dxn, 0, g, cfg.window_size, 1, t.dx, s.g_ln2_g, s.g_ln2_b, st));
    // attention
    RUN(launch_cast_bf16(t.dx, (long)M * D, t.gb, st));
    RUN(linear_wgrad(t.gb, s.attn, M, D, D, s.g_proj_w, s.g_proj_b, st));
    RUN(linear_dgrad(*this, t.gb, s.proj_wT, M, D, D, t.xn, 0, st));       // d(attention output), image order, over the xn scratch
    const __nv_bfloat16* d_attn = t.xn;
    if (!b.global) {
      RUN(launch_window_gather(t.xn, B, g, cfg.window_size, D, t.do_win, st));
      d_attn = t.do_win;
    }
    RUN(attention_backward(*this, t, b, s, d_attn, B, st));
    {
      LnArgs l;
      l.x = s.x_in; l.rows = M; l.D = D; l.gamma = b.ln1_g; l.beta = b.ln1_b; l.eps = 1e-6f; l.grid = g; l.ws = cfg.window_size;
      if (b.global) { l.out = t.xn; } else { l.out = t.xn_win; l.window_mode = 1; }
      RUN(launch_layernorm(l, st));
    }
    RUN(linear_wgrad(t.dqkv, b.global ? t.xn : t.xn_win, Mq, 3 * D, D, s.g_qkv_w, s.g_qkv_b, st));
    RUN(linear_dgrad(*this, t.dqkv, s.qkv_wT, Mq, 3 * D, D, t.dxn, 1, st));
    RUN(zero(s.g_ln1_g, D)); RUN(zero(s.g_ln1_b, D));
    RUN(launch_layernorm_bwd(s.x_in, M, D, b.ln1_g, 1e-6f, t.dxn, b.global ? 0 : 1, g, cfg.window_size, 1, t.dx, s.g_ln1_g, s.g_ln1_b, st));
  }
  // ---- patch embedding + positional embedding: x0 = patches W^T + b + pos
  RUN(launch_sum_batch(t.dx, B, (long)T * D, t.g_pos, 0, st));
  RUN(launch_cast_bf16(t.dx, (long)M * D, t.gb, st));
  RUN(linear_wgrad(t.gb, ws.patches, M, D, 768, t.g_patch_w, t.g_patch_b, st));
  return 0;
}

int Engine::encoder_grad(const char* name, float* dst, int64_t n, cudaStream_t st) {
  if (!train) return set_error("msam_encoder_grad: training mode was never entered");
  auto it = train->grads.find(name);
  if (it == train->grads.end()) return set_error("msam_encoder_grad: no gradient named '%s'", name);
  if (it->second.second != n) return set_error("msam_encoder_grad: '%s' has %lld elements, caller expects %lld", name, (long long)it->second.second, (long long)n);
  if (cudaMemcpyAsync(dst, it->second.first, (size_t)n * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return set_error("msam_encoder_grad: copy failed");
  return 0;
}

void Engine::train_free() {
  delete train;
  train = nullptr;
}

void Engine::train_invalidate() {
  if (train) { train->transposed = false; train->B = 0; }
}

}  // namespace msam
