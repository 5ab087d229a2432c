// ViT image encoder, training mode (BASELINE.json configs[4] "vit_b fine-tuning step: encoder fwd/bwd"): a forward pass that keeps
// what the backward pass needs, and the backward pass itself.  Reference: torch autograd over ImageEncoderViT (oracle/sam_ref.py)
// as driven by micro_sam/training/sam_trainer.py:393 (loss.backward()); gradients are checked tensor by tensor against it in
// tests/test_gpu_backward.py, and against a float64 mirror that rounds to bf16 where this file does in
// tests/test_gpu_encoder_train_mirror.py.  The backward pass reads the workspace of the inference forward (patches, neck
// activations), so any inference encode discards the saved forward pass (Engine::encode -> train_invalidate).
//
// Saved per block (bf16 unless noted): x_in (fp32), qkv, attention output, x_mid (fp32), fc1 pre-activation.  LayerNorm outputs and
// GELU(fc1) are recomputed (HBM-bound, cheaper than keeping them).  Per block, in reverse:
//   MLP    dW2 = dy^T h | dh = dy W2 | dpre = dh o gelu'(pre) | dW1 = dpre^T LN2(x_mid) | dxn = dpre W1 | dx += LN2'(dxn)
//   attn   dWp = dy^T a | da = dy Wp | (dq, dk, dv, drel) = attention'(qkv, da) | dWqkv = dqkv^T LN1(x_in) | dxn = dqkv Wqkv | dx += LN1'(dxn)
// The forward pass is Engine::vit_forward (engine.cu), the inference forward with those activations kept.
// dgrad products use the forward wgmma GEMMs on weights transposed once per weight update (W^T as the K-major operand: the
// GEMM of gemm.cu and its epilogues apply; built here at setup and rebuilt by optimizer_step), wgrad products the MN-major GEMM of gemm_tn.cu, the five attention products the batched
// GEMM of bgemm.cu (one launch per product for all windows / images and heads), with S / P / dS materialised in HBM per block
// (window blocks: 0.1 GB, global blocks: 0.07 GB per image and head).  Gradients are fp32, operands bf16.
#include "engine.h"

#include <algorithm>
#include <cmath>

namespace msam {

struct TrainSave {
  __nv_bfloat16 *qkv_wT = nullptr, *proj_wT = nullptr, *fc1_wT = nullptr, *fc2_wT = nullptr;
  float *g_ln1_g = nullptr, *g_ln1_b = nullptr, *g_ln2_g = nullptr, *g_ln2_b = nullptr, *g_qkv_w = nullptr, *g_qkv_b = nullptr,
        *g_proj_w = nullptr, *g_proj_b = nullptr, *g_fc1_w = nullptr, *g_fc1_b = nullptr, *g_fc2_w = nullptr, *g_fc2_b = nullptr,
        *g_rel_h = nullptr, *g_rel_w = nullptr;
};

struct TrainState {
  int B = 0;                 // batch of the saved forward pass (0 = none)
  std::vector<VitBlockActs> acts;
  std::vector<TrainSave> blk;
  __nv_bfloat16 *neck1_wT = nullptr, *neck2_wT = nullptr;
  float *g_patch_w = nullptr, *g_patch_b = nullptr, *g_pos = nullptr, *g_neck1_w = nullptr, *g_neck_ln1_g = nullptr, *g_neck_ln1_b = nullptr,
        *g_neck2_w = nullptr, *g_neck_ln2_g = nullptr, *g_neck_ln2_b = nullptr;
  // scratch
  float *dx = nullptr, *dxn = nullptr, *dtok = nullptr;
  __nv_bfloat16 *gb = nullptr, *hid = nullptr, *dhid = nullptr, *xn = nullptr, *xn_win = nullptr, *dqkv = nullptr, *do_win = nullptr,
                *dcol = nullptr;
  float *S = nullptr, *T = nullptr, *dq = nullptr, *dk = nullptr, *dv = nullptr, *drt = nullptr;
  __nv_bfloat16 *P = nullptr, *dS = nullptr, *dT = nullptr;
};

int Engine::train_setup(cudaStream_t st) {
  if (train) return 0;
  if (is_tinyvit()) return set_error("training mode: the TinyViT encoder has no backward pass");
  train = new TrainState();
  TrainState& t = *train;
  const int D = cfg.embed_dim, hd = D / cfg.num_heads, g = cfg.image_size / cfg.patch_size, T = g * g, B = cfg.max_batch, C = cfg.out_chans;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const size_t Tw = (size_t)wpr * wpr * cfg.window_size * cfg.window_size, M = (size_t)B * T, Mq = (size_t)B * Tw;
  const std::string e = "image_encoder.";
  t.acts.resize(cfg.depth);
  t.blk.resize(cfg.depth);
  // the registry (train_opt.cu): fp32 parameters are their own masters; bf16 operands (and their W^T) are refreshed from fp32 masters
  auto param = [&](const std::string& k, float* w, int64_t n) { OptParam q; q.key = k; q.w = w; q.n = n; return train_add(q); };
  auto operand = [&](const std::string& k, __nv_bfloat16* dst, int rows, int cols, __nv_bfloat16* dstT, const float* init = nullptr) -> float* {
    OptParam q; q.key = k; q.n = (int64_t)rows * cols; q.refresh = Refresh::Cast; q.dst = dst; q.dstT = dstT; q.rows = rows; q.cols = cols;
    if (dstT && launch_transpose_bf16(dst, rows, cols, dstT, st)) return nullptr;
    return train_add(q, init);
  };
  for (int i = 0; i < cfg.depth; ++i) {
    VitBlockActs& a = t.acts[i];
    TrainSave& s = t.blk[i];
    EncBlock& b = enc.blocks[i];
    const AttnBwdGeom geo = rel_table_geom(b.global, cfg.window_size, g);
    const std::string p = e + "blocks." + std::to_string(i) + ".";
    CHK(a.x_in = (float*)dalloc(M * D * 4));
    CHK(a.x_mid = (float*)dalloc(M * D * 4));
    CHK(a.qkv = (__nv_bfloat16*)dalloc((b.global ? M : Mq) * 3 * D * 2));
    CHK(a.attn = (__nv_bfloat16*)dalloc(M * D * 2));
    CHK(a.pre = (__nv_bfloat16*)dalloc(M * 4 * D * 2));
    CHK(s.qkv_wT = (__nv_bfloat16*)dalloc((size_t)3 * D * D * 2));
    CHK(s.proj_wT = (__nv_bfloat16*)dalloc((size_t)D * D * 2));
    CHK(s.fc1_wT = (__nv_bfloat16*)dalloc((size_t)4 * D * D * 2));
    CHK(s.fc2_wT = (__nv_bfloat16*)dalloc((size_t)4 * D * D * 2));
    CHK(s.g_ln1_g = param(p + "norm1.weight", b.ln1_g, D));
    CHK(s.g_ln1_b = param(p + "norm1.bias", b.ln1_b, D));
    CHK(s.g_ln2_g = param(p + "norm2.weight", b.ln2_g, D));
    CHK(s.g_ln2_b = param(p + "norm2.bias", b.ln2_b, D));
    CHK(s.g_qkv_w = operand(p + "attn.qkv.weight", b.qkv_w, 3 * D, D, s.qkv_wT));
    CHK(s.g_qkv_b = param(p + "attn.qkv.bias", b.qkv_b, 3 * D));
    CHK(s.g_proj_w = operand(p + "attn.proj.weight", b.proj_w, D, D, s.proj_wT));
    CHK(s.g_proj_b = param(p + "attn.proj.bias", b.proj_b, D));
    CHK(s.g_fc1_w = operand(p + "mlp.lin1.weight", b.fc1_w, 4 * D, D, s.fc1_wT));
    CHK(s.g_fc1_b = param(p + "mlp.lin1.bias", b.fc1_b, 4 * D));
    CHK(s.g_fc2_w = operand(p + "mlp.lin2.weight", b.fc2_w, D, 4 * D, s.fc2_wT));
    CHK(s.g_fc2_b = param(p + "mlp.lin2.bias", b.fc2_b, D));
    for (int hw = 0; hw < 2; ++hw) {
      OptParam q;
      q.key = p + (hw ? "attn.rel_pos_w" : "attn.rel_pos_h"); q.n = (int64_t)(2 * geo.side - 1) * hd; q.refresh = Refresh::RelPosRows;
      q.dst = b.rel_table; q.rows = 2 * geo.side - 1; q.cols = hd; q.cols_pad = rel_table_cols(hd); q.row_off = hw ? geo.woff : 0;
      CHK((hw ? s.g_rel_w : s.g_rel_h) = train_add(q));
    }
  }
  CHK(t.neck1_wT = (__nv_bfloat16*)dalloc((size_t)C * D * 2));
  CHK(t.neck2_wT = (__nv_bfloat16*)dalloc((size_t)9 * C * C * 2));
  CHK(t.g_patch_w = operand(e + "patch_embed.proj.weight", enc.patch_w, D, 768, nullptr));
  CHK(t.g_patch_b = param(e + "patch_embed.proj.bias", enc.patch_b, D));
  CHK(t.g_pos = param(e + "pos_embed", enc.pos_embed, (int64_t)T * D));
  CHK(t.g_neck1_w = operand(e + "neck.0.weight", enc.neck_conv1, C, D, t.neck1_wT));
  CHK(t.g_neck_ln1_g = param(e + "neck.1.weight", enc.neck_ln1_g, C));
  CHK(t.g_neck_ln1_b = param(e + "neck.1.bias", enc.neck_ln1_b, C));
  {   // master and gradient in the implicit GEMM's layout: the gradient is the wgrad GEMM's output itself
    auto it = dec_host.find(e + "neck.2.weight");
    if (it == dec_host.end()) return set_error("training: no host copy of '%sneck.2.weight'", e.c_str());
    const std::vector<float> w = conv3x3_gemm_layout(it->second.data, C);
    CHK(t.g_neck2_w = operand(e + "neck.2.weight@gemm", enc.neck_conv2, C, 9 * C, t.neck2_wT, w.data()));
  }
  CHK(t.g_neck_ln2_g = param(e + "neck.3.weight", enc.neck_ln2_g, C));
  CHK(t.g_neck_ln2_b = param(e + "neck.3.bias", enc.neck_ln2_b, C));
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
  RUN(train_setup(st));
  RUN(vit_forward(nullptr, f32, B, cfg.image_size, cfg.image_size, train->acts.data(), out, st));
  train->B = B;
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
static int attention_backward(Engine& e, TrainState& t, const EncBlock& b, const VitBlockActs& acts, TrainSave& s, const __nv_bfloat16* d_out,
                              int B, cudaStream_t st) {
  const msam_config& cfg = e.cfg;
  const int D = cfg.embed_dim, H = cfg.num_heads, hd = D / H, g = cfg.image_size / cfg.patch_size;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const AttnBwdGeom geo = rel_table_geom(b.global, cfg.window_size, g);
  const int outer = b.global ? B : B * wpr * wpr;
  const int Tk = geo.n_tok, pitch = (Tk + 7) & ~7, rt_cols = rel_table_cols(hd);
  const long nb = (long)outer * H;
  const float scale = 1.0f / sqrtf((float)hd);
  const __nv_bfloat16 *Q = acts.qkv, *K = acts.qkv + D, *V = acts.qkv + 2 * D;
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
    const VitBlockActs& a = t.acts[i];
    TrainSave& s = t.blk[i];
    const int Mq = b.global ? M : B * Tw;
    // MLP
    RUN(launch_cast_bf16(t.dx, (long)M * D, t.gb, st));
    RUN(launch_gelu_fwd(a.pre, (long)M * 4 * D, t.hid, st));
    RUN(linear_wgrad(t.gb, t.hid, M, D, 4 * D, s.g_fc2_w, s.g_fc2_b, st));
    RUN(linear_dgrad(*this, t.gb, s.fc2_wT, M, D, 4 * D, t.dhid, 0, st));
    RUN(launch_gelu_bwd(t.dhid, a.pre, (long)M * 4 * D, t.dhid, st));
    {
      LnArgs l;
      l.x = a.x_mid; l.rows = M; l.D = D; l.gamma = b.ln2_g; l.beta = b.ln2_b; l.eps = 1e-6f; l.out = t.xn;
      RUN(launch_layernorm(l, st));
    }
    RUN(linear_wgrad(t.dhid, t.xn, M, 4 * D, D, s.g_fc1_w, s.g_fc1_b, st));
    RUN(linear_dgrad(*this, t.dhid, s.fc1_wT, M, 4 * D, D, t.dxn, 1, st));
    RUN(zero(s.g_ln2_g, D)); RUN(zero(s.g_ln2_b, D));
    RUN(launch_layernorm_bwd(a.x_mid, M, D, b.ln2_g, 1e-6f, t.dxn, 0, g, cfg.window_size, 1, t.dx, s.g_ln2_g, s.g_ln2_b, st));
    // attention
    RUN(launch_cast_bf16(t.dx, (long)M * D, t.gb, st));
    RUN(linear_wgrad(t.gb, a.attn, M, D, D, s.g_proj_w, s.g_proj_b, st));
    RUN(linear_dgrad(*this, t.gb, s.proj_wT, M, D, D, t.xn, 0, st));       // d(attention output), image order, over the xn scratch
    const __nv_bfloat16* d_attn = t.xn;
    if (!b.global) {
      RUN(launch_window_gather(t.xn, B, g, cfg.window_size, D, t.do_win, st));
      d_attn = t.do_win;
    }
    RUN(attention_backward(*this, t, b, a, s, d_attn, B, st));
    {
      LnArgs l;
      l.x = a.x_in; l.rows = M; l.D = D; l.gamma = b.ln1_g; l.beta = b.ln1_b; l.eps = 1e-6f; l.grid = g; l.ws = cfg.window_size;
      if (b.global) { l.out = t.xn; } else { l.out = t.xn_win; l.window_mode = 1; }
      RUN(launch_layernorm(l, st));
    }
    RUN(linear_wgrad(t.dqkv, b.global ? t.xn : t.xn_win, Mq, 3 * D, D, s.g_qkv_w, s.g_qkv_b, st));
    RUN(linear_dgrad(*this, t.dqkv, s.qkv_wT, Mq, 3 * D, D, t.dxn, 1, st));
    RUN(zero(s.g_ln1_g, D)); RUN(zero(s.g_ln1_b, D));
    RUN(launch_layernorm_bwd(a.x_in, M, D, b.ln1_g, 1e-6f, t.dxn, b.global ? 0 : 1, g, cfg.window_size, 1, t.dx, s.g_ln1_g, s.g_ln1_b, st));
  }
  // ---- patch embedding + positional embedding: x0 = patches W^T + b + pos
  RUN(launch_sum_batch(t.dx, B, (long)T * D, t.g_pos, 0, st));
  RUN(launch_cast_bf16(t.dx, (long)M * D, t.gb, st));
  RUN(linear_wgrad(t.gb, ws.patches, M, D, 768, t.g_patch_w, t.g_patch_b, st));
  return 0;
}

void Engine::train_free() {
  delete train;
  train = nullptr;
}

void Engine::train_invalidate() {
  if (train) train->B = 0;
}

}  // namespace msam
