// C-ABI implementation (include/msam_b200.h): model container, weight packing, workspace, encoder forward.
#include "engine.h"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace msam {

// ------------------------------------------------------------------------------------------------ error / counters
static thread_local char g_err[1024] = "";
static thread_local int64_t g_launches = 0;

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return -1;
}
static void count_launch() { ++g_launches; }
int launch_check(const char* name) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch failed: %s", name, cudaGetErrorString(e));
  count_launch();
  return 0;
}
bool pdl_enabled() {
  // every kernel of the chain needs its predecessor's output at once, so only the short prologues could overlap -> off unless
  // MSAM_PDL=1
  static const bool on = getenv("MSAM_PDL") != nullptr;
  return on;
}

struct ProfRec { cudaEvent_t a, b; const char* name; double flops, bytes; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof;
void prof_begin(cudaStream_t st, const char* name, double flops, double bytes) {
  if (!g_prof_on) return;
  ProfRec r;
  cudaEventCreate(&r.a);
  cudaEventCreate(&r.b);
  r.name = name;
  r.flops = flops;
  r.bytes = bytes;
  cudaEventRecord(r.a, st);
  g_prof.push_back(r);
}
void prof_end(cudaStream_t st) {
  if (!g_prof_on || g_prof.empty()) return;
  cudaEventRecord(g_prof.back().b, st);
}

// ------------------------------------------------------------------------------------------------ tensor maps
PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  return make_tmap_2d(out, gptr, 2, rows, cols, ld, box_rows);
}

static int make_tmap_typed(CUtensorMap* out, const void* gptr, int elem_bytes, int f16, uint64_t rows, uint64_t cols,
                           uint64_t ld, uint32_t box_rows);
int make_tmap_2d(CUtensorMap* out, const void* gptr, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows) {
  return make_tmap_typed(out, gptr, elem_bytes, 0, rows, cols, ld, box_rows);
}
int make_tmap_f16_2d(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  return make_tmap_typed(out, gptr, 2, 1, rows, cols, ld, box_rows);
}
static int make_tmap_typed(CUtensorMap* out, const void* gptr, int elem_bytes, int f16, uint64_t rows, uint64_t cols,
                           uint64_t ld, uint32_t box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if (elem_bytes != 2 && elem_bytes != 4) return set_error("tensor map: unsupported element size %d", elem_bytes);
  if ((reinterpret_cast<uintptr_t>(gptr) & 15) != 0 || (ld * elem_bytes) % 16 != 0)
    return set_error("tensor map: base/stride must be 16-byte aligned (ptr=%p ld=%llu)", gptr, (unsigned long long)ld);
  if (box_rows > 256) return set_error("tensor map: box_rows=%u > 256", box_rows);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, elem_bytes == 2 ? (f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)
                                        : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                   const_cast<void*>(gptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error("cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu ld=%llu box_rows=%u", (int)r,
                     (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows);
  return 0;
}

// ------------------------------------------------------------------------------------------------ device memory
void* Engine::dalloc(size_t bytes, bool zero) {
  void* p = nullptr;
  if (bytes == 0) bytes = 16;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    set_error("cudaMalloc of %zu bytes failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  if (zero) cudaMemset(p, 0, bytes);
  allocs.push_back(p);
  return p;
}

const std::vector<float>* Engine::host(const std::string& name, std::initializer_list<int64_t> shape) {
  auto it = host_weights.find(name);
  if (it == host_weights.end()) {
    set_error("missing weight '%s'", name.c_str());
    return nullptr;
  }
  int64_t n = 1;
  for (auto s : shape) n *= s;
  if ((int64_t)it->second.data.size() != n) {
    set_error("weight '%s' has %zu elements, expected %lld", name.c_str(), it->second.data.size(), (long long)n);
    return nullptr;
  }
  return &it->second.data;
}

__nv_bfloat16* Engine::upload_bf16(const float* src, size_t n) {
  std::vector<__nv_bfloat16> tmp(n);
  for (size_t i = 0; i < n; ++i) tmp[i] = __float2bfloat16(src[i]);
  auto* d = static_cast<__nv_bfloat16*>(dalloc(n * 2));
  if (!d) return nullptr;
  if (cudaMemcpy(d, tmp.data(), n * 2, cudaMemcpyHostToDevice) != cudaSuccess) {
    set_error("H2D copy failed");
    return nullptr;
  }
  return d;
}
__half* Engine::upload_f16(const float* src, size_t n) {
  std::vector<__half> tmp(n);
  for (size_t i = 0; i < n; ++i) tmp[i] = __float2half(src[i]);
  auto* d = static_cast<__half*>(dalloc(n * 2));
  if (!d) return nullptr;
  if (cudaMemcpy(d, tmp.data(), n * 2, cudaMemcpyHostToDevice) != cudaSuccess) {
    set_error("H2D copy failed");
    return nullptr;
  }
  return d;
}
float* Engine::upload_f32(const float* src, size_t n) {
  auto* d = static_cast<float*>(dalloc(n * 4));
  if (!d) return nullptr;
  if (cudaMemcpy(d, src, n * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
    set_error("H2D copy failed");
    return nullptr;
  }
  return d;
}
__nv_bfloat16* Engine::up_bf16(const std::string& name, std::initializer_list<int64_t> shape) {
  const auto* h = host(name, shape);
  return h ? upload_bf16(h->data(), h->size()) : nullptr;
}
float* Engine::up_f32(const std::string& name, std::initializer_list<int64_t> shape) {
  const auto* h = host(name, shape);
  return h ? upload_f32(h->data(), h->size()) : nullptr;
}

std::vector<float> conv3x3_gemm_layout(const std::vector<float>& w, int C) {
  std::vector<float> r((size_t)C * 9 * C);
  for (int o = 0; o < C; ++o)
    for (int c = 0; c < C; ++c)
      for (int k = 0; k < 9; ++k) r[((size_t)o * 9 + k) * C + c] = w[((size_t)o * C + c) * 9 + k];
  return r;
}

// ------------------------------------------------------------------------------------------------ weights
int Engine::finalize_encoder() {
  const int D = cfg.embed_dim, hd = D / cfg.num_heads, g = cfg.image_size / cfg.patch_size;
  const std::string e = "image_encoder.";
  CHK(enc.patch_w = up_bf16(e + "patch_embed.proj.weight", {D, 3, 16, 16}));
  CHK(enc.patch_b = up_f32(e + "patch_embed.proj.bias", {D}));
  CHK(enc.pos_embed = up_f32(e + "pos_embed", {1, g, g, D}));
  enc.blocks.resize(cfg.depth);
  for (int i = 0; i < cfg.depth; ++i) {
    EncBlock& b = enc.blocks[i];
    const std::string p = e + "blocks." + std::to_string(i) + ".";
    b.global = false;
    for (int k = 0; k < 8 && cfg.global_attn[k] >= 0; ++k) b.global |= (cfg.global_attn[k] == i);
    const AttnBwdGeom geo = rel_table_geom(b.global, cfg.window_size, g);
    const int S = geo.side;
    CHK(b.ln1_g = up_f32(p + "norm1.weight", {D}));
    CHK(b.ln1_b = up_f32(p + "norm1.bias", {D}));
    CHK(b.qkv_w = up_bf16(p + "attn.qkv.weight", {3 * D, D}));
    CHK(b.qkv_b = up_f32(p + "attn.qkv.bias", {3 * D}));
    CHK(b.proj_w = up_bf16(p + "attn.proj.weight", {D, D}));
    CHK(b.proj_b = up_f32(p + "attn.proj.bias", {D}));
    CHK(b.ln2_g = up_f32(p + "norm2.weight", {D}));
    CHK(b.ln2_b = up_f32(p + "norm2.bias", {D}));
    CHK(b.fc1_w = up_bf16(p + "mlp.lin1.weight", {4 * D, D}));
    CHK(b.fc1_b = up_f32(p + "mlp.lin1.bias", {4 * D}));
    CHK(b.fc2_w = up_bf16(p + "mlp.lin2.weight", {D, 4 * D}));
    CHK(b.fc2_b = up_f32(p + "mlp.lin2.bias", {D}));
    // relative-position table tile in the layout of rel_table_geom (kernels.h).  get_rel_pos's interpolation branch (table length
    // != 2S-1, only hit when image_size != 1024) is not supported.
    const auto* rh = host(p + "attn.rel_pos_h", {2 * S - 1, hd});
    const auto* rw = host(p + "attn.rel_pos_w", {2 * S - 1, hd});
    CHK(rh && rw);
    const int cols = rel_table_cols(hd);
    std::vector<float> tab((size_t)geo.nt * cols, 0.f);
    for (int r = 0; r < 2 * S - 1; ++r)
      for (int c = 0; c < hd; ++c) {
        tab[(size_t)r * cols + c] = (*rh)[(size_t)r * hd + c];
        tab[(size_t)(geo.woff + r) * cols + c] = (*rw)[(size_t)r * hd + c];
      }
    CHK(b.rel_table = upload_bf16(tab.data(), tab.size()));
  }
  const int C = cfg.out_chans;
  CHK(enc.neck_conv1 = up_bf16(e + "neck.0.weight", {C, D, 1, 1}));
  CHK(enc.neck_ln1_g = up_f32(e + "neck.1.weight", {C}));
  CHK(enc.neck_ln1_b = up_f32(e + "neck.1.bias", {C}));
  {
    const auto* w = host(e + "neck.2.weight", {C, C, 3, 3});
    CHK(w);
    const std::vector<float> r = conv3x3_gemm_layout(*w, C);
    CHK(enc.neck_conv2 = upload_bf16(r.data(), r.size()));
  }
  CHK(enc.neck_ln2_g = up_f32(e + "neck.3.weight", {C}));
  CHK(enc.neck_ln2_b = up_f32(e + "neck.3.bias", {C}));
  return 0;
}

int Engine::alloc_encoder_ws() {
  const int D = cfg.embed_dim, g = cfg.image_size / cfg.patch_size, T = g * g, B = cfg.max_batch, C = cfg.out_chans;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const size_t Tw = (size_t)wpr * wpr * cfg.window_size * cfg.window_size;  // 4900 window-partitioned rows / image
  CHK(ws.patches = (__nv_bfloat16*)dalloc((size_t)B * T * 768 * 2));
  CHK(ws.x = (float*)dalloc((size_t)B * T * D * 4));
  CHK(ws.xn = (__nv_bfloat16*)dalloc((size_t)B * T * D * 2));
  CHK(ws.xn_win = (__nv_bfloat16*)dalloc((size_t)B * Tw * D * 2, /*zero=*/true));  // pad rows stay zero forever
  CHK(ws.qkv = (__nv_bfloat16*)dalloc((size_t)B * Tw * 3 * D * 2));
  CHK(ws.attn = (__nv_bfloat16*)dalloc((size_t)B * T * D * 2));
  CHK(ws.hidden = (__nv_bfloat16*)dalloc((size_t)B * T * 4 * D * 2));
  CHK(ws.neck1 = (float*)dalloc((size_t)B * T * C * 4));
  CHK(ws.neck1b = (__nv_bfloat16*)dalloc((size_t)B * T * C * 2));
  CHK(ws.neck_col = (__nv_bfloat16*)dalloc((size_t)B * T * 9 * C * 2));
  CHK(ws.neck2 = (float*)dalloc((size_t)B * T * C * 4));
  return 0;
}

// ------------------------------------------------------------------------------------------------ encoder forward
int Engine::encode(const uint8_t* u8, const float* f32, int B, int hh, int ww, float* out, cudaStream_t st, int stop_after,
                   float* x_out) {
  // the inference forward writes the workspace that msam_encode_backward reads (patches, neck activations): a saved training
  // forward pass does not survive it
  train_invalidate();
  if (is_tinyvit()) return encode_tinyvit(u8, f32, B, hh, ww, out, st, stop_after, x_out);
  if (!finalized) return set_error("msam_encode: weights not finalized");
  if (B <= 0) return set_error("msam_encode: empty batch");
  const int D = cfg.embed_dim, g = cfg.image_size / cfg.patch_size, T = g * g, C = cfg.out_chans;
  if (u8 && (hh > cfg.image_size || ww > cfg.image_size || hh <= 0 || ww <= 0))
    return set_error("msam_encode_u8: image %dx%d exceeds %d", hh, ww, cfg.image_size);
  for (int b0 = 0; b0 < B; b0 += cfg.max_batch) {
    const int nb = (B - b0 < cfg.max_batch) ? (B - b0) : cfg.max_batch;
    const uint8_t* u8p = u8 ? u8 + (size_t)b0 * hh * ww * 3 : nullptr;
    const float* f32p = f32 ? f32 + (size_t)b0 * 3 * cfg.image_size * cfg.image_size : nullptr;
    if (vit_forward(u8p, f32p, nb, hh, ww, nullptr, stop_after >= 0 ? nullptr : out + (size_t)b0 * C * T, st, stop_after)) return -1;
    if (stop_after >= 0 &&   // debug / parity localisation: the fp32 residual stream after `stop_after` blocks
        cudaMemcpyAsync(x_out + (size_t)b0 * T * D, ws.x, (size_t)nb * T * D * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return set_error("encode_blocks: copy failed");
  }
  return 0;
}

int Engine::vit_forward(const uint8_t* u8, const float* f32, int nb, int hh, int ww, const VitBlockActs* keep, float* out,
                        cudaStream_t st, int stop_after) {
  const int D = cfg.embed_dim, hd = D / cfg.num_heads, g = cfg.image_size / cfg.patch_size, T = g * g, C = cfg.out_chans;
  const int wpr = (g + cfg.window_size - 1) / cfg.window_size;
  const int Tw = wpr * wpr * cfg.window_size * cfg.window_size;
  const int M = nb * T;
  static const float mean[3] = {123.675f, 116.28f, 103.53f}, stdv[3] = {58.395f, 57.12f, 57.375f};
  auto keep_copy = [&](float* dst) {   // training: a copy of the fp32 residual stream for the backward pass
    if (cudaMemcpyAsync(dst, ws.x, (size_t)M * D * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("encode_train: copy failed");
    return 0;
  };
  if (launch_patchify(u8, f32, nb, hh, ww, cfg.image_size, mean, stdv, ws.patches, st)) return -1;
  {  // patch embed: conv 16x16/16 == GEMM, + bias + pos_embed (row % T)
    GemmArgs a;
    a.A = ws.patches; a.W = enc.patch_w; a.M = M; a.N = D; a.K = 768; a.lda = 768; a.ldw = 768;
    a.bias = enc.patch_b; a.residual = enc.pos_embed; a.res_rows = T; a.out = ws.x; a.out_fp32 = 1;
    if (launch_gemm(a, num_sms, st)) return -1;
  }
  const int n_blocks = stop_after >= 0 && stop_after < cfg.depth ? stop_after : cfg.depth;
  for (int i = 0; i < n_blocks; ++i) {
    const EncBlock& b = enc.blocks[i];
    __nv_bfloat16* qkv = keep ? keep[i].qkv : ws.qkv;
    __nv_bfloat16* attn = keep ? keep[i].attn : ws.attn;
    if (keep && keep_copy(keep[i].x_in)) return -1;
    LnArgs l;
    l.x = ws.x; l.rows = M; l.D = D; l.gamma = b.ln1_g; l.beta = b.ln1_b; l.eps = 1e-6f;
    l.grid = g; l.ws = cfg.window_size;
    if (b.global) { l.out = ws.xn; } else { l.out = ws.xn_win; l.window_mode = 1; }
    if (launch_layernorm(l, st)) return -1;
    const int Mq = b.global ? M : nb * Tw;
    {
      GemmArgs a;
      a.A = b.global ? ws.xn : ws.xn_win; a.W = b.qkv_w; a.M = Mq; a.N = 3 * D; a.K = D; a.lda = D; a.ldw = D;
      a.bias = b.qkv_b; a.out = qkv;
      if (launch_gemm(a, num_sms, st)) return -1;
    }
    {
      AttnArgs a;
      a.qkv = qkv; a.rel_table = b.rel_table; a.out = attn; a.batch = nb; a.heads = cfg.num_heads;
      a.head_dim = hd; a.grid = g; a.window = b.global ? 0 : cfg.window_size; a.scale = 1.0f / sqrtf((float)hd);
      if (launch_attention(a, st)) return -1;
    }
    {
      GemmArgs a;
      a.A = attn; a.W = b.proj_w; a.M = M; a.N = D; a.K = D; a.lda = D; a.ldw = D;
      a.bias = b.proj_b; a.residual = ws.x; a.out = ws.x; a.out_fp32 = 1;
      if (launch_gemm(a, num_sms, st)) return -1;
    }
    if (keep && keep_copy(keep[i].x_mid)) return -1;
    l = LnArgs();
    l.x = ws.x; l.rows = M; l.D = D; l.gamma = b.ln2_g; l.beta = b.ln2_b; l.eps = 1e-6f; l.out = ws.xn;
    if (launch_layernorm(l, st)) return -1;
    {
      GemmArgs a;
      a.A = ws.xn; a.W = b.fc1_w; a.M = M; a.N = 4 * D; a.K = D; a.lda = D; a.ldw = D; a.bias = b.fc1_b;
      if (keep) { a.out = keep[i].pre; } else { a.act = 1; a.out = ws.hidden; }   // training keeps the pre-activation for GELU'
      if (launch_gemm(a, num_sms, st)) return -1;
    }
    if (keep && launch_gelu_fwd(keep[i].pre, (long)M * 4 * D, ws.hidden, st)) return -1;
    {
      GemmArgs a;
      a.A = ws.hidden; a.W = b.fc2_w; a.M = M; a.N = D; a.K = 4 * D; a.lda = 4 * D; a.ldw = 4 * D;
      a.bias = b.fc2_b; a.residual = ws.x; a.out = ws.x; a.out_fp32 = 1;
      if (launch_gemm(a, num_sms, st)) return -1;
    }
  }
  if (stop_after >= 0) return 0;
  // neck: conv1x1 -> LN2d -> conv3x3 (im2col GEMM) -> LN2d (NCHW out); the training backward reads its intermediates from ws
  if (launch_cast_bf16(ws.x, (long)M * D, ws.xn, st)) return -1;
  {
    GemmArgs a;
    a.A = ws.xn; a.W = enc.neck_conv1; a.M = M; a.N = C; a.K = D; a.lda = D; a.ldw = D; a.out = ws.neck1; a.out_fp32 = 1;
    if (launch_gemm(a, num_sms, st)) return -1;
  }
  {
    LnArgs l;
    l.x = ws.neck1; l.rows = M; l.D = C; l.gamma = enc.neck_ln1_g; l.beta = enc.neck_ln1_b; l.eps = 1e-6f; l.out = ws.neck1b;
    if (launch_layernorm(l, st)) return -1;
  }
  if (launch_im2col3x3(ws.neck1b, nb, g, C, ws.neck_col, st)) return -1;
  {
    GemmArgs a;
    a.A = ws.neck_col; a.W = enc.neck_conv2; a.M = M; a.N = C; a.K = 9 * C; a.lda = 9 * C; a.ldw = 9 * C;
    a.out = ws.neck2; a.out_fp32 = 1;
    if (launch_gemm(a, num_sms, st)) return -1;
  }
  return launch_layernorm2d_nchw(ws.neck2, nb, T, enc.neck_ln2_g, enc.neck_ln2_b, 1e-6f, out, st);
}

}  // namespace msam

// =================================================================================================== C ABI
using namespace msam;

struct msam_handle {
  Engine eng;
};

extern "C" {

const char* msam_last_error(void) { return g_err; }
int64_t msam_launch_count(void) { return g_launches; }

int msam_profile(int enable) {
  for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
  g_prof_on = enable != 0;
  return 0;
}
// JSON array, one object per kernel name: {"name", "ms" (sum of CUDA-event times), "n" (launches), "flops", "bytes"
// (algorithmic work summed over the launches)}.  Synchronises the device.  Returns the length written, < 0 on error.
int msam_profile_report(char* buf, int cap) {
  if (!buf || cap < 4) return set_error("msam_profile_report: null argument");
  if (cudaDeviceSynchronize() != cudaSuccess) return set_error("profile: %s", cudaGetErrorString(cudaGetLastError()));
  struct Agg { double ms = 0, n = 0, flops = 0, bytes = 0; };
  std::vector<std::pair<std::string, Agg>> agg;
  for (auto& r : g_prof) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) continue;
    Agg* a = nullptr;
    for (auto& kv : agg) if (kv.first == r.name) { a = &kv.second; break; }
    if (!a) { agg.emplace_back(r.name, Agg()); a = &agg.back().second; }
    a->ms += ms; a->n += 1; a->flops += r.flops; a->bytes += r.bytes;
  }
  std::string s = "[";
  char tmp[512];
  for (size_t i = 0; i < agg.size(); ++i) {
    snprintf(tmp, sizeof(tmp), "%s{\"name\": \"%s\", \"ms\": %.6f, \"n\": %.0f, \"flops\": %.6e, \"bytes\": %.6e}", i ? ", " : "",
             agg[i].first.c_str(), agg[i].second.ms, agg[i].second.n, agg[i].second.flops, agg[i].second.bytes);
    s += tmp;
  }
  s += "]";
  if ((int)s.size() + 1 > cap) return set_error("msam_profile_report: buffer too small (%zu needed)", s.size() + 1);
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int)s.size();
}

int msam_create(const msam_config* cfg, int device, msam_handle** out) {
  if (!cfg || !out) return set_error("msam_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return set_error("msam_create: no CUDA device available (this library has no CPU fallback)");
  if (device < 0 || device >= ndev) return set_error("msam_create: bad device %d (have %d)", device, ndev);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9) return set_error("msam_create: device %d is sm_%d%d; this library is sm_90a only", device, prop.major, prop.minor);
  if (cfg->depth == 0) {   // MobileSAM TinyViT (vit_t): fixed architecture, see csrc/tinyvit.cu
    if (cfg->embed_dim != 320 || cfg->num_heads != 10) return set_error("vit_t (depth 0) takes embed_dim 320 / num_heads 10");
  } else {
    if (cfg->num_heads <= 0 || cfg->embed_dim % cfg->num_heads != 0) return set_error("embed_dim %% num_heads != 0");
    const int hd = cfg->embed_dim / cfg->num_heads;
    if (hd != 64 && hd != 80) return set_error("head_dim %d unsupported (64 or 80)", hd);
  }
  if (cfg->image_size != 1024 || cfg->patch_size != 16 || cfg->window_size != 14 || cfg->out_chans != 256)
    return set_error("only image_size 1024 / patch 16 / window 14 / out_chans 256 are supported");
  if (cfg->embed_dim % 32 != 0 || cfg->embed_dim > 1280) return set_error("embed_dim %d unsupported", cfg->embed_dim);
  if (cudaSetDevice(device) != cudaSuccess) return set_error("cudaSetDevice(%d) failed", device);
  auto* h = new msam_handle();
  h->eng.cfg = *cfg;
  if (h->eng.cfg.max_batch <= 0) h->eng.cfg.max_batch = 1;
  if (h->eng.cfg.max_prompts <= 0) h->eng.cfg.max_prompts = 64;
  h->eng.device = device;
  h->eng.num_sms = prop.multiProcessorCount;
  *out = h;
  return 0;
}

int msam_destroy(msam_handle* h) {
  if (!h) return 0;
  cudaSetDevice(h->eng.device);
  cudaDeviceSynchronize();
  h->eng.dec_train_free();
  h->eng.train_free();
  for (void* p : h->eng.allocs) cudaFree(p);
  delete h;
  return 0;
}

int msam_load_weight(msam_handle* h, const char* name, const float* host_data, const int64_t* shape, int ndim) {
  if (!h || !name || !host_data || !shape) return set_error("msam_load_weight: null argument");
  int64_t n = 1;
  HostTensor t;
  for (int i = 0; i < ndim; ++i) { n *= shape[i]; t.shape.push_back(shape[i]); }
  t.data.assign(host_data, host_data + n);
  h->eng.host_weights[name] = std::move(t);
  return 0;
}

int msam_finalize_weights(msam_handle* h) {
  if (!h) return set_error("null handle");
  cudaSetDevice(h->eng.device);
  if (h->eng.is_tinyvit()) {
    if (h->eng.finalize_tinyvit()) return -1;
    if (h->eng.alloc_tinyvit_ws()) return -1;
  } else {
    if (h->eng.finalize_encoder()) return -1;
    if (h->eng.alloc_encoder_ws()) return -1;
  }
  if (h->eng.finalize_decoder()) return -1;
  h->eng.dec_host = std::move(h->eng.host_weights);   // kept: fp32 masters / training-path operands are built from them on demand
  h->eng.host_weights.clear();
  if (cudaDeviceSynchronize() != cudaSuccess) return set_error("finalize: %s", cudaGetErrorString(cudaGetLastError()));
  h->eng.finalized = true;
  return 0;
}

int msam_encode_f32(msam_handle* h, const float* nchw, int B, float* out, void* stream) {
  if (!h || !nchw || !out) return set_error("msam_encode_f32: null argument");
  return h->eng.encode(nullptr, nchw, B, h->eng.cfg.image_size, h->eng.cfg.image_size, out, (cudaStream_t)stream);
}
int msam_encode_u8(msam_handle* h, const uint8_t* hwc, int B, int hh, int ww, float* out, void* stream) {
  if (!h || !hwc || !out) return set_error("msam_encode_u8: null argument");
  return h->eng.encode(hwc, nullptr, B, hh, ww, out, (cudaStream_t)stream);
}

int msam_encode_u8_blocks(msam_handle* h, const uint8_t* hwc, int B, int hh, int ww, int n_blocks, float* x_out, void* stream) {
  if (!h || !hwc || !x_out || n_blocks < 0) return set_error("msam_encode_u8_blocks: bad argument");
  return h->eng.encode(hwc, nullptr, B, hh, ww, nullptr, (cudaStream_t)stream, n_blocks, x_out);
}

int msam_set_image_embedding(msam_handle* h, const float* feat, void* stream) {
  if (!h || !feat) return set_error("msam_set_image_embedding: null argument");
  return h->eng.set_image_embedding(feat, (cudaStream_t)stream);
}
int msam_decode(msam_handle* h, const float* points, const float* labels, int n_points, const float* boxes, int P,
                int multimask, float* low_res, float* iou, void* stream) {
  if (!h || !low_res || !iou) return set_error("msam_decode: null argument");
  if (!points && !boxes) return set_error("msam_decode: need points and/or boxes");
  if (points && !labels) return set_error("msam_decode: points without labels");
  return h->eng.decode(points, labels, points ? n_points : 0, boxes, nullptr, P, multimask, low_res, iou, (cudaStream_t)stream);
}
int msam_decode_ex(msam_handle* h, const float* points, const float* labels, int n_points, const float* boxes,
                   const float* mask_input, int P, int multimask, float* low_res, float* iou, void* stream) {
  if (!h || !low_res || !iou) return set_error("msam_decode_ex: null argument");
  if (!points && !boxes && !mask_input) return set_error("msam_decode_ex: need points, boxes and/or mask prompts");
  if (points && !labels) return set_error("msam_decode_ex: points without labels");
  return h->eng.decode(points, labels, points ? n_points : 0, boxes, mask_input, P, multimask, low_res, iou, (cudaStream_t)stream);
}
int msam_prompt_encode(msam_handle* h, const float* points, const float* labels, int n_points, const float* boxes,
                       const float* mask_input, int P, float* sparse_out, float* dense_out, void* stream) {
  if (!h) return set_error("msam_prompt_encode: null handle");
  if (points && !labels) return set_error("msam_prompt_encode: points without labels");
  return h->eng.prompt_encode(points, labels, points ? n_points : 0, boxes, mask_input, P, sparse_out, dense_out, (cudaStream_t)stream);
}
int msam_get_dense_pe(msam_handle* h, float* out_4096x256, void* stream) {
  if (!h || !out_4096x256) return set_error("msam_get_dense_pe: null argument");
  return h->eng.dense_pe(out_4096x256, (cudaStream_t)stream);
}
int msam_mask_decode(msam_handle* h, const float* sparse, int n_sparse, const float* dense, int P, int multimask, float* low_res,
                     float* iou, void* stream) {
  if (!h || !low_res || !iou) return set_error("msam_mask_decode: null argument");
  return h->eng.mask_decode(sparse, n_sparse, dense, P, multimask, low_res, iou, (cudaStream_t)stream);
}
int msam_mask_stats(const float* low_res, int n_masks, int in_h, int in_w, int orig_h, int orig_w, float mask_threshold,
                    float stability_offset, int32_t* boxes_xyxy, float* stability, int32_t* area, void* stream) {
  // a negative stability_offset selects the generic (any-geometry) kernel with |offset| (used by the parity tests to
  // cross-check the 4x fast path)
  const bool generic = stability_offset < 0.f;
  return post_mask_stats(low_res, n_masks, in_h, in_w, orig_h, orig_w, mask_threshold, fabsf(stability_offset), boxes_xyxy,
                         stability, area, (cudaStream_t)stream, generic);
}
int msam_mask_stats_lazy(const float* low_res, int n_masks, int in_h, int in_w, int orig_h, int orig_w, float mask_threshold,
                         float stability_offset, const float* iou_preds, float pred_iou_thresh, uint8_t* done,
                         int32_t* boxes_xyxy, float* stability, int32_t* area, void* stream) {
  if (!iou_preds || !done) return set_error("msam_mask_stats_lazy: null argument");
  return post_mask_stats(low_res, n_masks, in_h, in_w, orig_h, orig_w, mask_threshold, fabsf(stability_offset), boxes_xyxy,
                         stability, area, (cudaStream_t)stream, stability_offset < 0.f, nullptr, iou_preds, pred_iou_thresh, done);
}
int msam_upsample_masks(const float* low_res, const int32_t* sel, int n_sel, int in_h, int in_w, int orig_h, int orig_w,
                        float mask_threshold, float* logits, uint8_t* binary, void* stream) {
  return post_upsample(low_res, sel, n_sel, in_h, in_w, orig_h, orig_w, mask_threshold, logits, binary, (cudaStream_t)stream);
}
int msam_remove_small_regions(uint8_t* masks, int n, int h, int w, int area_thresh, int holes, int32_t* changed,
                              int32_t* workspace, void* stream) {
  if (!masks || !changed || !workspace) return set_error("msam_remove_small_regions: null argument");
  return post_remove_small_regions(masks, n, h, w, area_thresh, holes, changed, workspace, (cudaStream_t)stream);
}
int msam_mask_boxes(const uint8_t* masks, int n, int h, int w, int32_t* boxes_xyxy, int32_t* area, void* stream) {
  if (!masks || !boxes_xyxy || !area) return set_error("msam_mask_boxes: null argument");
  return post_mask_boxes(masks, n, h, w, boxes_xyxy, area, (cudaStream_t)stream);
}
int msam_local_otsu_threshold(const float* low_res, int n_masks, float* thresholds, void* stream) {
  if (!low_res || !thresholds) return set_error("msam_local_otsu_threshold: null argument");
  return post_local_otsu(low_res, n_masks, thresholds, (cudaStream_t)stream);
}
int msam_mask_stats_ex(const float* low_res, int n_masks, int in_h, int in_w, int orig_h, int orig_w, const float* thresholds,
                       float stability_offset, int32_t* boxes_xyxy, float* stability, int32_t* area, void* stream) {
  if (!thresholds) return set_error("msam_mask_stats_ex: null thresholds");
  return post_mask_stats(low_res, n_masks, in_h, in_w, orig_h, orig_w, 0.f, fabsf(stability_offset), boxes_xyxy, stability, area,
                         (cudaStream_t)stream, stability_offset < 0.f, thresholds);
}
int msam_upsample_masks_ex(const float* low_res, const int32_t* sel, int n_sel, int in_h, int in_w, int orig_h, int orig_w,
                           const float* thresholds, float* logits, uint8_t* binary, void* stream) {
  if (!thresholds) return set_error("msam_upsample_masks_ex: null thresholds");
  return post_upsample(low_res, sel, n_sel, in_h, in_w, orig_h, orig_w, 0.f, logits, binary, (cudaStream_t)stream, thresholds);
}
int msam_paint_ex(const float* low_res, const int32_t* sel, const int32_t* boxes_xyxy, const int32_t* seg_ids, int n_sel,
                  int in_h, int in_w, int orig_h, int orig_w, const float* thresholds, int exclusive, uint32_t* label,
                  int ld_label, void* stream) {
  if (!thresholds) return set_error("msam_paint_ex: null thresholds");
  return post_paint(low_res, sel, boxes_xyxy, seg_ids, n_sel, in_h, in_w, orig_h, orig_w, 0.f, exclusive, label, ld_label,
                    (cudaStream_t)stream, thresholds);
}
int msam_paint(const float* low_res, const int32_t* sel, const int32_t* boxes_xyxy, const int32_t* seg_ids, int n_sel,
               int in_h, int in_w, int orig_h, int orig_w, float mask_threshold, int exclusive, uint32_t* label,
               int ld_label, void* stream) {
  return post_paint(low_res, sel, boxes_xyxy, seg_ids, n_sel, in_h, in_w, orig_h, orig_w, mask_threshold, exclusive, label,
                    ld_label, (cudaStream_t)stream);
}
int msam_amg_filter_nms(const int32_t* boxes_xyxy, const float* iou_preds, const float* stability, int n, int use_filters,
                        float pred_iou_thresh, float stability_thresh, float box_nms_thresh, const int32_t* crop_box_host,
                        const int32_t* orig_box_host, int32_t* keep, int32_t* n_keep, void* stream) {
  return post_filter_nms(boxes_xyxy, iou_preds, stability, n, use_filters, pred_iou_thresh, stability_thresh,
                         box_nms_thresh, crop_box_host, orig_box_host, keep, n_keep, (cudaStream_t)stream);
}

int msam_mask_loss_stats(const float* low_res, const uint8_t* targets, int n_obj, int M, int in_h, int in_w, int orig_h, int orig_w,
                         float* out5, void* stream) {
  if (!low_res || !targets || !out5) return set_error("msam_mask_loss_stats: null argument");
  return post_mask_loss_stats(low_res, targets, n_obj, M, in_h, in_w, orig_h, orig_w, out5, (cudaStream_t)stream);
}
int msam_prompt_targets(const void* labels, int label_dtype, int B, int H, int W, const int64_t* ids, const int32_t* n_ids, int n_obj,
                        double box_distortion, uint64_t seed, uint8_t* targets, int32_t* counts, int32_t* boxes, void* stream) {
  if (!labels || !ids || !n_ids || !targets || !counts || !boxes) return set_error("msam_prompt_targets: null argument");
  return prompt_targets(labels, label_dtype, B, H, W, ids, n_ids, n_obj, box_distortion, seed, targets, counts, boxes, (cudaStream_t)stream);
}
int msam_prompt_sample_points(const uint8_t* targets, const int32_t* counts, const int32_t* boxes, const int32_t* centers, int n,
                              int n_per_img, int H, int W, int n_pos, int n_neg, int dilation, uint64_t seed, uint8_t* scratch,
                              int32_t* coords, int32_t* labels, void* stream) {
  if (!targets || !counts || !boxes || !coords || !labels) return set_error("msam_prompt_sample_points: null argument");
  return prompt_sample_points(targets, counts, boxes, centers, n, n_per_img, H, W, n_pos, n_neg, dilation, seed, scratch, coords, labels,
                              (cudaStream_t)stream);
}
int msam_prompt_iterative(const uint8_t* targets, const float* low_res, const float* iou, int M, const uint8_t* pred, int n,
                          int n_per_img, int in_h, int in_w, int orig_h, int orig_w, uint64_t seed, int32_t* coords, int32_t* labels,
                          void* stream) {
  if (!targets || !coords || !labels) return set_error("msam_prompt_iterative: null argument");
  return prompt_iterative(targets, low_res, iou, M, pred, n, n_per_img, in_h, in_w, orig_h, orig_w, seed, coords, labels,
                          (cudaStream_t)stream);
}
int64_t msam_mask_prompts_workspace(int H, int W) { return H > 0 && W > 0 ? mask_prompts_workspace(H, W) : -1; }
int msam_mask_prompts(const uint8_t* mask, int H, int W, int ld, double box_extension, int want_logits, int point_mode, int max_points,
                      void* workspace, int64_t ws_bytes, int64_t* stats, float* box1024, float* logits, float* points, float* labels,
                      float* field, void* stream) {
  if (!mask || !workspace || !stats || (want_logits && !logits) || (point_mode && (!points || !labels)))
    return set_error("msam_mask_prompts: null argument");
  return mask_prompts(mask, H, W, ld, box_extension, want_logits, point_mode, max_points, workspace, ws_bytes, stats, box1024, logits,
                      points, labels, field, (cudaStream_t)stream);
}
int msam_mask_iou_counts(const uint8_t* a, int lda, const uint8_t* b, int ldb, int H, int W, int64_t* counts, void* stream) {
  if (!a || !b || !counts) return set_error("msam_mask_iou_counts: null argument");
  return mask_iou_counts(a, lda, b, ldb, H, W, counts, (cudaStream_t)stream);
}
int msam_shift_mask(const uint8_t* src, int ld_src, uint8_t* dst, int ld_dst, int H, int W, double dy, double dx, void* stream) {
  if (!src || !dst) return set_error("msam_shift_mask: null argument");
  return shift_mask(src, ld_src, dst, ld_dst, H, W, dy, dx, (cudaStream_t)stream);
}
int64_t msam_object_features_workspace(int n_ids) { return n_ids >= 0 ? object_features_workspace(n_ids) : -1; }
int msam_object_features(const float* emb, const int32_t* seg, int ld, int h, int w, int ry, int rx, int n_ids, void* workspace,
                         int64_t ws_bytes, double* sums, int64_t* areas, void* stream) {
  if (!emb || !seg || !workspace || !sums || !areas) return set_error("msam_object_features: null argument");
  return object_features(emb, seg, ld, h, w, ry, rx, n_ids, workspace, ws_bytes, sums, areas, (cudaStream_t)stream);
}
int msam_object_features_finish(const double* sums, const int64_t* areas, int n_ids, int out_f64, void* out, void* stream) {
  if (n_ids > 0 && (!sums || !areas || !out)) return set_error("msam_object_features_finish: null argument");
  return object_features_finish(sums, areas, n_ids, out_f64, out, (cudaStream_t)stream);
}
int msam_project_labels(const int64_t* seg, int64_t n, const int64_t* ids, const int64_t* values, int n_ids, int64_t* out, void* stream) {
  if (n > 0 && (!seg || !out || (n_ids > 0 && (!ids || !values)))) return set_error("msam_project_labels: null argument");
  return project_labels(seg, n, ids, values, n_ids, out, (cudaStream_t)stream);
}
int64_t msam_merge3d_workspace(int Z, int H, int W, int max_id, int max_edges) {
  return Z > 0 && H > 0 && W > 0 && max_id >= 0 && max_edges > 0 ? merge3d_workspace(Z, H, W, max_id, max_edges) : -1;
}
int msam_merge3d_range(const int32_t* seg, int Z, int H, int W, int32_t* out, void* stream) {
  if (!seg || !out) return set_error("msam_merge3d_range: null argument");
  return merge3d_range(seg, Z, H, W, out, (cudaStream_t)stream);
}
int msam_merge3d_close(const int32_t* seg, int Z, int H, int W, int gap_closing, int max_id, void* workspace, int64_t ws_bytes,
                       int32_t* out, uint8_t* closed, int32_t* out_max, void* stream) {
  if (!seg || !workspace || !out || !out_max) return set_error("msam_merge3d_close: null argument");
  return merge3d_close(seg, Z, H, W, gap_closing, max_id, workspace, ws_bytes, out, closed, out_max, (cudaStream_t)stream);
}
int msam_merge3d_edges(const int32_t* seg, int Z, int H, int W, void* workspace, int64_t ws_bytes, int max_edges, int32_t* edges,
                       int64_t* n_edges, void* stream) {
  if (!seg || !workspace || !edges || !n_edges) return set_error("msam_merge3d_edges: null argument");
  return merge3d_edges(seg, Z, H, W, workspace, ws_bytes, max_edges, edges, n_edges, (cudaStream_t)stream);
}
int msam_merge3d_gather(const int32_t* seg, int64_t n, const int32_t* node_labels, int n_nodes, int32_t* out, void* stream) {
  if (n > 0 && (!seg || !node_labels || !out)) return set_error("msam_merge3d_gather: null argument");
  return merge3d_gather(seg, n, node_labels, n_nodes, out, (cudaStream_t)stream);
}
int msam_merge3d_filter_z(int32_t* seg, int Z, int H, int W, int n_labels, int min_z_extent, void* workspace, int64_t ws_bytes,
                          void* stream) {
  if (!seg || !workspace) return set_error("msam_merge3d_filter_z: null argument");
  return merge3d_filter_z(seg, Z, H, W, n_labels, min_z_extent, workspace, ws_bytes, (cudaStream_t)stream);
}
int msam_stack_slice(const int32_t* src, int64_t n, int32_t* dst, int32_t* state, void* stream) {
  if (n > 0 && (!src || !dst || !state)) return set_error("msam_stack_slice: null argument");
  return stack_slice(src, n, dst, state, (cudaStream_t)stream);
}
int msam_multicut_gaec(int64_t n_nodes, int64_t n_edges, const int64_t* uv, const double* weights, int64_t* labels) {
  if (!labels || (n_edges > 0 && (!uv || !weights))) return set_error("msam_multicut_gaec: null argument");
  return multicut_gaec(n_nodes, n_edges, uv, weights, labels);
}
int msam_to_image(const void* src, int dtype, int h, int w, int c, uint8_t* out_hwc3, uint32_t* scratch6, void* stream) {
  return post_to_image(src, dtype, h, w, c, out_hwc3, scratch6, (cudaStream_t)stream);
}
int msam_paint_min_area(const float* low_res, const int32_t* sel, const int32_t* n_sel, const int32_t* boxes_xyxy,
                        const int32_t* area, int in_h, int in_w, int orig_h, int orig_w, float mask_threshold,
                        int32_t* label, int ld_label, void* stream) {
  return post_paint_min_area(low_res, sel, n_sel, boxes_xyxy, area, in_h, in_w, orig_h, orig_w, mask_threshold, label,
                             ld_label, (cudaStream_t)stream);
}
int msam_finish_segmentation(const int32_t* painted, int h, int w, int min_object_size, int with_background, uint32_t* out,
                             int32_t* workspace, void* stream) {
  return post_finish_segmentation(painted, h, w, min_object_size, with_background, out, workspace, (cudaStream_t)stream);
}

int msam_paint_canvas(const float* low_res, const int32_t* sel, const int32_t* global_pos, int n_sel,
                      const int32_t* boxes_xyxy, const int32_t* area, int in_h, int in_w, int crop_h, int crop_w,
                      float mask_threshold, int off_x, int off_y, uint64_t* canvas, int ld_canvas, void* stream) {
  return post_paint_canvas(low_res, sel, global_pos, n_sel, boxes_xyxy, area, in_h, in_w, crop_h, crop_w, mask_threshold,
                           off_x, off_y, reinterpret_cast<unsigned long long*>(canvas), ld_canvas, (cudaStream_t)stream);
}
int msam_canvas_to_label(const uint64_t* canvas, int64_t n, int32_t* label, void* stream) {
  return post_canvas_to_label(reinterpret_cast<const unsigned long long*>(canvas), (long)n, label, (cudaStream_t)stream);
}

int msam_mask_nms(const uint8_t* masks, int n, int h, int w, const float* boxes_xyxy, const float* scores, float nms_thresh,
                  int intersection_over_min, uint32_t* bits_ws, int32_t* areas, float* matrix_ws, int32_t* keep,
                  int32_t* n_keep, void* stream) {
  return post_mask_nms(masks, n, h, w, boxes_xyxy, scores, nms_thresh, intersection_over_min, bits_ws, areas, matrix_ws,
                       keep, n_keep, (cudaStream_t)stream);
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

int msam_op_gemm(const void* A, const void* W, int M, int N, int K, const float* bias, const float* residual,
                 int res_rows, void* out, int out_fp32, int act, void* stream) {
  GemmArgs a;
  a.A = (const __nv_bfloat16*)A; a.W = (const __nv_bfloat16*)W; a.M = M; a.N = N; a.K = K; a.lda = K; a.ldw = K;
  a.bias = bias; a.residual = residual; a.res_rows = res_rows; a.out = out; a.out_fp32 = out_fp32; a.act = act;
  return launch_gemm(a, sm_count(), (cudaStream_t)stream);
}

int msam_op_gemm_ex(const void* A, const void* W, int M, int N, int K, int lda, int ldw, const float* bias, const void* residual,
                    int res_rows, int ldr, int res_bf16, void* out, int ldc, int out_fp32, int act, int act_after_res, int epi,
                    const float* ln_gamma, const float* ln_beta, float ln_eps, int num_sms, void* stream) {
  return msam_op_gemm_ex2(A, W, M, N, K, lda, ldw, bias, residual, res_rows, ldr, res_bf16, out, ldc, out_fp32, act,
                          act_after_res, epi, ln_gamma, ln_beta, ln_eps, num_sms, GEMM_PATH_AUTO, stream);
}

int msam_op_gemm_ex2(const void* A, const void* W, int M, int N, int K, int lda, int ldw, const float* bias, const void* residual,
                     int res_rows, int ldr, int res_bf16, void* out, int ldc, int out_fp32, int act, int act_after_res, int epi,
                     const float* ln_gamma, const float* ln_beta, float ln_eps, int num_sms, int path, void* stream) {
  if (!A || !W || !out) return set_error("msam_op_gemm_ex: null argument");
  if (lda < K || ldw < K) return set_error("msam_op_gemm_ex: lda=%d / ldw=%d below K=%d", lda, ldw, K);
  if ((ldc > 0 && ldc < N) || (ldr > 0 && ldr < N)) return set_error("msam_op_gemm_ex: ldc=%d / ldr=%d below N=%d", ldc, ldr, N);
  GemmArgs a;
  a.A = (const __nv_bfloat16*)A; a.W = (const __nv_bfloat16*)W; a.M = M; a.N = N; a.K = K; a.lda = lda; a.ldw = ldw;
  a.bias = bias; a.residual = residual; a.res_rows = res_rows; a.ldr = ldr; a.res_bf16 = res_bf16;
  a.out = out; a.ldc = ldc; a.out_fp32 = out_fp32; a.act = act; a.act_after_res = act_after_res;
  a.epi = epi; a.ln_gamma = ln_gamma; a.ln_beta = ln_beta; a.ln_eps = ln_eps; a.path = path;
  return launch_gemm(a, num_sms > 0 ? num_sms : sm_count(), (cudaStream_t)stream);
}

int msam_op_gemm_tn(const void* A, const void* B, int M, int N, int K, float* out, void* stream) {
  if (!A || !B || !out) return set_error("msam_op_gemm_tn: null argument");
  return launch_gemm_tn((const __nv_bfloat16*)A, (const __nv_bfloat16*)B, M, N, K, M, N, out, N, (cudaStream_t)stream);
}

int msam_op_gemm_nn(const void* A, const void* B, int M, int N, int K, float* out, void* stream) {
  if (!A || !B || !out) return set_error("msam_op_gemm_nn: null argument");
  return launch_gemm_nn((const __nv_bfloat16*)A, (const __nv_bfloat16*)B, M, N, K, K, N, out, N, (cudaStream_t)stream);
}

int msam_op_layernorm(const float* x, int rows, int D, const float* gamma, const float* beta, float eps, void* out_bf16,
                      int window_mode, void* stream) {
  LnArgs l;
  l.x = x; l.rows = rows; l.D = D; l.gamma = gamma; l.beta = beta; l.eps = eps; l.out = (__nv_bfloat16*)out_bf16;
  l.window_mode = window_mode;
  return launch_layernorm(l, (cudaStream_t)stream);
}

int msam_op_attention(const void* qkv, const void* rel_table, void* out, int batch, int heads, int head_dim, int window,
                      float scale, void* stream) {
  AttnArgs a;
  a.qkv = (const __nv_bfloat16*)qkv; a.rel_table = (const __nv_bfloat16*)rel_table; a.out = (__nv_bfloat16*)out;
  a.batch = batch; a.heads = heads; a.head_dim = head_dim; a.grid = 64; a.window = window; a.scale = scale;
  return launch_attention(a, (cudaStream_t)stream);
}

// TinyViT kernels: every precondition the kernels rely on without checking it is refused here, before anything is launched.
static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int msam_op_tv_stem(const uint8_t* u8, const float* f32, int B, int hh, int ww, int img, const float* w27x32, const float* b32,
                    void* out_bf16, void* stream) {
  if ((u8 == nullptr) == (f32 == nullptr)) return set_error("msam_op_tv_stem: exactly one of u8 / f32 must be given");
  if (!w27x32 || !b32 || !out_bf16) return set_error("msam_op_tv_stem: null argument");
  if (B <= 0 || img <= 0 || img % 2) return set_error("msam_op_tv_stem: B=%d, img=%d (img must be even and positive)", B, img);
  if (u8 && (hh <= 0 || ww <= 0 || hh > img || ww > img))
    return set_error("msam_op_tv_stem: image %dx%d outside 1..%d", hh, ww, img);
  if (!aligned16(out_bf16)) return set_error("msam_op_tv_stem: out is not 16-byte aligned");
  return launch_tv_stem1(u8, f32, B, hh, ww, img, w27x32, b32, (__nv_bfloat16*)out_bf16, (cudaStream_t)stream);
}

static int tv_conv_args(const char* op, const void* x, int B, int Hin, int C, int stride, int cmul, const void* out) {
  if (!x || !out) return set_error("%s: null argument", op);
  if (B <= 0 || Hin <= 0 || C <= 0 || C % cmul) return set_error("%s: B=%d, Hin=%d, C=%d (C must be a multiple of %d)", op, B, Hin, C, cmul);
  if (stride != 1 && stride != 2) return set_error("%s: stride %d (1 or 2)", op, stride);
  if (stride == 2 && Hin % 2) return set_error("%s: odd Hin=%d with stride 2 (the kernel's output side is Hin / 2)", op, Hin);
  if (!aligned16(x) || !aligned16(out)) return set_error("%s: x / out not 16-byte aligned", op);
  return 0;
}

int msam_op_tv_im2col(const void* x_bf16, int B, int Hin, int C, int stride, void* out_bf16, void* stream) {
  if (tv_conv_args("msam_op_tv_im2col", x_bf16, B, Hin, C, stride, 8, out_bf16)) return -1;
  return launch_tv_im2col((const __nv_bfloat16*)x_bf16, B, Hin, C, stride, (__nv_bfloat16*)out_bf16, (cudaStream_t)stream);
}

int msam_op_tv_dwconv_bf16(const void* x_bf16, int B, int Hin, int C, int stride, const float* w9xC, const float* b, int act,
                           void* out_bf16, void* stream) {
  if (tv_conv_args("msam_op_tv_dwconv_bf16", x_bf16, B, Hin, C, stride, 8, out_bf16)) return -1;
  if (!w9xC || !b) return set_error("msam_op_tv_dwconv_bf16: null argument");
  if (!aligned16(w9xC) || !aligned16(b)) return set_error("msam_op_tv_dwconv_bf16: w / b not 16-byte aligned");
  return launch_tv_dwconv_bf16((const __nv_bfloat16*)x_bf16, B, Hin, C, stride, w9xC, b, act, (__nv_bfloat16*)out_bf16,
                               (cudaStream_t)stream);
}

int msam_op_tv_dwconv_f32(const float* x, int B, int Hin, int C, const float* w9xC, const float* b, float* out, void* stream) {
  if (tv_conv_args("msam_op_tv_dwconv_f32", x, B, Hin, C, 1, 4, out)) return -1;
  if (!w9xC || !b) return set_error("msam_op_tv_dwconv_f32: null argument");
  if (!aligned16(w9xC) || !aligned16(b)) return set_error("msam_op_tv_dwconv_f32: w / b not 16-byte aligned");
  return launch_tv_dwconv_f32(x, B, Hin, C, w9xC, b, out, (cudaStream_t)stream);
}

int msam_op_tv_ln_window(const float* x, int B, int H, int D, int ws, const float* gamma, const float* beta, float eps,
                         void* out_bf16, void* stream) {
  if (!x || !gamma || !beta || !out_bf16) return set_error("msam_op_tv_ln_window: null argument");
  if (B <= 0 || H <= 0 || D <= 0 || D % 4 || D > 384)
    return set_error("msam_op_tv_ln_window: B=%d, H=%d, D=%d (D a multiple of 4, at most 384)", B, H, D);
  if (ws != 7 && ws != 14) return set_error("msam_op_tv_ln_window: window %d (7 or 14)", ws);
  if (!aligned16(x) || !aligned16(gamma) || !aligned16(beta) || ((uintptr_t)out_bf16 & 7))
    return set_error("msam_op_tv_ln_window: misaligned pointer");
  return launch_tv_ln_window(x, B, H, D, ws, gamma, beta, eps, (__nv_bfloat16*)out_bf16, (cudaStream_t)stream);
}

int msam_op_tv_attention(const void* qkv_bf16, const float* bias_tab, int B, int H, int ws, int heads, void* out_bf16,
                         void* stream) {
  if (!qkv_bf16 || !bias_tab || !out_bf16) return set_error("msam_op_tv_attention: null argument");
  if (B <= 0 || H <= 0 || heads <= 0 || heads > 65535) return set_error("msam_op_tv_attention: B=%d, H=%d, heads=%d", B, H, heads);
  if (ws != 7 && ws != 14) return set_error("msam_op_tv_attention: window %d (7 or 14)", ws);
  if (!aligned16(qkv_bf16) || !aligned16(out_bf16)) return set_error("msam_op_tv_attention: qkv / out not 16-byte aligned");
  return launch_tv_attention((const __nv_bfloat16*)qkv_bf16, bias_tab, B, H, ws, heads, (__nv_bfloat16*)out_bf16,
                             (cudaStream_t)stream);
}

int msam_op_dec_t2i(msam_handle* h, int which, const void* q_pe, const void* keys, int P, int T, void* out, int num_sms,
                    void* stream) {
  if (!h) return set_error("msam_op_dec_t2i: null handle");
  return h->eng.op_dec_t2i(which, (const __nv_bfloat16*)q_pe, (const __nv_bfloat16*)keys, P, T, (__nv_bfloat16*)out, num_sms,
                           (cudaStream_t)stream);
}
int msam_op_dec_i2t(msam_handle* h, int layer, const void* queries, const void* q_pe, int shared, void* keys, int P, int T,
                    int num_sms, void* stream) {
  if (!h) return set_error("msam_op_dec_i2t: null handle");
  return h->eng.op_dec_i2t(layer, (const __nv_bfloat16*)queries, (const __nv_bfloat16*)q_pe, shared, (__nv_bfloat16*)keys, P, T,
                           num_sms, (cudaStream_t)stream);
}
int msam_op_dec_upscale(msam_handle* h, const void* keys, const float* hyper_in, int P, int multimask, float* low_res,
                        int num_sms, void* stream) {
  if (!h) return set_error("msam_op_dec_upscale: null handle");
  return h->eng.op_dec_upscale((const __nv_bfloat16*)keys, hyper_in, P, multimask, low_res, num_sms, (cudaStream_t)stream);
}

int msam_encode_train(msam_handle* h, const float* nchw, int B, float* out, void* stream) {
  if (!h || !nchw || !out) return set_error("msam_encode_train: null argument");
  return h->eng.encode_train(nchw, B, out, (cudaStream_t)stream);
}
int msam_encode_backward(msam_handle* h, const float* d_out, void* stream) {
  if (!h || !d_out) return set_error("msam_encode_backward: null argument");
  return h->eng.encode_backward(d_out, (cudaStream_t)stream);
}
int msam_decoder_train_forward(msam_handle* h, int slot, const float* emb_nchw, const float* sparse, const int32_t* emb_index, int n_sparse,
                               int P, int multimask, float* low_res, float* iou, void* stream) {
  return msam_decoder_train_forward_ex(h, slot, emb_nchw, sparse, emb_index, n_sparse, P, nullptr, multimask, low_res, iou, stream);
}
int msam_decoder_train_forward_ex(msam_handle* h, int slot, const float* emb_nchw, const float* sparse, const int32_t* emb_index,
                                  int n_sparse, int P, const float* mask_input, int multimask, float* low_res, float* iou, void* stream) {
  if (!h || !emb_nchw || !low_res || !iou) return set_error("msam_decoder_train_forward: null argument");
  return h->eng.decoder_train_forward(slot, emb_nchw, sparse, emb_index, n_sparse, P, mask_input, multimask, low_res, iou,
                                      (cudaStream_t)stream);
}
int msam_decoder_train_forward_images(msam_handle* h, int slot, const float* emb_nchw, int B, int multimask, float* low_res, float* iou,
                                      void* stream) {
  if (!h || !emb_nchw || !low_res || !iou) return set_error("msam_decoder_train_forward_images: null argument");
  return h->eng.decoder_train_forward_images(slot, emb_nchw, B, multimask, low_res, iou, (cudaStream_t)stream);
}
int msam_op_mask_downscaling_train(msam_handle* h, const float* mask, int P, const float* d_dense, float* dense_out, float* grads_out,
                                   void* stream) {
  if (!h || !mask || !d_dense || !dense_out || !grads_out) return set_error("msam_op_mask_downscaling_train: null argument");
  return h->eng.op_mask_downscaling_train(mask, P, d_dense, dense_out, grads_out, (cudaStream_t)stream);
}
int msam_decoder_train_backward(msam_handle* h, int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, void* stream) {
  if (!h || !d_emb_nchw) return set_error("msam_decoder_train_backward: null argument");
  return h->eng.decoder_train_backward(slot, d_low_res, d_iou, d_emb_nchw, (cudaStream_t)stream);
}
int msam_decoder_zero_grads(msam_handle* h, void* stream) {
  if (!h) return set_error("msam_decoder_zero_grads: null handle");
  return h->eng.decoder_zero_grads((cudaStream_t)stream);
}
int msam_mask_loss_backward(const float* low_res, const uint8_t* targets, const float* d_stats, int n_obj, int M, int in_h, int in_w,
                            int orig_h, int orig_w, float* d_low_res, void* stream) {
  return post_mask_loss_backward(low_res, targets, d_stats, n_obj, M, in_h, in_w, orig_h, orig_w, d_low_res, (cudaStream_t)stream);
}
int msam_optimizer_step(msam_handle* h, float lr, float beta1, float beta2, float eps, float weight_decay, void* stream) {
  if (!h) return set_error("msam_optimizer_step: null handle");
  return h->eng.optimizer_step(lr, beta1, beta2, eps, weight_decay, (cudaStream_t)stream);
}
int msam_optimizer_step_prefix(msam_handle* h, const char* prefix, float lr, float beta1, float beta2, float eps, float weight_decay,
                               void* stream) {
  if (!h || !prefix || !*prefix) return set_error("msam_optimizer_step_prefix: null handle or empty prefix");
  return h->eng.optimizer_step(lr, beta1, beta2, eps, weight_decay, (cudaStream_t)stream, prefix);
}
int msam_train_tensor_count(msam_handle* h) { return h ? (int)h->eng.opt.size() : -1; }
int msam_train_tensor_info(msam_handle* h, int i, char* key_buf, int cap, void** grad, void** master, int64_t* n) {
  if (!h || i < 0 || i >= (int)h->eng.opt.size() || !key_buf || cap < 2) return set_error("msam_train_tensor_info: bad argument");
  const OptParam& p = h->eng.opt[i];
  snprintf(key_buf, cap, "%s", p.key.c_str());
  if (grad) *grad = p.g;
  if (master) *master = p.w;
  if (n) *n = p.n;
  return 0;
}
int msam_op_bgemm(const void* A, const void* B, int a_mn, int b_mn, int M, int N, int K, int lda, int ldb, int64_t a_hstride,
                  int64_t a_wstride, int64_t b_hstride, int64_t b_wstride, int heads, int outer, float* out, int ldc,
                  int64_t o_hstride, int64_t o_wstride, float alpha, int accumulate, void* stream) {
  BGemmArgs a;
  a.A = (const __nv_bfloat16*)A; a.B = (const __nv_bfloat16*)B; a.a_mn = a_mn; a.b_mn = b_mn; a.M = M; a.N = N; a.K = K;
  a.lda = lda; a.ldb = ldb; a.a_hstride = a_hstride; a.a_wstride = a_wstride; a.b_hstride = b_hstride; a.b_wstride = b_wstride;
  a.heads = heads; a.outer = outer; a.out = out; a.ldc = ldc; a.o_hstride = o_hstride; a.o_wstride = o_wstride; a.alpha = alpha;
  a.accumulate = accumulate;
  return launch_bgemm(a, (cudaStream_t)stream);
}
int msam_op_layernorm_bwd(const float* x, int rows, int D, const float* gamma, float eps, const float* dy, int window_mode,
                          int accumulate, float* dx, float* dgamma, float* dbeta, void* stream) {
  return launch_layernorm_bwd(x, rows, D, gamma, eps, dy, window_mode, 64, 14, accumulate, dx, dgamma, dbeta, (cudaStream_t)stream);
}

// ---- element-wise / row-wise stages of the encoder backward pass (backward.cu), one entry point per launcher
static int attn_bwd_pitches_ok(const char* who, const AttnBwdGeom& g, long n_batch, int pitch_s, int pitch_p) {
  if (n_batch <= 0) return set_error("%s: n_batch=%ld", who, n_batch);
  if (pitch_s < g.n_tok || pitch_p < g.n_tok) return set_error("%s: pitch_s=%d / pitch_p=%d below %d keys", who, pitch_s, pitch_p, g.n_tok);
  return 0;
}
int msam_op_attn_probs(const float* S, const float* T, int64_t n_batch, int global, int pitch_s, int pitch_p, float scale, void* P,
                       void* stream) {
  if (!S || !T || !P) return set_error("msam_op_attn_probs: null argument");
  const AttnBwdGeom g = rel_table_geom(global != 0, 14, 64);
  if (attn_bwd_pitches_ok("msam_op_attn_probs", g, (long)n_batch, pitch_s, pitch_p)) return -1;
  return launch_attn_probs(S, T, (long)n_batch, g, pitch_s, pitch_p, scale, (__nv_bfloat16*)P, (cudaStream_t)stream);
}
int msam_op_attn_ds(const void* P, const float* dP, int64_t n_batch, int global, int pitch_s, int pitch_p, void* dS, void* dT,
                    void* stream) {
  if (!P || !dP || !dS || !dT) return set_error("msam_op_attn_ds: null argument");
  const AttnBwdGeom g = rel_table_geom(global != 0, 14, 64);
  if (attn_bwd_pitches_ok("msam_op_attn_ds", g, (long)n_batch, pitch_s, pitch_p)) return -1;
  return launch_attn_ds((const __nv_bfloat16*)P, dP, (long)n_batch, g, pitch_s, pitch_p, (__nv_bfloat16*)dS, (__nv_bfloat16*)dT,
                        (cudaStream_t)stream);
}
int msam_op_pack_dqkv(const float* dq, const float* dk, const float* dv, int outer, int heads, int T, int d, void* dqkv, void* stream) {
  if (!dq || !dk || !dv || !dqkv) return set_error("msam_op_pack_dqkv: null argument");
  if (outer <= 0 || heads <= 0 || T <= 0 || d <= 0 || d % 4) return set_error("msam_op_pack_dqkv: d=%d must be a positive multiple of 4", d);
  return launch_pack_dqkv(dq, dk, dv, outer, heads, T, d, (__nv_bfloat16*)dqkv, (cudaStream_t)stream);
}
int msam_op_gelu_bwd(const void* dh, const void* pre, int64_t n, void* dpre, void* stream) {
  if (!dh || !pre || !dpre) return set_error("msam_op_gelu_bwd: null argument");
  if (n <= 0) return set_error("msam_op_gelu_bwd: n=%lld", (long long)n);
  return launch_gelu_bwd((const __nv_bfloat16*)dh, (const __nv_bfloat16*)pre, (long)n, (__nv_bfloat16*)dpre, (cudaStream_t)stream);
}
int msam_op_colsum(const void* x, int64_t rows, int N, float* out, void* stream) {
  if (!x || !out) return set_error("msam_op_colsum: null argument");
  if (rows <= 0 || N <= 0) return set_error("msam_op_colsum: rows=%lld N=%d", (long long)rows, N);
  return launch_colsum((const __nv_bfloat16*)x, (long)rows, N, out, (cudaStream_t)stream);
}
int msam_op_window_gather(const void* x, int B, int D, void* out_win, void* stream) {
  if (!x || !out_win) return set_error("msam_op_window_gather: null argument");
  if (B <= 0 || D <= 0 || D % 8) return set_error("msam_op_window_gather: D=%d must be a positive multiple of 8", D);
  return launch_window_gather((const __nv_bfloat16*)x, B, 64, 14, D, (__nv_bfloat16*)out_win, (cudaStream_t)stream);
}
int msam_op_col2im3x3(const void* dcol, int B, int g, int C, float* out, void* stream) {
  if (!dcol || !out) return set_error("msam_op_col2im3x3: null argument");
  if (B <= 0 || g <= 0 || C <= 0 || C % 8) return set_error("msam_op_col2im3x3: C=%d must be a positive multiple of 8", C);
  return launch_col2im3x3((const __nv_bfloat16*)dcol, B, g, C, out, (cudaStream_t)stream);
}
int msam_op_sum_batch(const float* x, int64_t n_batch, int64_t n, float* out, int accumulate, void* stream) {
  if (!x || !out) return set_error("msam_op_sum_batch: null argument");
  if (n_batch <= 0 || n <= 0) return set_error("msam_op_sum_batch: n_batch=%lld n=%lld", (long long)n_batch, (long long)n);
  return launch_sum_batch(x, (long)n_batch, (long)n, out, accumulate, (cudaStream_t)stream);
}
int msam_op_transpose_bf16(const void* in, int rows, int cols, void* out, void* stream) {
  if (!in || !out) return set_error("msam_op_transpose_bf16: null argument");
  if (rows <= 0 || cols <= 0) return set_error("msam_op_transpose_bf16: rows=%d cols=%d", rows, cols);
  return launch_transpose_bf16((const __nv_bfloat16*)in, rows, cols, (__nv_bfloat16*)out, (cudaStream_t)stream);
}

// debug hook: device buffer of 64 x 16 uint64 phase timestamps, or NULL to switch off
int msam_debug_attn_trace(void* dev_buf) {
  set_attn_trace((unsigned long long*)dev_buf);
  return 0;
}

}  // extern "C"
