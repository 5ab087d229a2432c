// Optimizer of the fine-tuning step (cfg 5): AdamW (torch.optim.AdamW semantics: decoupled weight decay, bias-corrected moments) over
// fp32 master weights on the device, then refresh of the operands the training paths read (bf16 casts, transposes for the dgrad
// GEMMs, rel-pos tables, tiled conv-transpose biases).  The tensors are registered by encoder_train.cu / decoder_train.cu when
// their gradient buffers are created.  Reference: micro_sam/training/training.py:train_sam (AdamW) driven by sam_trainer.py:393.
#include "engine.h"

#include <cmath>
#include <cstring>

namespace msam {

namespace {

__global__ void adamw_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long n, float lr,
                             float b1, float b2, float eps, float wd, float c1, float c2) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  float wi = w[i];
  wi -= lr * wd * wi;
  const float mi = b1 * m[i] + (1.f - b1) * gi;
  const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi; v[i] = vi;
  wi -= lr * (mi / c1) / (sqrtf(vi / c2) + eps);
  w[i] = wi;
}
// out[s * co + o] = b[o] for the 4 sub-pixels s
__global__ void tile4_kernel(const float* __restrict__ b, int co, float* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= co) return;
  const float v = b[o];
  out[o] = v; out[co + o] = v; out[2 * co + o] = v; out[3 * co + o] = v;
}
// rows [row_off, row_off + rows) of a rel-pos table tile [NT, cols_pad] <- fp32 [rows, cols]
__global__ void rel_rows_kernel(const float* __restrict__ w, int rows, int cols, int cols_pad, int row_off, __nv_bfloat16* __restrict__ tab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  tab[(long)(row_off + i / cols) * cols_pad + i % cols] = __float2bfloat16(w[i]);
}

}  // namespace

float* Engine::train_add(OptParam p, const float* init) {
  if (!p.w) {
    if (!init) {
      auto it = dec_host.find(p.key);
      if (it == dec_host.end() || (int64_t)it->second.data.size() != p.n) {
        set_error("training: no host copy of '%s' with %lld elements", p.key.c_str(), (long long)p.n);
        return nullptr;
      }
      init = it->second.data.data();
    }
    if (!(p.w = upload_f32(init, (size_t)p.n))) return nullptr;
  }
  if (!p.g && !(p.g = (float*)dalloc((size_t)p.n * 4, true))) return nullptr;
  opt.push_back(p);
  return p.g;
}

int Engine::optimizer_step(float lr, float b1, float b2, float eps, float wd, cudaStream_t st, const char* prefix) {
  if (opt.empty()) return set_error("msam_optimizer_step: no trainable tensors registered (run a training forward / backward first)");
  if (prefix) per_tensor_counts = true;
  else ++opt_step_count;
  const float c1 = 1.f - powf(b1, (float)opt_step_count), c2 = 1.f - powf(b2, (float)opt_step_count);
  const size_t plen = prefix ? strlen(prefix) : 0;
  for (const OptParam& p : opt)   // a skipped tensor falls behind the step count: from now on each tensor counts its own updates
    if (p.skip && *p.skip) per_tensor_counts = true;
  for (OptParam& p : opt) {
    if (prefix && p.key.compare(0, plen, prefix) != 0) continue;
    if (p.skip && *p.skip) continue;
    float c1p = c1, c2p = c2;
    if (p.written) {
      if (!*p.written) continue;
      ++p.steps;
      c1p = 1.f - powf(b1, (float)p.steps); c2p = 1.f - powf(b2, (float)p.steps);
    }
    ++p.count;
    if (per_tensor_counts) {   // torch.optim.AdamW: a parameter's step counts only the steps that updated it
      c1p = 1.f - powf(b1, (float)p.count); c2p = 1.f - powf(b2, (float)p.count);
    }
    if (!p.m) {
      p.m = (float*)dalloc((size_t)p.n * 4, true);
      p.v = (float*)dalloc((size_t)p.n * 4, true);
      if (!p.m || !p.v) return -1;
    }
    adamw_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, st>>>(p.w, p.g, p.m, p.v, p.n, lr, b1, b2, eps, wd, c1p, c2p);
    LAUNCH_CHECK("adamw");
    switch (p.refresh) {
      case Refresh::None:
        break;
      case Refresh::Cast:
        RUN(launch_cast_bf16(p.w, p.n, p.dst, st));
        break;
      case Refresh::RelPosRows:
        rel_rows_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, st>>>(p.w, p.rows, p.cols, p.cols_pad, p.row_off, p.dst);
        LAUNCH_CHECK("rel_rows");
        break;
      case Refresh::TileBias4:
        tile4_kernel<<<(unsigned)((p.n + 127) / 128), 128, 0, st>>>(p.w, (int)p.n, p.dst4);
        LAUNCH_CHECK("tile4");
        break;
    }
    if (p.dstT) RUN(launch_transpose_bf16(p.dst, p.rows, p.cols, p.dstT, st));
  }
  RUN(dec_train_refresh_prompt_tables(st));
  train_invalidate();   // the saved encoder forward pass belongs to the old weights
  return 0;
}

}  // namespace msam

extern "C" int msam_op_adamw(float* w, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                             float weight_decay, int step, void* stream) {
  using namespace msam;
  if (!w || !g || !m || !v) return set_error("msam_op_adamw: null argument");
  if (n <= 0 || step <= 0) return set_error("msam_op_adamw: %lld elements, step %d", (long long)n, step);
  const float c1 = 1.f - powf(beta1, (float)step), c2 = 1.f - powf(beta2, (float)step);
  adamw_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, g, m, v, n, lr, beta1, beta2, eps, weight_decay, c1, c2);
  LAUNCH_CHECK("adamw");
  return 0;
}
