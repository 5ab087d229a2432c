// Optimizer of the fine-tuning step (cfg 5): AdamW (torch.optim.AdamW semantics: decoupled weight decay, bias-corrected moments) over
// fp32 master weights on the device, then refresh of the packed operands the training paths read (bf16 casts, transposes for the
// dgrad GEMMs, rel-pos tables, the 3x3 neck conv layout).  The tensors are registered by encoder_train.cu / decoder_train.cu when
// their gradient buffers are created.  Reference: micro_sam/training/training.py:train_sam (AdamW) driven by sam_trainer.py:393.
#include "engine.h"

#include <cmath>

namespace msam {

#define RUN(x) do { if (x) return -1; } while (0)

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
// conv-transpose bias kept as 4 tiles (one per sub-pixel): g[s * co + o] <- sum over the 4 tiles
__global__ void fold4_kernel(float* __restrict__ g, int co) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= co) return;
  const float s = g[o] + g[co + o] + g[2 * co + o] + g[3 * co + o];
  g[o] = s; g[co + o] = s; g[2 * co + o] = s; g[3 * co + o] = s;
}
// rows [row_off, row_off + rows) of a rel-pos table tile [NT, cols_pad] <- fp32 [rows, cols]
__global__ void rel_rows_kernel(const float* __restrict__ w, int rows, int cols, int cols_pad, int row_off, __nv_bfloat16* __restrict__ tab) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  tab[(long)(row_off + i / cols) * cols_pad + i % cols] = __float2bfloat16(w[i]);
}
// upstream conv weight [o][c][k] fp32 -> GEMM operand [o][k][c] bf16
__global__ void neck2_pack_kernel(const float* __restrict__ w, int C, __nv_bfloat16* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)C * C * 9) return;
  const int c = i % C, k = (i / C) % 9, o = i / (9 * C);
  out[i] = __float2bfloat16(w[((long)o * C + c) * 9 + k]);
}

}  // namespace

float* Engine::opt_master_from_host(const std::string& key, int64_t n) {
  auto it = dec_host.find(key);
  if (it == dec_host.end() || (int64_t)it->second.data.size() != n) {
    set_error("optimizer: no host copy of '%s' with %lld elements", key.c_str(), (long long)n);
    return nullptr;
  }
  return upload_f32(it->second.data.data(), (size_t)n);
}

int Engine::optimizer_step(float lr, float b1, float b2, float eps, float wd, cudaStream_t st) {
  if (opt.empty()) return set_error("msam_optimizer_step: no trainable tensors registered (run a training forward / backward first)");
  ++opt_step_count;
  const float c1 = 1.f - powf(b1, (float)opt_step_count), c2 = 1.f - powf(b2, (float)opt_step_count);
  for (OptParam& p : opt) {
    float c1p = c1, c2p = c2;
    if (p.written) {
      if (!*p.written) continue;
      ++p.steps;
      c1p = 1.f - powf(b1, (float)p.steps); c2p = 1.f - powf(b2, (float)p.steps);
    }
    if (!p.m) {
      p.m = (float*)dalloc((size_t)p.n * 4, true);
      p.v = (float*)dalloc((size_t)p.n * 4, true);
      if (!p.m || !p.v) return -1;
    }
    if (p.refresh == 6) fold4_kernel<<<(p.n / 4 + 127) / 128, 128, 0, st>>>(p.g, (int)(p.n / 4));
    adamw_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, st>>>(p.w, p.g, p.m, p.v, p.n, lr, b1, b2, eps, wd, c1p, c2p);
    count_launch();
    switch (p.refresh) {
      case 1:
        RUN(launch_cast_bf16(p.w, p.n, p.dst, st));
        break;
      case 3:
        rel_rows_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, st>>>(p.w, p.rows, p.cols, p.cols_pad, p.row_off, p.dst);
        break;
      case 4:
        neck2_pack_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, st>>>(p.w, p.rows, p.dst);
        break;
      default:
        break;
    }
    if (p.dstT) RUN(launch_transpose_bf16(p.dst, p.rows, p.cols, p.dstT, st));
  }
  // embedding tables shared with the inference prompt encoder (it produces the sparse tokens of the training path as well)
  const float *pe = nullptr, *nap = nullptr;
  for (const OptParam& p : opt)
    if (p.refresh == 5) { if (p.n == 4 * 256) pe = p.w; else nap = p.w; }
  if (pe || nap) RUN(dec_set_prompt_tables(pe, nap, st));
  train_invalidate();   // the saved encoder forward pass belongs to the old weights
  if (cudaGetLastError() != cudaSuccess) return set_error("optimizer step: kernel launch failed");
  return 0;
}

int Engine::train_param(const char* key, float* dst, int64_t n, cudaStream_t st) {
  for (const OptParam& p : opt)
    if (p.key == key) {
      if (p.n != n) return set_error("msam_train_param: '%s' has %lld elements, caller expects %lld", key, (long long)p.n, (long long)n);
      if (cudaMemcpyAsync(dst, p.w, (size_t)n * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) return set_error("msam_train_param: copy failed");
      return 0;
    }
  return set_error("msam_train_param: no trainable tensor named '%s'", key);
}

}  // namespace msam
