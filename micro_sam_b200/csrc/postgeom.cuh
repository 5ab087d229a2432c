// Sam.postprocess_masks evaluated per pixel from the 256 x 256 low-res logits (bilinear 256 -> 1024, crop to input_size,
// bilinear -> original_size, align_corners=False), shared by the post-processing kernels (postprocess.cu) and the prompt
// sampler (prompts.cu) so that every consumer sees the same value at every pixel.
#pragma once
#include "kernels.h"

namespace msam {

struct Interp {  // one axis of F.interpolate(mode="bilinear", align_corners=False)
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Interp interp_axis(int dst, float scale, int in_size) {
  float src = scale * ((float)dst + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  Interp r;
  r.i0 = (int)src;
  if (r.i0 > in_size - 1) r.i0 = in_size - 1;
  r.i1 = r.i0 + ((r.i0 < in_size - 1) ? 1 : 0);
  r.l1 = src - (float)r.i0;
  r.l0 = 1.f - r.l1;
  return r;
}
__device__ __forceinline__ float bilerp(float v00, float v01, float v10, float v11, const Interp& y, const Interp& x) {
  return y.l0 * (x.l0 * v00 + x.l1 * v01) + y.l1 * (x.l0 * v10 + x.l1 * v11);
}

struct PostGeom {
  int lr;              // low-res side (256)
  int img;             // model input side (1024)
  int in_h, in_w;      // input_size (resized image before padding)
  int out_h, out_w;    // original_size
  float s1;            // lr / img
  float s2y, s2x;      // in_h / out_h, in_w / out_w
  int identity2;       // second interpolation is the identity (in == out)
};

// stage 1 value at (Y, X) of the img x img grid
__device__ __forceinline__ float stage1(const float* __restrict__ lr, const PostGeom& g, int Y, int X) {
  const Interp iy = interp_axis(Y, g.s1, g.lr), ix = interp_axis(X, g.s1, g.lr);
  const float* r0 = lr + iy.i0 * g.lr;
  const float* r1 = lr + iy.i1 * g.lr;
  return bilerp(__ldg(r0 + ix.i0), __ldg(r0 + ix.i1), __ldg(r1 + ix.i0), __ldg(r1 + ix.i1), iy, ix);
}
__device__ __forceinline__ float full_res(const float* __restrict__ lr, const PostGeom& g, int y, int x) {
  if (g.identity2) return stage1(lr, g, y, x);
  const Interp iy = interp_axis(y, g.s2y, g.in_h), ix = interp_axis(x, g.s2x, g.in_w);
  return bilerp(stage1(lr, g, iy.i0, ix.i0), stage1(lr, g, iy.i0, ix.i1), stage1(lr, g, iy.i1, ix.i0),
                stage1(lr, g, iy.i1, ix.i1), iy, ix);
}

static inline int make_geom(int in_h, int in_w, int out_h, int out_w, PostGeom* g) {
  if (in_h <= 0 || in_w <= 0 || out_h <= 0 || out_w <= 0 || in_h > 1024 || in_w > 1024)
    return set_error("postprocess: bad sizes input=(%d,%d) original=(%d,%d)", in_h, in_w, out_h, out_w);
  g->lr = 256; g->img = 1024; g->in_h = in_h; g->in_w = in_w; g->out_h = out_h; g->out_w = out_w;
  g->s1 = 256.f / 1024.f;
  g->s2y = (float)in_h / (float)out_h;
  g->s2x = (float)in_w / (float)out_w;
  g->identity2 = (in_h == out_h && in_w == out_w);
  return 0;
}

}  // namespace msam
