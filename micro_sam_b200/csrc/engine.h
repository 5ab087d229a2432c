// Engine: model container behind the opaque msam_handle.
#pragma once
#include <initializer_list>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_fp16.h>

#include "../../include/msam_b200.h"
#include "kernels.h"
#include "tensormap.h"

namespace msam {

struct HostTensor {
  std::vector<int64_t> shape;
  std::vector<float> data;
};

struct EncBlock {
  bool global = false;
  float *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
  __nv_bfloat16 *qkv_w = nullptr, *proj_w = nullptr, *fc1_w = nullptr, *fc2_w = nullptr, *rel_table = nullptr;
  float *qkv_b = nullptr, *proj_b = nullptr, *fc1_b = nullptr, *fc2_b = nullptr;
};

struct EncoderWeights {
  __nv_bfloat16* patch_w = nullptr;
  float *patch_b = nullptr, *pos_embed = nullptr;
  std::vector<EncBlock> blocks;
  __nv_bfloat16 *neck_conv1 = nullptr, *neck_conv2 = nullptr;
  float *neck_ln1_g = nullptr, *neck_ln1_b = nullptr, *neck_ln2_g = nullptr, *neck_ln2_b = nullptr;
};

struct EncoderWorkspace {
  __nv_bfloat16 *patches = nullptr, *xn = nullptr, *xn_win = nullptr, *qkv = nullptr, *attn = nullptr, *hidden = nullptr;
  float* x = nullptr;
  float *neck1 = nullptr, *neck2 = nullptr;
  __nv_bfloat16 *neck1b = nullptr, *neck_col = nullptr;
};

// ---- TinyViT (vit_t) encoder, tinyvit.cu
struct TvConv {                       // Conv2d_BN with the BatchNorm folded in
  __nv_bfloat16* w = nullptr;         // dense / 1x1: GEMM operand [out, in * k * k]
  float* wf = nullptr;                // depth-wise 3x3: [9][C]; stem conv 1: [27][32]
  float* b = nullptr;
};
struct TvMBConv { TvConv conv1, conv2, conv3; };
struct TvMerge { TvConv conv1, conv2, conv3; };
struct TvBlock {
  float *an_g = nullptr, *an_b = nullptr, *mn_g = nullptr, *mn_b = nullptr, *bias_tab = nullptr;
  __nv_bfloat16 *qkv_w = nullptr, *proj_w = nullptr, *fc1_w = nullptr, *fc2_w = nullptr;
  float *qkv_b = nullptr, *proj_b = nullptr, *fc1_b = nullptr, *fc2_b = nullptr;
  TvConv local;
};
struct TvStage { int dim = 0, heads = 0, ws = 0; std::vector<TvBlock> blocks; };
struct TinyVit {
  TvConv stem1, stem2;
  TvMBConv mb[2];
  TvMerge merge[3];
  TvStage stage[4];                   // [1..3] used
  __nv_bfloat16 *s1 = nullptr, *col = nullptr, *a0 = nullptr, *a1 = nullptr, *h1 = nullptr, *h2 = nullptr, *xw = nullptr,
                *qkv = nullptr, *attn = nullptr, *xn = nullptr;
  float *x = nullptr, *x2 = nullptr;
};

// One trainable tensor of the optimizer (train_opt.cu): fp32 master weights (the live parameter buffer itself when the kernels read
// fp32: biases, LayerNorm, embedding tables), its gradient, AdamW moments, and how the packed operands are refreshed after an update.
struct OptParam {
  std::string key;              // gradient key: upstream name, or "<name>@gemm" / "@stack" for packed layouts
  float *w = nullptr, *g = nullptr, *m = nullptr, *v = nullptr;
  int64_t n = 0;
  const bool* written = nullptr;  // non-null: AdamW skips the tensor while *written is false (no gradient since the last zeroing)
  int64_t steps = 0;              // ... and counts its own steps for the bias correction (with written only)
  int refresh = 0;              // 0 none | 1 cast -> dst | 2 cast -> dst + transpose -> dstT | 3 rows of a rel-pos table | 4 neck 3x3 conv
                                // relayout | 5 prompt-encoder tables of the inference decoder | 6 conv-transpose bias (fold the 4 tiles first)
  __nv_bfloat16 *dst = nullptr, *dstT = nullptr;
  int rows = 0, cols = 0, cols_pad = 0, row_off = 0;
};

struct DecoderState;  // decoder.cu
struct TrainState;    // encoder_train.cu
struct DecTrain;      // decoder_train.cu

struct Engine {
  msam_config cfg{};
  int device = 0, num_sms = 132;
  bool finalized = false;
  std::unordered_map<std::string, HostTensor> host_weights;
  std::vector<void*> allocs;
  EncoderWeights enc;
  EncoderWorkspace ws;
  TinyVit tv;
  bool is_tinyvit() const { return cfg.depth == 0; }
  DecoderState* dec = nullptr;
  TrainState* train = nullptr;
  DecTrain* dtrain = nullptr;
  std::unordered_map<std::string, HostTensor> dec_host;   // host fp32 copies of every weight, kept for the training paths (masters, decoder_train.cu operands)
  std::vector<OptParam> opt;
  int64_t opt_step_count = 0;

  void* dalloc(size_t bytes, bool zero = false);
  const std::vector<float>* host(const std::string& name, std::initializer_list<int64_t> shape);
  __nv_bfloat16* upload_bf16(const float* src, size_t n);
  __half* upload_f16(const float* src, size_t n);
  float* upload_f32(const float* src, size_t n);
  __nv_bfloat16* up_bf16(const std::string& name, std::initializer_list<int64_t> shape);
  float* up_f32(const std::string& name, std::initializer_list<int64_t> shape);

  int finalize_encoder();
  int alloc_encoder_ws();
  int finalize_decoder();  // decoder.cu
  int finalize_tinyvit();   // tinyvit.cu
  int alloc_tinyvit_ws();
  int encode_tinyvit(const uint8_t* u8, const float* f32, int B, int hh, int ww, float* out, cudaStream_t st, int stop_after = -1,
                     float* x_out = nullptr);
  int encode(const uint8_t* u8, const float* f32, int B, int hh, int ww, float* out, cudaStream_t st, int stop_after = -1,
             float* x_out = nullptr);
  // encoder_train.cu (cfg 5): forward keeping activations, backward, gradient read-out by upstream key name
  int train_setup();
  int encode_train(const float* f32, int B, float* out, cudaStream_t st);
  int encode_backward(const float* d_out, cudaStream_t st);
  int encoder_grad(const char* name, float* dst, int64_t n, cudaStream_t st);
  void train_invalidate();
  void train_free();       // encoder_train.cu: host-side training state (device buffers are in `allocs`)
  void dec_train_free();   // decoder_train.cu: per-slot arenas + host-side state
  // decoder_train.cu (cfg 5): mask decoder forward keeping activations (one image's prompts per call and slot) + backward
  int dec_train_setup();
  int decoder_train_forward(int slot, const float* emb_nchw, const float* sparse, const int* emb_index, int Ts, int P,
                            const float* mask_in, int multimask, float* low_res, float* iou, cudaStream_t st);
  int decoder_train_backward(int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, cudaStream_t st);
  int decoder_grad(const char* name, float* dst, int64_t n, cudaStream_t st);
  int decoder_zero_grads(cudaStream_t st);
  int md_setup();      // mask_downscaling masters + gradient buffer
  int md_register();   // ... joining the gradient table and the optimizer (first masked training forward)
  int op_mask_downscaling_train(const float* mask, int P, const float* d_dense, float* dense_out, float* grads_out, cudaStream_t st);
  const float* dec_pos();   // decoder.cu: dense positional encoding, token-major [4096, 256] fp32
  int dec_set_prompt_tables(const float* point_emb_4x256, const float* not_a_point, cudaStream_t st);   // decoder.cu
  // train_opt.cu: AdamW over every registered tensor + refresh of the packed operands; read-out of the master weights
  float* opt_master_from_host(const std::string& key, int64_t n);
  void opt_add(const OptParam& p) { opt.push_back(p); }
  int optimizer_step(float lr, float beta1, float beta2, float eps, float weight_decay, cudaStream_t st);
  int train_param(const char* key, float* dst, int64_t n, cudaStream_t st);
  int set_image_embedding(const float* feat, cudaStream_t st);  // decoder.cu
  int decode(const float* points, const float* labels, int np, const float* boxes, const float* mask_in, int P, int multimask,
             float* low_res, float* iou, cudaStream_t st);  // decoder.cu
  int prompt_encode(const float* points, const float* labels, int np, const float* boxes, const float* mask_in, int P,
                    float* sparse_out, float* dense_out, cudaStream_t st);  // decoder.cu
  int mask_decode(const float* sparse, int n_sparse, const float* dense, int P, int multimask, float* low_res, float* iou,
                  cudaStream_t st);  // decoder.cu
  int dense_pe(float* out_tokmajor, cudaStream_t st);  // decoder.cu
  // decoder.cu: the three fused decoder blocks on explicit inputs (msam_op_dec_*); sms > 0 overrides num_sms for the call
  int op_dec_t2i(int which, const __nv_bfloat16* qpe, const __nv_bfloat16* keys, int P, int T, __nv_bfloat16* out, int sms,
                 cudaStream_t st);
  int op_dec_i2t(int layer, const __nv_bfloat16* q, const __nv_bfloat16* qpe, int shared, __nv_bfloat16* keys, int P, int T,
                 int sms, cudaStream_t st);
  int op_dec_upscale(const __nv_bfloat16* keys, const float* hyper, int P, int multimask, float* low_res, int sms,
                     cudaStream_t st);
};

// postprocess.cu
int post_remove_small_regions(uint8_t* masks, int n, int h, int w, int area_thresh, int holes, int32_t* changed, int32_t* ws,
                              cudaStream_t st);
int post_mask_boxes(const uint8_t* masks, int n, int h, int w, int32_t* boxes, int32_t* area, cudaStream_t st);
int post_local_otsu(const float* low_res, int n, float* thr_out, cudaStream_t st);
int post_mask_stats(const float* low_res, int n, int in_h, int in_w, int out_h, int out_w, float thr, float off,
                    int32_t* boxes, float* stability, int32_t* area, cudaStream_t st, bool force_generic = false,
                    const float* thr_arr = nullptr, const float* lazy_iou = nullptr, float lazy_iou_thresh = 0.f,
                    uint8_t* lazy_done = nullptr);
int post_upsample(const float* low_res, const int32_t* sel, int n_sel, int in_h, int in_w, int out_h, int out_w, float thr,
                  float* logits, uint8_t* bin, cudaStream_t st, const float* thr_arr = nullptr);
int post_paint(const float* low_res, const int32_t* sel, const int32_t* boxes, const int32_t* seg_ids, int n_sel, int in_h,
               int in_w, int out_h, int out_w, float thr, int exclusive, uint32_t* label, int ld_label, cudaStream_t st,
               const float* thr_arr = nullptr);
int post_to_image(const void* src, int dtype, int h, int w, int c, uint8_t* out, uint32_t* scratch6, cudaStream_t st);
int post_paint_min_area(const float* low_res, const int32_t* sel, const int32_t* n_sel, const int32_t* boxes,
                        const int32_t* area, int in_h, int in_w, int out_h, int out_w, float thr, int32_t* label,
                        int ld_label, cudaStream_t st);
int post_finish_segmentation(const int32_t* seg, int h, int w, int min_size, int with_background, uint32_t* out,
                             int32_t* ws, cudaStream_t st);
int post_mask_nms(const uint8_t* masks, int n, int h, int w, const float* boxes_xyxy, const float* scores, float thresh,
                  int iomin, uint32_t* bits_ws, int32_t* areas, float* matrix_ws, int32_t* keep, int32_t* n_keep,
                  cudaStream_t st);
int post_paint_canvas(const float* low_res, const int32_t* sel, const int32_t* gpos, int n_sel, const int32_t* boxes,
                      const int32_t* area, int in_h, int in_w, int out_h, int out_w, float thr, int off_x, int off_y,
                      unsigned long long* canvas, int ld_canvas, cudaStream_t st);
int post_canvas_to_label(const unsigned long long* canvas, long n, int32_t* label, cudaStream_t st);
int post_mask_loss_stats(const float* low_res, const uint8_t* targets, int n_obj, int M, int in_h, int in_w, int out_h, int out_w,
                         float* out, cudaStream_t st);
int post_mask_loss_backward(const float* low_res, const uint8_t* targets, const float* d_stats, int n_obj, int M, int in_h, int in_w,
                            int out_h, int out_w, float* d_low_res, cudaStream_t st);
int post_filter_nms(const int32_t* boxes, const float* scores, const float* stab, int n, int use_filters, float iou_thresh,
                    float stab_thresh, float nms_thresh, const int32_t* crop_box, const int32_t* orig_box, int32_t* keep,
                    int32_t* n_keep, cudaStream_t st);

// ---- prompts.cu: training prompts from label images and predictions (micro_sam/prompt_generators.py)
int prompt_targets(const void* labels, int label_dtype, int B, int H, int W, const int64_t* ids, const int32_t* n_ids, int n_obj,
                   double box_distortion, uint64_t seed, uint8_t* targets, int32_t* counts, int32_t* boxes, cudaStream_t st);
int prompt_sample_points(const uint8_t* targets, const int32_t* counts, const int32_t* boxes, const int32_t* centers, int n, int n_per_img,
                         int H, int W, int n_pos, int n_neg, int dilation, uint64_t seed, uint8_t* scratch, int32_t* coords,
                         int32_t* labels, cudaStream_t st);
int prompt_iterative(const uint8_t* targets, const float* low_res, const float* iou, int M, const uint8_t* pred, int n, int n_per_img,
                     int in_h, int in_w, int H, int W, uint64_t seed, int32_t* coords, int32_t* labels, cudaStream_t st);

}  // namespace msam
