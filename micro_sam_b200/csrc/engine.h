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

// Early returns (-1) of the int-returning host functions: CHK when a result is null / false, RUN when a return code is nonzero.
#define CHK(p) do { if (!(p)) return -1; } while (0)
#define RUN(x) do { if (x) return -1; } while (0)

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

// Activations of one ViT block that the training forward keeps for the backward pass (encoder_train.cu): the fp32 residual stream
// before the block (x_in) and before the MLP (x_mid), qkv, the attention output and the fc1 pre-activation (bf16).
struct VitBlockActs {
  float *x_in = nullptr, *x_mid = nullptr;
  __nv_bfloat16 *qkv = nullptr, *attn = nullptr, *pre = nullptr;
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

// How the operand a kernel reads is rebuilt from an updated fp32 master (train_opt.cu)
enum class Refresh {
  None,        // the kernels read the master itself
  Cast,        // dst [n] = bf16(master)
  RelPosRows,  // rows [row_off, row_off + rows) of the bf16 rel-pos table dst [*, cols_pad] = master [rows, cols]
  TileBias4,   // dst4 [4, n] = master [n] repeated: a conv-transpose bias as the GEMM epilogue reads it, one tile per sub-pixel
};

// One trainable tensor (the registry Engine::opt, train_opt.cu): fp32 master weights (the live parameter buffer itself when the
// kernels read fp32: biases, LayerNorm, embedding tables), its gradient, AdamW moments, and how the operands are refreshed after
// an update.  Every entry is an upstream tensor with its upstream element count; a key "<name>@gemm" holds it in the GEMM layout
// of its convolution, a permutation of the upstream layout (micro_sam_b200/sam.py:B200Sam._upstream).
struct OptParam {
  std::string key;
  float *w = nullptr, *g = nullptr, *m = nullptr, *v = nullptr;
  int64_t n = 0;
  bool decoder = false;           // the gradient accumulates until msam_decoder_zero_grads; else msam_encode_backward overwrites it
  const bool* written = nullptr;  // non-null: AdamW skips the tensor while *written is false (no gradient since the last zeroing)
  int64_t steps = 0;              // ... and counts its own steps for the bias correction (with written only)
  const bool* skip = nullptr;     // non-null: AdamW skips the tensor while *skip is true (its upstream .grad would be None)
  int64_t count = 0;              // updates of the tensor; the bias correction once a subset step has run (per_tensor_counts)
  Refresh refresh = Refresh::None;
  __nv_bfloat16 *dst = nullptr;
  __nv_bfloat16* dstT = nullptr;  // non-null: after the refresh, dstT [cols, rows] = dst [rows, cols]^T (W^T of the dgrad GEMMs)
  float* dst4 = nullptr;
  int rows = 0, cols = 0, cols_pad = 0, row_off = 0;
};

// 3x3 conv weight [o][c][ky][kx] -> the layout of its implicit GEMM, [o][ky * 3 + kx][c] (engine.cu)
std::vector<float> conv3x3_gemm_layout(const std::vector<float>& w, int C);

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
  bool per_tensor_counts = false;  // set by the first subset step: from then on each tensor's bias correction uses its own count

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
  // ViT forward of nb <= max_batch images: patch embedding, blocks, neck -> out (NCHW).  stop_after >= 0: only the first stop_after
  // blocks, no neck (the fp32 residual stream is left in ws.x).  keep: null for inference, else one VitBlockActs per block.
  int vit_forward(const uint8_t* u8, const float* f32, int nb, int hh, int ww, const VitBlockActs* keep, float* out, cudaStream_t st,
                  int stop_after = -1);
  // encoder_train.cu (cfg 5): forward keeping activations, backward
  int train_setup(cudaStream_t st);
  int encode_train(const float* f32, int B, float* out, cudaStream_t st);
  int encode_backward(const float* d_out, cudaStream_t st);
  void train_invalidate();
  void train_free();       // encoder_train.cu: host-side training state (device buffers are in `allocs`)
  void dec_train_free();   // decoder_train.cu: per-slot arenas + host-side state
  // decoder_train.cu (cfg 5): mask decoder forward keeping activations (one image's prompts per call and slot) + backward
  int dec_train_setup();
  int decoder_train_forward(int slot, const float* emb_nchw, const float* sparse, const int* emb_index, int Ts, int P,
                            const float* mask_in, int multimask, float* low_res, float* iou, cudaStream_t st);
  // B images with no prompts in one slot (one prompt of 5 tokens per image)
  int decoder_train_forward_images(int slot, const float* emb_nchw, int B, int multimask, float* low_res, float* iou, cudaStream_t st);
  int dec_train_run(int slot, const float* emb_nchw, const float* sparse, const int* emb_index, int Ts, int P, const float* mask_in,
                    bool images, int multimask, float* low_res, float* iou, cudaStream_t st);
  int decoder_train_backward(int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, cudaStream_t st);
  int decoder_zero_grads(cudaStream_t st);
  int dec_train_refresh_prompt_tables(cudaStream_t st);   // the inference prompt encoder's tables <- the training masters
  int md_setup();      // mask_downscaling masters + gradient buffer
  int md_register();   // ... joining the registry (first masked training forward)
  int op_mask_downscaling_train(const float* mask, int P, const float* d_dense, float* dense_out, float* grads_out, cudaStream_t st);
  const float* dec_pos();   // decoder.cu: dense positional encoding, token-major [4096, 256] fp32
  int dec_set_prompt_tables(const float* point_emb_4x256, const float* not_a_point, cudaStream_t st);   // decoder.cu
  // train_opt.cu: registration of a trainable tensor, AdamW over every registered tensor + refresh of the operands.
  // train_add returns the gradient buffer of p, or null on error.  p.g null: a zeroed buffer of p.n floats is allocated.
  // p.w null: the master is an fp32 upload of p.n floats from `init`, or from the host copy dec_host[p.key] when init is null.
  float* train_add(OptParam p, const float* init = nullptr);
  // prefix non-null: only the tensors whose key starts with it (a subset step: torch skips the parameters without a gradient)
  int optimizer_step(float lr, float beta1, float beta2, float eps, float weight_decay, cudaStream_t st, const char* prefix = nullptr);
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
// Connected components of equal non-zero labels of seg int32 [h, w] (4-connectivity): parent [h * w] = the component's root,
// its first pixel in raster order (-1 on label 0); size [h * w] = pixel count at the roots; *bg_count += count of label 0.
// The caller zeroes *bg_count.  h * w < 2^31 - 1024.  img_h > 0: no links between rows of different blocks of img_h rows (a
// batch of images); conn8: 8-connectivity.
int post_label_components(const int32_t* seg, int h, int w, int* parent, int* size, int* bg_count, cudaStream_t st, int img_h = 0,
                          int conn8 = 0);
// flag [n] = 1 at the roots of the components of post_label_components with at least min_size pixels, else 0.
int post_flag_components(int n, const int* parent, const int* size, int min_size, int* flag, cudaStream_t st);
// Objects of B label images seg int32 [B, h, w] (ids >= 0, 0 background): apply_label = 1 the 8-connected components of equal
// non-zero ids, 0 the distinct non-zero ids of each image.  Objects of fewer than min_size pixels become 0; the others are
// numbered 1.. over the whole batch, image by image, within an image by first pixel in raster order (apply_label = 1) or by
// ascending id (0).  out int32 [B, h, w]; *n_objects (device) = their count.  ws: post_label_objects_ws bytes, 8-byte aligned.
int64_t post_label_objects_ws(int B, int h, int w, int apply_label);
int post_label_objects(const int32_t* seg, int B, int h, int w, int apply_label, int min_size, int32_t* out, int* n_objects, void* ws,
                       cudaStream_t st);
// Inclusive prefix sum of in [n]: the sum up to i is out[i] + block_sums[i >> 10]; block_sums holds ceil(n / 1024) ints.
int post_inclusive_scan(const int* in, int n, int* out, int* block_sums, cudaStream_t st);
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

// ---- volume.cu: segment_from_mask's prompt derivation and compute_iou's counts (segment_mask_in_volume)
int64_t mask_prompts_workspace(int H, int W);
int mask_prompts(const uint8_t* mask, int H, int W, int ld, double box_extension, int want_logits, int point_mode, int max_points,
                 void* workspace, int64_t ws_bytes, int64_t* stats, float* box1024, float* logits, float* points, float* labels,
                 float* field, cudaStream_t st);
int mask_iou_counts(const uint8_t* a, int lda, const uint8_t* b, int ldb, int H, int W, int64_t* counts, cudaStream_t st);
int shift_mask(const uint8_t* src, int ld_src, uint8_t* dst, int ld_dst, int H, int W, double dy, double dx, cudaStream_t st);

// ---- objfeat.cu: per-object embedding features of object classification and the projection of object predictions
int64_t object_features_workspace(int n_ids);
int object_features(const float* emb, const int32_t* seg, int ld, int h, int w, int ry, int rx, int n_ids, void* workspace,
                    int64_t ws_bytes, double* sums, int64_t* areas, cudaStream_t st);
int object_features_finish(const double* sums, const int64_t* areas, int n_ids, int out_f64, void* out, cudaStream_t st);
int project_labels(const int64_t* seg, int64_t n, const int64_t* ids, const int64_t* values, int n_ids, int64_t* out,
                   cudaStream_t st);

// ---- merge3d.cu: merge_instance_segmentation_3d's slice merge and _segment_slices' stacking (automatic_3d_segmentation)
int64_t merge3d_workspace(int Z, int H, int W, int max_id, int max_edges);
int merge3d_range(const int32_t* seg, int Z, int H, int W, int32_t* out, cudaStream_t st);
int merge3d_close(const int32_t* seg, int Z, int H, int W, int gap, int max_id, void* ws, int64_t ws_bytes, int32_t* out,
                  uint8_t* closed_out, int32_t* out_max, cudaStream_t st);
int merge3d_edges(const int32_t* seg, int Z, int H, int W, void* ws, int64_t ws_bytes, int max_edges, int32_t* edges,
                  int64_t* n_edges, cudaStream_t st);
int merge3d_gather(const int32_t* seg, int64_t n, const int32_t* node_labels, int n_nodes, int32_t* out, cudaStream_t st);
int merge3d_filter_z(int32_t* seg, int Z, int H, int W, int n_labels, int min_z_extent, void* ws, int64_t ws_bytes, cudaStream_t st);
int stack_slice(const int32_t* src, int64_t n, int32_t* dst, int32_t* state, cudaStream_t st);
int multicut_gaec(int64_t n_nodes, int64_t n_edges, const int64_t* uv, const double* w, int64_t* labels);

}  // namespace msam
