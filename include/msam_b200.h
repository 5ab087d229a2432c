/* msam_b200.h -- C ABI of libmsam_b200.so: the sm_90a (H100) SAM inference core behind micro-sam's predictor seam.
 *
 * The reference (micro-sam) has no FFI; its seam is the Python `SamPredictor`/`Sam` duck type returned by
 * micro_sam/util.py:318 (get_sam_model).  Each entry point below names the reference call it replaces.
 * Conventions: opaque handle; int return code (0 = ok, <0 = error, text via msam_last_error()); plain pointers and
 * sizes only.  Unless stated otherwise pointers are DEVICE pointers on the handle's CUDA device, `stream` is a
 * cudaStream_t passed as void*, calls are asynchronous on that stream.  One handle = one predictor = one stream at a
 * time (the reference predictor is stateful and not re-entrant either, SURVEY.md 8b).
 */
#ifndef MSAM_B200_H
#define MSAM_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct msam_handle msam_handle;

/* Architecture, mirrors the constructor arguments of micro_sam/models/build_sam.py:87-142 (_build_sam). */
typedef struct msam_config {
  int32_t embed_dim;          /* 768 / 1024 / 1280 */
  int32_t depth;              /* 12 / 24 / 32; 0 selects MobileSAM's TinyViT encoder (vit_t: embed_dim 320, num_heads 10) */
  int32_t num_heads;          /* 12 / 16 / 16  (head_dim must be 64 or 80) */
  int32_t global_attn[8];     /* indexes of global-attention blocks, -1 terminated */
  int32_t window_size;        /* 14 */
  int32_t image_size;         /* 1024 */
  int32_t patch_size;         /* 16 */
  int32_t out_chans;          /* 256 */
  int32_t max_batch;          /* tiles per msam_encode call the workspace is sized for */
  int32_t max_prompts;        /* prompts per msam_decode call the workspace is sized for */
} msam_config;

const char* msam_last_error(void);
/* number of CUDA kernels this library has launched from the calling thread since load */
int64_t msam_launch_count(void);

/* bench instrumentation: when enabled, CUDA events are recorded on the launching stream around every instrumented kernel
 * launch; msam_profile_report synchronises and writes a JSON array with one object per kernel name
 * {"name", "ms", "n", "flops", "bytes"} (CUDA-event time, launches, ALGORITHMIC flops / bytes summed over the launches)
 * into buf[cap]; returns the length, < 0 on error. */
int msam_profile(int enable);
int msam_profile_report(char* buf, int cap);

/* util.get_sam_model (util.py:441-458): build the model on `device`. */
int msam_create(const msam_config* cfg, int device, msam_handle** out);
int msam_destroy(msam_handle* h);

/* sam.load_state_dict (util.py:457): one tensor, upstream SAM key name (e.g. "image_encoder.blocks.0.attn.qkv.weight"),
 * fp32, HOST pointer, row-major, `shape[ndim]`.  Call once per tensor, then msam_finalize_weights. */
int msam_load_weight(msam_handle* h, const char* name, const float* host_data, const int64_t* shape, int ndim);
int msam_finalize_weights(msam_handle* h);

/* ImageEncoderViT.forward as called from util.py:674 (_compute_embeddings_batched) / SamPredictor.set_torch_image:
 * (B,3,S,S) fp32 preprocessed (normalised + padded) NCHW -> (B,256,64,64) fp32 NCHW. */
int msam_encode_f32(msam_handle* h, const float* nchw, int B, float* out, void* stream);
/* Same, fusing Sam.preprocess (util.py:670; trainable_sam.py:24-47): B resized uint8 HWC images, each (hh, ww, 3)
 * with max(hh, ww) <= S, contiguous [B, hh, ww, 3]. */
int msam_encode_u8(msam_handle* h, const uint8_t* hwc, int B, int hh, int ww, float* out, void* stream);

/* Parity localisation (tests): patch embedding + the first n_blocks transformer blocks of msam_encode_u8; x_out receives the
 * fp32 residual stream [B*4096, embed_dim] (token-major), to be compared with the oracle's activations block by block. */
int msam_encode_u8_blocks(msam_handle* h, const uint8_t* hwc, int B, int hh, int ww, int n_blocks, float* x_out, void* stream);
/* (vit_t: n_blocks counts TinyViT stages 1..4; x_out = the token stream [B*H*H, dim] after layers.{n_blocks-1}.) */

/* SamPredictor.features assignment (util.py:676-679 / set_precomputed util.py:1248-1256): bind a (256,64,64) fp32
 * NCHW image embedding as the decoder's current image; precomputes the prompt-independent layer-0 projections. */
int msam_set_image_embedding(msam_handle* h, const float* feat_256x64x64, void* stream);

/* SamPredictor.predict_torch up to the low-res logits (inference.py:248, instance_segmentation.py:361):
 * prompt_encoder(points=(coords,labels)|None, boxes|None, masks=None) -> mask_decoder(multimask_output).
 * points [P,n_points,2] / labels [P,n_points] (fp32; -1 pad, 0 neg, 1 pos) in the 1024-frame (already
 * ResizeLongestSide.apply_coords'ed), boxes [P,4] xyxy; either may be NULL, not both.
 * Outputs: low_res [P,M,256,256] fp32, iou [P,M] fp32, M = 3 (multimask) or 1. */
int msam_decode(msam_handle* h, const float* points, const float* labels, int n_points, const float* boxes, int P,
                int multimask, float* low_res, float* iou, void* stream);
/* Same with mask prompts (predict_torch(mask_input=...), prompt_based_segmentation.py:289-493; PromptEncoder._embed_masks):
 * mask_input [P,1,256,256] fp32 low-res logits of a previous prediction, or NULL.  With a mask prompt the dense prompt
 * embedding differs per prompt, so the layer-0 image-side work is no longer shared between prompts. */
int msam_decode_ex(msam_handle* h, const float* points, const float* labels, int n_points, const float* boxes,
                   const float* mask_input, int P, int multimask, float* low_res, float* iou, void* stream);

/* The model-level calls of the Sam duck type (SURVEY.md 8b; training/trainable_sam.py:88-106, models/build_sam.py:115-133):
 * sam.prompt_encoder(points=(coords, labels)|None, boxes|None, masks|None) -> sparse [P, n_sparse, 256] (n_sparse = n_points
 * (+1 padding point when no box is given) + 2 box corners) and, for mask prompts, dense [P, 256, 64, 64] (NCHW fp32; without
 * a mask prompt the dense embedding is the broadcast no_mask_embed and dense_out is not written);
 * sam.prompt_encoder.get_dense_pe() -> token-major [4096, 256] (the caller views it as (1, 256, 64, 64));
 * sam.mask_decoder(image_embeddings = the bound embedding, image_pe = get_dense_pe(), sparse, dense|NULL = no mask,
 * multimask_output) -> low_res [P, M, 256, 256], iou [P, M].  n_sparse = 0 with dense = NULL (an empty prompt) decodes the 5
 * output tokens alone, as upstream does. */
int msam_prompt_encode(msam_handle* h, const float* points, const float* labels, int n_points, const float* boxes,
                       const float* mask_input, int P, float* sparse_out, float* dense_out, void* stream);
int msam_get_dense_pe(msam_handle* h, float* out_4096x256, void* stream);
int msam_mask_decode(msam_handle* h, const float* sparse, int n_sparse, const float* dense, int P, int multimask, float* low_res,
                     float* iou, void* stream);

/* Sam.postprocess_masks + calculate_stability_score + threshold + batched_mask_to_box + area, fused, never
 * materialising the upsampled logits (instance_segmentation.py:229-255; inference.py:137-151; _vendored.py:33-85).
 * low_res [n,256,256]; boxes int32 [n,4] xyxy ([0,0,0,0] if empty); stability fp32 [n]; area int32 [n]. */
int msam_mask_stats(const float* low_res, int n_masks, int in_h, int in_w, int orig_h, int orig_w, float mask_threshold,
                    float stability_offset, int32_t* boxes_xyxy, float* stability, int32_t* area, void* stream);
/* The same, evaluated lazily for automatic mask generation: AMGBase._postprocess_batch (instance_segmentation.py:99-132)
 * applies the predicted-IoU filter first, so the statistics of a mask are only ever read once `iou_preds[k] >
 * pred_iou_thresh` holds (pred_iou_thresh <= 0: no filter).  Masks with done[k] != 0 or failing the filter are skipped,
 * the others are computed and marked in `done` (uint8 [n_masks], device, zero-initialised by the caller). */
int msam_mask_stats_lazy(const float* low_res, int n_masks, int in_h, int in_w, int orig_h, int orig_w, float mask_threshold,
                         float stability_offset, const float* iou_preds, float pred_iou_thresh, uint8_t* done,
                         int32_t* boxes_xyxy, float* stability, int32_t* area, void* stream);
/* segment_anything.utils.amg.remove_small_regions for a batch of materialised masks (AMGBase._postprocess_small_regions,
 * instance_segmentation.py:146-186): masks uint8 [n,h,w] (0/1) are edited in place -- holes != 0: 8-connected background
 * components smaller than area_thresh are filled; holes == 0: foreground components smaller than area_thresh are removed
 * (the largest one is kept if all are small).  changed int32 [n]; workspace int32 [n*(2*h*w + 4)]. */
int msam_remove_small_regions(uint8_t* masks, int n, int h, int w, int area_thresh, int holes, int32_t* changed,
                              int32_t* workspace, void* stream);
/* batched_mask_to_box (_vendored.py:33-85) + area for materialised uint8 masks [n,h,w]: boxes int32 [n,4] xyxy. */
int msam_mask_boxes(const uint8_t* masks, int n, int h, int w, int32_t* boxes_xyxy, int32_t* area, void* stream);
/* mask_threshold = "auto" (inference._local_otsu_threshold, inference.py:70-134): thresholds[n] = max over the pixels of the
 * Otsu threshold of the 31x31 window (64 bins) of the min-max normalised low-res logits, mapped back and clamped at 0. */
int msam_local_otsu_threshold(const float* low_res, int n_masks, float* thresholds, void* stream);
/* msam_mask_stats / msam_upsample_masks / msam_paint with one threshold per mask (device fp32, indexed by the mask's
 * position in low_res) instead of the scalar mask_threshold (inference._process_masks_for_batch, inference.py:137-151). */
int msam_mask_stats_ex(const float* low_res, int n_masks, int in_h, int in_w, int orig_h, int orig_w, const float* thresholds,
                       float stability_offset, int32_t* boxes_xyxy, float* stability, int32_t* area, void* stream);
int msam_upsample_masks_ex(const float* low_res, const int32_t* sel, int n_sel, int in_h, int in_w, int orig_h, int orig_w,
                           const float* thresholds, float* logits, uint8_t* binary, void* stream);
int msam_paint_ex(const float* low_res, const int32_t* sel, const int32_t* boxes_xyxy, const int32_t* seg_ids, int n_sel,
                  int in_h, int in_w, int orig_h, int orig_w, const float* thresholds, int exclusive, uint32_t* label,
                  int ld_label, void* stream);
/* Sam.postprocess_masks materialised for the selected masks `sel` (int32 [n_sel] device, or NULL = first n_sel):
 * logits fp32 [n_sel,H,W] and/or binary uint8 [n_sel,H,W] (either may be NULL). */
int msam_upsample_masks(const float* low_res, const int32_t* sel, int n_sel, int in_h, int in_w, int orig_h, int orig_w,
                        float mask_threshold, float* logits, uint8_t* binary, void* stream);
/* util.mask_data_to_segmentation painting loop (util.py:1799-1829): paint masks sel[0..n_sel) in that order with ids
 * seg_ids[k] into label (uint32, row pitch ld_label); exclusive=1: first painter wins, 0: last wins (AMG). */
int msam_paint(const float* low_res, const int32_t* sel, const int32_t* boxes_xyxy, const int32_t* seg_ids, int n_sel,
               int in_h, int in_w, int orig_h, int orig_w, float mask_threshold, int exclusive, uint32_t* label,
               int ld_label, void* stream);
/* AMGBase._postprocess_batch (instance_segmentation.py:99-132): iou_pred > t, stability >= t, not
 * is_box_near_crop_edge(atol 20), then torchvision-semantics greedy box NMS by iou_pred.  crop/orig boxes are HOST
 * int32[4] xyxy.  keep: int32 [n] device (descending score order), n_keep: int32 [1] device.  use_filters=0: NMS only. */
int msam_amg_filter_nms(const int32_t* boxes_xyxy, const float* iou_preds, const float* stability, int n, int use_filters,
                        float pred_iou_thresh, float stability_thresh, float box_nms_thresh, const int32_t* crop_box_host,
                        const int32_t* orig_box_host, int32_t* keep, int32_t* n_keep, void* stream);

/* Loss statistics of the fine-tuning step (training/sam_trainer.py:122-172: dice loss on sigmoid(masks) + true IoU for the
 * IoU-regression target), fused with Sam.postprocess_masks: low_res [n_obj*M, 256, 256] logits, targets uint8 [n_obj, H, W]
 * (0/1 object masks; mask k belongs to object k / M) -> out5 fp32 [n_obj*M, 5] = {sum sigmoid(v) t, sum sigmoid(v)^2, sum t,
 * |{v>0} and t|, |{v>0} or t|} over the H x W pixels of the up-sampled logits v (never materialised). */
int msam_mask_loss_stats(const float* low_res, const uint8_t* targets, int n_obj, int M, int in_h, int in_w, int orig_h, int orig_w,
                         float* out5, void* stream);

/* util._to_image (util.py:618-651): H x W x C raw image (device; dtype 0 u8, 1 u16, 2 f32, 3 i16, 4 f64; C = 1..)
 * -> H x W x 3 uint8 with per-channel min-max normalisation in the reference's exact float32 arithmetic.
 * scratch6: 6 x uint32 device scratch. */
int msam_to_image(const void* src, int dtype, int h, int w, int c, uint8_t* out_hwc3, uint32_t* scratch6, void* stream);
/* AMG painting (mask_data_to_segmentation(..., merge_exclusively=False), util.py:1799-1829) of the masks sel[0..*n_sel)
 * (n_sel read on the device: chain it to msam_amg_filter_nms without a host sync); per pixel the covering mask with the
 * smallest area wins (later position on ties); label = position + 1, int32 [orig_h, ld_label]. */
int msam_paint_min_area(const float* low_res, const int32_t* sel, const int32_t* n_sel, const int32_t* boxes_xyxy,
                        const int32_t* area, int in_h, int in_w, int orig_h, int orig_w, float mask_threshold,
                        int32_t* label, int ld_label, void* stream);
/* util.mask_data_to_segmentation tail (util.py:1831-1848): connected components of equal labels (4-connectivity), drop
 * components smaller than min_object_size and (with_background) the largest segment, relabel consecutively in raster
 * order.  workspace: int32 [4*h*w + max(4096, ceil(h*w/1024)) + 8] (any image size below 2^31 pixels). */
int msam_finish_segmentation(const int32_t* painted, int h, int w, int min_object_size, int with_background, uint32_t* out,
                             int32_t* workspace, void* stream);

/* Multi-crop / tiled AMG painting (instance_segmentation.py:499-529 + util.py:1799-1829): each crop paints its
 * surviving masks sel[0..n_sel) (global list positions global_pos[k]) into a uint64 canvas [H, ld_canvas] initialised to
 * all-ones with atomicMin((area << 32) | ~pos): smallest area wins, later position on ties.  msam_canvas_to_label turns
 * the canvas into int32 ids (position + 1, 0 = empty). */
int msam_paint_canvas(const float* low_res, const int32_t* sel, const int32_t* global_pos, int n_sel,
                      const int32_t* boxes_xyxy, const int32_t* area, int in_h, int in_w, int crop_h, int crop_w,
                      float mask_threshold, int off_x, int off_y, uint64_t* canvas, int ld_canvas, void* stream);
int msam_canvas_to_label(const uint64_t* canvas, int64_t n, int32_t* label, void* stream);

/* util._batched_mask_nms (util.py:1647-1676) with _calculate_ious_/_iomin_between_pred_masks (:1601-1644): masks uint8
 * [n,h,w]; boxes fp32 xyxy [n,4]; scores fp32 [n].  Workspaces: bits_ws uint32 [n*ceil(h*w/32)], areas int32 [n] (out:
 * popcount areas), matrix_ws fp32 [n*n] (out: the overlap matrix).  keep int32 [n] in greedy order, n_keep int32 [1]. */
int msam_mask_nms(const uint8_t* masks, int n, int h, int w, const float* boxes_xyxy, const float* scores, float nms_thresh,
                  int intersection_over_min, uint32_t* bits_ws, int32_t* areas, float* matrix_ws, int32_t* keep,
                  int32_t* n_keep, void* stream);

/* ---- single-op entry points (unit tests / profiling; the same kernels the calls above are built from) ---- */
/* out[M,N] = act(A[M,K] @ W[N,K]^T + bias) + residual[row % res_rows];  A, W bf16; bias/residual fp32 or NULL;
 * out bf16 (out_fp32=0) or fp32; act: 0 none, 1 GELU(erf), 2 ReLU. */
int msam_op_gemm(const void* A, const void* W, int M, int N, int K, const float* bias, const float* residual,
                 int res_rows, void* out, int out_fp32, int act, void* stream);
/* Weight gradient of a linear layer (first piece of msam_*_backward, cfg 5): out[M,N] fp32 = A[K,M]^T B[K,N], A = dY
 * (tokens x out-features), B = X (tokens x in-features), both bf16 row-major -- torch autograd's dW = dY^T X. */
int msam_op_gemm_tn(const void* A, const void* B, int M, int N, int K, float* out, void* stream);
/* Input gradient of the same layer: out[M,N] fp32 = A[M,K] B[K,N], A = dY (tokens x out-features), B = W (out-features x
 * in-features, the forward weight as stored) -- torch autograd's dX = dY W. */
int msam_op_gemm_nn(const void* A, const void* B, int M, int N, int K, float* out, void* stream);
/* LayerNorm over rows of fp32 x[rows, D] -> bf16; window_mode=1 scatters into the 14x14 window-partitioned layout. */
int msam_op_layernorm(const float* x, int rows, int D, const float* gamma, const float* beta, float eps, void* out_bf16,
                      int window_mode, void* stream);
/* Encoder attention on a packed qkv buffer (see csrc/attention.cu). rel_table: bf16 [NT, 64*ceil(hd/64)]. */
int msam_op_attention(const void* qkv_bf16, const void* rel_table_bf16, void* out_bf16, int batch, int heads, int head_dim,
                      int window, float scale, void* stream);
/* The three fused mask-decoder blocks, running the code msam_decode runs for them, on explicit bf16 inputs with the weights as
 * loaded.  P <= max_prompts prompts of T tokens (5 <= T <= 16).  num_sms caps the grid of the persistent kernels (0 = the
 * device's SM count): results must not depend on it.
 * t2i: token -> image attention instance `which` (0 / 1 = cross_attn_token_to_image of layer 0 / 1, 2 =
 * final_attn_token_to_image), q_pe = queries + query_pe [P*T, 256], keys [P*4096, 256] or NULL = the bound image embedding
 * shared by every prompt -> out [P*T, 128]: the per-head attention output before out_proj. */
int msam_op_dec_t2i(msam_handle* h, int which, const void* q_pe, const void* keys, int P, int T, void* out, int num_sms,
                    void* stream);
/* i2t: image -> token block of `layer`, keys <- norm4(keys + cross_attn_image_to_token(q = keys + pe, k = q_pe, v = queries)),
 * queries / q_pe [P*T, 256]; keys [P*4096, 256] is updated in place.  shared = 1 (layer 0 only): the block's input is the bound
 * image embedding (no mask prompt) and keys is only written. */
int msam_op_dec_i2t(msam_handle* h, int layer, const void* queries, const void* q_pe, int shared, void* keys, int P, int T,
                    int num_sms, void* stream);
/* upscale: output_upscaling(keys [P*4096, 256] bf16) times hyper_in [P, 4, 32] fp32 -> low_res [P, M, 256, 256] fp32 (multimask:
 * masks 1..3, M = 3; else mask 0, M = 1). */
int msam_op_dec_upscale(msam_handle* h, const void* keys, const float* hyper_in, int P, int multimask, float* low_res,
                        int num_sms, void* stream);

/* ---- fine-tuning (BASELINE.json configs[4], micro_sam/training/sam_trainer.py:393: loss.backward() through the image encoder).
 * msam_encode_train = msam_encode_f32 that keeps the activations of B <= max_batch images (ViT encoders only);
 * msam_encode_backward takes dL/d(embedding) (B,256,64,64) fp32 NCHW and fills one fp32 gradient per encoder parameter;
 * msam_encoder_grad copies the gradient of the parameter with upstream key `name` (e.g. "image_encoder.blocks.0.attn.qkv.weight",
 * n = its element count, upstream layout) into a device buffer.  The decoder-side backward (dL/d embedding from the mask loss) is
 * not part of this library yet (DESIGN.md). */
int msam_encode_train(msam_handle* h, const float* nchw, int B, float* out, void* stream);
int msam_encode_backward(msam_handle* h, const float* d_out_nchw, void* stream);
int msam_encoder_grad(msam_handle* h, const char* name, float* dst, int64_t n, void* stream);
/* Mask decoder + prompt encoder in training mode (micro_sam/training/trainable_sam.py:62-114): MaskDecoder.forward for the P prompts of
 * ONE image keeping the activations in `slot` (0..7), and its backward pass.  sparse = prompt_encoder's sparse embeddings
 * [P, n_sparse, 256] (msam_prompt_encode), emb_index [P, n_sparse] int32 = the embedding-table row behind each sparse token (0..3 =
 * point_embeddings.{0..3}, 4 = not_a_point_embed) so that their gradients can be formed; the dense prompt is no_mask_embed.
 * backward: d_low_res [P, M, 256, 256] / d_iou [P, M] (either may be NULL) -> parameter gradients ACCUMULATE (msam_decoder_zero_grads),
 * d_emb_nchw [256, 64, 64] = dL/d(image embedding) is overwritten.  msam_decoder_grad reads a gradient by upstream key
 * ("....weight@gemm" / "@stack" keys carry packed layouts that micro_sam_b200/sam.py:decoder_grads folds back). */
int msam_decoder_train_forward(msam_handle* h, int slot, const float* emb_nchw, const float* sparse, const int32_t* emb_index, int n_sparse,
                               int P, int multimask, float* low_res, float* iou, void* stream);
int msam_decoder_train_backward(msam_handle* h, int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, void* stream);
/* msam_decoder_train_forward with mask prompts: mask_input [P, 1, 256, 256] fp32 low-res logits (PromptEncoder._embed_masks), or NULL
 * (= msam_decoder_train_forward).  The dense prompt is then mask_downscaling(mask_input) instead of no_mask_embed.  The first call with
 * masks adds the ten "prompt_encoder.mask_downscaling.*" tensors (upstream keys and layouts) to the gradient table and the optimizer;
 * msam_decoder_train_backward of such a slot accumulates their gradients (none w.r.t. the mask) and none for no_mask_embed, and
 * msam_optimizer_step updates them only when a masked backward has run since the last msam_decoder_zero_grads. */
int msam_decoder_train_forward_ex(msam_handle* h, int slot, const float* emb_nchw, const float* sparse, const int32_t* emb_index,
                                  int n_sparse, int P, const float* mask_input, int multimask, float* low_res, float* iou, void* stream);
/* mask_downscaling alone, forward and backward, with the training masters (op-level tests): mask [P, 1, 256, 256] -> dense_out
 * [P, 4096, 256] (token-major: the layout that is added to the image embedding); d_dense [P, 4096, 256] = upstream gradient ->
 * grads_out [4684] = the gradients of the ten tensors, overwritten, concatenated in the order 0.weight, 0.bias, 1.weight, 1.bias,
 * 3.weight, 3.bias, 4.weight, 4.bias, 6.weight, 6.bias (each in its upstream layout).  Leaves the engine's gradients alone. */
int msam_op_mask_downscaling_train(msam_handle* h, const float* mask, int P, const float* d_dense, float* dense_out, float* grads_out,
                                   void* stream);
int msam_decoder_grad(msam_handle* h, const char* name, float* dst, int64_t n, void* stream);
int msam_decoder_zero_grads(msam_handle* h, void* stream);
/* torch.optim.AdamW semantics (micro_sam/training/training.py:train_sam's default optimizer) over every tensor that has received
 * gradients through msam_encode_backward / msam_decoder_train_backward: fp32 master weights, moments and decoupled weight decay on the
 * device, then the bf16 / transposed / packed operands of the training paths are refreshed.  msam_train_param reads a master tensor
 * (same keys and layouts as the gradient read-outs).  The packed operands of the INFERENCE decoder are refreshed by load_state_dict. */
int msam_optimizer_step(msam_handle* h, float lr, float beta1, float beta2, float eps, float weight_decay, void* stream);
int msam_train_param(msam_handle* h, const char* key, float* dst, int64_t n, void* stream);
/* Enumeration of the trainable tensors (after the first training forward passes): key, DEVICE pointers of the fp32 gradient and master
 * buffers, element count -- so that a data-parallel driver can all-reduce the gradients in place (torch.distributed / NCCL on views of
 * these buffers) before msam_optimizer_step. */
int msam_train_tensor_count(msam_handle* h);
int msam_train_tensor_info(msam_handle* h, int i, char* key_buf, int cap, void** grad, void** master, int64_t* n);
/* Adjoint of msam_mask_loss_stats w.r.t. the low-res logits: d_stats [n_obj*M, 5] (only columns 0, 1 = dL/d sum(p t), dL/d sum(p^2)
 * matter) -> d_low_res [n_obj*M, 256, 256] accumulated (zero it first).  sam_trainer.py:131-172 backward. */
int msam_mask_loss_backward(const float* low_res, const uint8_t* targets, const float* d_stats, int n_obj, int M, int in_h, int in_w,
                            int orig_h, int orig_w, float* d_low_res, void* stream);
/* Batched GEMM of the attention backward pass (csrc/bgemm.cu), exposed for the op-level parity tests. */
int msam_op_bgemm(const void* A, const void* B, int a_mn, int b_mn, int M, int N, int K, int lda, int ldb, int64_t a_hstride,
                  int64_t a_wstride, int64_t b_hstride, int64_t b_wstride, int heads, int outer, float* out, int ldc,
                  int64_t o_hstride, int64_t o_wstride, float alpha, int accumulate, void* stream);
/* LayerNorm backward over fp32 rows (csrc/backward.cu); dgamma / dbeta are ACCUMULATED into (zero them first). */
int msam_op_layernorm_bwd(const float* x, int rows, int D, const float* gamma, float eps, const float* dy, int window_mode,
                          int accumulate, float* dx, float* dgamma, float* dbeta, void* stream);
/* Training prompts (csrc/prompts.cu).  Random draws come from Philox4x32-10 keyed by `seed`, counter (image, object, draw): the
 * result depends on the seed and the inputs only.
 *
 * ConvertToSamInputs._get_prompt_lists minus the host-side id sampling (micro_sam/training/util.py:174-211,
 * segmentation_to_one_hot and get_centers_and_bounding_boxes(mode="p")): label images [B, H, W] (label_dtype 0 int32,
 * 1 int64), sorted ids [B, n_obj] int64 of which the first n_ids[b] (int32 [B]) are used -> uint8 one-hot targets
 * [B, n_obj, H, W], int32 pixel counts [B, n_obj] and int32 boxes [B, n_obj, 4] (min_row, min_col, max_row + 1, max_col + 1;
 * 0 for unused slots).  box_distortion >= 0 applies _distort_boxes with that factor; < 0 leaves the boxes as they are. */
int msam_prompt_targets(const void* labels, int label_dtype, int B, int H, int W, const int64_t* ids, const int32_t* n_ids, int n_obj,
                        double box_distortion, uint64_t seed, uint8_t* targets, int32_t* counts, int32_t* boxes, void* stream);
/* PointAndBoxPromptGenerator._sample_points (micro_sam/prompt_generators.py:105-205): n = n_img * n_per_img objects, uint8 masks
 * [n, H, W], pixel counts [n], boxes [n, 4] (row / col, exclusive max, as passed by the caller), optional int32 centres [n, 2]
 * (row, col; NULL = none) -> int32 coords [n, n_pos + n_neg, 2] (x, y) and labels [n, n_pos + n_neg].  n_pos + n_neg <= 64.
 * scratch: 2 * n * H * W bytes when n_neg > 0 and dilation > 0, else NULL. */
int msam_prompt_sample_points(const uint8_t* targets, const int32_t* counts, const int32_t* boxes, const int32_t* centers, int n,
                              int n_per_img, int H, int W, int n_pos, int n_neg, int dilation, uint64_t seed, uint8_t* scratch,
                              int32_t* coords, int32_t* labels, void* stream);
/* IterativePromptGenerator.__call__ for 2-D objects (micro_sam/prompt_generators.py:252-377) with SamTrainer._get_best_masks
 * (sam_trainer.py:178-204): uint8 targets [n, H, W] and EITHER low_res [n, M, 256, 256] logits with iou [n, M] (argmax, NULL
 * when M == 1; the prediction is Sam.postprocess_masks(low_res) > 0 for input_size (in_h, in_w), evaluated per pixel) OR a
 * binary prediction pred [n, H, W] uint8 -> int32 coords [n, 2, 2] (x, y; positive then negative) and labels [n, 2]. */
int msam_prompt_iterative(const uint8_t* targets, const float* low_res, const float* iou, int M, const uint8_t* pred, int n,
                          int n_per_img, int in_h, int in_w, int orig_h, int orig_w, uint64_t seed, int32_t* coords, int32_t* labels,
                          void* stream);
/* debug: device buffer of 64 x 16 uint64 %globaltimer stamps written by the window-attention kernels, NULL = off */
int msam_debug_attn_trace(void* dev_buf);

#ifdef __cplusplus
}
#endif
#endif
