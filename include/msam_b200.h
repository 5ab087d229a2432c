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
/* The same kernel with every field of its argument block (csrc/kernels.h:GemmArgs): row pitches lda / ldw (>= K, multiples of 8),
 * ldc / ldr (0 = N; ldc even), residual fp32 or bf16 (res_bf16) indexed by row % res_rows (0 = M), act_after_res = apply `act` after
 * the residual add, epi = 1: LayerNorm over the N = 256 columns of each row (ln_gamma / ln_beta / ln_eps; bf16 out, bf16 residual or
 * none, no act).  num_sms caps the grid of the persistent kernel (<= 0 = the device's SM count): results must not depend on it. */
int msam_op_gemm_ex(const void* A, const void* W, int M, int N, int K, int lda, int ldw, const float* bias, const void* residual,
                    int res_rows, int ldr, int res_bf16, void* out, int ldc, int out_fp32, int act, int act_after_res, int epi,
                    const float* ln_gamma, const float* ln_beta, float ln_eps, int num_sms, void* stream);
/* msam_op_gemm_ex with the kernel chosen by `path`: 0 = the choice every other caller gets (the 128 x 256 wide-tile kernel for
 * plain-epilogue products with N % 256 == 0 and at least one such tile per SM of the device, else the tiled kernel), 1 = the
 * tiled kernel (column groups of 64, BN = 256 / 128 / 64), 2 = the wide-tile kernel (N % 256 == 0, epi = 0; -1 otherwise). */
int msam_op_gemm_ex2(const void* A, const void* W, int M, int N, int K, int lda, int ldw, const float* bias, const void* residual,
                     int res_rows, int ldr, int res_bf16, void* out, int ldc, int out_fp32, int act, int act_after_res, int epi,
                     const float* ln_gamma, const float* ln_beta, float ln_eps, int num_sms, int path, void* stream);
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
/* The TinyViT (vit_t) encoder's CUDA-core kernels, launched as msam_encode launches them (csrc/tinyvit.cu).  Each returns -1 with
 * a message and launches nothing when an argument breaks what its kernel assumes.
 * stem: Sam.preprocess of uint8 HWC [B, hh, ww, 3] (zero pad to img x img; hh, ww <= img) or of nothing (f32 = preprocessed
 * NCHW [B, 3, img, img]; exactly one of u8 / f32), conv3x3/2 pad 1 with w27x32 [(ky*3+kx)*3 + c][32] and b32 (BatchNorm
 * folded), GELU -> bf16 NHWC [B, img/2, img/2, 32].  img even. */
int msam_op_tv_stem(const uint8_t* u8, const float* f32, int B, int hh, int ww, int img, const float* w27x32, const float* b32,
                    void* out_bf16, void* stream);
/* im2col of a 3x3 / pad 1 conv on bf16 NHWC [B, Hin, Hin, C] -> [B * Ho * Ho, 9 * C] (column (ky*3+kx)*C + c), Ho = Hin / stride;
 * C % 8 == 0, stride 1 or 2, Hin even with stride 2. */
int msam_op_tv_im2col(const void* x_bf16, int B, int Hin, int C, int stride, void* out_bf16, void* stream);
/* Depth-wise conv3x3 pad 1 + bias (w9xC [9][C] fp32, BatchNorm folded), GELU when act, on bf16 NHWC; shapes as im2col. */
int msam_op_tv_dwconv_bf16(const void* x_bf16, int B, int Hin, int C, int stride, const float* w9xC, const float* b, int act,
                           void* out_bf16, void* stream);
/* The same with stride 1 on fp32 NHWC (the blocks' local_conv); C % 4 == 0. */
int msam_op_tv_dwconv_f32(const float* x, int B, int Hin, int C, const float* w9xC, const float* b, float* out, void* stream);
/* LayerNorm of fp32 [B, H, H, D] into the window-partitioned bf16 rows [B * nw * nw * ws * ws, D], nw = ceil(H / ws); the rows
 * of the zero pad tokens are LayerNorm(0) = beta.  D % 4 == 0, D <= 384, ws 7 or 14. */
int msam_op_tv_ln_window(const float* x, int B, int H, int D, int ws, const float* gamma, const float* beta, float eps,
                         void* out_bf16, void* stream);
/* Window attention, head_dim 32, scale 32^-0.5: qkv bf16 [B * nw * nw * ws * ws, heads * 96] (per head [q | k | v], pad tokens
 * included as keys), bias_tab fp32 [heads, ws * ws] indexed by |dy| * ws + |dx| -> bf16 [B * H * H, heads * 32] in image order. */
int msam_op_tv_attention(const void* qkv_bf16, const float* bias_tab, int B, int H, int ws, int heads, void* out_bf16,
                         void* stream);
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

/* ---- fine-tuning (BASELINE.json configs[4], micro_sam/training/sam_trainer.py:393: loss.backward() through the image encoder and
 * the mask decoder).  Every trainable tensor has one fp32 gradient buffer and one fp32 master buffer in the engine, listed by
 * msam_train_tensor_count / _info (below); that list is the only way to read gradients and master weights.
 * msam_encode_train = msam_encode_f32 that keeps the activations of B <= max_batch images (ViT encoders only);
 * msam_encode_backward takes dL/d(embedding) (B,256,64,64) fp32 NCHW and overwrites the gradient of every encoder parameter.  It
 * needs the latest forward pass to be that training forward: an inference encode (msam_encode_f32 / _u8 / _u8_blocks) or an
 * optimizer step in between discards the saved pass, and the backward then fails. */
int msam_encode_train(msam_handle* h, const float* nchw, int B, float* out, void* stream);
int msam_encode_backward(msam_handle* h, const float* d_out_nchw, void* stream);
/* Mask decoder + prompt encoder in training mode (micro_sam/training/trainable_sam.py:62-114): MaskDecoder.forward for the P prompts of
 * ONE image keeping the activations in `slot` (0..7), and its backward pass.  sparse = prompt_encoder's sparse embeddings
 * [P, n_sparse, 256] (msam_prompt_encode), emb_index [P, n_sparse] int32 = the embedding-table row behind each sparse token (0..3 =
 * point_embeddings.{0..3}, 4 = not_a_point_embed) so that their gradients can be formed; the dense prompt is no_mask_embed.
 * backward: d_low_res [P, M, 256, 256] / d_iou [P, M] (either may be NULL) -> parameter gradients ACCUMULATE (msam_decoder_zero_grads),
 * d_emb_nchw = dL/d(image embedding) is overwritten: [256, 64, 64] for a slot of msam_decoder_train_forward(_ex), [B, 256, 64, 64]
 * (one gradient per image, not summed) for a slot of msam_decoder_train_forward_images. */
int msam_decoder_train_forward(msam_handle* h, int slot, const float* emb_nchw, const float* sparse, const int32_t* emb_index, int n_sparse,
                               int P, int multimask, float* low_res, float* iou, void* stream);
/* Prompt-free training decode of B images in one slot (micro_sam's SemanticSamTrainer: no prompts, so the sparse embeddings are
 * empty and the dense prompt is no_mask_embed): emb_nchw [B, 256, 64, 64] -> low_res [B, M, 256, 256], iou [B, M], one prompt of the
 * 5 output tokens per image, image b keyed by its own embedding.  Its backward gives no_mask_embed a gradient and none to
 * point_embeddings.*, not_a_point_embed or mask_downscaling.*.  While only such backwards have run since the last
 * msam_decoder_zero_grads, msam_optimizer_step skips (masters, moments and update counts untouched) the tensors a prompt-free loss
 * cannot reach: iou_prediction_head.*, point_embeddings.*, not_a_point_embed and mask_downscaling.*; once any other backward has
 * run, the step updates every tensor as before. */
int msam_decoder_train_forward_images(msam_handle* h, int slot, const float* emb_nchw, int B, int multimask, float* low_res, float* iou,
                                      void* stream);
int msam_decoder_train_backward(msam_handle* h, int slot, const float* d_low_res, const float* d_iou, float* d_emb_nchw, void* stream);
/* msam_decoder_train_forward with mask prompts: mask_input [P, 1, 256, 256] fp32 low-res logits (PromptEncoder._embed_masks), or NULL
 * (= msam_decoder_train_forward).  The dense prompt is then mask_downscaling(mask_input) instead of no_mask_embed.  The first call with
 * masks adds the ten "prompt_encoder.mask_downscaling.*" tensors (upstream keys and layouts) to the trainable tensors;
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
/* Zeroes the gradients of the prompt-encoder and mask-decoder tensors (the encoder's are overwritten by each backward). */
int msam_decoder_zero_grads(msam_handle* h, void* stream);
/* torch.optim.AdamW semantics (micro_sam/training/training.py:train_sam's default optimizer) over every tensor that has received
 * gradients through msam_encode_backward / msam_decoder_train_backward: fp32 master weights, moments and decoupled weight decay on the
 * device, then the bf16 / transposed / tiled operands of the training paths are refreshed.  No gradient buffer is written, so a
 * second step without a new backward applies the same gradients again, as torch.optim.AdamW does.  The packed operands of the
 * INFERENCE decoder are refreshed by load_state_dict. */
int msam_optimizer_step(msam_handle* h, float lr, float beta1, float beta2, float eps, float weight_decay, void* stream);
/* The same AdamW update restricted to the tensors whose key starts with `prefix` (e.g. "image_encoder."): the step of an optimizer
 * whose other parameters have no gradient, which torch skips.  After the first such call every tensor's bias correction uses its
 * own number of updates, as torch.optim.AdamW's per-parameter step does; without it msam_optimizer_step is unchanged. */
int msam_optimizer_step_prefix(msam_handle* h, const char* prefix, float lr, float beta1, float beta2, float eps, float weight_decay,
                               void* stream);
/* Enumeration of the trainable tensors (after the first training forward passes): key, DEVICE pointers of the fp32 gradient and master
 * buffers, element count -- to read gradients and weights, and so that a data-parallel driver can all-reduce (or clip) the gradients in
 * place before msam_optimizer_step.  Each tensor is an upstream one with its upstream element count.  The key is its upstream name,
 * except for the three convolution weights kept in the layout of their GEMM, a permutation of the upstream layout:
 * "mask_decoder.output_upscaling.{0,3}.weight@gemm" (ConvTranspose2d [ci, co, 2, 2] as [(dy * 2 + dx) * co + o][ci]) and
 * "image_encoder.neck.2.weight@gemm" (Conv2d [o, c, 3, 3] as [o][ky * 3 + kx][c]). */
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
/* Row-wise / element-wise stages of the encoder backward pass (csrc/backward.cu), exposed for the op-level tests.  `global` selects
 * the geometry of csrc/kernels.h:rel_table_geom: 0 = 14 x 14 window (196 keys, T rows of nt = 64 columns, rel_pos_w at woff = 32),
 * 1 = 64 x 64 global (4096 keys, nt = 256, woff = 128).  n_batch = (windows | images) * heads; a batch entry has n_tok query rows.
 * attn_probs: P[row, :pitch_p] bf16 = softmax_k(scale * S[row, k] + T[row, qh - kh + side - 1] + T[row, woff + qw - kw + side - 1]),
 * zero in columns [n_tok, pitch_p); S fp32 rows of pitch_s, T fp32 rows of nt.
 * attn_ds: dS = P o (dP - sum_k P dP) (bf16, pitch_p, zero pad columns) and dT bf16 rows of nt = the bias gradient summed into the
 * table-row index of each key (every other entry zero). */
int msam_op_attn_probs(const float* S, const float* T, int64_t n_batch, int global, int pitch_s, int pitch_p, float scale, void* P_bf16,
                       void* stream);
int msam_op_attn_ds(const void* P_bf16, const float* dP, int64_t n_batch, int global, int pitch_s, int pitch_p, void* dS_bf16,
                    void* dT_bf16, void* stream);
/* dq / dk / dv fp32 [outer, heads, T, d] -> dqkv bf16 [outer * T, 3 * heads * d]; d % 4 == 0. */
int msam_op_pack_dqkv(const float* dq, const float* dk, const float* dv, int outer, int heads, int T, int d, void* dqkv_bf16, void* stream);
/* dpre = dh * GELU'(pre) (exact erf form), bf16, n % 8 == 0; dpre may alias dh. */
int msam_op_gelu_bwd(const void* dh_bf16, const void* pre_bf16, int64_t n, void* dpre_bf16, void* stream);
/* out[N] fp32 += column sums of bf16 x[rows, N] (bias gradients). */
int msam_op_colsum(const void* x_bf16, int64_t rows, int N, float* out, void* stream);
/* image-order bf16 [B * 4096, D] -> 14 x 14 window-partitioned [B * 25 * 196, D], zero pad rows; D % 8 == 0. */
int msam_op_window_gather(const void* x_bf16, int B, int D, void* out_win_bf16, void* stream);
/* Adjoint of the 3 x 3 / pad 1 im2col of the neck: dcol bf16 [B * g * g, 9 * C] -> out fp32 [B * g * g, C]; C % 8 == 0. */
int msam_op_col2im3x3(const void* dcol_bf16, int B, int g, int C, float* out, void* stream);
/* out[n] (+)= sum_b x[b, n], fp32. */
int msam_op_sum_batch(const float* x, int64_t n_batch, int64_t n, float* out, int accumulate, void* stream);
/* out bf16 [cols, rows] = in [rows, cols]^T. */
int msam_op_transpose_bf16(const void* in_bf16, int rows, int cols, void* out_bf16, void* stream);
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
/* segment_from_mask's mask -> prompt derivation on the device (csrc/volume.cu; prompt_based_segmentation.py:24-101 here,
 * micro_sam/prompt_based_segmentation.py:28-140 upstream), for multi_dimensional_segmentation.segment_mask_in_volume.
 * mask: uint8 [H, W] with row pitch ld >= W (a tile's outer block may be a view into a larger frame); pixels == 1 are the
 * object.  H, W <= 8192; with want_logits, shapes whose resize to the longest side 256 needs more than 72 taps per output
 * pixel (2 * ceil(in / out) + 1, e.g. 8192 x 111) are refused.  workspace: msam_mask_prompts_workspace(H, W) bytes of device memory.
 * stats int64 [12]: count, sum_y, sum_x, (y0, x0, y1, x1) python box of the object (exclusive ends), (x0, y0, x1, y1) the
 * _process_box(box_extension) box (rounded half to even, clipped to the mask), n_points (-1: more than 8192 peak candidates).
 * box1024 fp32 [4] (or NULL): that box through ResizeLongestSide(1024).apply_boxes for original size (H, W).
 * want_logits: logits fp32 [256, 256] = _compute_logits_from_mask, bit-identical to torch's CPU antialiased resize.
 * point_mode 0: none; 1: use_single_point; 2: _compute_points_from_mask's inner (d = 3) + outer (d = 5) peaks.  points fp32
 * [max_points, 2] (x, y) in the 1024 frame, labels fp32 [max_points] (1 / 0); only the first max_points are written, stats[11]
 * holds the full count.  field fp32 [H * W] (or NULL): the smoothed distance field of the box crop, row-major with the crop's
 * width as pitch.  An empty mask gives count 0, zero boxes, no points and all -hi logits. */
int64_t msam_mask_prompts_workspace(int H, int W);
int msam_mask_prompts(const uint8_t* mask, int H, int W, int ld, double box_extension, int want_logits, int point_mode, int max_points,
                      void* workspace, int64_t ws_bytes, int64_t* stats, float* box1024, float* logits, float* points, float* labels,
                      float* field, void* stream);
/* util.compute_iou's counts (micro_sam/util.py:1266-1280): counts int64 [2] = (|a == 1 & b == 1|, |a == 1 | b == 1|) of two
 * uint8 [H, W] masks with row pitches lda, ldb.  The ratio is formed by the caller in fp64. */
int msam_mask_iou_counts(const uint8_t* a, int lda, const uint8_t* b, int ldb, int H, int W, int64_t* counts, void* stream);
/* The tracking annotator's _shift_object (micro_sam/sam_annotator/util.py:576-579): dst = scipy.ndimage.shift(src, (dy, dx),
 * order=0, prefilter=False) with mode 'constant', cval 0, bit for bit, for multi_dimensional_segmentation.track_from_prompts.
 * src, dst: uint8 [H, W] with row pitches ld_src, ld_dst >= W; they must not overlap.  Per axis x = o - s in fp64; dst[o] is 0
 * unless 0 <= x <= n - 1 on both axes, else src[floor(x + 0.5)].  A NaN shift gives an all-zero plane. */
int msam_shift_mask(const uint8_t* src, int ld_src, uint8_t* dst, int ld_dst, int H, int W, double dy, double dx, void* stream);
/* Object features of micro-sam's object classification (csrc/objfeat.cu; micro_sam/object_classification.py:20-193): one unit
 * (image, slice or tile) of _compute_object_features_impl with resize_embedding_shape's grid (ry, rx), accumulated.
 * emb: fp32 [256, 64, 64] contiguous.  seg: int32 [h, w] with row pitch ld >= w, dense label indices: 0 is background, v in
 * [1, n_ids] is object v - 1 (other values are ignored).  The segmentation is padded to S = max(h, w) and both it (nearest) and
 * the embedding (bilinear, Gaussian prefilter on axes with r < 64) are resized to ry x rx as skimage's resize does;
 * 1 <= ry, rx <= min(S, 8192).  Adds each object's sum of the resized embedding over its resized pixels to sums fp64
 * [n_ids, 256] and its pixel count to areas int64 [n_ids]; the caller zeroes both before the first unit.  Bit-identical from
 * run to run.  workspace: msam_object_features_workspace(n_ids) bytes of device memory. */
int64_t msam_object_features_workspace(int n_ids);
int msam_object_features(const float* emb, const int32_t* seg, int ld, int h, int w, int ry, int rx, int n_ids, void* workspace,
                         int64_t ws_bytes, double* sums, int64_t* areas, void* stream);
/* out [n_ids, 257] (fp64 with out_f64, else fp32): column 0 the area, columns 1..256 sums / area; rows of area 0 are zero. */
int msam_object_features_finish(const double* sums, const int64_t* areas, int n_ids, int out_f64, void* out, void* stream);
/* project_prediction_to_segmentation (object_classification.py:196-217): out[i] = values[k] where ids[k] == seg[i], else 0.
 * seg, out int64 [n]; ids int64 [n_ids] sorted ascending without repeats; values [n_ids] of any 8-byte type, copied bitwise. */
int msam_project_labels(const int64_t* seg, int64_t n, const int64_t* ids, const int64_t* values, int n_ids, int64_t* out, void* stream);
/* merge_instance_segmentation_3d (micro_sam/multi_dimensional_segmentation.py:312-382) on the device (csrc/merge3d.cu), for
 * multi_dimensional_segmentation.automatic_3d_segmentation.  Stacks are int32 [Z, H, W] contiguous, ids >= 0, Z * H * W <
 * 2^31 - 1024.  workspace: msam_merge3d_workspace(Z, H, W, max_id, max_edges) bytes of device memory serve every stage. */
int64_t msam_merge3d_workspace(int Z, int H, int W, int max_id, int max_edges);
/* out int32 [2] (device) = (min, max) of the stack. */
int msam_merge3d_range(const int32_t* seg, int Z, int H, int W, int32_t* out, void* stream);
/* _preprocess_closing (:236-296): scipy.ndimage.binary_closing(seg > 0, 3x1x1 structure along z, iterations=gap_closing) bit
 * for bit (border 0, so slices within gap_closing of either end are open), written to closed uint8 [Z, H, W] when not NULL.
 * out = the relabelled stack: an edge slice (z < g or z >= Z - g) is relabel_sequential(seg[z], offset); a middle slice keeps
 * the 4-connected components of its closed plane that overlap at most one non-zero id, numbered in raster order of their
 * first pixel, and takes the ids under the other components relabelled in ascending order after them; then
 * relabel_sequential(offset).  offset starts at 1; an edge slice sets it to max + 1 (1 when empty), a middle slice advances it
 * only when non-empty.  max_id >= the largest id of seg; out_max int32 [1] (device) = the largest id of out. */
int msam_merge3d_close(const int32_t* seg, int Z, int H, int W, int gap_closing, int max_id, void* workspace, int64_t ws_bytes,
                       int32_t* out, uint8_t* closed, int32_t* out_max, void* stream);
/* elf.tracking.tracking_utils.compute_edges_from_overlap's counts: edges int32 [max_edges, 4] (device) = (t, u, v, count) for
 * every source u of slice t (every id of the slice but its smallest, np.unique(seg[t])[1:]) and id v of slice t + 1, count =
 * pixels with seg[t] == u and seg[t + 1] == v, v = 0 included (the counts of one (t, u) sum to its size).  Entries are unordered.
 * Synchronises the stream; *n_edges (host) = the entries found.  More than max_edges is an error, the list stays bounded. */
int msam_merge3d_edges(const int32_t* seg, int Z, int H, int W, void* workspace, int64_t ws_bytes, int max_edges, int32_t* edges,
                       int64_t* n_edges, void* stream);
/* segmentation = node_labels[slice_segmentation] (:375): out[i] = node_labels[seg[i]] int32 [n_nodes] (device); ids outside
 * [0, n_nodes) give 0.  seg and out int32 [n]. */
int msam_merge3d_gather(const int32_t* seg, int64_t n, const int32_t* node_labels, int n_nodes, int32_t* out, void* stream);
/* _filter_z_extent (:299-309) in place: every label in [1, n_labels) whose z extent (last slice - first slice + 1) is below
 * min_z_extent is set to 0.  Labels are not renumbered.  workspace as above with max_id >= n_labels - 1. */
int msam_merge3d_filter_z(int32_t* seg, int Z, int H, int W, int n_labels, int min_z_extent, void* workspace, int64_t ws_bytes,
                          void* stream);
/* _segment_slices' offset loop (:401-414): dst = src + offset where src != 0, else 0, then offset += max(src).  src, dst int32
 * [n] (device); state int32 [2] (device): state[0] is the offset (the caller zeroes it before the first slice), state[1] scratch. */
int msam_stack_slice(const int32_t* src, int64_t n, int32_t* dst, int32_t* state, void* stream);
/* The multicut of merge_instance_segmentation_3d (:360-373), on the host: greedy additive edge contraction over uv int64
 * [n_edges, 2] with weights fp64 [n_edges] (the 1 - costs the reference passes): contract the edge of largest positive weight
 * (ties: smallest (min rep, max rep)) into the smaller representative, parallel edges summed as w(rep, x) + w(other, x), until
 * no positive weight is left.  labels int64 [n_nodes]: elf's multicut_decomposition numbering, clusters ordered by the smallest
 * node of their component of positive edges, then by their own smallest node, from 0. */
int msam_multicut_gaec(int64_t n_nodes, int64_t n_edges, const int64_t* uv, const double* weights, int64_t* labels);
/* ---- decoder-based automatic instance segmentation (AIS): UNETR decoder layers and generate() on the device ----
 * Activations are bf16 NHWC, 16-byte aligned.  Convolution as an implicit GEMM on wgmma: sources x0 [B, H, W, C0] and
 * x1 [B, H, W, C1] (C1 = 0: none) are read as their channel concatenation; w bf16 [N][ks * ks * (C0 + C1)] with K index
 * (ky * 3 + kx) * (C0 + C1) + c; ks 3 (pad 1, zero padding) or 1; out = bias + conv, ReLU when relu.  transposed (ks = 1):
 * the 2x2 / stride 2 transposed convolution, N = 4 Cout with row (i * 2 + j) * Cout + co of w, out [B, 2H, 2W, Cout].
 * C0, C1 multiples of 64, Cout a multiple of 64.  stats (optional, msam_ais_conv_stats_size bytes): per image, 64 x 2-pixel
 * tile (and 2x2 position when transposed) and channel, the sum and sum of squares of the stored outputs, for
 * msam_op_ais_norm_forward with nchunk = size / (16 B Cout). */
int64_t msam_ais_conv_stats_size(int B, int H, int W, int Cout, int transposed);
int msam_op_ais_conv(const void* x0, int C0, const void* x1, int C1, int B, int H, int W, int ks, const void* w_bf16,
                     const float* bias, int Cout, int relu, int transposed, void* out, double* stats, void* stream);
/* bilinear x2 (align_corners=False) of [B, H, W, C] -> [B, 2H, 2W, C]; C % 8 == 0 */
int msam_op_ais_upsample2(const void* x, int B, int H, int W, int C, void* out, void* stream);
/* out_conv (1x1, C -> 3, w fp32 [3][C]) + sigmoid of [B, HW, C] -> fp32 [B, 3, HW]; C % 8 == 0, C <= 512 */
int msam_op_ais_head(const void* x, int B, int HW, int C, const float* w, const float* bias, float* out, void* stream);
/* fp32 planes [P, Hs, Ws] cropped to [ih, iw], then bilinear (align_corners=False) to [P, oh, ow] */
int msam_op_ais_resize(const float* x, int P, int Hs, int Ws, int ih, int iw, int oh, int ow, float* out, void* stream);
/* generate() of one image from fp32 maps fg / cd / bd [H, W]: separable gaussian smoothing in fp64 (taps [2r + 1] on the host,
 * r = 0: none; taps_fg for fg, taps_d for both distances), fg = fg_s > t_fg, markers = cd_s < t_cd & bd_s < t_bd & fg, their
 * 8-connected components numbered 1.. in raster order, the seeded watershed on bd_s inside fg (DESIGN.md section 2), then ids
 * of fewer than min_size pixels removed and the rest renumbered.  labels int32 [H, W] (device); n_ids and sweeps (host): the
 * number of ids and of watershed sweeps.  ws: msam_ais_postprocess_workspace bytes, 256-byte aligned.  Synchronises stream. */
int64_t msam_ais_postprocess_workspace(int H, int W);
int msam_ais_postprocess(const float* fg, const float* cd, const float* bd, int H, int W, const double* taps_fg, int r_fg,
                         const double* taps_d, int r_d, float t_fg, float t_cd, float t_bd, int min_size, void* ws,
                         int64_t ws_bytes, int32_t* labels, int* n_ids, int* sweeps, void* stream);
/* per id 1..n_ids of labels [H, W]: props int32 [n_ids][5] = area, x0, y0, x1, y1 (inclusive) */
int msam_ais_props(const int32_t* labels, int H, int W, int n_ids, int32_t* props, void* stream);
/* ---- training of the AIS decoder (csrc/ais_train.cu).  Every reduction runs in a fixed order: repeats are bit-identical. ----
 * Weight gradient of msam_op_ais_conv (ks 3 or 1, not transposed): dw fp32 [Cout][ks * ks * (C0 + C1)] (the forward's layout) =
 * sum over the pixels of dy [B, H, W, Cout] times the sources x0 / x1 shifted by the tap, zero outside the image.  ws:
 * msam_ais_wgrad_workspace bytes (the split-K partials), 16-byte aligned.  The data gradient is msam_op_ais_conv on dy with the
 * weights rotated by 180 degrees and the channel roles swapped. */
int64_t msam_ais_wgrad_workspace(int Cout, int C0, int C1, int B, int H, int W, int ks);
int msam_op_ais_wgrad(const void* dy, int Cout, const void* x0, int C0, const void* x1, int C1, int B, int H, int W, int ks, void* ws,
                      int64_t ws_bytes, float* dw, void* stream);
/* Norm of x [B, HW, C] bf16, C % 8 == 0: per_image 1 = InstanceNorm (biased variance per image and channel), 0 = BatchNorm
 * on batch statistics (over B * HW per channel; run_mean / run_var, if given, updated as torch does: momentum, unbiased
 * variance); optional affine gamma / beta; out = (relu of) the normalised x.  stats: the partial sums msam_op_ais_conv wrote for
 * x (nchunk per image), or null: computed here.  The partial sums are reduced in a fixed order.  mean and rstd ([B * C] or [C],
 * for the backward pass) are optional, both or neither.  ws: msam_ais_norm_workspace bytes, 256-byte aligned. */
int64_t msam_ais_norm_workspace(int B, int HW, int C);
int msam_op_ais_norm_forward(const void* x, int B, int HW, int C, int per_image, const double* stats, int nchunk, const float* gamma,
                             const float* beta, float eps, int relu, float momentum, float* run_mean, float* run_var, void* ws,
                             int64_t ws_bytes, float* mean, float* rstd, void* out, void* stream);
/* Its backward pass: g = dy (bf16, or fp32 when dy_f32; row stride ldd) times [relu_out > 0] when relu_out is given;
 * dx = gamma rstd (g - mean(g) - xhat mean(g xhat)), times [x > 0] when in_mask; out_mode 0: bf16 store, 1: fp32 store,
 * 2: fp32 add, row stride ldo.  dgamma / dbeta (optional): sum g xhat, sum g per channel. */
int msam_op_ais_norm_backward(const void* x, int ldx, const void* dy, int dy_f32, int ldd, const void* relu_out, int B, int HW, int C,
                              int per_image, const float* gamma, const float* mean, const float* rstd, int in_mask, void* ws,
                              int64_t ws_bytes, void* dx, int out_mode, int ldo, float* dgamma, float* dbeta, void* stream);
/* out[c] = sum over the B * HW pixels of g [B, HW, C] bf16 (a bias gradient); ws: msam_ais_norm_workspace bytes */
int msam_op_ais_chan_sum(const void* g, int B, int HW, int C, void* ws, int64_t ws_bytes, float* out, void* stream);
/* adjoint of msam_op_ais_upsample2: dy [B, 2H, 2W, C] -> dx [B, H, W, C], bf16 */
int msam_op_ais_upsample2_backward(const void* dy, int B, int H, int W, int C, void* dx, void* stream);
/* out[b, y, x, (i * 2 + j) * C + c] = dy[b, 2y + i, 2x + j, c] (bf16): the transposed convolution's output as GEMM columns */
int msam_op_ais_space_to_depth(const void* dy, int B, int H, int W, int C, void* out, void* stream);
/* acc[i] (fp32) += x[i] (bf16) */
int msam_op_ais_add_bf16(float* acc, const void* x, int64_t n, void* stream);
/* g[i] (bf16) = 0 where out[i] <= 0: the ReLU mask of the layer that wrote out */
int msam_op_ais_relu_mask(void* g, const void* out, int64_t n, void* stream);
/* backward of msam_op_ais_head from its input h, weights w and sigmoid maps: dh (bf16, times [h > 0]: the ReLU before the head),
 * dw fp32 [3][C], db [3].  ws: msam_ais_head_backward_workspace bytes, 256-byte aligned. */
int64_t msam_ais_head_backward_workspace(int B, int HW, int C);
int msam_op_ais_head_backward(const void* h, int B, int HW, int C, const float* w, const float* maps, const float* dmaps, void* ws,
                              int64_t ws_bytes, void* dh, float* dw, float* db, void* stream);
/* adjoint of msam_op_ais_resize: dout [P, oh, ow] -> dsrc [P, Hs, Ws] (zero outside the crop); tmp: P * oh * iw floats */
int msam_op_ais_resize_backward(const float* dout, int P, int Hs, int Ws, int ih, int iw, int oh, int ow, float* tmp, float* dsrc,
                                void* stream);
/* Distance-based Dice loss sums of prediction x and target y (fp32 [B, 3, HW]); mask: channels 1, 2 of both times y[:, 0].
 * stats (device, fp64 [3][3]): per channel sum x y, sum x^2, sum y^2 over the batch.  The backward pass takes
 * coef (device, fp32 [3][2]) = dL / d(sum x y), dL / d(sum x^2) per channel and writes dx. */
int64_t msam_ais_dist_loss_workspace(int B, int HW);
int msam_op_ais_dist_loss_stats(const float* x, const float* y, int B, int HW, int mask, void* ws, int64_t ws_bytes, double* stats,
                                void* stream);
int msam_op_ais_dist_loss_backward(const float* x, const float* y, int B, int HW, int mask, const float* coef, float* dx, void* stream);
/* ---- loss of semantic fine-tuning (csrc/semantic_loss.cu; micro_sam/training/semantic_sam_trainer.py:11-86) ----
 * low_res fp32 [B, C, 256, 256] logits (1 <= C <= 15), labels [B, H, W] (label_dtype 0 int32, 1 int64), (in_h, in_w) the
 * input_size and (H, W) the original_size of Sam.postprocess_masks, evaluated per pixel and never materialised.  With
 * p = softmax over the C full-resolution logits, stats (device, fp64 [3 C + 3]) = per class c { sum p_c [l == c], sum p_c^2,
 * sum [l == c] }, then { sum of -log p_l over the labels l in [0, C), their count, the count of labels outside [0, C) other
 * than -100 }.  Label -100 is ignored by the cross entropy and in no class.  The backward pass takes d_stats (device, fp64, the
 * layout of stats; reads dL/d sum p_c t_c, dL/d sum p_c^2 and dL/d ce sum) and WRITES d_low_res.  fp64 partials reduced in a
 * fixed order and no float atomics: repeats are bit-identical.  ws: msam_semantic_loss_workspace(..., backward) bytes of
 * device memory, 256-byte aligned (backward = 1 sizes it for both calls). */
int64_t msam_semantic_loss_workspace(int B, int C, int in_h, int in_w, int H, int W, int backward);
int msam_semantic_loss_stats(const float* low_res, const void* labels, int label_dtype, int B, int C, int in_h, int in_w, int H, int W,
                             void* ws, int64_t ws_bytes, double* stats, void* stream);
int msam_semantic_loss_backward(const float* low_res, const void* labels, int label_dtype, const double* d_stats, int B, int C, int in_h,
                                int in_w, int H, int W, void* ws, int64_t ws_bytes, float* d_low_res, void* stream);
/* One AdamW step (torch.optim.AdamW) of fp32 masters w with gradients g and moments m, v at bias-correction step `step` (>= 1),
 * for tensors kept outside the engine's table. */
int msam_op_adamw(float* w, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int step, void* stream);
/* ---- object centres, bounding boxes and one-hot masks of a label image (csrc/centers.cu; micro_sam/util.py:1283-1396) ----
 * labels: int32 ids in [0, 2^31), 0 background, C order, ndim 2 ([H, W]) or 3 ([Z, H, W]) with host extents dims; the grid padded
 * by one pixel per side must have fewer than 2^31 pixels.  ws: msam_centers_workspace bytes of device memory, 256-byte aligned.
 * msam_centers_boxes: for the n_ids objects of ids (int32, sorted ascending, unique, non-zero; pixels with other ids are ignored)
 * boxes int32 [n_ids][2 ndim] = (min per axis, max + 1 per axis) and centers [n_ids][ndim]: mode 'v' int32, the object pixel of
 * largest Euclidean distance to the inner boundaries of the padded labels (the first in raster order on ties); mode 'p' fp64,
 * the mean pixel coordinate (int64 sums divided once).  Integer atomics only: bit-identical from run to run. */
int64_t msam_centers_workspace(int ndim, const int* dims, int n_ids);
int msam_centers_boxes(const int32_t* labels, int ndim, const int* dims, int mode, void* ws, int64_t ws_bytes, const int32_t* ids,
                       int n_ids, void* centers, int32_t* boxes, void* stream);
/* out uint8 over the padded grid ([H + 2, W + 2] or [Z + 2, H + 2, W + 2]): 1 where skimage's find_boundaries(np.pad(labels, 1),
 * mode="inner") is true (foreground with a different label among its in-grid cross / 6-neighbours) */
int msam_op_label_boundaries(const int32_t* labels, int ndim, const int* dims, uint8_t* out, void* stream);
/* out int32 = scipy's distance_transform_edt(mask)^2 exactly, for a uint8 mask of 1 to 3 dims (< 2^31 pixels): the squared
 * distance of every pixel to the nearest zero of mask (0 on the zeros), saturated at INT32_MAX (also where mask has no zero).
 * ws: 3 x (4 n bytes rounded up to 256) of device memory, 256-byte aligned. */
int msam_op_edt_squared(const uint8_t* mask, int ndim, const int* dims, void* ws, int64_t ws_bytes, int32_t* out, void* stream);
/* segmentation_to_one_hot's planes: out fp32 [n_planes, n], plane p = (plane(labels[i]) == p).  ids NULL: plane(v) = v - 1;
 * else ids int32 [n_tab] sorted ascending and unique, plane(v) = the index of v in ids (none when absent or v == 0). */
int msam_segmentation_one_hot(const int32_t* labels, int64_t n, const int32_t* ids, int n_tab, int n_planes, float* out, void* stream);
/* ---- the UNETR decoder's training targets: torch_em's PerObjectDistanceTransform for B 2-D label images (csrc/distance_targets.cu;
 * DESIGN.md section 2) ----
 * labels [B, H, W] C order, label_dtype 0 int32 / 1 int64, ids in [0, 2^31) (0 background); H, W <= 32768 and B H W < 2^31 - 1024.
 * apply_label 1: objects are the 8-connected components of equal ids (skimage.measure.label), numbered in raster order of their
 * first pixel; 0: the distinct ids in ascending order.  Objects of fewer than min_size pixels become background.  channels: bit
 * 1 instances (per-image object number), 2 foreground, 4 centre distances, 8 boundary distances, each normalised within its
 * object; out fp32 [B, popcount(channels), H, W] in that order, fill at background pixels of the distance channels.
 * ws: msam_distance_targets_workspace bytes of device memory, 256-byte aligned (-1: shape refused).  Integer atomics only:
 * bit-identical from run to run. */
int64_t msam_distance_targets_workspace(int B, int H, int W, int apply_label);
int msam_distance_targets(const void* labels, int label_dtype, int B, int H, int W, int apply_label, int min_size, int channels,
                          float fill, void* ws, int64_t ws_bytes, float* out, void* stream);
/* debug: device buffer of 64 x 16 uint64 %globaltimer stamps written by the window-attention kernels, NULL = off */
int msam_debug_attn_trace(void* dev_buf);

#ifdef __cplusplus
}
#endif
#endif
