"""Automatic mask generation (AMG) with the reference's class surface and initialize/generate split
(micro_sam/instance_segmentation.py:65-680), re-expressed so that no full-resolution logit, bool mask or RLE ever leaves
the GPU unless asked for:

* initialize(): encoder -> decoder over the point grid.  The per-crop state keeps the 256x256 low-res logits on the device
  instead of CPU RLEs (the reference's `_to_mask_data` D2H-copies every mask for CPU RLE, instance_segmentation.py:229-255).
  The per-mask statistics (`msam_mask_stats`: fused upsample + stability + threshold + box + area) are evaluated LAZILY:
  `_postprocess_batch` (:99-132) filters by predicted IoU first, so generate() computes them -- once, cached in the state --
  only for the masks that pass that filter; `crop_list` / `get_state()` materialise all of them, so the state a caller sees
  is always complete.
* generate(): `msam_amg_filter_nms` (pred-IoU / stability / crop-edge filters + box NMS, one kernel) -> survivors are
  painted straight from their low-res logits (`msam_paint`), then connected components / background removal / relabel
  on the host like the reference (util.py:1831-1848).  RLEs / binary masks are produced lazily for the survivors only.
"""
from __future__ import annotations

import ctypes
from abc import ABC
from typing import Any, Callable, Dict, List, Optional, Union

import numpy as np
import torch

from . import _amg_utils as amg_utils
from . import _lib, util

DEFAULT_SEGMENTATION_MODE_WITH_DECODER = "ais"


class AMGBase(ABC):
    """instance_segmentation.py:65-285."""

    def __init__(self):
        self._is_initialized = False
        self._crop_list = None
        self._crop_boxes = None
        self._original_size = None

    @property
    def is_initialized(self):
        return self._is_initialized

    @property
    def crop_list(self):
        """The per-crop state with every statistic materialised (pending lazy statistics are computed first)."""
        if self._crop_list is not None and getattr(self, "_predictor", None) is not None:
            lo = getattr(self, "_tile_lo", 0)      # multi-rank tiled state: this rank's tiles are crop_boxes[lo : lo + n]
            for k, data in enumerate(self._crop_list):
                self._ensure_stats(data, self._crop_boxes[lo + k], 0.0)
        return self._crop_list

    def _geom_of(self, crop_box):
        from .sam import get_preprocess_shape
        H, W = self.original_size
        x0, y0, x1, y1 = crop_box
        h, w = min(int(y1), H) - int(y0), min(int(x1), W) - int(x0)
        return dict(inp=get_preprocess_shape(h, w, self._predictor.transform.target_length), orig=(h, w))

    def _ensure_stats(self, data, crop_box, pred_iou_thresh: float) -> None:
        """Compute the pending mask statistics of a crop for the masks with iou_pred > pred_iou_thresh (<= 0: all of them);
        no host synchronisation (`msam_mask_stats_lazy` skips per mask on the device)."""
        done = data["stats_done"] if "stats_done" in data else None
        if done is None or getattr(data, "_all_done", False):
            return
        low = data["low_res"]
        if low.device != done.device:      # offloaded state: statistics were completed before the logits left the device
            return
        g = self._geom_of(crop_box)
        n = int(low.shape[0])
        if n:
            _lib.check(_lib.lib().msam_mask_stats_lazy(
                _lib.ptr(low), n, int(g["inp"][0]), int(g["inp"][1]), int(g["orig"][0]), int(g["orig"][1]),
                float(self._predictor.model.mask_threshold), float(getattr(self, "_stability_score_offset", 1.0)),
                _lib.ptr(data["iou_preds"]), float(pred_iou_thresh), _lib.ptr(done), _lib.ptr(data["boxes"]),
                _lib.ptr(data["stability_score"]), _lib.ptr(data["area"]), _lib.cur_stream()))
        if pred_iou_thresh <= 0.0:
            data._all_done = True

    @property
    def crop_boxes(self):
        return self._crop_boxes

    @property
    def original_size(self):
        return self._original_size

    # ---- device-side equivalents of _postprocess_batch (instance_segmentation.py:99-144)
    def _filter_nms(self, data, crop_box, original_size, pred_iou_thresh, stability_score_thresh, box_nms_thresh,
                    sync: bool = True):
        orig_h, orig_w = original_size
        n = int(data["iou_preds"].shape[0])
        dev = data["iou_preds"].device
        self._ensure_stats(data, crop_box, pred_iou_thresh)   # statistics of the masks the predicted-IoU filter lets through
        keep = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        n_keep = torch.zeros(1, dtype=torch.int32, device=dev)
        crop = (ctypes.c_int32 * 4)(*[int(c) for c in crop_box])
        orig = (ctypes.c_int32 * 4)(0, 0, int(orig_w), int(orig_h))
        _lib.check(_lib.lib().msam_amg_filter_nms(
            _lib.ptr(data["boxes"]), _lib.ptr(data["iou_preds"]), _lib.ptr(data["stability_score"]), n, 1,
            float(pred_iou_thresh), float(stability_score_thresh), float(box_nms_thresh), crop, orig, _lib.ptr(keep),
            _lib.ptr(n_keep), _lib.cur_stream()))
        self._n_keep_dev = n_keep
        if not sync:
            return keep
        self._last_n_keep = int(n_keep.item())
        return keep[: self._last_n_keep].long()

    def _records(self, data, keep, crop_box, output_mode, geom):
        """Annotation dicts for the kept masks (instance_segmentation.py:188-227)."""
        x0, y0 = int(crop_box[0]), int(crop_box[1])
        boxes = data["boxes"][keep].cpu().numpy().astype(np.int64) + np.array([x0, y0, x0, y0])
        iou = data["iou_preds"][keep].cpu().numpy()
        stab = data["stability_score"][keep].cpu().numpy()
        area = data["area"][keep].cpu().numpy()
        pts = data["points"][keep.cpu()].numpy() + np.array([x0, y0]) if "points" in data else None
        segs = None
        if output_mode in ("binary_mask", "rle", "coco_rle"):
            H, W = geom["orig"]
            sel = keep.to(torch.int32).contiguous()
            binm = torch.empty(len(keep), H, W, dtype=torch.uint8, device=sel.device)
            low_dev, sel = self._logits_rows(data, keep, sel.device)
            _lib.check(_lib.lib().msam_upsample_masks(_lib.ptr(low_dev), _lib.ptr(sel), len(keep), geom["inp"][0],
                                                      geom["inp"][1], H, W, 0.0, None, _lib.ptr(binm), _lib.cur_stream()))
            segs = binm.cpu().numpy().astype(bool)
            if output_mode != "binary_mask":
                segs = amg_utils.mask_to_rle(segs)
            if output_mode == "coco_rle":
                segs = [amg_utils.coco_encode_rle(r) for r in segs]
        anns = []
        for k in range(len(keep)):
            ann = {
                "segmentation": None if segs is None else segs[k],
                "area": int(area[k]),
                "bbox": amg_utils.box_xyxy_to_xywh(boxes[k]).tolist(),
                "predicted_iou": float(iou[k]),
                "stability_score": float(stab[k]),
                "crop_box": amg_utils.box_xyxy_to_xywh(list(crop_box)),
            }
            if pts is not None:
                ann["point_coords"] = [pts[k].tolist()]
            anns.append(ann)
        return anns

    def _crop_geoms(self):
        """Per-crop (input_size, original_size) of the predictor while the crop was decoded -- a pure function of the crop
        boxes (the crop is what `set_image` / the tile embedding saw; input_size = ResizeLongestSide of it), so a state
        restored with set_state() needs nothing beyond the reference's three keys."""
        return [self._geom_of(cb) for cb in self.crop_boxes]

    @staticmethod
    def _logits_rows(data, rows: torch.Tensor, device):
        """Low-res logits of the given masks on `device` + their row indices in the returned tensor.  The state normally
        keeps all logits on the device (rows index them directly); an OFFLOADED state (`offload_state`, pinned host memory)
        ships only the requested rows -- the survivors of filters + NMS, a few hundred of the 3072 masks of a tile."""
        low = data["low_res"]
        if low.device == device:
            return low, rows.to(torch.int32).contiguous()
        picked = low.index_select(0, rows.to("cpu", torch.long))
        return picked.to(device, non_blocking=True), torch.arange(len(rows), dtype=torch.int32, device=device)

    def _offload(self, data, crop_box) -> None:
        """Move a crop's low-res logits (805 MB per 32x32-grid tile) to pinned host memory; the small per-mask statistics stay
        on the device.  This is the reference's memory model (its state holds CPU RLEs, instance_segmentation.py:229-255)."""
        low = data["low_res"]
        self._ensure_stats(data, crop_box, 0.0)   # the statistics need the logits on the device: complete them first
        host = torch.empty(low.shape, dtype=low.dtype, pin_memory=True)
        host.copy_(low, non_blocking=False)
        data["low_res"] = host

    def get_state(self) -> Dict[str, Any]:
        if not self.is_initialized:
            raise RuntimeError("The state has not been computed yet. Call initialize first.")
        return {"crop_list": self.crop_list, "crop_boxes": self.crop_boxes, "original_size": self.original_size}

    def set_state(self, state: Dict[str, Any]) -> None:
        """A cached state (precompute_state.cache_amg_state) holds CPU tensors: what the kernels read goes back to the
        predictor's device (`points` stay on the host, as `initialize` keeps them), except the low-res logits when they would
        take more than half of the free device memory (then they stay in pinned host memory, the offloaded layout of
        `initialize(offload_state=None)`)."""
        dev = self._predictor.device
        crops = state["crop_list"]
        need = sum(d["low_res"].numel() * d["low_res"].element_size() for d in crops
                   if "low_res" in d and torch.is_tensor(d["low_res"]))
        offload = need > 0 and need > 0.5 * torch.cuda.mem_get_info(dev)[0]

        def place(k, v):
            if not torch.is_tensor(v) or k not in ("low_res", "iou_preds", "stability_score", "boxes", "area", "stats_done"):
                return v
            if k == "low_res" and offload:
                return v if v.is_pinned() else v.cpu().pin_memory()
            return v.to(dev)
        self._crop_list = []
        for d in crops:
            data = amg_utils.MaskData()
            data._stats.update({k: place(k, v) for k, v in d.items()})
            self._crop_list.append(data)
        self._crop_boxes = state["crop_boxes"]
        self._original_size = state["original_size"]
        self._is_initialized = True

    def clear_state(self):
        self._crop_list = None
        self._crop_boxes = None
        self._original_size = None
        self._is_initialized = False


class AutomaticMaskGenerator(AMGBase):
    """instance_segmentation.py:288-530.  Same constructor / initialize / generate signatures."""

    def __init__(self, predictor, points_per_side: Optional[int] = 32, points_per_batch: Optional[int] = None,
                 crop_n_layers: int = 0, crop_overlap_ratio: float = 512 / 1500,
                 crop_n_points_downscale_factor: int = 1, point_grids: Optional[List[np.ndarray]] = None,
                 stability_score_offset: float = 1.0):
        super().__init__()
        if points_per_side is not None:
            self.point_grids = amg_utils.build_all_layer_point_grids(points_per_side, crop_n_layers,
                                                                     crop_n_points_downscale_factor)
        elif point_grids is not None:
            self.point_grids = point_grids
        else:
            raise ValueError("Can't have both points_per_side and point_grid be None or not None.")
        self._predictor = predictor
        self._points_per_side = points_per_side
        # the whole grid fits one decoder launch sequence; the engine chunks internally by its max_prompts
        self._points_per_batch = 1024 if points_per_batch is None else points_per_batch
        self._crop_n_layers = crop_n_layers
        self._crop_overlap_ratio = crop_overlap_ratio
        self._crop_n_points_downscale_factor = crop_n_points_downscale_factor
        self._stability_score_offset = stability_score_offset

    def _process_batch(self, points, im_size, crop_box, original_size):
        """instance_segmentation.py:356-369 + _to_mask_data :229-255, fused on the device."""
        pred = self._predictor
        transformed = pred.transform.apply_coords(points, im_size)
        in_points = torch.as_tensor(transformed, dtype=torch.float, device=pred.device)
        in_labels = torch.ones(in_points.shape[0], dtype=torch.float, device=pred.device)
        low, iou = pred.decode_low_res(in_points[:, None, :], in_labels[:, None], None, multimask_output=True)
        P, M = low.shape[:2]
        low = low.view(P * M, 256, 256)
        dev = low.device
        # statistics pending: filled by _ensure_stats for the masks a generate() call actually looks at
        data = amg_utils.MaskData(low_res=low, iou_preds=iou.reshape(-1),
                                  stability_score=torch.zeros(P * M, dtype=torch.float32, device=dev),
                                  boxes=torch.zeros(P * M, 4, dtype=torch.int32, device=dev),
                                  area=torch.zeros(P * M, dtype=torch.int32, device=dev),
                                  stats_done=torch.zeros(P * M, dtype=torch.uint8, device=dev))
        data["points"] = torch.as_tensor(points.repeat(M, axis=0), dtype=torch.float)
        return data

    def _process_crop(self, image_size, crop_box, crop_layer_idx, pbar_init=None, pbar_update=None):
        x0, y0, x1, y1 = crop_box
        cropped_im_size = (min(y1, image_size[0]) - y0, min(x1, image_size[1]) - x0)
        points_scale = np.array(cropped_im_size)[None, ::-1]
        points_for_image = self.point_grids[crop_layer_idx] * points_scale
        data = amg_utils.MaskData()
        n_batches = len(points_for_image) // self._points_per_batch + int(len(points_for_image) % self._points_per_batch != 0)
        if pbar_init is not None:
            pbar_init(n_batches, "Predict masks for point grid prompts")
        for (points,) in amg_utils.batch_iterator(self._points_per_batch, points_for_image):
            data.cat(self._process_batch(points, cropped_im_size, crop_box, self.original_size), copy=False)
            if pbar_update is not None:
                pbar_update(1)
        return data

    @torch.no_grad()
    def initialize(self, image: np.ndarray, image_embeddings: Optional[util.ImageEmbeddings] = None,
                   i: Optional[int] = None, verbose: bool = False, pbar_init: Optional[Callable] = None,
                   pbar_update: Optional[Callable] = None) -> None:
        original_size = image.shape[:2]
        self._original_size = original_size
        crop_boxes, layer_idxs = amg_utils.generate_crop_boxes(original_size, self._crop_n_layers,
                                                               self._crop_overlap_ratio)
        # a single crop (default) uses the (pre)computed embedding of the whole image; with crop layers every crop of the
        # globally normalised image is embedded on its own (instance_segmentation.py:433-441, :371-378)
        precomputed = len(crop_boxes) == 1
        if precomputed:
            if image_embeddings is None:
                image_embeddings = util.precompute_image_embeddings(self._predictor, image, to_numpy=False)
            util.set_precomputed(self._predictor, image_embeddings, i=i)
        else:
            image_u8 = util._to_image(image)
        _, pbar_init, pbar_update, pbar_close = util.handle_pbar(verbose, pbar_init, pbar_update)
        crop_list = []
        for crop_box, layer_idx in zip(crop_boxes, layer_idxs):
            if not precomputed:
                x0, y0, x1, y1 = crop_box
                self._predictor.set_image(np.ascontiguousarray(image_u8[y0:y1, x0:x1, :]))
            crop_list.append(self._process_crop(original_size, crop_box, layer_idx, pbar_init, pbar_update))
        if not precomputed:
            self._predictor.reset_image()
        pbar_close()
        self._is_initialized = True
        self._crop_list = crop_list
        self._crop_boxes = crop_boxes

    @torch.no_grad()
    def generate(self, pred_iou_thresh: float = 0.88, stability_score_thresh: float = 0.95, box_nms_thresh: float = 0.7,
                 crop_nms_thresh: float = 0.7, min_mask_region_area: int = 0,
                 output_mode: str = "instance_segmentation", with_background: bool = True):
        if not self.is_initialized:
            raise RuntimeError("AutomaticMaskGenerator has not been initialized. Call initialize first.")
        if output_mode not in ("instance_segmentation", "binary_mask", "rle", "coco_rle"):
            raise ValueError(f"Invalid output mode {output_mode}.")
        geoms = self._crop_geoms()
        if min_mask_region_area > 0:
            return self._generate_small_regions(pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh,
                                                min_mask_region_area, output_mode, with_background, geoms)
        if output_mode == "instance_segmentation" and len(self._crop_list) == 1 and geoms and \
                self._crop_list[0]["low_res"].device == self._crop_list[0]["iou_preds"].device and \
                tuple(self.crop_boxes[0]) == (0, 0, self.original_size[1], self.original_size[0]):
            out = self.generate_device(pred_iou_thresh, stability_score_thresh, box_nms_thresh, with_background)
            return out.cpu().numpy().view(np.uint32)
        return self._generate_multi(pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh, output_mode,
                                    with_background, geoms)

    def _generate_multi(self, pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh, output_mode,
                        with_background, geoms):
        """generate() for any number of crops / tiles (instance_segmentation.py:499-529): per-crop filters + NMS, then the
        cross-crop NMS that prefers masks from smaller crops, then records or painting."""
        H, W = self.original_size
        dev = self._predictor.device
        keeps, gboxes, crop_id = [], [], []
        for ci, (data, crop_box) in enumerate(zip(self._crop_list, self.crop_boxes)):
            keep = self._filter_nms(data, crop_box, self.original_size, pred_iou_thresh, stability_score_thresh,
                                    box_nms_thresh)
            keeps.append(keep)
            off = torch.tensor([crop_box[0], crop_box[1], crop_box[0], crop_box[1]], dtype=torch.int32, device=dev)
            gboxes.append(data["boxes"][keep] + off)
            crop_id.append(torch.full((len(keep),), ci, dtype=torch.int64, device=dev))
        gboxes = torch.cat(gboxes).contiguous() if gboxes else torch.zeros(0, 4, dtype=torch.int32, device=dev)
        crop_id = torch.cat(crop_id) if crop_id else torch.zeros(0, dtype=torch.int64, device=dev)
        local = torch.cat(keeps) if keeps else torch.zeros(0, dtype=torch.int64, device=dev)
        n = int(gboxes.shape[0])
        order = torch.arange(n, device=dev)
        if len(self.crop_boxes) > 1 and n > 0:
            cb = torch.tensor(self.crop_boxes, dtype=torch.float32, device=dev)
            scores = (1.0 / ((cb[:, 2] - cb[:, 0]) * (cb[:, 3] - cb[:, 1])))[crop_id].contiguous()
            keep2 = torch.empty(n, dtype=torch.int32, device=dev)
            n2 = torch.zeros(1, dtype=torch.int32, device=dev)
            zero4 = (ctypes.c_int32 * 4)(0, 0, 0, 0)
            _lib.check(_lib.lib().msam_amg_filter_nms(_lib.ptr(gboxes), _lib.ptr(scores), _lib.ptr(scores), n, 0, 0.0, 0.0,
                                                      float(crop_nms_thresh), zero4, zero4, _lib.ptr(keep2), _lib.ptr(n2),
                                                      _lib.cur_stream()))
            order = keep2[: int(n2.item())].long()
        crop_id, local, gboxes = crop_id[order], local[order], gboxes[order]
        n = len(order)
        if output_mode != "instance_segmentation":
            out = [None] * n
            for ci, (data, crop_box) in enumerate(zip(self._crop_list, self.crop_boxes)):
                pos = (crop_id == ci).nonzero()[:, 0]
                if len(pos) == 0:
                    continue
                recs = self._records(data, local[pos], crop_box, output_mode, geoms[ci])
                x0, y0, x1, y1 = crop_box
                for k, r in zip(pos.tolist(), recs):
                    if output_mode == "binary_mask" and (x1 - x0, y1 - y0) != (W, H):  # uncrop_masks
                        full = np.zeros((H, W), dtype=bool)
                        full[y0:y1, x0:x1] = r["segmentation"]
                        r["segmentation"] = full
                    elif output_mode in ("rle", "coco_rle") and (x1 - x0, y1 - y0) != (W, H):
                        rl = r["segmentation"] if output_mode == "rle" else amg_utils.coco_decode_rle(r["segmentation"])
                        full = np.zeros((H, W), dtype=bool)
                        full[y0:y1, x0:x1] = amg_utils.rle_to_mask(rl)
                        rl = amg_utils.mask_to_rle(full[None])[0]
                        r["segmentation"] = rl if output_mode == "rle" else amg_utils.coco_encode_rle(rl)
                    out[k] = r
            return out
        canvas = torch.full((H, W), -1, dtype=torch.int64, device=dev)
        L = _lib.lib()
        for ci, (data, crop_box) in enumerate(zip(self._crop_list, self.crop_boxes)):
            pos = (crop_id == ci).nonzero()[:, 0]
            if len(pos) == 0:
                continue
            low_dev, sel = self._logits_rows(data, local[pos], dev)
            gpos = pos.to(torch.int32).contiguous()
            g = geoms[ci]
            bx_t, ar_t = data["boxes"], data["area"]
            if low_dev is not data["low_res"]:   # offloaded state: the compacted logits are indexed 0..n-1, so are box / area
                bx_t, ar_t = data["boxes"][local[pos]].contiguous(), data["area"][local[pos]].contiguous()
            _lib.check(L.msam_paint_canvas(_lib.ptr(low_dev), _lib.ptr(sel), _lib.ptr(gpos), len(sel),
                                           _lib.ptr(bx_t), _lib.ptr(ar_t), g["inp"][0], g["inp"][1],
                                           g["orig"][0], g["orig"][1], 0.0, int(crop_box[0]), int(crop_box[1]),
                                           _lib.ptr(canvas), W, _lib.cur_stream()))
        label = torch.empty(H, W, dtype=torch.int32, device=dev)
        out = torch.empty(H, W, dtype=torch.int32, device=dev)
        ws = torch.empty(util.finish_ws_size(H, W), dtype=torch.int32, device=dev)
        _lib.check(L.msam_canvas_to_label(_lib.ptr(canvas), H * W, _lib.ptr(label), _lib.cur_stream()))
        _lib.check(L.msam_finish_segmentation(_lib.ptr(label), H, W, 0, int(with_background), _lib.ptr(out), _lib.ptr(ws),
                                              _lib.cur_stream()))
        return out.cpu().numpy().view(np.uint32)

    def _generate_small_regions(self, pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh, min_area,
                                output_mode, with_background, geoms):
        """generate(min_mask_region_area > 0): AMGBase._postprocess_small_regions (instance_segmentation.py:146-186) on the
        device -- holes then islands smaller than `min_area` are filled / removed per mask (8-connected components,
        `msam_remove_small_regions`), boxes are recomputed, and a box NMS that prefers unchanged masks drops new duplicates."""
        recs = self._generate_multi(pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh, "binary_mask",
                                    with_background, geoms)
        H, W = self.original_size
        dev = self._predictor.device
        L = _lib.lib()
        n = len(recs)
        if n > 0:
            masks = torch.from_numpy(np.stack([r["segmentation"] for r in recs])).to(dev).to(torch.uint8).contiguous()
            changed = torch.zeros(n, dtype=torch.bool, device=dev)
            CH = 128
            ws = torch.empty(min(n, CH) * (2 * H * W + 4), dtype=torch.int32, device=dev)
            for s0 in range(0, n, CH):
                m = masks[s0:s0 + CH]
                for holes in (1, 0):
                    ch = torch.zeros(m.shape[0], dtype=torch.int32, device=dev)
                    _lib.check(L.msam_remove_small_regions(_lib.ptr(m), m.shape[0], H, W, int(min_area), holes, _lib.ptr(ch),
                                                           _lib.ptr(ws), _lib.cur_stream()))
                    changed[s0:s0 + CH] |= ch != 0
            boxes = torch.empty(n, 4, dtype=torch.int32, device=dev)
            area = torch.empty(n, dtype=torch.int32, device=dev)
            _lib.check(L.msam_mask_boxes(_lib.ptr(masks), n, H, W, _lib.ptr(boxes), _lib.ptr(area), _lib.cur_stream()))
            scores = (~changed).to(torch.float32).contiguous()
            keep = torch.empty(n, dtype=torch.int32, device=dev)
            nk = torch.zeros(1, dtype=torch.int32, device=dev)
            z4 = (ctypes.c_int32 * 4)(0, 0, 0, 0)
            _lib.check(L.msam_amg_filter_nms(_lib.ptr(boxes), _lib.ptr(scores), _lib.ptr(scores), n, 0, 0.0, 0.0,
                                             float(max(box_nms_thresh, crop_nms_thresh)), z4, z4, _lib.ptr(keep), _lib.ptr(nk),
                                             _lib.cur_stream()))
            keep = keep[: int(nk.item())].long()
            ch_h, bx_h, ar_h = changed.cpu().numpy(), boxes.cpu().numpy().astype(np.int64), area.cpu().numpy()
            out = []
            for k in keep.tolist():
                r = recs[k]
                if ch_h[k]:   # only changed masks get a new mask / box / area (:176-182)
                    r = dict(r, segmentation=masks[k].bool().cpu().numpy(), area=int(ar_h[k]),
                             bbox=amg_utils.box_xyxy_to_xywh(bx_h[k]).tolist())
                out.append(r)
            recs = out
        if output_mode == "binary_mask":
            return recs
        if output_mode in ("rle", "coco_rle"):
            rl = [amg_utils.mask_to_rle(r["segmentation"][None])[0] for r in recs]
            if output_mode == "coco_rle":
                rl = [amg_utils.coco_encode_rle(x) for x in rl]
            return [dict(r, segmentation=x) for r, x in zip(recs, rl)]
        # instance segmentation: mask_data_to_segmentation(..., merge_exclusively=False): descending area, later overwrites
        label = torch.zeros(H, W, dtype=torch.int32, device=dev)
        order = sorted(range(len(recs)), key=lambda k: recs[k]["area"], reverse=True)
        for sid, k in enumerate(order, 1):
            label[torch.from_numpy(recs[k]["segmentation"]).to(dev)] = sid
        out_t = torch.empty(H, W, dtype=torch.int32, device=dev)
        ws2 = torch.empty(util.finish_ws_size(H, W), dtype=torch.int32, device=dev)
        _lib.check(L.msam_finish_segmentation(_lib.ptr(label), H, W, 0, int(with_background), _lib.ptr(out_t), _lib.ptr(ws2),
                                              _lib.cur_stream()))
        return out_t.cpu().numpy().view(np.uint32)

    @torch.no_grad()
    def generate_device(self, pred_iou_thresh: float = 0.88, stability_score_thresh: float = 0.95,
                        box_nms_thresh: float = 0.7, with_background: bool = True, finish: bool = True, **_):
        """generate(output_mode="instance_segmentation") entirely on the device and without any host synchronisation:
        filter+NMS -> per-pixel min-area painting (n_keep read on the device) -> connected components / background
        removal / consecutive relabel (msam_finish_segmentation).  Returns a uint32-valued int32 (H, W) device tensor."""
        if not self.is_initialized:
            raise RuntimeError("AutomaticMaskGenerator has not been initialized. Call initialize first.")
        if len(self._crop_list) != 1:
            raise NotImplementedError("device-side generate supports a single crop")
        data, crop_box, geom = self._crop_list[0], self.crop_boxes[0], self._crop_geoms()[0]
        H, W = self.original_size
        dev = data["iou_preds"].device
        if data["low_res"].device != dev:
            raise NotImplementedError("device-side generate needs the state on the device (offload_state=False)")
        keep = self._filter_nms(data, crop_box, self.original_size, pred_iou_thresh, stability_score_thresh,
                                box_nms_thresh, sync=False)
        bufs = getattr(self, "_dev_bufs", None)
        if bufs is None or bufs[0].shape != (H, W) or bufs[0].device != dev:
            bufs = (torch.empty(H, W, dtype=torch.int32, device=dev), torch.empty(H, W, dtype=torch.int32, device=dev),
                    torch.empty(util.finish_ws_size(H, W), dtype=torch.int32, device=dev))
            self._dev_bufs = bufs
        painted, out, ws = bufs
        L = _lib.lib()
        _lib.check(L.msam_paint_min_area(_lib.ptr(data["low_res"]), _lib.ptr(keep), _lib.ptr(self._n_keep_dev),
                                         _lib.ptr(data["boxes"]), _lib.ptr(data["area"]), geom["inp"][0], geom["inp"][1],
                                         geom["orig"][0], geom["orig"][1], 0.0, _lib.ptr(painted), W, _lib.cur_stream()))
        if not finish:
            return painted
        _lib.check(L.msam_finish_segmentation(_lib.ptr(painted), H, W, 0, int(with_background), _lib.ptr(out), _lib.ptr(ws),
                                              _lib.cur_stream()))
        return out



class TiledAutomaticMaskGenerator(AutomaticMaskGenerator):
    """instance_segmentation.py:564-680: AMG over tiled embeddings; every (outer) tile acts as a crop, `generate` is the
    inherited multi-crop path (per-tile filters + NMS, cross-tile NMS, global painting)."""

    @torch.no_grad()
    def generate(self, pred_iou_thresh: float = 0.88, stability_score_thresh: float = 0.95, box_nms_thresh: float = 0.7,
                 crop_nms_thresh: float = 0.7, min_mask_region_area: int = 0, output_mode: str = "instance_segmentation",
                 with_background: bool = True, group=None):
        if self._world_size == 1:
            return super().generate(pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh,
                                    min_mask_region_area, output_mode, with_background)
        if not self.is_initialized:
            raise RuntimeError("TiledAutomaticMaskGenerator has not been initialized. Call initialize first.")
        if output_mode != "instance_segmentation" or min_mask_region_area > 0:
            raise NotImplementedError("multi-rank generate() produces the stitched instance segmentation")
        return self._generate_distributed(pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh,
                                          with_background, group)

    def _generate_distributed(self, pred_iou_thresh, stability_score_thresh, box_nms_thresh, crop_nms_thresh, with_background,
                              group):
        """instance_segmentation.py:499-529 across ranks: per-tile filters + box NMS on the owner rank, ONE all-gather of
        the survivors' instance tables (global box, tile id, tile-local box, area, low-res logits), then the cross-tile
        NMS that prefers smaller tiles (:511-521) and the painting (util.py:1799-1829) on the gathered list, identically
        on every rank (so every rank returns the full label image)."""
        from . import distributed as D
        local = self._local_instance_tables(pred_iou_thresh, stability_score_thresh, box_nms_thresh)
        tab, _ = D.gather_instance_tables(local, group)          # <- the one collective of the stitched path
        return self._stitch_gathered(tab, crop_nms_thresh, with_background)

    def _local_instance_tables(self, pred_iou_thresh, stability_score_thresh, box_nms_thresh):
        """This rank's contribution to the exchange: per-tile filters + box NMS on the tiles it owns."""
        dev = self._predictor.device
        tabs = dict(gbox=[], lbox=[], area=[], tile=[], low=[])
        for k, data in enumerate(self._crop_list):
            ci = self._tile_lo + k
            crop_box = self.crop_boxes[ci]
            keep = self._filter_nms(data, crop_box, self.original_size, pred_iou_thresh, stability_score_thresh, box_nms_thresh)
            off = torch.tensor([crop_box[0], crop_box[1], crop_box[0], crop_box[1]], dtype=torch.int32, device=dev)
            tabs["gbox"].append(data["boxes"][keep] + off)
            tabs["lbox"].append(data["boxes"][keep])
            tabs["area"].append(data["area"][keep])
            tabs["tile"].append(torch.full((len(keep),), ci, dtype=torch.int32, device=dev))
            tabs["low"].append(self._logits_rows(data, keep, dev)[0] if data["low_res"].device != dev else data["low_res"][keep])
        empty = dict(gbox=(0, 4), lbox=(0, 4), area=(0,), tile=(0,), low=(0, 256, 256))
        return {k: (torch.cat(v) if v else torch.zeros(empty[k], dtype=torch.float32 if k == "low" else torch.int32, device=dev))
                for k, v in tabs.items()}

    def _stitch_gathered(self, tab, crop_nms_thresh, with_background):
        """Cross-tile NMS + painting on the gathered instance tables (rank order = tile order), identical on every rank."""
        H, W = self.original_size
        dev = self._predictor.device
        geoms = self._crop_geoms()
        n = int(tab["gbox"].shape[0])
        crop_id = tab["tile"].long()
        order = torch.arange(n, device=dev)
        L = _lib.lib()
        if len(self.crop_boxes) > 1 and n > 0:
            cb = torch.tensor(self.crop_boxes, dtype=torch.float32, device=dev)
            scores = (1.0 / ((cb[:, 2] - cb[:, 0]) * (cb[:, 3] - cb[:, 1])))[crop_id].contiguous()
            keep2 = torch.empty(n, dtype=torch.int32, device=dev)
            n2 = torch.zeros(1, dtype=torch.int32, device=dev)
            zero4 = (ctypes.c_int32 * 4)(0, 0, 0, 0)
            gb = tab["gbox"].contiguous()
            _lib.check(L.msam_amg_filter_nms(_lib.ptr(gb), _lib.ptr(scores), _lib.ptr(scores), n, 0, 0.0, 0.0,
                                             float(crop_nms_thresh), zero4, zero4, _lib.ptr(keep2), _lib.ptr(n2),
                                             _lib.cur_stream()))
            order = keep2[: int(n2.item())].long()
        crop_id = crop_id[order]
        low, lbox, area = tab["low"].contiguous(), tab["lbox"].contiguous(), tab["area"].contiguous()
        canvas = torch.full((H, W), -1, dtype=torch.int64, device=dev)
        for ci, crop_box in enumerate(self.crop_boxes):
            pos = (crop_id == ci).nonzero()[:, 0]
            if len(pos) == 0:
                continue
            sel = order[pos].to(torch.int32).contiguous()      # rows of the gathered table
            gpos = pos.to(torch.int32).contiguous()            # position in the NMS-ordered global list
            g = geoms[ci]
            _lib.check(L.msam_paint_canvas(_lib.ptr(low), _lib.ptr(sel), _lib.ptr(gpos), len(sel), _lib.ptr(lbox), _lib.ptr(area),
                                           g["inp"][0], g["inp"][1], g["orig"][0], g["orig"][1], 0.0, int(crop_box[0]),
                                           int(crop_box[1]), _lib.ptr(canvas), W, _lib.cur_stream()))
        label = torch.empty(H, W, dtype=torch.int32, device=dev)
        out = torch.empty(H, W, dtype=torch.int32, device=dev)
        ws = torch.empty(util.finish_ws_size(H, W), dtype=torch.int32, device=dev)
        _lib.check(L.msam_canvas_to_label(_lib.ptr(canvas), H * W, _lib.ptr(label), _lib.cur_stream()))
        _lib.check(L.msam_finish_segmentation(_lib.ptr(label), H, W, 0, int(with_background), _lib.ptr(out), _lib.ptr(ws),
                                              _lib.cur_stream()))
        return out.cpu().numpy().view(np.uint32)

    def __init__(self, predictor, points_per_side: Optional[int] = 32, points_per_batch: Optional[int] = None,
                 point_grids: Optional[List[np.ndarray]] = None, stability_score_offset: float = 1.0) -> None:
        super().__init__(predictor=predictor, points_per_side=points_per_side, points_per_batch=points_per_batch,
                         point_grids=point_grids, stability_score_offset=stability_score_offset)
        self._rank, self._world_size, self._tile_lo = 0, 1, 0

    @torch.no_grad()
    def initialize(self, image: np.ndarray, image_embeddings: Optional[util.ImageEmbeddings] = None,
                   i: Optional[int] = None, tile_shape=None, halo=None, verbose: bool = False,
                   pbar_init: Optional[Callable] = None, pbar_update: Optional[Callable] = None, batch_size: int = 1,
                   mask=None, rank: int = 0, world_size: int = 1, offload_state: Optional[bool] = None) -> None:
        """rank / world_size (one process per GPU, `torch.distributed` initialised): this rank embeds and decodes only its
        contiguous share of the tiles; `generate()` then all-gathers the per-tile instance tables (one exchange, NCCL) so
        that the cross-tile NMS and the painting see every instance -- the result is the single-process result bit for bit.
        offload_state: keep the per-tile low-res logits (805 MB per tile at the default 32x32 grid) in pinned host memory
        instead of HBM; None = automatically when this rank's tiles would need more than half of the free device memory."""
        original_size = image.shape[:2]
        self._original_size = original_size
        self._rank, self._world_size = int(rank), int(world_size)
        if image_embeddings is None:
            if tile_shape is None or halo is None:
                raise ValueError("To compute tiled embeddings the parameters tile_shape and halo have to be passed.")
            image_embeddings = util.precompute_image_embeddings(self._predictor, image, tile_shape=tile_shape, halo=halo,
                                                                verbose=verbose, batch_size=batch_size, mask=mask,
                                                                to_numpy=False, rank=rank, world_size=world_size)
        feats = image_embeddings["features"]
        tile_shape_, halo_ = tuple(feats.attrs["tile_shape"]), tuple(feats.attrs["halo"])
        if tile_shape is not None and tuple(tile_shape) != tile_shape_:
            raise ValueError(f"Inconsistent tile_shape parameter {tile_shape} with precomputed embeedings: {tile_shape_}.")
        if halo is not None and tuple(halo) != halo_:
            raise ValueError(f"Inconsistent halo parameter {halo} with precomputed embeedings: {halo_}.")
        tile_shape, halo = tile_shape_, halo_
        tiles_in_mask = feats.attrs.get("tiles_in_mask", None)
        if tiles_in_mask is not None and i is not None:
            tiles_in_mask = tiles_in_mask[str(i)]
        tiling = amg_utils.Blocking([0, 0], original_size, tile_shape)
        tile_ids = list(range(tiling.number_of_blocks) if tiles_in_mask is None else tiles_in_mask)
        tiles = [tiling.get_block_with_halo(t, list(halo)).outer_block for t in tile_ids]
        crop_boxes = [[t.begin[1], t.begin[0], t.end[1], t.end[0]] for t in tiles]
        # this rank's contiguous share of the tile list (the same partition precompute_image_embeddings uses in 2-D)
        lo, hi = (len(tile_ids) * self._rank) // self._world_size, (len(tile_ids) * (self._rank + 1)) // self._world_size
        self._tile_lo = lo
        _, pbar_init, pbar_update, pbar_close = util.handle_pbar(verbose, pbar_init, pbar_update)
        pbar_init(hi - lo, "Compute masks for tile")
        mask_data = []
        if offload_state is None:
            n_pts = sum(len(g) for g in self.point_grids[:1])
            need = (hi - lo) * n_pts * 3 * 256 * 256 * 4
            offload_state = need > 0.5 * torch.cuda.mem_get_info(self._predictor.device)[0]
        for idx, tile_id in list(enumerate(tile_ids))[lo:hi]:
            f = feats[str(tile_id)]
            util.set_precomputed(self._predictor, {"features": f, "input_size": f.attrs["input_size"],
                                                   "original_size": f.attrs["original_size"]}, i)
            mask_data.append(self._process_crop(original_size, crop_boxes[idx], 0))
            if offload_state:
                self._offload(mask_data[-1], crop_boxes[idx])
            pbar_update(1)
        pbar_close()
        self._is_initialized = True
        self._crop_list = mask_data
        self._crop_boxes = crop_boxes


def get_instance_segmentation_generator(predictor, is_tiled: bool, decoder=None, segmentation_mode: Optional[str] = None,
                                        **kwargs):
    """instance_segmentation.py:1631: only the AMG mode exists on this path (AIS/APG need the UNETR decoder, 8f-2)."""
    if decoder is not None or segmentation_mode not in (None, "amg"):
        raise NotImplementedError("only segmentation_mode='amg' is available on the GPU path")
    return (TiledAutomaticMaskGenerator if is_tiled else AutomaticMaskGenerator)(predictor, **kwargs)
