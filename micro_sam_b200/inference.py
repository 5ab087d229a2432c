"""micro_sam.inference.batched_inference (inference.py:155-286) on the H100 core.

`batched_tiled_inference` / `_stitch_segmentation` (inference.py:315-538) route prompts to tiles and call it per tile.

Same signature and return values; the per-batch `predict_torch` + `_process_masks_for_batch` (:137-151, three passes
over (P,1,H,W) fp32 logits) + per-mask `.item()` record building + CPU painting are replaced by: decode -> fused
`msam_mask_stats` -> `msam_paint` (exclusive, descending area) on the device; only the uint32 label image is copied back.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Union

import numpy as np
import torch

from . import _amg_utils as amg_utils
from . import _lib, util
from .sam import ResizeLongestSide, local_otsu_threshold, mask_stats


def _validate_inputs(boxes, points, point_labels, multimasking, return_instance_segmentation, segmentation_ids,
                     logits_masks):
    """inference.py:22-67."""
    if multimasking and (segmentation_ids is not None) and (not return_instance_segmentation):
        raise NotImplementedError
    if (points is None) != (point_labels is None):
        raise ValueError("If you have point prompts both `points` and `point_labels` have to be passed, "
                         "but you passed only one of them.")
    have_points, have_boxes, have_logits = points is not None, boxes is not None, logits_masks is not None
    if (not have_points) and (not have_boxes):
        raise ValueError("Point and/or box prompts have to be passed, you passed neither.")
    if have_points and (len(point_labels) != len(points)):
        raise ValueError(f"The number of point coordinates and labels does not match: {len(point_labels)} != {len(points)}")
    if (have_points and have_boxes) and (len(points) != len(boxes)):
        raise ValueError(f"The number of point and box prompts does not match: {len(points)} != {len(boxes)}")
    n_prompts = boxes.shape[0] if have_boxes else points.shape[0]
    if (segmentation_ids is not None) and (len(segmentation_ids) != n_prompts):
        raise ValueError(f"The number of segmentation ids and prompts does not match: {len(segmentation_ids)} != {n_prompts}")
    return n_prompts, have_boxes, have_points, have_logits


@torch.no_grad()
def batched_inference(predictor, image: Optional[np.ndarray], batch_size: int, boxes: Optional[np.ndarray] = None,
                      points: Optional[np.ndarray] = None, point_labels: Optional[np.ndarray] = None,
                      multimasking: bool = False, embedding_path=None, return_instance_segmentation: bool = True,
                      segmentation_ids: Optional[list] = None, reduce_multimasking: bool = True,
                      logits_masks: Optional[torch.Tensor] = None, verbose_embeddings: bool = False,
                      mask_threshold: Optional[Union[float, str]] = None, return_highres_logits: bool = False,
                      i: Optional[int] = None, device_result: bool = False):
    """`device_result=True` (extension): the instance segmentation stays on the device (int32 (H, W) tensor holding the
    uint32 ids), skipping the D2H copy the reference's numpy return implies."""
    n_prompts, have_boxes, have_points, have_logits = _validate_inputs(
        boxes, points, point_labels, multimasking, return_instance_segmentation, segmentation_ids, logits_masks)
    if image is None:
        predictor.get_image_embedding()
    else:
        input_ = image if i is None else image[i]
        emb = util.precompute_image_embeddings(predictor, input_, embedding_path, verbose=verbose_embeddings, to_numpy=False)
        util.set_precomputed(predictor, emb)
    device = predictor.device
    tf = ResizeLongestSide(1024)
    image_shape = predictor.original_size
    if have_boxes:
        boxes_t = torch.tensor(tf.apply_boxes(boxes, image_shape), dtype=torch.float32).to(device)
    if have_points:
        points_t = torch.tensor(tf.apply_coords(points, image_shape), dtype=torch.float32).to(device)
        labels_t = torch.tensor(point_labels, dtype=torch.float32).to(device)
    auto = isinstance(mask_threshold, str)
    if auto and mask_threshold != "auto":
        raise ValueError(f"Invalid mask_threshold {mask_threshold}")
    thr = predictor.model.mask_threshold if (mask_threshold is None or auto) else float(mask_threshold)

    lows, ious = [], []
    for s in range(0, n_prompts, batch_size):
        e = min(s + batch_size, n_prompts)
        low, iou = predictor.decode_low_res(points_t[s:e] if have_points else None, labels_t[s:e] if have_points else None,
                                            boxes_t[s:e] if have_boxes else None, multimask_output=multimasking,
                                            mask_input=logits_masks[s:e] if have_logits else None)
        if multimasking and reduce_multimasking:  # keep the mask with the highest predicted IoU (inference.py:259-263)
            best = iou.argmax(dim=1)
            sel = torch.arange(low.shape[0], device=device)
            low, iou = low[sel, best][:, None], iou[sel, best][:, None]
        # without the reduction all three masks of every prompt become records (flattened prompt-major, :266-269)
        lows.append(low.flatten(0, 1))
        ious.append(iou.flatten(0, 1))
    low = torch.cat(lows).contiguous()
    iou = torch.cat(ious)
    if low.shape[0] != n_prompts:
        if segmentation_ids is not None:
            raise ValueError("segmentation_ids cannot be combined with multimasking without reduce_multimasking")
        n_prompts = low.shape[0]
    thr_t = local_otsu_threshold(low) if auto else None   # one threshold per mask (inference.py:137-151)
    bxs, stab, area = mask_stats(low, predictor.input_size, image_shape, thr_t if auto else thr, 1.0)
    H, W = image_shape
    inp = predictor.input_size
    seg_ids = np.arange(1, n_prompts + 1) if segmentation_ids is None else np.asarray(segmentation_ids, dtype=np.int64)

    if return_instance_segmentation:
        # mask_data_to_segmentation(masks, min_object_size=0): descending area (stable), first painter wins, CC, relabel
        order = torch.argsort(area, descending=True, stable=True)
        sel = order.to(torch.int32).contiguous()
        ids = torch.as_tensor(seg_ids, device=device)[order].to(torch.int32).contiguous()
        label = torch.zeros(H, W, dtype=torch.int32, device=device)
        if auto:
            _lib.check(_lib.lib().msam_paint_ex(_lib.ptr(low), _lib.ptr(sel), _lib.ptr(bxs), _lib.ptr(ids), n_prompts,
                                                int(inp[0]), int(inp[1]), H, W, _lib.ptr(thr_t), 1, _lib.ptr(label), W,
                                                _lib.cur_stream()))
        else:
            _lib.check(_lib.lib().msam_paint(_lib.ptr(low), _lib.ptr(sel), _lib.ptr(bxs), _lib.ptr(ids), n_prompts, int(inp[0]),
                                             int(inp[1]), H, W, float(thr), 1, _lib.ptr(label), W, _lib.cur_stream()))
        # connected components + consecutive relabelling on the device (util.py:1831-1848), like the AMG path
        out = torch.empty(H, W, dtype=torch.int32, device=device)
        ws = torch.empty(util.finish_ws_size(H, W), dtype=torch.int32, device=device)
        _lib.check(_lib.lib().msam_finish_segmentation(_lib.ptr(label), H, W, 0, 0, _lib.ptr(out), _lib.ptr(ws),
                                                       _lib.cur_stream()))
        return out if device_result else out.cpu().numpy().view(np.uint32)

    binm = torch.empty(n_prompts, H, W, dtype=torch.uint8, device=device)
    logits = torch.empty(n_prompts, H, W, dtype=torch.float32, device=device) if return_highres_logits else None
    if auto:
        _lib.check(_lib.lib().msam_upsample_masks_ex(_lib.ptr(low), None, n_prompts, int(inp[0]), int(inp[1]), H, W,
                                                     _lib.ptr(thr_t), _lib.ptr(logits), _lib.ptr(binm), _lib.cur_stream()))
    else:
        _lib.check(_lib.lib().msam_upsample_masks(_lib.ptr(low), None, n_prompts, int(inp[0]), int(inp[1]), H, W, float(thr),
                                                  _lib.ptr(logits), _lib.ptr(binm), _lib.cur_stream()))
    binm = binm.bool()
    bx, io, st, ar = bxs.cpu().numpy(), iou.cpu().numpy(), stab.cpu().numpy(), area.cpu().numpy()
    return [{
        "segmentation": binm[k], "area": int(ar[k]), "bbox": amg_utils.box_xyxy_to_xywh(bx[k].astype(np.int64)).tolist(),
        "predicted_iou": float(io[k]), "stability_score": float(st[k]), "seg_id": int(seg_ids[k]),
        "logits": (logits[k][None] if return_highres_logits else low[k][None]),
    } for k in range(n_prompts)]


def _require_tiled_embeddings(predictor, image, image_embeddings, embedding_path, tile_shape, halo, verbose_embeddings):
    """inference.py:289-312."""
    if image_embeddings is None:
        assert image is not None
        assert (tile_shape is not None) and (halo is not None)
        shape = image.shape[:2]
        image_embeddings = util.precompute_image_embeddings(predictor, image, embedding_path, ndim=2, tile_shape=tile_shape,
                                                            halo=halo, verbose=verbose_embeddings, to_numpy=False)
    else:
        attrs = image_embeddings["features"].attrs
        tile_shape_, halo_, shape = attrs["tile_shape"], attrs["halo"], attrs["shape"]
        if tile_shape is None:
            tile_shape = tile_shape_
        elif any(ts != ts_ for ts, ts_ in zip(tile_shape, tile_shape_)):
            raise ValueError(f"Incompatible tile shapes: {tile_shape} != {tile_shape_}")
        if halo is None:
            halo = halo_
        elif any(ts != ts_ for ts, ts_ in zip(halo, halo_)):
            raise ValueError(f"Incompatible tile shapes: {halo} != {halo_}")
    return image_embeddings, tuple(shape), tuple(tile_shape), tuple(halo)


def _merge_segmentations(this_seg, prev_seg, overlap_threshold=0.75):
    """inference.py:315-332.  The reference computes the ids to discard (overlap > threshold) but never applies them, so the
    observable behaviour -- reproduced here -- is: the previous segmentation is fully preserved."""
    captured = prev_seg != 0
    this_seg[captured] = prev_seg[captured]
    return this_seg


def _stitch_segmentation(masks, tile_ids, tiling, halo, output_shape, verbose=False):
    """inference.py:337-356: first come, first served."""
    assert len(masks) == len(tile_ids), f"{len(masks)}, {len(tile_ids)}"
    segmentation = np.zeros(output_shape, dtype="uint32")
    for tile_id, this_seg in zip(tile_ids, masks):
        tile = tiling.get_block_with_halo(tile_id, list(halo)).outer_block
        bb = tuple(slice(begin, end) for begin, end in zip(tile.begin, tile.end))
        if tile_id == 0:
            segmentation[bb] = this_seg
        else:
            prev_seg = segmentation[bb]
            assert prev_seg.shape == this_seg.shape, f"{tile_id}: {prev_seg.shape}, {this_seg.shape}"
            segmentation[bb] = _merge_segmentations(this_seg, prev_seg)
    return segmentation


def _route_prompts_to_tiles(tiling, halo, boxes, points, point_labels):
    """Prompt -> tile assignment of batched_tiled_inference (inference.py:424-470), vectorised: every prompt goes to the tile
    that holds its anchor (box centre, else the point) and keeps its original order inside the tile.  Tile-local boxes are
    assembled exactly like the reference does (inference.py:438-445), i.e. as (y0, x0, y1, x1) clipped to the outer tile --
    kept as is so that results stay identical.  Returns (sorted tile ids, boxes / points / labels per tile)."""
    have_boxes, have_points = boxes is not None, points is not None
    if have_boxes:
        anchors = np.stack([(boxes[:, 1] + boxes[:, 3]) / 2, (boxes[:, 0] + boxes[:, 2]) / 2], axis=1)
    else:
        anchors = points[:, 0, ::-1]
    anchors = np.asarray(anchors).round().astype("int")
    tile_of = np.array([tiling.coordinates_to_block_id(a.tolist()) for a in anchors], dtype=np.int64)
    if have_boxes and have_points:
        pt_tiles = [tiling.coordinates_to_block_id(pt.tolist()) for pt in np.asarray(points[:, 0, ::-1]).round().astype("int")]
        assert np.array_equal(tile_of, np.array(pt_tiles)), "box and point prompts of a pair must fall into the same tile"
    tile_ids = sorted(set(tile_of.tolist()))
    box_to_tile, point_to_tile, label_to_tile = {}, {}, {}
    for tile_id in tile_ids:
        sel = np.flatnonzero(tile_of == tile_id)
        outer = tiling.get_block_with_halo(tile_id, list(halo)).outer_block
        (oy, ox), (th, tw) = outer.begin, outer.shape
        if have_boxes:
            bx = boxes[sel]
            box_to_tile[tile_id] = np.stack([np.maximum(bx[:, 1] - oy, 0), np.maximum(bx[:, 0] - ox, 0),
                                             np.minimum(bx[:, 3] - oy, th), np.minimum(bx[:, 2] - ox, tw)], axis=1)
        if have_points:
            point_to_tile[tile_id] = points[sel] - np.array([ox, oy])[None, None]
            label_to_tile[tile_id] = point_labels[sel]
    return tile_ids, box_to_tile, point_to_tile, label_to_tile


@torch.no_grad()
def batched_tiled_inference(predictor, image: Optional[np.ndarray], batch_size: int, image_embeddings=None,
                            boxes: Optional[np.ndarray] = None, points: Optional[np.ndarray] = None,
                            point_labels: Optional[np.ndarray] = None, multimasking: bool = False, embedding_path=None,
                            return_instance_segmentation: bool = True, reduce_multimasking: bool = True,
                            logits_masks: Optional[torch.Tensor] = None, verbose_embeddings: bool = True,
                            mask_threshold: Optional[Union[float, str]] = None, tile_shape=None, halo=None,
                            optimize_memory: bool = False, i: Optional[int] = None, **nms_kwargs):
    """inference.py:359-538: prompts are assigned to the tile that contains the box centre / the point, decoded per tile
    (tile-local coordinates, tile embeddings switched with `set_precomputed`), and either returned with a `global_bbox`
    (painted by `mask_data_to_segmentation`) or, with `optimize_memory`, reduced per tile by `apply_nms` and stitched."""
    segmentation_ids = None
    n_prompts, have_boxes, have_points, have_logits = _validate_inputs(
        boxes, points, point_labels, multimasking, return_instance_segmentation, segmentation_ids, logits_masks)
    if have_logits:
        raise NotImplementedError
    image_embeddings, shape, tile_shape, halo = _require_tiled_embeddings(
        predictor, image, image_embeddings, embedding_path, tile_shape, halo, verbose_embeddings)

    tiling = amg_utils.Blocking([0, 0], shape, tile_shape)
    tile_ids, box_to_tile, point_to_tile, label_to_tile = _route_prompts_to_tiles(tiling, halo, boxes, points, point_labels)

    masks, id_offset = [], 0
    for tile_id in tile_ids:
        predictor = util.set_precomputed(predictor, image_embeddings, tile_id=tile_id, i=i)
        this_masks = batched_inference(
            predictor=predictor, image=None, batch_size=batch_size, boxes=box_to_tile.get(tile_id),
            points=point_to_tile.get(tile_id), point_labels=label_to_tile.get(tile_id), multimasking=multimasking,
            return_instance_segmentation=False, segmentation_ids=segmentation_ids, reduce_multimasking=reduce_multimasking,
            logits_masks=None, mask_threshold=mask_threshold)
        if optimize_memory:
            segmentation = util.apply_nms(this_masks, **nms_kwargs)
            fg_mask = segmentation != 0
            segmentation[fg_mask] += id_offset
            id_offset = segmentation.max()
            masks.append(segmentation)
        else:
            tile = tiling.get_block_with_halo(tile_id, list(halo)).outer_block
            offset = np.array(tile.begin[::-1] + [0, 0])
            masks.extend({**mask, "global_bbox": (np.array(mask["bbox"]) + offset).tolist()} for mask in this_masks)

    if optimize_memory:
        return _stitch_segmentation(masks, tile_ids, tiling, halo, output_shape=shape)
    if return_instance_segmentation:
        masks = util.mask_data_to_segmentation(masks, shape=shape, min_object_size=0)
    return masks
