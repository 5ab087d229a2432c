"""Interactive (prompt-based) segmentation on the GPU predictor: `segment_from_points / _box / _box_and_points / _mask`
with the reference's signatures (micro_sam/prompt_based_segmentation.py:251-506), including the tiled-embedding routing
(`_initialize_predictor`, :209-231) and the mask -> (box, points, logits) prompt derivation (:28-113).

Everything numeric runs in `B200SamPredictor.predict` (one decoder pass on the device); this module is the host glue around
it.  `_compute_points_from_mask` needs skimage / bioimage_cpp in the reference (boundaries, distance transform, Gaussian
smoothing, `peak_local_max`); they are absent here and restated with scipy -- same definitions, parity unpinned for that
helper only (DESIGN.md).
"""
from __future__ import annotations

import warnings
from typing import Optional, Tuple

import numpy as np
import torch

from . import util
from ._amg_utils import Blocking
from .sam import ResizeLongestSide


# ------------------------------------------------------------------------------------------------ prompt derivation
def _process_box(box, shape, original_size=None, box_extension=0):
    """(y0, x0, y1, x1) python-convention box -> SAM's XYXY, optionally extended and rescaled (:119-140)."""
    if box_extension == 0:
        ext_y = ext_x = 0
    elif box_extension >= 1:
        ext_y = ext_x = box_extension
    else:
        ext_y, ext_x = box_extension * (box[2] - box[0]), box_extension * (box[3] - box[1])
    out = np.array([max(box[1] - ext_x, 0), max(box[0] - ext_y, 0),
                    min(box[3] + ext_x, shape[1]), min(box[2] + ext_y, shape[0])])
    if original_size is not None:
        out = ResizeLongestSide(max(original_size)).apply_boxes(out[None], (256, 256)).squeeze()
    return np.round(out).astype(int)


def _compute_box_from_mask(mask, original_size=None, box_extension=0):
    ys, xs = np.where(mask == 1)
    box = np.array([ys.min(), xs.min(), ys.max() + 1, xs.max() + 1])
    return _process_box(box, mask.shape, original_size=original_size, box_extension=box_extension)


def _peak_local_max(img: np.ndarray, min_distance: int) -> np.ndarray:
    """skimage.feature.peak_local_max(img, exclude_border=False, min_distance=d) semantics: pixels that equal the maximum of
    their (2d+1)^2 neighbourhood and are > 0 (threshold_abs defaults to the image minimum for non-negative inputs),
    strongest first, thinned so that no two peaks are closer than d (Chebyshev)."""
    from scipy import ndimage
    size = 2 * min_distance + 1
    is_peak = (ndimage.maximum_filter(img, size=size, mode="nearest") == img) & (img > img.min())
    coords = np.argwhere(is_peak)
    if len(coords) == 0:
        return coords.reshape(0, 2)
    order = np.argsort(-img[tuple(coords.T)], kind="stable")
    coords = coords[order]
    keep = []
    for c in coords:
        if all(np.abs(c - k).max() > min_distance for k in keep):
            keep.append(c)
    return np.array(keep).reshape(-1, 2)


def _compute_points_from_mask(mask, original_size, box_extension, use_single_point=False):
    """Positive points at the inner distance maxima, negative ones at the outer maxima inside the (extended) box (:41-83)."""
    from scipy import ndimage
    box = _compute_box_from_mask(mask, box_extension=box_extension)
    bb = (slice(box[1], box[3]), slice(box[0], box[2]))
    offset = np.array([box[1], box[0]])
    crop = mask[bb].astype(bool)
    # find_boundaries(mode="outer"): background pixels that touch the object (4-neighbourhood dilation minus the object)
    # plus object pixels touching other labels -- for a binary mask the former
    boundaries = ndimage.binary_dilation(crop) & ~crop
    distances = ndimage.gaussian_filter(ndimage.distance_transform_edt(~boundaries).astype("float32"), sigma=1.0)
    inner = np.where(crop, distances, 0.0)
    if use_single_point:
        center = np.array(np.unravel_index(inner.argmax(), inner.shape))
        return (center + offset)[None][:, ::-1], np.ones(1, dtype="uint8")
    outer = np.where(crop, 0.0, distances)
    inner_max, outer_max = _peak_local_max(inner, 3), _peak_local_max(outer, 5)
    coords = np.concatenate([inner_max, outer_max]).astype("float64") + offset
    if original_size is not None:
        coords *= np.array([original_size[0] / float(mask.shape[0]), original_size[1] / float(mask.shape[1])])[None]
    labels = np.concatenate([np.ones(len(inner_max), dtype="uint8"), np.zeros(len(outer_max), dtype="uint8")])
    return coords[:, ::-1], labels


def _compute_logits_from_mask(mask, eps=1e-3):
    """Binary mask -> (1, 256, 256) mask-prompt logits: resize the BINARY mask with the model's transform, pad with zeros,
    re-binarise at 0.5, map to +-logit(1 - eps) (:86-113)."""
    assert mask.ndim == 2
    binary = (mask == 1).astype("float32")
    if binary.shape != (256, 256):
        binary = ResizeLongestSide(256).apply_image_torch(torch.from_numpy(binary[None, None])).numpy().squeeze()
        if binary.shape != (256, 256):
            binary = np.pad(binary, ((0, 256 - binary.shape[0]), (0, 256 - binary.shape[1])), mode="constant",
                            constant_values=0)
    hi = np.log((1 - eps) / eps)
    logits = np.where(binary > 0.5, hi, -hi).astype("float32")[None]
    assert logits.shape == (1, 256, 256), f"{logits.shape}"
    return logits


# ------------------------------------------------------------------------------------------------ tiled routing
def _tile_of(center, shape, tile_shape, halo):
    tiling = Blocking([0, 0], shape, tile_shape)
    tile_id = tiling.coordinates_to_block_id(np.asarray(center).round().astype("int").tolist())
    return tile_id, tiling.get_block_with_halo(tile_id, list(halo)).outer_block


def _points_to_tile(prompts, shape, tile_shape, halo):
    points, labels = prompts
    tile_id, tile = _tile_of(np.mean(points, axis=0), shape, tile_shape, halo)
    local = points - np.array(tile.begin)
    valid = (local >= 0).all(axis=1) & (local[:, 0] < tile.shape[0]) & (local[:, 1] < tile.shape[1])
    if not valid.all():
        warnings.warn(f"{(~valid).sum()} points were not in the tile and are dropped")
        local, labels = local[valid], labels[valid]
    return tile_id, tile, (local, labels)


def _box_to_tile(box, shape, tile_shape, halo):
    tile_id, tile = _tile_of([(box[0] + box[2]) / 2, (box[1] + box[3]) / 2], shape, tile_shape, halo)
    off, ts = tile.begin, tile.shape
    local = np.array([max(box[0] - off[0], 0), max(box[1] - off[1], 0), min(box[2] - off[0], ts[0]), min(box[3] - off[1], ts[1])])
    return tile_id, tile, local


def _mask_to_tile(mask, shape, tile_shape, halo):
    ys, xs = np.where(mask)
    tile_id, tile = _tile_of([np.mean(ys), np.mean(xs)], shape, tile_shape, halo)
    return tile_id, tile, mask[tuple(slice(b, e) for b, e in zip(tile.begin, tile.end))]


def _initialize_predictor(predictor, image_embeddings, i, prompts, to_tile):
    """Bind the right embedding: the tile that contains the prompts for tiled embeddings (prompts moved to tile
    coordinates), the (slice of the) precomputed embedding otherwise, or whatever the predictor already holds (:209-231)."""
    tile = None
    if image_embeddings is not None and image_embeddings["input_size"] is None:
        attrs = image_embeddings["features"].attrs
        shape = tuple(attrs["shape"])
        tile_id, tile, prompts = to_tile(prompts, shape, tuple(attrs["tile_shape"]), tuple(attrs["halo"]))
        util.set_precomputed(predictor, image_embeddings, i, tile_id=tile_id)
    elif image_embeddings is not None:
        shape = image_embeddings["original_size"]
        util.set_precomputed(predictor, image_embeddings, i)
    else:
        shape = predictor.original_size
    return predictor, tile, prompts, shape


def _finish(mask, scores, logits, tile, shape, return_all):
    if tile is not None:  # paste the tile-local masks into the full image frame
        full = np.zeros(mask.shape[0:1] + tuple(shape), dtype=mask.dtype)
        full[(slice(None),) + tuple(slice(b, e) for b, e in zip(tile.begin, tile.end))] = mask
        mask = full
    return (mask, scores, logits) if return_all else mask


# ------------------------------------------------------------------------------------------------ public functions
def segment_from_points(predictor, points: np.ndarray, labels: np.ndarray, image_embeddings=None, i: Optional[int] = None,
                        multimask_output: bool = False, return_all: bool = False, use_best_multimask: Optional[bool] = None):
    """Point prompts (row, col) + labels -> binary mask (1, H, W) (:251-305).  A single positive point uses the multi-mask
    output and keeps the mask with the best predicted IoU unless `use_best_multimask` says otherwise."""
    predictor, tile, (points, labels), shape = _initialize_predictor(predictor, image_embeddings, i, (points, labels),
                                                                      _points_to_tile)
    if use_best_multimask is None:
        use_best_multimask = len(points) == 1 and labels[0] == 1
    mask, scores, logits = predictor.predict(point_coords=points[:, ::-1], point_labels=labels,
                                             multimask_output=multimask_output or use_best_multimask)
    if use_best_multimask:
        mask = mask[np.argmax(scores)][None]
    return _finish(mask, scores, logits, tile, shape, return_all)


def segment_from_box(predictor, box: np.ndarray, image_embeddings=None, i: Optional[int] = None, multimask_output: bool = False,
                     return_all: bool = False, box_extension: float = 0.0):
    """Box prompt (y0, x0, y1, x1) -> binary mask (:411-447)."""
    predictor, tile, box, shape = _initialize_predictor(predictor, image_embeddings, i, box, _box_to_tile)
    mask, scores, logits = predictor.predict(box=_process_box(box, shape, box_extension=box_extension),
                                             multimask_output=multimask_output)
    return _finish(mask, scores, logits, tile, shape, return_all)


def segment_from_box_and_points(predictor, box: np.ndarray, points: np.ndarray, labels: np.ndarray, image_embeddings=None,
                                i: Optional[int] = None, multimask_output: bool = False, return_all: bool = False):
    """Box + point prompts -> binary mask (:450-506)."""
    def to_tile(prompts, shape, tile_shape, halo):
        b, p, l = prompts
        tid_p, tile, (p, l) = _points_to_tile((p, l), shape, tile_shape, halo)
        tid_b, tile, b = _box_to_tile(b, shape, tile_shape, halo)
        if tid_b != tid_p:
            raise RuntimeError(f"Inconsistent tile ids for box and point annotations: {tid_b} != {tid_p}.")
        return tid_p, tile, (b, p, l)

    predictor, tile, (box, points, labels), shape = _initialize_predictor(predictor, image_embeddings, i, (box, points, labels),
                                                                           to_tile)
    mask, scores, logits = predictor.predict(point_coords=points[:, ::-1], point_labels=labels, box=_process_box(box, shape),
                                             multimask_output=multimask_output)
    return _finish(mask, scores, logits, tile, shape, return_all)


def segment_from_mask(predictor, mask: np.ndarray, image_embeddings=None, i: Optional[int] = None, use_box: bool = True,
                      use_mask: bool = True, use_points: bool = False, original_size: Optional[Tuple[int, ...]] = None,
                      multimask_output: bool = False, return_all: bool = False, return_logits: bool = False,
                      box_extension: float = 0.0, box: Optional[np.ndarray] = None, points: Optional[np.ndarray] = None,
                      labels: Optional[np.ndarray] = None, use_single_point: bool = False):
    """Mask prompt, optionally with the box / points derived from it (or given) (:308-408)."""
    def to_tile(prompts, shape, tile_shape, halo):
        m, b, p, l = prompts
        tile_id, tile, m = _mask_to_tile(m, shape, tile_shape, halo)
        if p is not None:
            tid, tile, (p, l) = _points_to_tile((p, l), shape, tile_shape, halo)
            if tid != tile_id:
                raise RuntimeError(f"Inconsistent tile ids for mask and point prompts: {tid} != {tile_id}.")
        if b is not None:
            tid, tile, b = _box_to_tile(b, shape, tile_shape, halo)
            if tid != tile_id:
                raise RuntimeError(f"Inconsistent tile ids for mask and box prompts: {tid} != {tile_id}.")
        return tile_id, tile, (m, b, p, l)

    predictor, tile, (mask, box, points, labels), shape = _initialize_predictor(predictor, image_embeddings, i,
                                                                                 (mask, box, points, labels), to_tile)
    if points is not None:
        if labels is None:
            raise ValueError("If points are passed you also need to pass labels.")
        point_coords, point_labels = points, labels
    elif use_points and mask.sum() != 0:
        point_coords, point_labels = _compute_points_from_mask(mask, original_size=original_size, box_extension=box_extension,
                                                               use_single_point=use_single_point)
    else:
        point_coords = point_labels = None
    if box is None:
        box = _compute_box_from_mask(mask, original_size=original_size, box_extension=box_extension) \
            if use_box and mask.sum() != 0 else None
    else:
        box = _process_box(box, mask.shape, original_size=original_size, box_extension=box_extension)
    logits_in = _compute_logits_from_mask(mask) if use_mask else None
    out, scores, logits = predictor.predict(point_coords=point_coords, point_labels=point_labels, mask_input=logits_in, box=box,
                                            multimask_output=multimask_output, return_logits=return_logits)
    return _finish(out, scores, logits, tile, shape, return_all)
