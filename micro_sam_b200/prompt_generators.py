"""micro_sam.prompt_generators on the GPU (micro_sam/prompt_generators.py:58-377): the point and box prompts of micro-sam's training
loop, sampled by the kernels of csrc/prompts.cu.

The candidate sets and the distributions over them are the reference's: positive points uniform over the object (without replacement
unless more points than pixels are asked for), negative points uniform over the ring around it, fill-up points uniform over the
background; the iterative corrections uniform over the false negatives / false positives with the reference's fallbacks.  The
individual draws are not numpy's: they come from Philox4x32-10 keyed by a 64-bit seed, which `seed=None` draws from numpy's global
RNG -- so `np.random.seed(s)` reproduces a run.  Outputs are device tensors (the reference returns CPU tensors).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib


MAX_POINTS = 64          # points per object and call of the sampling kernel (csrc/prompts.cu, kMaxPts)


def draw_seed(seed: Optional[int] = None) -> int:
    """the 64-bit Philox key: `seed` itself, or a draw from numpy's global RNG"""
    if seed is None:
        return int(np.random.randint(0, 2 ** 64, dtype=np.uint64))
    return int(seed) & (2 ** 64 - 1)


def _device(t) -> torch.device:
    if isinstance(t, torch.Tensor) and t.is_cuda:
        return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _planes(x, dev) -> torch.Tensor:
    """(N, 1, H, W) masks (torch or numpy, any dtype) -> contiguous uint8 (N, H, W) {0, 1} on `dev`"""
    x = torch.as_tensor(x)
    if x.ndim == 5:
        raise NotImplementedError("3-D prompts (NUM_OBJECTS x 1 x Z x H x W) are not supported")
    if x.ndim != 4 or x.shape[1] != 1:
        raise ValueError(f"expected masks of shape NUM_OBJECTS x 1 x H x W, got {tuple(x.shape)}")
    return (x.to(dev)[:, 0] != 0).to(torch.uint8).contiguous()


def sample_points(targets: torch.Tensor, counts: torch.Tensor, boxes: torch.Tensor, n_pos: int, n_neg: int, dilation: int, seed: int,
                  centers: Optional[torch.Tensor] = None, n_per_img: Optional[int] = None):
    """`msam_prompt_sample_points` on uint8 masks (N, H, W), int32 counts (N,) and int32 row / col boxes (N, 4) -> int32 (x, y)
    coords (N, n_pos + n_neg, 2) and int32 labels (N, n_pos + n_neg)"""
    N, H, W = targets.shape
    dev = targets.device
    npts = n_pos + n_neg
    coords = torch.empty(N, npts, 2, device=dev, dtype=torch.int32)
    labels = torch.empty(N, npts, device=dev, dtype=torch.int32)
    scratch = torch.empty(2 * N * H * W, device=dev, dtype=torch.uint8) if (n_neg > 0 and dilation > 0 and N > 0) else None
    _lib.check(_lib.lib().msam_prompt_sample_points(
        _lib.ptr(targets), _lib.ptr(counts), _lib.ptr(boxes), _lib.ptr(centers), N, n_per_img or max(N, 1), H, W, n_pos, n_neg,
        dilation, seed, _lib.ptr(scratch), _lib.ptr(coords), _lib.ptr(labels), _lib.cur_stream()))
    return coords, labels


def iterative_points(targets: torch.Tensor, seed: int, low_res: Optional[torch.Tensor] = None, iou: Optional[torch.Tensor] = None,
                     input_size=None, pred: Optional[torch.Tensor] = None, n_per_img: Optional[int] = None):
    """`msam_prompt_iterative`: uint8 targets (N, H, W) and either fp32 low-res logits (N, M, 256, 256) (+ iou (N, M) when M > 1;
    the prediction is postprocess_masks(logits) > 0 for `input_size`) or a uint8 prediction (N, H, W) -> int32 (x, y) coords
    (N, 2, 2) and int32 labels (N, 2), positive point first"""
    N, H, W = targets.shape
    dev = targets.device
    coords = torch.empty(N, 2, 2, device=dev, dtype=torch.int32)
    labels = torch.empty(N, 2, device=dev, dtype=torch.int32)
    M = 1 if low_res is None else int(low_res.shape[1])
    in_h, in_w = (H, W) if input_size is None else (int(input_size[0]), int(input_size[1]))
    _lib.check(_lib.lib().msam_prompt_iterative(
        _lib.ptr(targets), _lib.ptr(low_res), _lib.ptr(iou), M, _lib.ptr(pred), N, n_per_img or max(N, 1), in_h, in_w, H, W, seed,
        _lib.ptr(coords), _lib.ptr(labels), _lib.cur_stream()))
    return coords, labels


class PointAndBoxPromptGenerator:
    """micro_sam.prompt_generators.PointAndBoxPromptGenerator (prompt_generators.py:58-249).

    `__call__(segmentation, bbox_coordinates, center_coordinates=None)`: segmentation (N, 1, H, W) object masks, bbox_coordinates
    N tuples (min_row, min_col, max_row + 1, max_col + 1) -> (coords (N, n, 2) int64 in (x, y) order, labels (N, n) int64, boxes
    (N, 4) int64 (min_x, min_y, max_x, max_y), None), with n = n_positive_points + n_negative_points; coords / labels are None
    without point prompts and boxes None without box prompts.  With `center_coordinates` the first positive point of each object
    is int(centre).  All outputs are device tensors.  An object mask without pixels gets coordinates -1 (the reference raises).
    n_positive_points + n_negative_points is at most 64 (the reference has no limit); more raises ValueError.
    """

    def __init__(self, n_positive_points: int, n_negative_points: int, dilation_strength: int, get_point_prompts: bool = True,
                 get_box_prompts: bool = False) -> None:
        self.n_positive_points = n_positive_points
        self.n_negative_points = n_negative_points
        self.dilation_strength = dilation_strength
        self.get_box_prompts = get_box_prompts
        self.get_point_prompts = get_point_prompts
        if self.get_point_prompts is False and self.get_box_prompts is False:
            raise ValueError("You need to request box prompts, point prompts or both.")
        if self.get_point_prompts and not 0 < n_positive_points + n_negative_points <= MAX_POINTS:
            raise ValueError(f"n_positive_points + n_negative_points must be in 1..{MAX_POINTS}, got "
                             f"{n_positive_points} + {n_negative_points}")

    def __call__(self, segmentation, bbox_coordinates: Sequence, center_coordinates: Optional[List[np.ndarray]] = None,
                 seed: Optional[int] = None, **kwargs):
        dev = _device(segmentation)
        tg = _planes(segmentation, dev)
        boxes = torch.as_tensor(np.asarray([[int(v) for v in b] for b in bbox_coordinates], dtype=np.int32).reshape(-1, 4)).to(dev)
        coords = labels = None
        if self.get_point_prompts:
            counts = tg.flatten(1).sum(1, dtype=torch.int32)
            centers = None
            if center_coordinates is not None:
                centers = torch.as_tensor(np.asarray([[int(v) for v in c] for c in center_coordinates], dtype=np.int32)).to(dev)
            coords, labels = sample_points(tg, counts, boxes, self.n_positive_points, self.n_negative_points, self.dilation_strength,
                                           draw_seed(seed), centers=centers)
            coords, labels = coords.long(), labels.long()
        bbox_list = boxes[:, [1, 0, 3, 2]].long() if self.get_box_prompts else None
        return coords, labels, bbox_list, None


class IterativePromptGenerator:
    """micro_sam.prompt_generators.IterativePromptGenerator (prompt_generators.py:252-377), 2-D.

    `__call__(segmentation, prediction)`: targets and binary predictions, both (N, 1, H, W) -> (coords (N, 2, 2) int64 (x, y),
    labels (N, 2) int64, None, None): per object one positive point uniform over the false negatives (else the overlap) and one
    negative point uniform over the false positives (else the box ring of _get_negative_locations_in_obj_bbox, else the true
    background).  Device tensors.  3-D input raises NotImplementedError.
    """

    def __call__(self, segmentation, prediction, seed: Optional[int] = None, **kwargs):
        seg, pred = torch.as_tensor(segmentation), torch.as_tensor(prediction)
        if seg.shape != pred.shape:
            raise AssertionError("The segmentation and prediction tensors should have the same shape.")
        dev = _device(pred)
        coords, labels = iterative_points(_planes(seg, dev), draw_seed(seed), pred=_planes(pred, dev))
        return coords.long(), labels.long(), None, None
