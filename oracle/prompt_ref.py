"""ORACLE (test infrastructure, NOT product code) -- numpy / scipy restatement of the candidate regions of micro-sam's prompt
generators (micro_sam/prompt_generators.py:58-377, micro_sam/training/util.py:153-265).  It returns the SETS each point is drawn
from, not samples: the library's draws come from another generator, so a test checks membership, counts and distributions.

The reference dilates with kornia.morphology.dilation (3 x 3 ones, engine="convolution", geodesic border: nothing outside the
image); kornia is not installed, so `iterated_dilation` uses scipy.ndimage.binary_dilation with a 3 x 3 element and
`iterations=ds`, which is the same operation.  Also here: Philox4x32-10 in numpy, to recompute the library's box distortion
(`_distort_boxes`) from its seed.
"""
from __future__ import annotations

import random

import numpy as np
import torch
from scipy import ndimage


def iterated_dilation(mask: np.ndarray, ds: int) -> np.ndarray:
    """`ds` iterations of a 3 x 3 binary dilation, zero outside the image (ds = 0: the mask itself)"""
    mask = np.asarray(mask, dtype=bool)
    if ds == 0:
        return mask.copy()
    return ndimage.binary_dilation(mask, structure=np.ones((3, 3), dtype=bool), iterations=ds, border_value=0)


def square_dilation(mask: np.ndarray, ds: int) -> np.ndarray:
    """the (2 ds + 1)^2 square dilation as the kernels compute it: a windowed OR along the rows, then along the columns, nothing
    outside the image"""
    m = np.asarray(mask, dtype=bool)
    H, W = m.shape
    rows = np.zeros_like(m)
    for x in range(W):
        rows[:, x] = m[:, max(x - ds, 0):min(x + ds, W - 1) + 1].any(1)
    out = np.zeros_like(m)
    for y in range(H):
        out[y] = rows[max(y - ds, 0):min(y + ds, H - 1) + 1].any(0)
    return out


def one_hot_counts_boxes(label: np.ndarray, ids):
    """segmentation_to_one_hot + get_centers_and_bounding_boxes(mode="p") boxes: (n, H, W) bool, (n,) counts, (n, 4)
    (min_row, min_col, max_row + 1, max_col + 1)"""
    planes = np.stack([label == i for i in ids]) if len(ids) else np.zeros((0,) + label.shape, bool)
    counts = planes.reshape(len(ids), -1).sum(1)
    boxes = np.zeros((len(ids), 4), np.int64)
    for k, p in enumerate(planes):
        ys, xs = np.nonzero(p)
        if len(ys):
            boxes[k] = (ys.min(), xs.min(), ys.max() + 1, xs.max() + 1)
    return planes, counts, boxes


def point_box_regions(object_mask: np.ndarray, box, ds: int):
    """PointAndBoxPromptGenerator._sample_points (prompt_generators.py:105-189): the positive set (the object), the ring
    |box widened by ds and clipped - object dilated ds times| the negatives come from, and the fill-up set (the background)"""
    obj = np.asarray(object_mask, dtype=bool)
    H, W = obj.shape
    inbox = np.zeros_like(obj)
    inbox[max(box[0] - ds, 0):min(box[2] + ds, H), max(box[1] - ds, 0):min(box[3] + ds, W)] = True
    ring = inbox != iterated_dilation(obj, ds)
    return {"positive": obj, "ring": ring, "fill": ~obj}


def iterative_regions(target: np.ndarray, pred: np.ndarray):
    """IterativePromptGenerator.__call__ (prompt_generators.py:252-377), 2-D: the set the positive point comes from (false negatives,
    else the overlap) and the set of the negative point (false positives, else the box of the target widened by 3 minus the target,
    else the true background), with the name of the set chosen"""
    t, p = np.asarray(target, dtype=bool), np.asarray(pred, dtype=bool)
    fn, fp, ov = t & ~p, p & ~t, t & p
    pos, pos_name = (fn, "fn") if fn.any() else (ov, "overlap")
    if fp.any():
        neg, neg_name = fp, "fp"
    else:
        neg, neg_name = np.zeros_like(t), "ring"
        if t.any():
            ys, xs = np.nonzero(t)
            H, W = t.shape
            box = np.zeros_like(t)
            box[max(ys.min() - 3, 0):min(ys.max() + 1 + 3, H), max(xs.min() - 3, 0):min(xs.max() + 1 + 3, W)] = True
            neg = box & ~t
        if not neg.any():
            neg, neg_name = ~t, "background"
    return {"positive": pos, "positive_set": pos_name, "negative": neg, "negative_set": neg_name}


# ---- Philox4x32-10 (Salmon et al., SC'11), counter (draw, object, image, stream), key = 64-bit seed
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
TAG_BOX = 0


def philox4x32_10(ctr, seed: int):
    c = [int(v) & 0xFFFFFFFF for v in ctr]
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c[3] ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return c


def uniform01(seed: int, tag: int, img: int, obj: int, draw: int) -> float:
    r = philox4x32_10((draw, obj, img, tag), seed)
    return float(((r[0] << 32) | r[1]) >> 11) * 2.0 ** -53


def distort_box(box, factor: float, shape, u4) -> list:
    """ConvertToSamInputs._distort_boxes (training/util.py:174-185) for one box with the uniforms U of its four draws
    (y0, y1, x0, x1): numpy's uniform(0, f) is f * U"""
    y0, x0, y1, x1 = (int(v) for v in box)
    ly, lx = y1 - y0, x1 - x0
    u = [factor * v for v in u4]
    return [int(round(max(0, y0 - u[0] * ly))), int(round(max(0, x0 - u[2] * lx))),
            int(round(min(shape[0], y1 + u[1] * ly))), int(round(min(shape[1], x1 + u[3] * lx)))]


# ---- the reference's iterative prompt update, as micro-sam runs it (timing baseline of tests/time_prompt_update.py)
class ReferenceStyleUpdate:
    """IterativePromptGenerator.__call__ + SamTrainer._update_prompts as micro-sam runs them: per object torch.where on the
    full-size (B, n, 1, H, W) masks, np.random.choice on the host"""

    def __init__(self, y_one_hot, transform, mask_prob=0.5):
        self.y, self.transform, self.mask_prob = y_one_hot, transform, mask_prob

    @staticmethod
    def _negative_in_bbox(t):
        loc = torch.where(t)
        box = torch.stack([torch.min(loc[1]), torch.min(loc[2]), torch.max(loc[1]) + 1, torch.max(loc[2]) + 1])
        m = torch.zeros_like(t).squeeze(0)
        m[max(box[0] - 3, 0):min(box[2] + 3, t.shape[-2]), max(box[1] - 3, 0):min(box[3] + 3, t.shape[-1])] = 1
        return torch.where(torch.abs(m[None] - t))

    def generate(self, seg, pred):
        diff = pred - seg
        neg_region, pos_region = (diff == 1).float(), diff == -1
        overlap = torch.logical_and(pred == 1, seg == 1).float()
        pos, neg = [], []
        for pr_, ov, nr, t in zip(pos_region, overlap, neg_region, seg):
            loc = torch.where(pr_)
            if len(loc[0]) == 0:
                loc = torch.where(ov)
            i = np.random.choice(len(loc[0]))
            pos.append([loc[-1][i], loc[-2][i]])
            loc = torch.where(nr)
            if len(loc[0]) == 0:
                loc = self._negative_in_bbox(t)
            if len(loc[0]) == 0:
                loc = torch.where(t == 0)
            i = np.random.choice(len(loc[0]))
            neg.append([loc[-1][i], loc[-2][i]])
        coords = torch.cat([torch.tensor(pos)[:, None], torch.tensor(neg)[:, None]], 1)
        labels = torch.tensor([[1, 0]] * len(pos))
        return coords, labels

    def __call__(self, batched_inputs, masks, logits):
        for x1, x2, rec, lg in zip(masks, self.y, batched_inputs, logits):
            coords, labels = self.generate(x2, x1)
            coords = self.transform.apply_coords_torch(coords, self.y.shape[-2:]).to(rec["point_coords"].device if "point_coords" in rec else lg.device)
            labels = labels.to(coords.device)
            rec["point_coords"] = torch.cat([rec["point_coords"], coords], 1) if "point_coords" in rec else coords
            rec["point_labels"] = torch.cat([rec["point_labels"], labels], 1) if "point_labels" in rec else labels
            if self.mask_prob > 0 and random.random() < self.mask_prob:
                rec["mask_inputs"] = lg
            else:
                rec.pop("mask_inputs", None)
        return batched_inputs
