"""ORACLE (test infrastructure, NOT product code) -- fp64 restatement of micro-sam's object features
(micro_sam/object_classification.py:20-217).

The reference resizes with skimage, which is not installed here, so its calls are restated through what skimage runs:
- `resize(embeddings (64, 64, 256), (ry, rx, 256), preserve_range=True)` (order 1, mode 'reflect', anti-aliasing because an
  axis may shrink): `scipy.ndimage.gaussian_filter(x, max(0, (64 / r - 1) / 2) per axis, mode='mirror')` when any axis shrinks,
  then `scipy.ndimage.zoom(x, r / 64, order=1, mode='mirror', grid_mode=True)` (skimage maps 'reflect' to scipy's 'mirror');
- `resize(seg, (ry, rx), order=0, anti_aliasing=False, preserve_range=True)`: `scipy.ndimage.zoom(seg, r / S, order=0,
  mode='mirror', grid_mode=True)`;
- `regionprops_table(label, area, mean_intensity)`: per-label pixel counts and means by `np.bincount`, labels > 0 ascending.
This mapping is not pinned against skimage (unpinned restatement).  Everything runs in fp64 here; the reference's skimage
resize and means run in fp32, well inside the 1e-5 x max|E| the tests allow.  Slices and tiles are combined from the
specification -- areas add up, means are area-weighted -- as fp64 totals rounded to float32 once.  `nearest_index` / `linear_taps` / `gaussian_weights` state the index and
weight rules the device follows; tests/test_object_features_cpu.py checks them against scipy.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage

N_FEATURES = 257


def pad_to_square(seg: np.ndarray) -> np.ndarray:
    """object_classification.py:24-32: pad bottom or right with 0 to the longer side."""
    h, w = seg.shape
    if h > w:
        return np.pad(seg, ((0, 0), (0, h - w)))
    if w > h:
        return np.pad(seg, ((0, w - h), (0, 0)))
    return seg


def resize_shape(seg_shape, resize_embedding_shape=(256, 256)):
    S = max(seg_shape)
    return tuple(min(int(r), S) for r in resize_embedding_shape)


def resize_embeddings(emb: np.ndarray, shape) -> np.ndarray:
    """skimage resize of the (64, 64, 256) embedding to (ry, rx, 256), fp64."""
    x = np.asarray(emb, np.float64).transpose(1, 2, 0)
    out_shape = tuple(shape) + (x.shape[-1],)
    factors = np.divide(x.shape, out_shape)
    if any(o < i for o, i in zip(out_shape, x.shape)):
        x = ndimage.gaussian_filter(x, np.maximum(0, (factors - 1) / 2), cval=0, mode="mirror")
    return ndimage.zoom(x, [1 / f for f in factors], order=1, mode="mirror", cval=0, grid_mode=True)


def resize_segmentation(seg: np.ndarray, shape) -> np.ndarray:
    """skimage resize with order=0 of the padded square segmentation."""
    factors = np.divide(seg.shape, shape)
    return ndimage.zoom(seg, [1 / f for f in factors], order=0, mode="mirror", cval=0, grid_mode=True)


def nearest_index(S: int, r: int) -> np.ndarray:
    """source index of each of r outputs, as scipy's zoom computes it: floor(((o + 0.5) * (S / r) - 0.5) + 0.5)"""
    z = np.float64(S) / np.float64(r)
    cc = (np.arange(r, dtype=np.float64) + 0.5) * z - 0.5
    return np.floor(cc + 0.5).astype(np.int64)


def fold(i, n: int = 64):
    """scipy's 'mirror' extension into [0, n): -i, 2 (n - 1) - i, periodically"""
    p = 2 * (n - 1)
    i = np.mod(i, p)
    return np.where(i > n - 1, p - i, i)


def linear_taps(r: int, n: int = 64):
    """bilinear taps of r outputs from n inputs: (floor(c), c - floor(c)) of c = (o + 0.5) * (n / r) - 0.5; tap t has weight
    1 - frac, tap t + 1 weight frac, both folded"""
    c = (np.arange(r, dtype=np.float64) + 0.5) * (np.float64(n) / np.float64(r)) - 0.5
    t = np.floor(c)
    return t.astype(np.int64), c - t


def gaussian_weights(r: int, n: int = 64):
    """skimage's anti-aliasing Gaussian for an axis resized from n to r: scipy's kernel of sigma (n / r - 1) / 2, radius
    int(4 sigma + 0.5); None when the axis is not filtered"""
    sigma = max(0.0, (n / r - 1) / 2)
    if sigma <= 1e-15:
        return None
    radius = int(4.0 * sigma + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


def compute_unit(emb: np.ndarray, seg: np.ndarray, resize_embedding_shape=(256, 256)):
    """_compute_object_features_impl: (seg_ids int64 [n], features float64 [n, 257]) of the labels in the resized segmentation"""
    seg = pad_to_square(np.asarray(seg))
    shape = resize_shape(seg.shape, resize_embedding_shape)
    E = resize_embeddings(emb, shape).reshape(-1, np.asarray(emb).shape[0])
    lab = resize_segmentation(seg, shape).ravel()
    ids = np.unique(lab)
    ids = ids[ids > 0]
    fg = lab > 0
    inv = np.searchsorted(ids, lab[fg])
    area = np.bincount(inv, minlength=len(ids)).astype(np.float64)
    sums = np.stack([np.bincount(inv, weights=E[fg, c], minlength=len(ids)) for c in range(E.shape[1])], axis=1)
    means = sums / np.maximum(area, 1)[:, None]
    feats = np.concatenate([area[:, None], means], axis=1) if len(ids) else np.zeros((0, N_FEATURES))
    return ids.astype(np.int64), feats


def tile_outer_boxes(shape, tile_shape, halo):
    """Blocking([0, 0], shape, tile_shape).get_block_with_halo(i, halo).outer_block as slices, block ids in C order"""
    nb = [int(math.ceil(s / t)) for s, t in zip(shape, tile_shape)]
    out = []
    for by in range(nb[0]):
        for bx in range(nb[1]):
            sl = []
            for p, s, t, h in zip((by, bx), shape, tile_shape, halo):
                b, e = p * t, min(p * t + t, s)
                sl.append(slice(max(b - h, 0), min(e + h, s)))
            out.append(tuple(sl))
    return out


def units(embeddings: dict, segmentation: np.ndarray):
    """(segmentation crop, embedding [256, 64, 64]) of every unit, in the reference generator's order
    (object_classification.py:60-106); embeddings hold numpy arrays"""
    feats = embeddings["features"]
    is_3d = segmentation.ndim == 3
    if embeddings["input_size"] is not None:
        for z in range(segmentation.shape[0]):
            yield segmentation[z], np.asarray(feats[z]).squeeze()
        return
    boxes = tile_outer_boxes(feats.attrs["shape"], feats.attrs["tile_shape"], feats.attrs["halo"])
    for z in range(segmentation.shape[0] if is_3d else 1):
        for i, bb in enumerate(boxes):
            if is_3d:
                yield segmentation[z][bb], np.asarray(feats[str(i)][z]).squeeze()
            else:
                yield segmentation[bb], np.asarray(feats[str(i)][:]).squeeze()


def compute_object_features(embeddings: dict, segmentation: np.ndarray, resize_embedding_shape=(256, 256)):
    """object features of a 2-D image (one unit, fp64) or of slices / tiles (`merge` of the units, float32)"""
    if embeddings["input_size"] is not None and segmentation.ndim == 2:
        return compute_unit(np.asarray(embeddings["features"]).squeeze(), segmentation, resize_embedding_shape)
    return merge(units(embeddings, segmentation), segmentation, resize_embedding_shape)


def merge(unit_iter, segmentation, resize_embedding_shape=(256, 256), unit_fn=None):
    """Slices and tiles combined: the ids are every nonzero label of the whole segmentation; an id's area is the sum of its
    per-unit areas and its mean the area-weighted mean of its per-unit means, both totalled in fp64 and rounded to float32
    once; an id that no unit keeps has an all-zero row.  `unit_fn(unit_iter)` yields the per-unit (ids, features) in place
    of compute_unit (e.g. from a process pool)."""
    ids = np.unique(np.asarray(segmentation))
    ids = ids[ids != 0].astype(np.int64)
    area = np.zeros(len(ids))
    weighted = np.zeros((len(ids), N_FEATURES - 1))
    results = unit_fn(unit_iter) if unit_fn is not None else (
        compute_unit(emb, seg, resize_embedding_shape) for seg, emb in unit_iter)
    for unit_ids, unit_feats in results:
        rows = np.searchsorted(ids, unit_ids)
        area[rows] += unit_feats[:, 0]
        weighted[rows] += unit_feats[:, :1] * unit_feats[:, 1:]
    feats = np.zeros((len(ids), N_FEATURES))
    feats[:, 0] = area
    kept = area > 0
    feats[kept, 1:] = weighted[kept] / area[kept, None]
    return ids, feats.astype(np.float32)


def project_prediction_to_segmentation(segmentation, object_prediction, seg_ids):
    """each pixel takes the prediction of its label, looked up in the sorted ids; labels without a prediction give 0; for an
    id listed twice the later prediction counts"""
    pred = np.asarray(object_prediction)
    ids_rev = np.asarray(seg_ids, dtype=np.int64)[::-1]
    ids, first_in_rev = np.unique(ids_rev, return_index=True)   # first in the reversed list = last in the given one
    vals = pred[::-1][first_in_rev]
    seg = np.asarray(segmentation).astype(np.int64)
    out = np.zeros(seg.shape, dtype=pred.dtype)
    if len(ids):
        pos = np.minimum(np.searchsorted(ids, seg), len(ids) - 1)
        hit = ids[pos] == seg
        out[hit] = vals[pos[hit]]
    return out
