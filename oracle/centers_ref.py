"""ORACLE (test infrastructure, NOT product code) -- numpy / scipy restatement of micro-sam's util.get_centers_and_bounding_boxes
and util.segmentation_to_one_hot (micro_sam/util.py:1283-1396), 2-D and 3-D.  skimage and bioimage_cpp are absent, so the
steps they take are restated here (DESIGN.md section 2, unpinned):
  1. pad     : np.pad(segmentation, 1) -- objects on the image border get a boundary there;
  2. boundary: find_boundaries(padded, mode="inner"), connectivity 1: foreground pixels whose cross / 6-neighbourhood (itself
               included, neighbours outside the padded array ignored) has max != min;
  3. distance: distance_transform(boundaries == 0) taken as scipy's distance_transform_edt; used here as integer squared
               distances (rounded), which order as the reference's fp64 distances do;
  4. centre v: per object, the object pixel of largest distance, ties to the first in raster order of its bounding box;
  5. centre p: the mean coordinate, int64 sums divided once in fp64 (numpy's float64 mean while the sums stay below 2^53).
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage


def inner_boundaries(padded: np.ndarray) -> np.ndarray:
    """rule 2 on an already padded label array (any ndim)"""
    lab = np.asarray(padded)
    hi, lo = lab.copy(), lab.copy()
    for ax in range(lab.ndim):
        n = lab.shape[ax]
        for src, dst in ((slice(1, n), slice(0, n - 1)), (slice(0, n - 1), slice(1, n))):
            s = [slice(None)] * lab.ndim
            d = [slice(None)] * lab.ndim
            s[ax], d[ax] = src, dst
            hi[tuple(d)] = np.maximum(hi[tuple(d)], lab[tuple(s)])
            lo[tuple(d)] = np.minimum(lo[tuple(d)], lab[tuple(s)])
    return (lab != 0) & (hi != lo)


def edt_squared(mask: np.ndarray) -> np.ndarray:
    """scipy's distance_transform_edt(mask) ** 2 as int64 (distance of every pixel to the nearest zero of mask)"""
    return np.rint(ndimage.distance_transform_edt(mask) ** 2).astype(np.int64)


def center_distances(segmentation: np.ndarray) -> np.ndarray:
    """rules 1-3: int64 squared distance to the nearest inner boundary pixel over the padded grid"""
    return edt_squared(~inner_boundaries(np.pad(segmentation, 1)))


def _dense(segmentation: np.ndarray):
    ids, inv = np.unique(segmentation, return_inverse=True)
    dense = inv.reshape(segmentation.shape).astype(np.int64)
    if ids[0] != 0:   # no background: index 0 must stay background for find_objects
        ids, dense = np.concatenate([[0], ids]), dense + 1
    return ids[1:].astype(np.int64), dense


def get_centers_and_bounding_boxes(segmentation: np.ndarray, mode: str = "v"):
    """-> ids int64 (n,), centers (n, ndim) (int64 for "v", float64 for "p"), boxes int64 (n, 2 ndim) in skimage's bbox layout"""
    seg = np.asarray(segmentation)
    nd = seg.ndim
    ids, dense = _dense(seg)
    slices = ndimage.find_objects(dense)
    d2 = center_distances(seg) if mode == "v" else None
    centers = np.zeros((len(ids), nd), np.int64 if mode == "v" else np.float64)
    boxes = np.zeros((len(ids), 2 * nd), np.int64)
    for k, sl in enumerate(slices):
        start = np.array([s.start for s in sl])
        boxes[k] = np.concatenate([start, [s.stop for s in sl]])
        obj = dense[sl] == k + 1
        if mode == "v":
            region = d2[tuple(slice(s.start + 1, s.stop + 1) for s in sl)]
            masked = np.where(obj, region, -1)
            centers[k] = np.array(np.unravel_index(int(np.argmax(masked)), masked.shape)) + start
        else:
            coords = np.stack(np.nonzero(obj), 1).astype(np.int64) + start
            centers[k] = coords.sum(0).astype(np.float64) / np.float64(len(coords))
    return ids, centers, boxes


def relabel_sequential(seg: np.ndarray) -> np.ndarray:
    """skimage's relabel_sequential(seg)[0] for non-negative labels: the non-zero ids present become 1, 2, ... in ascending order"""
    ids = np.unique(seg)
    ids = ids[ids != 0]
    return np.where(seg != 0, np.searchsorted(ids, seg) + 1, 0)


def segmentation_to_one_hot(segmentation: np.ndarray, segmentation_ids=None) -> np.ndarray:
    """float32 (n_ids, 1, *shape), the reference's rule (its quirk with absent selected ids included)"""
    seg = np.asarray(segmentation).astype(np.int64)
    if segmentation_ids is None:
        n_ids, masks = int(seg.max()), seg
    else:
        sel = np.sort(np.asarray(segmentation_ids))
        if len(sel) == 0 or 0 in sel:
            raise RuntimeError("No foreground objects were found.")
        masks = np.where(np.isin(seg, sel), seg, 0)
        masks = relabel_sequential(masks)
        n_ids = len(sel)
    out = np.zeros((n_ids, 1) + seg.shape, np.float32)
    for k in range(n_ids):
        out[k, 0] = masks == k + 1
    return out
