"""torch_em's PerObjectDistanceTransform (torch_em/transform/label.py), restated in numpy / scipy for one 2-D label image.

torch_em is not available here, so this follows the structure of its __call__ / compute_normalized_object_distances as DESIGN.md
section 2 restates it (unpinned): label, size filter, inner boundaries, then per object a loop over its bounding box (the crop)
with a Euclidean distance transform of the crop's boundary pixels, np.argmax for the corrected centre and the normalisation
v / (max v + 1e-7).  It deliberately does not use the device's whole-image EDT, so the tests can compare the two.
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage

EPS = np.float32(1e-7)
_CROSS = ndimage.generate_binary_structure(2, 1)
_SQUARE = np.ones((3, 3), dtype=bool)


def label_components(labels: np.ndarray) -> np.ndarray:
    """skimage.measure.label(labels) for 2-D: 8-connected components of equal non-zero values, numbered 1.. in raster order of
    their first pixel."""
    labels = np.asarray(labels)
    out = np.zeros(labels.shape, dtype=np.int64)
    ids, dense = np.unique(labels, return_inverse=True)
    dense = dense.reshape(labels.shape)
    firsts, pieces = [], []
    for d, sl in enumerate(ndimage.find_objects(dense + 1)):
        if sl is None or ids[d] == 0:
            continue
        lab, n = ndimage.label(dense[sl] == d, structure=_SQUARE)
        for c in range(1, n + 1):
            yy, xx = np.nonzero(lab == c)
            yy, xx = yy + sl[0].start, xx + sl[1].start
            firsts.append(int(np.min(yy * labels.shape[1] + xx)))
            pieces.append((yy, xx))
    for k, j in enumerate(np.argsort(firsts, kind="stable")):
        out[pieces[j]] = k + 1
    return out


def relabel_consecutive(labels: np.ndarray) -> np.ndarray:
    """The non-zero ids numbered 1.. in ascending order (0 stays 0)."""
    ids, inv = np.unique(labels, return_inverse=True)
    new = np.arange(len(ids)) + (0 if ids[0] == 0 else 1)
    return new[inv.reshape(labels.shape)]


def size_filter(labels: np.ndarray, min_size: int) -> np.ndarray:
    """Objects of fewer than min_size pixels set to 0, the rest renumbered consecutively in ascending order."""
    counts = np.bincount(labels.ravel())
    small = np.nonzero(counts < min_size)[0]
    labels = np.where(np.isin(labels, small[small > 0]), 0, labels)
    return relabel_consecutive(labels)


def find_boundaries_inner(labels: np.ndarray) -> np.ndarray:
    """skimage.segmentation.find_boundaries(labels, mode="inner"), connectivity 1: foreground pixels whose cross neighbourhood
    (themselves included, neighbours outside the image ignored) holds more than one value."""
    hi = ndimage.grey_dilation(labels, footprint=_CROSS, mode="nearest")
    lo = ndimage.grey_erosion(labels, footprint=_CROSS, mode="nearest")
    return (hi != lo) & (labels != 0)


def _crop_edt(boundary_crop: np.ndarray) -> np.ndarray:
    """vigra.filters.distanceTransform of the crop's boundary map in float32: the distance to the nearest boundary pixel.  A
    crop without any boundary pixel (one object covering the whole image) is defined as 0."""
    if not boundary_crop.any():
        return np.zeros(boundary_crop.shape, dtype=np.float32)
    return ndimage.distance_transform_edt(~boundary_crop).astype(np.float32)


def per_object_distance_transform(labels, distances: bool = True, boundary_distances: bool = True,
                                  directed_distances: bool = False, foreground: bool = True, instances: bool = False,
                                  apply_label: bool = True, min_size: int = 0, distance_fill_value: float = 1.0,
                                  sampling=None) -> np.ndarray:
    """float32 (C, H, W): instances, foreground, centre distances, boundary distances (the selected ones, in that order)."""
    if directed_distances or sampling is not None:
        raise NotImplementedError("directed distances and sampling are not restated")
    labels = np.asarray(labels).astype(np.int64)
    if labels.ndim != 2:
        raise ValueError("2-D labels only")
    labels = label_components(labels) if apply_label else relabel_consecutive(labels)
    if min_size > 0:
        labels = size_filter(labels, min_size)
    shape = labels.shape
    fill = np.float32(distance_fill_value)
    cdist = np.full(shape, fill, dtype=np.float32)
    bdist = np.full(shape, fill, dtype=np.float32)
    if distances or boundary_distances:
        boundaries = find_boundaries_inner(labels)
        for k, bb in enumerate(ndimage.find_objects(labels)):
            if bb is None:
                continue
            mask = labels[bb] == k + 1
            yy, xx = np.nonzero(mask)
            centre = (int(np.round(np.mean(yy + bb[0].start))) - bb[0].start,
                      int(np.round(np.mean(xx + bb[1].start))) - bb[1].start)
            correct = not mask[centre]
            if correct or boundary_distances:
                edt = _crop_edt(boundaries[bb])
                edt[~mask] = 0
                if correct:
                    centre = np.unravel_index(np.argmax(edt), edt.shape)
            if distances:
                gy, gx = np.meshgrid(np.arange(mask.shape[0]), np.arange(mask.shape[1]), indexing="ij")
                vec = np.stack([gy - centre[0], gx - centre[1]]).astype(np.float32)
                cd = np.linalg.norm(vec, axis=0).astype(np.float32)
                cd = cd / (cd[mask].max() + EPS)
                cdist[bb][mask] = cd[mask]
            if boundary_distances:
                bd = edt / (edt[mask].max() + EPS)
                bdist[bb][mask] = bd[mask]
    out = []
    if instances:
        out.append(labels.astype(np.float32))
    if foreground:
        out.append((labels > 0).astype(np.float32))
    if distances:
        out.append(cdist)
    if boundary_distances:
        out.append(bdist)
    return np.stack(out) if out else np.zeros((0,) + shape, dtype=np.float32)
