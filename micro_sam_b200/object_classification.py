"""micro-sam's object classification (micro_sam/object_classification.py): SAM embeddings pooled over the objects of a
segmentation as object features, a classifier's object predictions painted back onto the segmentation, and the two together
for a pretrained random forest.

Each unit (the image, a slice or a tile) runs on the device (csrc/objfeat.cu): the segmentation is read through skimage's
nearest-neighbour resize in place and the embedding's bilinear resize is folded into per-object weights, so the resized
embedding (256 x 256 x 256 per unit) is never built.  The segmentation is relabelled to dense indices once, on the device;
sums and areas stay on the device across units, in fp64 and int64, and are divided once at the end.  Results are the same
bit for bit from run to run.  Outputs have the reference's types: numpy `seg_ids` (int64) and `features` of shape (n, 257) --
float64 for a 2-D image without tiling, float32 for slices and tiles.

Embeddings may be numpy arrays, device tensors (`precompute_image_embeddings(..., to_numpy=False)`, read in place), in-memory
tiled groups or saved containers, loaded or lazy.  Containers computed with a `mask` hold only some tiles and are refused.
"""
from __future__ import annotations

import ctypes
import os
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib, util
from ._amg_utils import Blocking

N_FEATURES = 257
_EMBEDDING_SHAPE = (256, 64, 64)


def _device(*xs) -> torch.device:
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return torch.device("cuda", torch.cuda.current_device())


def _labels_int64(segmentation, dev) -> torch.Tensor:
    """the label image as a device int64 tensor (uint32 is widened on the device)"""
    if torch.is_tensor(segmentation):
        return segmentation.to(dev).to(torch.int64)
    a = np.ascontiguousarray(segmentation)
    if a.dtype == np.uint32:
        return torch.from_numpy(a.view(np.int32)).to(dev).to(torch.int64) & 0xFFFFFFFF
    if a.dtype.kind not in "biu":
        raise ValueError(f"segmentation must hold integer labels, got {a.dtype}")
    if a.dtype not in (np.int64, np.int32, np.int16, np.int8, np.uint8, np.bool_):
        a = a.astype(np.int64)
    return torch.from_numpy(a).to(dev).to(torch.int64)


def _relabel(segmentation, dev) -> Tuple[torch.Tensor, torch.Tensor]:
    """dense int32 labels (0 background, k >= 1 the k-th nonzero id) and the sorted nonzero ids, both on the device"""
    s = _labels_int64(segmentation, dev)
    ids = torch.unique(s)
    if ids.numel() and int(ids[0]) < 0:
        raise ValueError("segmentation labels must be non-negative")
    ids = ids[ids != 0]
    table = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), ids])
    return torch.searchsorted(table, s).to(torch.int32), ids


def _unit_embedding(x, dev) -> torch.Tensor:
    t = x if torch.is_tensor(x) else torch.from_numpy(np.asarray(x, dtype=np.float32))
    t = t.to(dev, torch.float32).squeeze().contiguous()
    if tuple(t.shape) != _EMBEDDING_SHAPE:
        raise ValueError(f"expected embeddings of shape {_EMBEDDING_SHAPE} per image, slice or tile, got {tuple(t.shape)}")
    return t


class _Pool:
    """per-object fp64 sums and int64 areas on the device, accumulated unit by unit (msam_object_features)"""

    def __init__(self, n_ids: int, dev):
        L = _lib.lib()
        self.n, self.dev = n_ids, dev
        self.sums = torch.zeros((max(n_ids, 1), _EMBEDDING_SHAPE[0]), dtype=torch.float64, device=dev)
        self.areas = torch.zeros(max(n_ids, 1), dtype=torch.int64, device=dev)
        self.ws = torch.empty(int(L.msam_object_features_workspace(n_ids)), dtype=torch.uint8, device=dev)

    def add(self, emb: torch.Tensor, seg: torch.Tensor, resize_embedding_shape) -> None:
        """one unit: emb [256, 64, 64], seg a 2-D view of the dense labels (rows may be strided)"""
        h, w = seg.shape
        if h == 0 or w == 0:
            return
        S = max(h, w)
        ry, rx = (min(int(r), S) for r in resize_embedding_shape)
        assert seg.stride(1) == 1
        _lib.check(_lib.lib().msam_object_features(_lib.ptr(emb), ctypes.c_void_p(seg.data_ptr()), seg.stride(0), h, w, ry, rx, self.n,
                                                   _lib.ptr(self.ws), self.ws.numel(), _lib.ptr(self.sums), _lib.ptr(self.areas),
                                                   _lib.cur_stream()))

    def finish(self, out_f64: bool) -> torch.Tensor:
        out = torch.zeros((self.n, N_FEATURES), dtype=torch.float64 if out_f64 else torch.float32, device=self.dev)
        _lib.check(_lib.lib().msam_object_features_finish(_lib.ptr(self.sums), _lib.ptr(self.areas), self.n, int(out_f64),
                                                          _lib.ptr(out), _lib.cur_stream()))
        return out


def _units(image_embeddings, dense: torch.Tensor, is_tiled: bool, is_3d: bool):
    """(generator of (segmentation view, embedding) per unit, number of units), in the order of the reference's generator
    (object_classification.py:60-106); tiles take their outer block (with halo), so halo pixels count once in each tile that
    contains them"""
    feats = image_embeddings["features"]
    if not is_tiled:
        return ((dense[z], feats[z]) for z in range(dense.shape[0])), dense.shape[0]
    tiling = Blocking([0, 0], feats.attrs["shape"], feats.attrs["tile_shape"])
    halo = list(feats.attrs["halo"])
    boxes = []
    for block_id in range(tiling.number_of_blocks):
        outer = tiling.get_block_with_halo(block_id, halo).outer_block
        boxes.append(tuple(slice(b, e) for b, e in zip(outer.begin, outer.end)))
    if is_3d:
        gen = ((dense[z][bb], feats[str(i)][z]) for z in range(dense.shape[0]) for i, bb in enumerate(boxes))
        return gen, dense.shape[0] * len(boxes)
    return ((dense[bb], feats[str(i)][:]) for i, bb in enumerate(boxes)), len(boxes)


def compute_object_features(
    image_embeddings: util.ImageEmbeddings,
    segmentation: Union[np.ndarray, torch.Tensor],
    resize_embedding_shape: Tuple[int, int] = (256, 256),
    verbose: bool = True,
) -> Tuple[np.ndarray, np.ndarray]:
    """Pool SAM embeddings over each object of a label image (micro-sam's compute_object_features, same signature).

    Args:
        image_embeddings: what `util.precompute_image_embeddings` returned for the image or volume the labels belong to --
            one image, a stack of slices, or tiles; arrays, device tensors or a saved container.
        segmentation: integer labels (0 is background), 2-D or 3-D, numpy or a device tensor.
        resize_embedding_shape: the grid both the embedding and the labels are resized to before pooling, capped per axis at
            the padded square side of the labels.
        verbose: show a progress bar over slices and tiles.

    Returns:
        The object ids (int64).  For a single 2-D image without tiling these are the ids still present after the labels are
        resized; otherwise every nonzero id of `segmentation`, and an id no slice or tile keeps has a row of zeros.
        The features (n, 257): the object's pixel count on the resized grid, then its mean of each of the 256 channels --
        float64 for a single image, float32 for slices and tiles.
    """
    is_tiled = image_embeddings["input_size"] is None
    is_3d = segmentation.ndim == 3
    if segmentation.ndim not in (2, 3):
        raise ValueError(f"expected a 2-D or 3-D segmentation, got {segmentation.ndim} dimensions")
    if is_tiled and image_embeddings["features"].attrs.get("tiles_in_mask", None) is not None:
        raise ValueError("object features need the embeddings of every tile; these were computed with a mask and hold only "
                         "the tiles inside it")
    dev = _device(segmentation, image_embeddings["features"])
    dense, ids = _relabel(segmentation, dev)
    pool = _Pool(int(ids.numel()), dev)

    if not is_tiled and not is_3d:
        pool.add(_unit_embedding(image_embeddings["features"], dev), dense, resize_embedding_shape)
        feats = pool.finish(out_f64=True).cpu().numpy()
        present = feats[:, 0] > 0
        return ids.cpu().numpy()[present], feats[present]

    units, n_units = _units(image_embeddings, dense, is_tiled, is_3d)
    if verbose:
        from tqdm import tqdm
        units = tqdm(units, total=n_units, desc="Compute object features")
    for seg, emb in units:
        pool.add(_unit_embedding(emb, dev), seg, resize_embedding_shape)
    return ids.cpu().numpy(), pool.finish(out_f64=False).cpu().numpy()


def _projection_table(seg_ids, object_prediction):
    """sorted unique ids and their predictions as 8-byte payloads (int64, or float64 bits); the last prediction of a repeated
    id wins"""
    pred = np.asarray(object_prediction)
    if pred.dtype.kind not in "biuf":
        raise TypeError(f"object predictions must be numeric to be projected on the device, got {pred.dtype}")
    payload = (pred.astype(np.float64) if pred.dtype.kind == "f" else pred.astype(np.int64)).view(np.int64)
    ids = np.asarray(seg_ids).astype(np.int64)
    order = np.argsort(ids, kind="stable")
    ids, payload = ids[order], payload[order]
    last = np.ones(len(ids), dtype=bool)
    last[:-1] = ids[1:] != ids[:-1]
    return np.ascontiguousarray(ids[last]), np.ascontiguousarray(payload[last]), pred.dtype


def project_prediction_to_segmentation(
    segmentation: Union[np.ndarray, torch.Tensor],
    object_prediction: np.ndarray,
    seg_ids: np.ndarray,
) -> Union[np.ndarray, torch.Tensor]:
    """Paint per-object predictions onto the label image (micro-sam's project_prediction_to_segmentation, same signature).

    Args:
        segmentation: integer labels, numpy or a device tensor, any shape.
        object_prediction: one numeric prediction per entry of `seg_ids` (class ids, scores).
        seg_ids: the object id each prediction belongs to; for an id listed twice the later prediction counts.

    Returns:
        An array of the labels' shape holding each pixel's object prediction, and 0 where the label has none (background,
        objects dropped by the resize).  numpy in the prediction's dtype, or for a device segmentation a device tensor (int64,
        or float64 for float predictions).
    """
    assert len(object_prediction) == len(seg_ids)
    ids, payload, dtype = _projection_table(seg_ids, object_prediction)
    dev = _device(segmentation)
    seg = _labels_int64(segmentation, dev).contiguous()
    ids_t, payload_t = torch.from_numpy(ids).to(dev), torch.from_numpy(payload).to(dev)
    out = torch.empty_like(seg)
    _lib.check(_lib.lib().msam_project_labels(_lib.ptr(seg), seg.numel(), _lib.ptr(ids_t), _lib.ptr(payload_t), len(ids),
                                              _lib.ptr(out), _lib.cur_stream()))
    if dtype.kind == "f":
        out = out.view(torch.float64)
    if torch.is_tensor(segmentation):
        return out
    return out.cpu().numpy().astype(dtype, copy=False)


def run_prediction_with_object_classifier(
    images: Sequence[Union[str, os.PathLike, np.ndarray]],
    segmentations: Sequence[Union[str, os.PathLike, np.ndarray]],
    predictor,
    rf_path: Union[str, os.PathLike],
    image_key: Optional[str] = None,
    segmentation_key: Optional[str] = None,
    project_prediction: bool = True,
    ndim: Optional[int] = None,
) -> List[np.ndarray]:
    """run_prediction_with_object_classifier (object_classification.py:224-261): embeddings, object features and the
    predictions of the random forest saved with joblib at `rf_path`, per image; projected onto the segmentation if
    `project_prediction`.  Images and segmentations are arrays; file paths are not loaded (neither does the reference)."""
    assert len(images) == len(segmentations)
    if any(isinstance(x, (str, os.PathLike)) for x in list(images) + list(segmentations)):
        raise NotImplementedError("run_prediction_with_object_classifier takes images and segmentations as arrays, not paths")
    from joblib import load
    rf = load(rf_path)
    predictions = []
    for image, segmentation in zip(images, segmentations):
        embeddings = util.precompute_image_embeddings(predictor, image, verbose=False, ndim=ndim, to_numpy=False)
        seg_ids, features = compute_object_features(embeddings, segmentation, verbose=False)
        prediction = rf.predict(features)
        if project_prediction:
            prediction = project_prediction_to_segmentation(segmentation, prediction, seg_ids)
        predictions.append(prediction)
    return predictions
