"""micro_sam.precompute_state on the H100 core (micro_sam/precompute_state.py:27-279): precompute the image embeddings of a file /
folder into the reference's zarr layout and, optionally, the state of the automatic mask generator next to them
(`<embeddings>.zarr/amg_state.pickle`, or `amg_state/state-<i>.pkl` per slice), so that a later session -- the annotator, a batch
script -- loads instead of recomputing.  Same function names, arguments and file names as the reference.

Differences: (1) the cached AMG state holds this implementation's `crop_list` (low-res logits + per-mask statistics, moved to the
CPU for pickling: ~0.8 GB per 32 x 32-grid tile) instead of CPU RLEs -- `set_state` of either implementation only accepts its own
pickles; (2) `cache_is_state` (AIS: UNETR decoder) is not built (SURVEY.md 8f-2) and raises; (3) image files are read with numpy
(`.npy`), PIL or -- if importable -- imageio / tifffile; container files (`key=`) need h5py / zarr, which this image does not have.
"""
from __future__ import annotations

import os
import pickle
from functools import partial
from glob import glob
from pathlib import Path
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from . import instance_segmentation, util


def load_image_data(path, key: Optional[str] = None, lazy_loading: bool = False) -> np.ndarray:
    """util.load_image_data (util.py:1334-1353)."""
    path = str(path)
    if key is not None:
        if os.path.isdir(path) and ("*" in key or "?" in key):       # a folder of images loaded as a volume
            return np.stack([load_image_data(p) for p in sorted(glob(os.path.join(path, key)))])
        try:
            import h5py
            with h5py.File(path, "r") as f:
                return f[key] if lazy_loading else f[key][:]
        except ImportError as e:
            raise RuntimeError(f"reading '{key}' from the container {path} needs h5py / zarr, which are not installed") from e
    if path.endswith(".npy"):
        return np.load(path)
    try:
        import imageio.v3 as iio
        return np.asarray(iio.imread(path))
    except ImportError:
        pass
    if path.endswith((".tif", ".tiff")):
        try:
            import tifffile
            return tifffile.imread(path)
        except ImportError:
            pass
    from PIL import Image
    return np.asarray(Image.open(path))


def _state_to_cpu(state):
    crops = []
    for mask_data in state["crop_list"]:
        crops.append({k: (v.cpu() if torch.is_tensor(v) else v) for k, v in mask_data.items()})
    return {**state, "crop_list": crops}


def cache_amg_state(predictor, raw: np.ndarray, image_embeddings: util.ImageEmbeddings, save_path: Union[str, os.PathLike],
                    verbose: bool = True, i: Optional[int] = None, **kwargs) -> instance_segmentation.AMGBase:
    """precompute_state.py:27-87: compute and cache -- or load -- the state of the automatic mask generator."""
    is_tiled = image_embeddings["input_size"] is None
    amg = instance_segmentation.get_instance_segmentation_generator(predictor, is_tiled=is_tiled, **kwargs)
    if i is None:
        save_path_amg = os.path.join(save_path, "amg_state.pickle")
    else:
        os.makedirs(os.path.join(save_path, "amg_state"), exist_ok=True)
        save_path_amg = os.path.join(save_path, "amg_state", f"state-{i}.pkl")
    if os.path.exists(save_path_amg):
        if verbose:
            print("Load the AMG state from", save_path_amg)
        with open(save_path_amg, "rb") as f:
            amg.set_state(pickle.load(f))
        return amg
    if verbose:
        print("Precomputing the state for instance segmentation.")
    amg.initialize(raw if i is None else raw[i], image_embeddings=image_embeddings, verbose=verbose, i=i)
    with open(save_path_amg, "wb") as f:
        pickle.dump(_state_to_cpu(amg.get_state()), f)     # on the CPU: the pickle loads without a GPU
    return amg


def cache_is_state(*args, **kwargs):
    """precompute_state.py:90-155 (AIS: UNETR decoder outputs)."""
    raise NotImplementedError("the AIS decoder is not part of the GPU path (SURVEY.md 8f-2)")


def _precompute_state_for_file(predictor, input_path, output_path, key, ndim, tile_shape, halo, precompute_amg_state, decoder, verbose):
    image_data = input_path if isinstance(input_path, np.ndarray) else load_image_data(input_path, key)
    output_path = Path(output_path).with_suffix(".zarr")
    embeddings = util.precompute_image_embeddings(predictor, image_data, str(output_path), ndim=ndim, tile_shape=tile_shape, halo=halo,
                                                  verbose=verbose)
    if precompute_amg_state:
        if decoder is not None:
            cache_is_state()
        cache_function = partial(cache_amg_state, predictor=predictor, image_embeddings=embeddings, save_path=str(output_path))
        nd = image_data.ndim if ndim is None else ndim
        if nd == 2:
            cache_function(raw=image_data, verbose=verbose)
        else:
            for i in range(image_data.shape[0]):
                cache_function(raw=image_data, i=i, verbose=False)
    return embeddings


def _precompute_state_for_files(predictor, input_files: Union[List[Union[os.PathLike, str]], List[np.ndarray]],
                                output_path: Union[os.PathLike, str], key: Optional[str] = None, ndim: Optional[int] = None,
                                tile_shape: Optional[Tuple[int, int]] = None, halo: Optional[Tuple[int, int]] = None,
                                precompute_amg_state: bool = False, decoder=None):
    os.makedirs(output_path, exist_ok=True)
    for idx, file_path in enumerate(input_files):
        out_path = os.path.join(output_path, f"embedding_{idx:05}.tif" if isinstance(file_path, np.ndarray) else os.path.basename(file_path))
        _precompute_state_for_file(predictor, file_path, out_path, key=key, ndim=ndim, tile_shape=tile_shape, halo=halo,
                                   precompute_amg_state=precompute_amg_state, decoder=decoder, verbose=False)


def precompute_state(input_path: Union[os.PathLike, str], output_path: Union[os.PathLike, str], pattern: Optional[str] = None,
                     model_type: str = "vit_b", checkpoint_path: Optional[Union[os.PathLike, str]] = None, key: Optional[str] = None,
                     ndim: Optional[int] = None, tile_shape: Optional[Tuple[int, int]] = None, halo: Optional[Tuple[int, int]] = None,
                     precompute_amg_state: bool = False, predictor=None) -> None:
    """precompute_state.py:224-279.  `predictor=` passes an already built GPU predictor (no download here: without it
    `checkpoint_path` is required)."""
    if predictor is None:
        predictor, state = util.get_sam_model(model_type=model_type, checkpoint_path=checkpoint_path, return_state=True)
        if state is not None and "decoder_state" in state:
            raise NotImplementedError("checkpoints with an AIS decoder: only the AMG state can be precomputed on the GPU path")
    if pattern is None:
        _precompute_state_for_file(predictor, input_path, output_path, key, ndim=ndim, tile_shape=tile_shape, halo=halo,
                                   precompute_amg_state=precompute_amg_state, decoder=None, verbose=True)
    else:
        _precompute_state_for_files(predictor, sorted(glob(os.path.join(input_path, pattern))), output_path, key=key, ndim=ndim,
                                    tile_shape=tile_shape, halo=halo, precompute_amg_state=precompute_amg_state, decoder=None)
