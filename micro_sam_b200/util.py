"""micro_sam.util's hot-path functions with their reference signatures, on the H100 core.

Mirrors (reference file:line): get_sam_model util.py:318-476, _to_image :618-651, _compute_embeddings_batched
:654-681, tiled / 3-D drivers :765-1041, precompute_image_embeddings :1133-1212, set_precomputed :1215-1258,
mask_data_to_segmentation :1773-1848.
`save_path` stores the embeddings in the reference's zarr layout (group attrs = embedding signature, `features` dataset or
per-tile datasets, util.py:684-747 / :1044-1096) through micro_sam_b200/zarr_store.py (zarr itself is not in this image; the
written directory is a plain zarr-v2 store), including the signature check and the resume of partial 3-D runs.  Without
`save_path` embeddings stay in memory (optionally on the device, `to_numpy=False`) with the same dict / group layout.
Out of scope: pooch downloads.
"""
from __future__ import annotations

import ctypes
import hashlib
import os
import warnings
from concurrent import futures
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib, zarr_store
from ._amg_utils import Blocking
from .sam import ARCH, B200Sam, B200SamPredictor, validate_model_type

ImageEmbeddings = Dict[str, Any]


# ------------------------------------------------------------------------------------------------ model loading
def get_device(device: Optional[Union[str, torch.device]] = None) -> torch.device:
    """util.py:204-246 restricted to what this core can run on: a CUDA (sm_90a) device."""
    if device is None or str(device) == "auto":
        device = "cuda"
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"micro_sam_b200 only runs on CUDA sm_90a devices, not {device!r} (no CPU fallback).")
    if not torch.cuda.is_available():
        raise RuntimeError("PyTorch CUDA backend is not available.")
    return dev


class _TolerantPickle:
    """`pickle_module` for torch.load that resolves classes it cannot import to placeholders instead of failing (util.py:246-257):
    torch_em training checkpoints pickle trainer / loss / logger objects next to the weights, and only the weights are
    wanted here.  A private namespace instead of the reference's in-place patch of `pickle.Unpickler`."""
    import pickle as _p
    __name__ = "pickle"
    load, loads, dump, dumps = _p.load, _p.loads, _p.dump, _p.dumps
    HIGHEST_PROTOCOL, DEFAULT_PROTOCOL, Pickler = _p.HIGHEST_PROTOCOL, _p.DEFAULT_PROTOCOL, _p.Pickler
    PickleError, UnpicklingError, PicklingError = _p.PickleError, _p.UnpicklingError, _p.PicklingError

    class Unpickler(_p.Unpickler):
        def find_class(self, module, name):
            try:
                return super().find_class(module, name)
            except (AttributeError, ModuleNotFoundError) as e:
                warnings.warn(f"Did not find {module}:{name} and will skip it, due to error {e}")
                # a placeholder class (the reference returns None, which fails for pickled INSTANCES of the class)
                return type(name, (), {"__init__": lambda self, *a, **k: None, "__setstate__": lambda self, state: None,
                                       "__reduce_ex__": None, "__module__": module})


def _load_checkpoint(checkpoint_path):
    """util.py:273-290: torch_em checkpoints carry {"model_state": {"sam.<key>": ...}, "decoder_state": ...}."""
    state = torch.load(checkpoint_path, map_location="cpu", weights_only=False, pickle_module=_TolerantPickle)
    if "model_state" in state:
        model_state = state["model_state"]
        model_state = {k[len("module."):] if k.startswith("module.") else k: v for k, v in model_state.items()}
        model_state = {k[len("sam."):] if k.startswith("sam.") else k: v for k, v in model_state.items()}
    else:
        model_state = state
    return state, model_state


SUPPORTED_MULTIMASK_OUTPUTS = 3   # the mask decoder has 4 mask tokens: the single mask and 3 multimask outputs


def _check_model_kwargs(kwargs) -> None:
    """The model keywords of micro-sam's get_sam_model (util.py:434-476) that this port cannot honour are refused, not ignored:
    a mask decoder with another mask-token count (semantic models, `num_multimask_outputs=C`) is not built, and
    `flexible_load_checkpoint` only matters for such models."""
    n = kwargs.get("num_multimask_outputs")
    if n is not None and n != SUPPORTED_MULTIMASK_OUTPUTS:
        raise NotImplementedError(f"get_sam_model(num_multimask_outputs={n}): only {SUPPORTED_MULTIMASK_OUTPUTS} is supported (the "
                                  "mask decoder is built with 4 mask tokens; semantic models with other class counts are not)")
    if kwargs.get("flexible_load_checkpoint"):
        raise NotImplementedError("get_sam_model(flexible_load_checkpoint=True) is not implemented: checkpoints load strictly")


def check_mask_token_count(state_dict) -> None:
    """A checkpoint whose mask decoder has another mask-token count than 4 (a semantic model trained with
    num_multimask_outputs = C has C + 1) is refused with the limit named, before the weight loader's shape check."""
    w = state_dict.get("mask_decoder.mask_tokens.weight")
    if w is not None and tuple(w.shape)[:1] != (SUPPORTED_MULTIMASK_OUTPUTS + 1,):
        raise NotImplementedError(f"checkpoint has {tuple(w.shape)[0]} mask tokens (a model with num_multimask_outputs="
                                  f"{tuple(w.shape)[0] - 1}); only {SUPPORTED_MULTIMASK_OUTPUTS + 1} mask tokens "
                                  f"(num_multimask_outputs={SUPPORTED_MULTIMASK_OUTPUTS}) are supported")


def get_sam_model(model_type: str = "vit_b", device: Optional[Union[str, torch.device]] = None,
                  checkpoint_path: Optional[Union[str, os.PathLike]] = None, return_sam: bool = False,
                  return_state: bool = False, state_dict: Optional[Dict[str, torch.Tensor]] = None,
                  max_batch: int = 16, max_prompts: int = 256, **unsupported):
    """util.get_sam_model (util.py:318).  Weights come from `checkpoint_path` (upstream SAM or micro-sam/torch_em
    checkpoint layouts) or from an in-memory upstream-keyed `state_dict`.  There is no download (no network)."""
    for k in ("peft_kwargs", "decoder_path"):
        if unsupported.get(k) is not None:
            raise NotImplementedError(f"get_sam_model({k}=...) is outside the GPU hot path (SURVEY.md 8f)")
    _check_model_kwargs(unsupported)
    device = get_device(device)
    state = None
    if state_dict is None:
        if checkpoint_path is None:
            raise RuntimeError("No weights: pass checkpoint_path=... or state_dict=... (model download needs network).")
        state, state_dict = _load_checkpoint(checkpoint_path)
    abbrev = model_type[:5]
    detected = validate_model_type(state_dict)
    if detected in ARCH and detected != abbrev and abbrev in ("vit_b", "vit_l", "vit_h"):
        raise RuntimeError(f"model_type {model_type!r} does not match the checkpoint ({detected!r})")
    if detected == "vit_t" and abbrev in ("vit_b", "vit_l", "vit_h"):
        raise RuntimeError(f"model_type {model_type!r} does not match the checkpoint (MobileSAM 'vit_t')")
    check_mask_token_count(state_dict)
    sam = B200Sam(detected, state_dict, device=device, max_batch=max_batch, max_prompts=max_prompts)
    predictor = B200SamPredictor(sam)
    predictor.model_type = model_type
    predictor._hash = None
    predictor.model_name = model_type if checkpoint_path is None else os.path.basename(str(checkpoint_path))
    predictor.checkpoint_path = checkpoint_path
    ret = (predictor,)
    if return_sam:
        ret = ret + (sam,)
    if return_state:
        ret = ret + (state,)
    return ret[0] if len(ret) == 1 else ret


# ------------------------------------------------------------------------------------------------ input pipeline
def _normalize_channel(ch: np.ndarray) -> np.ndarray:
    """One channel of util._to_image (util.py:643-647): uint8(((x - min) / (max(x - min) + 1e-7)) * 255) in float32 arithmetic.
    Integer inputs go through a lookup table (the map is a pure function of the pixel value once min / max are known, so
    the table -- built with the very same float32 operations -- gives bit-identical results at a fraction of the passes)."""
    eps = np.float32(1e-7)
    if ch.dtype.kind in "ui" and ch.dtype.itemsize <= 2:
        info = np.iinfo(ch.dtype)
        mn = ch.min()
        span = np.float32(ch.max()) - np.float32(mn)           # exact: |values| < 2^24
        vals = np.arange(info.min, info.max + 1, dtype=np.int32).astype(np.float32)
        vals -= np.float32(mn)
        vals /= (span + eps)
        lut = (vals * 255).astype(np.uint8)                     # entries outside [min, max] are never read
        return lut[ch.astype(np.int32) - info.min] if info.min < 0 else lut[ch]
    x = np.ascontiguousarray(ch, dtype=np.float32)
    x = x - x.min()
    x /= (x.max() + eps)
    return (x * 255).astype(np.uint8)


def _to_image(image):
    """util._to_image (util.py:618-651): grey / 1-3(+) channel input of any dtype -> uint8 H x W x 3, every channel min-max
    normalised on its own; a 2-channel input gets an all-zero third channel (normalised like the others: 0 / 1e-7 = 0), more
    than 3 channels are cut with a warning.  Channel-wise formulation of the reference's whole-array expression (the
    reductions run over contiguous planes); pinned bit for bit on vectors produced by the reference's own function
    (tests/golden/util.npz)."""
    ndim = image.ndim
    if ndim == 2:
        c = _normalize_channel(image)
        return np.stack([c, c, c], axis=-1)
    if ndim != 3:
        raise ValueError(
            f"Invalid input dimensionality {ndim}. Expect either a 2D input (=grayscale image) "
            "or a 3D input (= image with channels)."
        )
    n_channels = image.shape[-1]
    if n_channels == 1:
        c = _normalize_channel(image[..., 0])
        return np.stack([c, c, c], axis=-1)
    if n_channels > 3:
        warnings.warn(f"You provided an input with {n_channels} channels. Only the first three will be used.")
    chans = [_normalize_channel(image[..., k]) for k in range(min(n_channels, 3))]
    if n_channels == 2:
        chans.append(np.zeros(image.shape[:2], dtype=np.uint8))
    return np.stack(chans, axis=-1)


_DTYPE_CODES = {np.dtype("uint8"): 0, np.dtype("uint16"): 1, np.dtype("float32"): 2, np.dtype("int16"): 3,
                np.dtype("float64"): 4}


def _to_image_device(image, device) -> torch.Tensor:
    """`_to_image` on the GPU (msam_to_image): raw host (numpy) or device (torch) image -> uint8 (H, W, 3) device tensor,
    bit-identical to the host function for the supported dtypes (u8/u16/i16/f32/f64, 1-3+ channels)."""
    if isinstance(image, torch.Tensor):
        t = image.to(device).contiguous()
        np_dtype = np.dtype(str(t.dtype).replace("torch.", ""))
    else:
        arr = np.ascontiguousarray(image)
        np_dtype = arr.dtype
        if np_dtype not in _DTYPE_CODES:
            return torch.from_numpy(_to_image(arr)).to(device)
        if np_dtype == np.dtype("uint16"):  # torch has no full uint16 support: ship the bytes
            t = torch.from_numpy(arr.view(np.int16)).to(device, non_blocking=True)
        else:
            t = torch.from_numpy(arr).to(device, non_blocking=True)
    if np_dtype not in _DTYPE_CODES or t.ndim not in (2, 3):
        raise ValueError(f"Invalid input for _to_image: shape {tuple(t.shape)}, dtype {np_dtype}")
    h, w = t.shape[:2]
    c = 1 if t.ndim == 2 else t.shape[2]
    out = torch.empty(h, w, 3, dtype=torch.uint8, device=device)
    scratch = torch.empty(6, dtype=torch.int32, device=device)
    _lib.check(_lib.lib().msam_to_image(_lib.ptr(t), _DTYPE_CODES[np_dtype], h, w, c, _lib.ptr(out), _lib.ptr(scratch),
                                        _lib.cur_stream()))
    return out


@torch.no_grad()
def _compute_embeddings_batched_raw(predictor, raw_images):
    """_to_image + _compute_embeddings_batched for raw images that need no resize (longest side == model input size):
    normalisation runs on the device, so the host only ships the raw bytes."""
    sam = predictor.model
    predictor.reset_image()
    u8 = torch.stack([_to_image_device(im, sam.device) for im in raw_images])
    features = sam.encode_u8(u8)
    sizes = [tuple(im.shape[:2]) for im in raw_images]
    predictor.original_size = sizes[-1]
    predictor.input_size = sizes[-1]
    predictor.features = features[-1:]
    predictor.is_image_set = True
    return features, sizes, sizes


def _needs_no_resize(predictor, image) -> bool:
    h, w = image.shape[:2]
    return max(h, w) == predictor.transform.target_length and (image.ndim == 2 or image.shape[2] >= 1) \
        and np.dtype(image.dtype) in _DTYPE_CODES


def _host_pool() -> futures.ThreadPoolExecutor:
    """Host threads for the per-tile numpy / PIL work (min-max normalisation, ResizeLongestSide): both release the GIL, and
    at H100 encoder speeds (a few ms per tile) a single Python thread would be the bottleneck (SURVEY.md 8a, a4)."""
    global _POOL
    if _POOL is None:
        _POOL = futures.ThreadPoolExecutor(max(1, min(32, (os.cpu_count() or 2) - 1)))
    return _POOL


_POOL = None


def _prepare_tiles(predictor, raw_tiles):
    """_to_image + ResizeLongestSide.apply_image for a list of raw tiles, in parallel on the host pool."""
    def one(raw):
        img = _to_image(raw)
        return img.shape[:2], predictor.transform.apply_image(img)
    return list(_host_pool().map(one, raw_tiles)) if len(raw_tiles) > 1 else [one(t) for t in raw_tiles]


@torch.no_grad()
def _compute_embeddings_batched(predictor, batched_images, prepared=None):
    """util.py:654-681: resize each image, then ONE encoder call for the batch (preprocess is fused in the kernel when
    all resized images share a shape, which is always the case for tiles of one tiling).  `prepared`: output of
    `_prepare_tiles` for the same images (then `batched_images` is ignored)."""
    predictor.reset_image()
    resized, original_sizes, input_sizes = [], [], []
    if prepared is None:
        prepared = [(image.shape[:2], predictor.transform.apply_image(image)) for image in batched_images]
    for osz, t in prepared:
        original_sizes.append(tuple(osz))
        input_sizes.append(tuple(t.shape[:2]))
        resized.append(t)
    sam = predictor.model
    if len(set(input_sizes)) == 1:
        batch = torch.from_numpy(np.stack(resized))
        if batch.numel() > 0:
            batch = batch.pin_memory() if torch.cuda.is_available() else batch
        features = sam.encode_u8(batch.to(sam.device, non_blocking=True))
    else:  # ragged border tiles: normalise + pad on the device, one fp32 batch
        tensors = [sam.preprocess(torch.from_numpy(t).to(sam.device).permute(2, 0, 1)[None]) for t in resized]
        features = sam.image_encoder(torch.cat(tensors))
    predictor.original_size = original_sizes[-1]
    predictor.input_size = input_sizes[-1]
    predictor.features = features[-1:]  # NB: the reference leaves features[-1] (3-D); kept 4-D for the decoder
    predictor.is_image_set = True
    return features, original_sizes, input_sizes


class _MemDataset:
    """Stand-in for a zarr array with `.attrs` (util.py:720-729)."""

    def __init__(self, data, attrs=None):
        self.data = data
        self.attrs = dict(attrs or {})

    @property
    def ndim(self):
        return self.data.ndim

    @property
    def shape(self):
        return self.data.shape

    def __getitem__(self, idx):
        return self.data[idx]

    def __setitem__(self, idx, val):
        self.data[idx] = val


class _MemGroup(dict):
    """Stand-in for a zarr group: datasets by name + attrs."""

    def __init__(self):
        super().__init__()
        self.attrs = {}


def handle_pbar(verbose, pbar_init, pbar_update):
    """util.py:1098-1130 without tqdm dependency on the hot path."""
    if verbose and pbar_init is None:
        from tqdm import tqdm
        pbar = tqdm()

        def pbar_init(total, description):  # noqa: F811
            pbar.total = total
            pbar.set_description(description)

        def pbar_update(update):  # noqa: F811
            pbar.update(update)

        def pbar_close():
            pbar.close()
    elif pbar_init is not None and pbar_update is not None:
        pbar = None

        def pbar_close():
            pass
    else:
        pbar = None

        def pbar_init(total, description):  # noqa: F811
            pass

        def pbar_update(update):  # noqa: F811
            pass

        def pbar_close():
            pass
    return pbar, pbar_init, pbar_update, pbar_close


def _get_tiles_in_mask(mask, tiling, halo, z=None):
    out = []
    for tile_id in range(tiling.number_of_blocks):
        tile = tiling.get_block_with_halo(tile_id, list(halo))
        outer = tuple(slice(b, e) for b, e in zip(tile.outer_block.begin, tile.outer_block.end))
        if z is not None:
            outer = (z,) + outer
        if np.asarray(mask[outer]).astype(bool).sum() != 0:
            out.append(tile_id)
    return out


def _compute_data_signature(input_) -> str:
    """util.py:1044-1046."""
    return hashlib.sha1(np.asarray(input_).tobytes()).hexdigest()


def _get_embedding_signature(input_, predictor, tile_shape, halo, data_signature=None):
    """util.py:1050-1064."""
    from . import __version__
    if data_signature is None:
        data_signature = _compute_data_signature(input_)
    return {
        "data_signature": data_signature,
        "tile_shape": tile_shape if tile_shape is None else list(tile_shape),
        "halo": halo if halo is None else list(halo),
        "model_type": predictor.model_type,
        "model_name": predictor.model_name,
        "micro_sam_version": __version__,
        "model_hash": getattr(predictor, "_hash", None),
    }


def _write_embedding_signature(f, input_, predictor, tile_shape, halo, input_size, original_size):
    """util.py:1070-1074: the signature is written LAST -- its `input_size` key is what marks a container as complete."""
    signature = _get_embedding_signature(input_, predictor, tile_shape, halo)
    signature.update({"input_size": None if input_size is None else list(input_size),
                      "original_size": None if original_size is None else list(original_size)})
    f.attrs.update(signature)


def _check_saved_embeddings(input_, predictor, f, save_path, tile_shape, halo):
    """util.py:1077-1102."""
    if "input_size" not in f.attrs:   # empty / partial container: embeddings will be (re)computed
        return
    signature = _get_embedding_signature(input_, predictor, tile_shape, halo)
    for key, val in signature.items():
        if key not in f.attrs or f.attrs[key] != val:
            if key in ("micro_sam_version", "model_hash", "model_name"):
                warnings.warn(f"The signature for {key} in embeddings file {save_path} has a mismatch: "
                              f"{f.attrs.get(key)} != {val}. This key was recently added, so your embeddings are likely "
                              "correct. But please recompute them if model predictions don't look as expected.")
            else:
                raise RuntimeError(f"Embeddings file {save_path} is invalid due to mismatch in {key}: "
                                   f"{f.attrs.get(key)} != {val}. Please recompute embeddings in a new file.")


def _write_chunks(jobs):
    """util._write_batch's thread pool (util.py:743-747): jobs = [(dataset, index, host array)]; chunk files are
    independent, so the writes run concurrently while the GPU computes the next batch."""
    if not jobs:
        return
    with futures.ThreadPoolExecutor(min(8, len(jobs))) as tp:
        list(tp.map(lambda j: j[0].__setitem__(j[1], j[2]), jobs))


def _compute_tiled_features(predictor, input_, is3d, tile_shape, halo, pbar_init, pbar_update, batch_size, mask, to_numpy,
                            rank: int = 0, world_size: int = 1, zgroup=None):
    """util.py:765-899 (_compute_tiled_features_2d/_3d + _BatchProvider): (z, tile) pairs in row-major order, batches of
    `batch_size`, each tile normalised on its own (_to_image) -- tiled embeddings are NOT crops of a global embedding.
    rank/world_size: static block partition of that order for multi-GPU sharding (SURVEY.md 8e) -- each rank fills only
    its own (z, tile) entries; no collective.  zgroup: zarr group to write into (`save_path`), else an in-memory group."""
    plane_shape = input_.shape[1:3] if is3d else input_.shape[:2]
    tiling = Blocking([0, 0], plane_shape, tile_shape)
    if zgroup is not None:
        features = zgroup.require_group("features")
        to_numpy = True
    else:
        features = _MemGroup()
    features.attrs["shape"] = tuple(plane_shape)
    features.attrs["tile_shape"] = tuple(tile_shape)
    features.attrs["halo"] = tuple(halo)
    n_slices = input_.shape[0] if is3d else 1
    work = []
    tiles_in_mask = {}
    for z in range(n_slices):
        ids = range(tiling.number_of_blocks) if mask is None else _get_tiles_in_mask(mask, tiling, halo, z if is3d else None)
        tiles_in_mask[str(z)] = list(ids)
        work += [(z, t) for t in ids]
    lo, hi = (len(work) * rank) // world_size, (len(work) * (rank + 1)) // world_size
    my_work = work[lo:hi]
    pbar_init(len(my_work), "Compute Image Embeddings tiled")

    def prepare(chunk):   # host side of a batch: crop, normalise per tile, resize -- runs one batch ahead of the GPU
        raw = []
        for z, tile_id in chunk:
            tile = tiling.get_block_with_halo(tile_id, list(halo))
            outer = tuple(slice(b, e) for b, e in zip(tile.outer_block.begin, tile.outer_block.end))
            raw.append(input_[(z,) + outer] if is3d else input_[outer])
        return _prepare_tiles(predictor, raw)

    chunks = [my_work[b0:b0 + batch_size] for b0 in range(0, len(my_work), batch_size)]
    ahead = futures.ThreadPoolExecutor(1)
    ahead_w, pending = futures.ThreadPoolExecutor(1), []
    nxt = ahead.submit(prepare, chunks[0]) if chunks else None
    for ci, chunk in enumerate(chunks):
        prepared = nxt.result()
        nxt = ahead.submit(prepare, chunks[ci + 1]) if ci + 1 < len(chunks) else None
        emb, original_sizes, input_sizes = _compute_embeddings_batched(predictor, None, prepared=prepared)
        if zgroup is not None:   # _write_batch (util.py:710-747): datasets first (creation is not thread-safe), then chunks
            targets = []
            for k, (z, tile_id) in enumerate(chunk):
                name = str(tile_id)
                eshape = tuple(emb.shape[1:])
                if name not in features:
                    shape = ((n_slices, 1) if is3d else (1,)) + eshape
                    ds = features.create_dataset(name, shape=shape, dtype="float32", chunks=((1, 1) if is3d else (1,)) + eshape)
                    ds.attrs["original_size"] = original_sizes[k]
                    ds.attrs["input_size"] = input_sizes[k]
                targets.append((features[name], z if is3d else slice(None)))

            def flush(emb=emb, targets=targets):   # D2H + chunk files off the critical path: the GPU encodes the next batch
                host = emb.cpu().numpy()
                _write_chunks([(ds, idx, host[k][None]) for k, (ds, idx) in enumerate(targets)])
            pending.append(ahead_w.submit(flush))
            if len(pending) > 2:                   # bound the embeddings held on the device to a few batches
                pending.pop(0).result()
            pbar_update(len(chunk))
            continue
        emb_host = emb.cpu().numpy() if to_numpy else emb
        for k, (z, tile_id) in enumerate(chunk):
            name = str(tile_id)
            if is3d:
                if name not in features:
                    shape = (n_slices, 1) + tuple(emb.shape[1:])
                    data = np.zeros(shape, dtype="float32") if to_numpy else torch.zeros(shape, device=emb.device)
                    features[name] = _MemDataset(data, {"original_size": original_sizes[k], "input_size": input_sizes[k]})
                features[name][z] = emb_host[k][None]
            else:
                features[name] = _MemDataset(emb_host[k][None], {"original_size": original_sizes[k],
                                                                   "input_size": input_sizes[k]})
        pbar_update(len(chunk))
    ahead.shutdown()
    for fut in pending:
        fut.result()
    ahead_w.shutdown()
    if mask is not None:
        features.attrs["tiles_in_mask"] = tiles_in_mask if is3d else tiles_in_mask["0"]
    if zgroup is not None and rank == 0:   # every rank's chunks are in place once the caller's barrier has passed
        _write_embedding_signature(zgroup, input_, predictor, tile_shape, halo, input_size=None, original_size=None)
    return features


def _precompute_saved(predictor, input_, save_path, lazy_loading, ndim, tile_shape, halo, pbar_init, pbar_update, batch_size,
                      mask, rank, world_size):
    """precompute_image_embeddings with a zarr container (util.py:1183-1211 + _compute_2d / _compute_3d / _compute_tiled_*)."""
    existed = os.path.exists(save_path)
    f = zarr_store.open_group(save_path, mode="a")
    if existed:
        _check_saved_embeddings(input_, predictor, f, save_path, tile_shape, halo)
    complete = "input_size" in f.attrs
    if tile_shape is not None:
        if complete:   # _compute_tiled_2d/_3d: cached
            return {"features": f["features"], "input_size": f.attrs["input_size"], "original_size": f.attrs["original_size"]}
        feats = _compute_tiled_features(predictor, input_, ndim == 3, tuple(tile_shape), tuple(halo), pbar_init, pbar_update,
                                        batch_size, mask, True, rank, world_size, zgroup=f)
        return {"features": feats, "input_size": None, "original_size": None}
    if ndim == 2:
        if complete:   # _compute_2d: load and set
            emb = {"features": f["features"][:], "input_size": tuple(f.attrs["input_size"]),
                   "original_size": tuple(f.attrs["original_size"])}
            set_precomputed(predictor, emb)
            return emb
        pbar_init(1, "Compute Image Embeddings 2D")
        if _needs_no_resize(predictor, input_):
            _compute_embeddings_batched_raw(predictor, [input_])
        else:
            predictor.reset_image()
            predictor.set_image(_to_image(input_))
        feats = predictor.get_image_embedding().cpu().numpy()
        pbar_update(1)
        f.create_dataset("features", data=feats)
        _write_embedding_signature(f, input_, predictor, None, None, predictor.input_size, predictor.original_size)
        return {"features": feats, "input_size": predictor.input_size, "original_size": predictor.original_size}
    # ---- 3-D (util.py:950-1022), resumable: slices whose chunk is already non-zero are skipped
    if complete:
        feats = f["features"] if lazy_loading else f["features"][:]
        return {"features": feats, "input_size": tuple(f.attrs["input_size"]), "original_size": tuple(f.attrs["original_size"])}
    n = input_.shape[0]
    eshape = (1, 256, 64, 64)
    shape, chunks = (n,) + eshape, (1,) + eshape
    partial = "features" in f
    if partial:
        feats = f["features"]
        if feats.shape != shape or feats.chunks != chunks:
            raise RuntimeError("Invalid partial features")
    else:
        feats = f.create_dataset("features", shape=shape, chunks=chunks, dtype="float32")
    todo = [z for z in range(n) if not (partial and np.count_nonzero(feats[z]) != 0)]
    lo, hi = (len(todo) * rank) // world_size, (len(todo) * (rank + 1)) // world_size
    todo = todo[lo:hi]
    pbar_init(len(todo), "Compute Image Embeddings 3D")
    original_sizes = input_sizes = None
    for b0 in range(0, len(todo), batch_size):
        zs = todo[b0:b0 + batch_size]
        raw = [input_[z] for z in zs]
        if all(_needs_no_resize(predictor, im) for im in raw):
            e, original_sizes, input_sizes = _compute_embeddings_batched_raw(predictor, raw)
        else:
            e, original_sizes, input_sizes = _compute_embeddings_batched(predictor, [_to_image(im) for im in raw])
        host = e.cpu().numpy()
        _write_chunks([(feats, z, host[k][None]) for k, z in enumerate(zs)])
        pbar_update(len(zs))
    if original_sizes is None:   # nothing left to compute on this rank: sizes follow from the geometry
        from .sam import get_preprocess_shape
        h, w = input_.shape[1:3]
        original_sizes, input_sizes = [(h, w)], [get_preprocess_shape(h, w, predictor.transform.target_length)]
    if rank == 0:
        _write_embedding_signature(f, input_, predictor, None, None, input_sizes[-1], original_sizes[-1])
    out = feats if (lazy_loading or world_size > 1) else feats[:]
    return {"features": out, "input_size": tuple(input_sizes[-1]), "original_size": tuple(original_sizes[-1])}


def precompute_image_embeddings(predictor, input_: np.ndarray, save_path=None, lazy_loading: bool = False,
                                ndim: Optional[int] = None, tile_shape: Optional[Tuple[int, int]] = None,
                                halo: Optional[Tuple[int, int]] = None, verbose: bool = False, batch_size: int = 1,
                                mask=None, pbar_init: Optional[Callable] = None, pbar_update: Optional[Callable] = None,
                                to_numpy: bool = True, rank: int = 0, world_size: int = 1) -> ImageEmbeddings:
    """util.precompute_image_embeddings (util.py:1133).  `to_numpy=False` keeps the embeddings on the device (skips the
    reference's D2H, util.py:917); rank/world_size shard tiled work across processes."""
    ndim = input_.ndim if ndim is None else ndim
    _, pbar_init, pbar_update, pbar_close = handle_pbar(verbose, pbar_init, pbar_update)
    if tile_shape is not None and halo is None:
        raise ValueError("To compute tiled embeddings the parameters tile_shape and halo have to be passed.")
    if ndim not in (2, 3):
        raise ValueError(f"Invalid dimesionality {input_.ndim}, expect 2 or 3 dim data.")
    if save_path is not None:
        emb = _precompute_saved(predictor, input_, save_path, lazy_loading, ndim, tile_shape, halo, pbar_init, pbar_update,
                                batch_size, mask, rank, world_size)
        pbar_close()
        return emb
    if ndim == 2 and tile_shape is None:
        pbar_init(1, "Compute Image Embeddings 2D")
        if _needs_no_resize(predictor, input_):
            _compute_embeddings_batched_raw(predictor, [input_])
        else:
            predictor.reset_image()
            predictor.set_image(_to_image(input_))
        feats = predictor.get_image_embedding()
        feats = feats.cpu().numpy() if to_numpy else feats
        pbar_update(1)
        emb = {"features": feats, "input_size": predictor.input_size, "original_size": predictor.original_size}
    elif ndim == 3 and tile_shape is None:
        n = input_.shape[0]
        pbar_init(n, "Compute Image Embeddings 3D")
        outs = []
        for z0 in range(0, n, batch_size):
            raw = [input_[z] for z in range(z0, min(z0 + batch_size, n))]
            if all(_needs_no_resize(predictor, im) for im in raw):
                e, original_sizes, input_sizes = _compute_embeddings_batched_raw(predictor, raw)
            else:
                e, original_sizes, input_sizes = _compute_embeddings_batched(predictor, [_to_image(im) for im in raw])
            images = raw
            outs.append(e[:, None])
            pbar_update(len(images))
        feats = torch.cat(outs)  # (Z,1,256,64,64) (util.py:968-970)
        feats = feats.cpu().numpy() if to_numpy else feats
        emb = {"features": feats, "input_size": input_sizes[-1], "original_size": original_sizes[-1]}
    elif ndim in (2, 3):
        feats = _compute_tiled_features(predictor, input_, ndim == 3, tuple(tile_shape), tuple(halo), pbar_init, pbar_update,
                                        batch_size, mask, to_numpy, rank, world_size)
        emb = {"features": feats, "input_size": None, "original_size": None}
    else:
        raise ValueError(f"Invalid dimesionality {input_.ndim}, expect 2 or 3 dim data.")
    pbar_close()
    return emb


def set_precomputed(predictor, image_embeddings: ImageEmbeddings, i: Optional[int] = None, tile_id: Optional[int] = None):
    """util.py:1215-1258."""
    if tile_id is not None:
        tile_features = image_embeddings["features"][str(tile_id)]
        return set_precomputed(predictor, {"features": tile_features, "input_size": tile_features.attrs["input_size"],
                                           "original_size": tile_features.attrs["original_size"]}, i=i)
    device = predictor.device
    features = image_embeddings["features"]
    assert features.ndim in (4, 5), f"{features.ndim}"
    if features.ndim == 5 and i is None:
        raise ValueError("The data is 3D so an index i is needed.")
    elif features.ndim == 4 and i is not None:
        raise ValueError("The data is 2D so an index is not needed.")
    f = features[:] if i is None else features[i]
    predictor.features = f.to(device) if torch.is_tensor(f) else torch.from_numpy(np.asarray(f)).to(device)
    predictor.original_size = tuple(image_embeddings["original_size"])
    predictor.input_size = tuple(image_embeddings["input_size"])
    predictor.is_image_set = True
    return predictor


def compute_iou(mask1: np.ndarray, mask2: np.ndarray) -> float:
    """util.compute_iou (util.py:1266-1280): overlap / (union + 1e-7) of the pixels == 1, in fp64."""
    overlap = np.logical_and(mask1 == 1, mask2 == 1).sum()
    union = np.logical_or(mask1 == 1, mask2 == 1).sum()
    return float(overlap) / (float(union) + 1e-7)


# ------------------------------------------------------------------------------------------------ centres, boxes and one-hot
def _check_label_shape(shape) -> None:
    if len(shape) not in (2, 3):
        raise ValueError(f"segmentation must be 2-D or 3-D, got {len(shape)} dimensions")
    padded = int(np.prod([int(v) + 2 for v in shape]))
    if min(shape) == 0 or padded >= 2 ** 31:
        raise ValueError(f"segmentation of shape {tuple(shape)}: the image padded by one pixel per side must have fewer than 2^31 "
                         f"pixels (int32 linear indices), got {padded}, and no axis may be empty")


def _labels_for_centers(segmentation):
    """A 2-D or 3-D integer label image (numpy or torch, host or device) -> (int32 labels on the device, C order; the sorted
    unique ids present, int64 on the device, 0 included when present; the largest id).  Refuses non-integer labels, negative
    labels, ids >= 2^31 and images whose grid padded by one pixel per side has 2^31 pixels or more."""
    wrapped = False   # unsigned values reinterpreted as signed: a negative value is one >= 2^31 (uint32) or >= 2^63 (uint64)
    if torch.is_tensor(segmentation):
        t = segmentation
        if t.is_floating_point() or t.is_complex():
            raise ValueError(f"segmentation must hold integer labels, got {t.dtype}")
        _check_label_shape(t.shape)
        if t.dtype in (torch.uint32, torch.uint64):
            t = t.to(torch.int64)   # uint32 widens exactly; uint64 >= 2^63 wraps negative
            wrapped = True
        dev = t.device if t.is_cuda else torch.device("cuda", torch.cuda.current_device())
        t = t.to(dev)
    else:
        a = np.asarray(segmentation)
        if a.dtype.kind not in "biu":
            raise ValueError(f"segmentation must hold integer labels, got {a.dtype}")
        _check_label_shape(a.shape)
        if a.dtype == np.uint32:
            a, wrapped = a.view(np.int32), True
        elif a.dtype == np.uint64:
            a, wrapped = a.view(np.int64), True
        dev = torch.device("cuda", torch.cuda.current_device())
        t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if t.dtype == torch.bool:
        t = t.to(torch.uint8)
    ids = torch.unique(t)
    lo, hi = (int(v) for v in ids[[0, -1]].tolist())
    if lo < 0:
        raise ValueError("segmentation ids must be below 2^31" if wrapped else "segmentation labels must be non-negative")
    if hi >= 2 ** 31:
        raise ValueError(f"segmentation ids must be below 2^31, got {hi}")
    return t.to(torch.int32).contiguous(), ids.to(torch.int64), hi


def get_centers_and_bounding_boxes(segmentation, mode: str = "v", device_result: bool = False):
    """util.get_centers_and_bounding_boxes (micro_sam/util.py:1283-1331) on the device (csrc/centers.cu), 2-D and 3-D.

    Returns (centers, boxes): two dicts keyed by object id in ascending order.  mode "v": the object pixel of largest distance to
    the object boundary (ties: the first in raster order), as a tuple of ints; "p": the centroid, a tuple of float64.  Boxes are
    skimage's bbox tuples (min per axis, then max + 1 per axis).  `segmentation` holds integer labels (numpy or torch, host or
    device; 0 is background, ids below 2^31).  The rules are restated in DESIGN.md section 2.

    `device_result=True` (extension): returns device tensors (ids int64 (n,), centers (n, ndim) int32 for "v" / float64 for "p",
    boxes int32 (n, 2 ndim)) and builds no dicts.
    """
    if mode not in ("p", "v"):
        raise AssertionError("Choose either 'p' for regionprops centroids or 'v' for distance-based centers")
    labels, ids, _ = _labels_for_centers(segmentation)
    dev, ndim = labels.device, labels.ndim
    ids = ids[ids != 0]
    n = int(ids.numel())
    centers = torch.empty((n, ndim), dtype=torch.int32 if mode == "v" else torch.float64, device=dev)
    boxes = torch.empty((n, 2 * ndim), dtype=torch.int32, device=dev)
    if n:
        L = _lib.lib()
        dims = (ctypes.c_int * ndim)(*labels.shape)
        ws = torch.empty(int(L.msam_centers_workspace(ndim, dims, n)), dtype=torch.uint8, device=dev)
        ids32 = ids.to(torch.int32)
        with torch.cuda.device(dev):
            _lib.check(L.msam_centers_boxes(_lib.ptr(labels), ndim, dims, ord(mode), _lib.ptr(ws), ws.numel(), _lib.ptr(ids32), n,
                                            _lib.ptr(centers), _lib.ptr(boxes), _lib.cur_stream()))
    if device_result:
        return ids, centers, boxes
    keys = ids.cpu().tolist()
    cast = int if mode == "v" else float
    center_coordinates = {k: tuple(cast(v) for v in c) for k, c in zip(keys, centers.cpu().tolist())}
    bbox_coordinates = {k: tuple(b) for k, b in zip(keys, boxes.cpu().tolist())}
    return center_coordinates, bbox_coordinates


def segmentation_to_one_hot(segmentation, segmentation_ids: Optional[np.ndarray] = None) -> torch.Tensor:
    """util.segmentation_to_one_hot (micro_sam/util.py:1356-1396) on the device (csrc/centers.cu), 2-D and 3-D.

    Returns float32 masks (n_ids, 1, *shape) as a device tensor (the reference returns a CPU tensor).  Without
    `segmentation_ids`, n_ids = segmentation.max() and plane k holds label k + 1.  With them (not empty, no 0), n_ids =
    len(segmentation_ids) and the selected ids present in the image fill the planes in ascending order, as the reference's
    relabel_sequential does: a selected id that is absent shifts the later ones forward and leaves an empty plane at the end.
    """
    if segmentation_ids is not None:
        sel = np.asarray(segmentation_ids).ravel()
        if len(sel) == 0 or 0 in sel:
            raise RuntimeError("No foreground objects were found.")
    labels, present, hi = _labels_for_centers(segmentation)
    dev = labels.device
    table, n_tab = None, 0
    if segmentation_ids is None:
        n_planes = hi
    else:
        n_planes = len(sel)
        wanted = torch.as_tensor(np.sort(sel).astype(np.int64), device=dev)
        table = present[torch.isin(present, wanted) & (present != 0)].to(torch.int32)
        n_tab = int(table.numel())
        if n_tab == 0:   # no selected id is present: every plane is empty, but the table pointer must still be set
            table = torch.zeros(1, dtype=torch.int32, device=dev)
    out = torch.empty((n_planes, 1) + tuple(labels.shape), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().msam_segmentation_one_hot(_lib.ptr(labels), labels.numel(), _lib.ptr(table), n_tab,
                                                        n_planes, _lib.ptr(out), _lib.cur_stream()))
    return out


# ------------------------------------------------------------------------------------------------ label image assembly
def finish_ws_size(h: int, w: int) -> int:
    """int32 workspace elements of msam_finish_segmentation (include/msam_b200.h)."""
    return 4 * h * w + max(4096, (h * w + 1023) // 1024) + 8


def _label_connected(seg: np.ndarray) -> np.ndarray:
    """Connected components of a label image (what elf.parallel.label does at util.py:1831-1834): 4-connectivity,
    components of equal non-zero label, ids in raster order of first pixel."""
    from scipy import ndimage
    h, w = seg.shape
    # edges exist only between equal labels: label the foreground with horizontal/vertical links masked out where the
    # neighbour differs, by labelling a 2x up-sampled "pixels + links" grid.
    big = np.zeros((2 * h - 1, 2 * w - 1), dtype=bool)
    fg = seg != 0
    big[::2, ::2] = fg
    big[::2, 1::2] = fg[:, :-1] & (seg[:, :-1] == seg[:, 1:])
    big[1::2, ::2] = fg[:-1, :] & (seg[:-1, :] == seg[1:, :])
    lab, _ = ndimage.label(big)  # default 4-connectivity; raster-order ids
    lab = lab[::2, ::2]
    ids = np.unique(lab)
    ids = ids[ids != 0]
    lut = np.zeros(int(lab.max()) + 1, dtype=np.uint32)
    lut[ids] = np.arange(1, len(ids) + 1, dtype=np.uint32)
    return lut[lab]


def _finish_segmentation(segmentation: np.ndarray, min_object_size: int, label_masks: bool, with_background: bool):
    """util.py:1831-1848: CC-label, drop small objects (and the largest one if with_background), relabel."""
    if label_masks:
        segmentation = _label_connected(segmentation)
    seg_ids, sizes = np.unique(segmentation, return_counts=True)
    filter_ids = seg_ids[sizes < min_object_size]
    if with_background:
        filter_ids = np.concatenate([filter_ids, [seg_ids[np.argmax(sizes)]]])
    if len(filter_ids):
        segmentation = segmentation.copy()
        segmentation[np.isin(segmentation, filter_ids)] = 0
    ids = np.unique(segmentation)
    ids = ids[ids != 0]
    lut = np.zeros(int(segmentation.max()) + 1, dtype=np.uint32)
    lut[ids] = np.arange(1, len(ids) + 1, dtype=np.uint32)
    return lut[segmentation]


def mask_data_to_segmentation(masks: List[Dict[str, Any]], shape: Optional[Tuple[int, int]] = None,
                              min_object_size: int = 0, max_object_size: Optional[int] = None, label_masks: bool = True,
                              with_background: bool = False, merge_exclusively: bool = True) -> np.ndarray:
    """util.mask_data_to_segmentation (util.py:1773-1848) for host-side binary-mask records (API parity; the AMG /
    batched-inference fast path paints on the device instead, see instance_segmentation.py)."""
    # paint in descending-area order (stable for equal areas): with merge_exclusively the first -- largest -- mask owns a pixel,
    # without it later -- smaller -- masks overwrite (what AMG asks for, instance_segmentation.py:527-529)
    order = sorted(range(len(masks)), key=lambda i: -masks[i]["area"])
    if shape is None:
        shape = masks[order[0]]["segmentation"].shape
    label = np.zeros(shape, dtype=np.uint32)
    next_id = 1
    for i in order:
        rec = masks[i]
        if rec["area"] < min_object_size or (max_object_size is not None and rec["area"] > max_object_size):
            continue
        m = rec["segmentation"]
        m = (m.cpu().numpy() if torch.is_tensor(m) else np.asarray(m)).astype(bool, copy=False)
        sid = rec.get("seg_id", next_id)
        if "global_bbox" in rec:     # tiled records: the tile-local box content goes to the global box position
            x, y, w, h = (int(v) for v in rec["bbox"])
            gx, gy, gw, gh = (int(v) for v in rec["global_bbox"])
            window = label[gy:gy + gh, gx:gx + gw]
            piece = m[y:y + h, x:x + w]
            window[piece & (window == 0) if merge_exclusively else piece] = sid
        else:
            label[m & (label == 0) if merge_exclusively else m] = sid
        next_id = sid + 1
    segmentation = label
    return _finish_segmentation(segmentation, min_object_size, label_masks, with_background)


# ------------------------------------------------------------------------------------------------ mask NMS
def _xywh_to_xyxy(boxes):
    boxes = boxes.clone() if isinstance(boxes, torch.Tensor) else torch.tensor(np.asarray(boxes))
    boxes = boxes.to(torch.float32)
    boxes[:, 2] += boxes[:, 0]
    boxes[:, 3] += boxes[:, 1]
    return boxes


def batched_mask_nms(masks: torch.Tensor, boxes_xyxy: torch.Tensor, scores: torch.Tensor, nms_thresh: float,
                     intersection_over_min: bool = False, return_matrix: bool = False):
    """util._batched_mask_nms (util.py:1647-1676) on the device (the reference forces this to the CPU, :1648-1656):
    bit-packed popcount intersections, the same float32 ratios, greedy `keep iou <= thresh`."""
    dev = torch.device("cuda") if not masks.is_cuda else masks.device
    m = masks.to(dev).to(torch.uint8).contiguous()
    n, h, w = m.shape
    bx = boxes_xyxy.to(dev, torch.float32).contiguous()
    sc = scores.to(dev, torch.float32).contiguous()
    words = (h * w + 31) // 32
    bits = torch.empty(max(n, 1) * words, dtype=torch.int32, device=dev)
    areas = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    mat = torch.empty(max(n * n, 1), dtype=torch.float32, device=dev)
    keep = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    nk = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().msam_mask_nms(_lib.ptr(m), n, h, w, _lib.ptr(bx), _lib.ptr(sc), float(nms_thresh),
                                        int(intersection_over_min), _lib.ptr(bits), _lib.ptr(areas), _lib.ptr(mat),
                                        _lib.ptr(keep), _lib.ptr(nk), _lib.cur_stream()))
    out = keep[: int(nk.item())].long()
    return (out, mat.view(n, n)) if return_matrix else out


def _tiled_mask_nms_sparse(predictions, idx, scores, nms_thresh: float, intersection_over_min: bool, areas, device=None):
    """Greedy mask NMS over tiled predictions WITHOUT the dense (N, H, W) canvas (util.py:1697-1770 compares overlap windows
    only): intersections are evaluated on the overlap window of the two global boxes, for box-overlapping pairs only -- pairs whose
    boxes are disjoint have IoU 0 and never suppress.  Same order and rule as `batched_mask_nms` (descending score, keep
    `iou <= thresh`).  Used when the canvas would not fit (`apply_nms`)."""
    n = len(idx)
    gb = np.array([predictions[k]["global_bbox"] for k in idx], dtype=np.int64)    # xywh, global
    lb = np.array([predictions[k]["bbox"] for k in idx], dtype=np.int64)           # xywh, tile-local
    x0, y0, x1, y1 = gb[:, 0], gb[:, 1], gb[:, 0] + gb[:, 2], gb[:, 1] + gb[:, 3]
    order = np.argsort(-np.asarray(scores, dtype=np.float64), kind="stable")
    masks = [torch.as_tensor(predictions[k]["segmentation"]).to(device).bool() if device is not None
             else torch.as_tensor(predictions[k]["segmentation"]).bool() for k in idx]
    a = np.asarray([float(areas[k]) for k in idx], dtype=np.float32)
    alive = np.ones(n, dtype=bool)
    keep = []
    for pos, i in enumerate(order):
        if not alive[i]:
            continue
        keep.append(int(i))
        rest = order[pos + 1:]
        rest = rest[alive[rest]]
        if len(rest) == 0:
            break
        ov = rest[(x0[rest] < x1[i]) & (x1[rest] > x0[i]) & (y0[rest] < y1[i]) & (y1[rest] > y0[i])]
        oi = (gb[i, 1] - lb[i, 1], gb[i, 0] - lb[i, 0])                                # global offset of tile-local (0, 0)
        for j in ov:
            wx0, wy0, wx1, wy1 = max(x0[i], x0[j]), max(y0[i], y0[j]), min(x1[i], x1[j]), min(y1[i], y1[j])
            oj = (gb[j, 1] - lb[j, 1], gb[j, 0] - lb[j, 0])
            mi = masks[i][wy0 - oi[0]:wy1 - oi[0], wx0 - oi[1]:wx1 - oi[1]]
            mj = masks[j][wy0 - oj[0]:wy1 - oj[0], wx0 - oj[1]:wx1 - oj[1]]
            inter = np.float32(int((mi & mj).sum()))
            den = np.float32(min(a[i], a[j])) if intersection_over_min else np.float32(a[i] + a[j] - inter)
            if den > 0 and np.float32(inter / den) > np.float32(nms_thresh):
                alive[j] = False
    return torch.as_tensor(keep, dtype=torch.long)


# dense canvases above this many bytes (N x H x W uint8) switch the tiled mask NMS to the box-overlap formulation
_DENSE_NMS_BYTES = 8 << 30


def apply_nms(predictions: List[Dict[str, Any]], min_size: int, shape: Optional[Tuple[int, int]] = None,
              perform_box_nms: bool = False, nms_thresh: float = 0.9, max_size: Optional[int] = None,
              intersection_over_min: bool = False) -> np.ndarray:
    """util.apply_nms (util.py:1851-1957).  Tiled predictions (records with a `global_bbox`, util.py:1687-1770) are placed
    at their global offset (global_bbox - bbox) on canvases of the full shape: masks are zero outside their boxes, so the
    intersection over the overlap window that the reference crops out equals the global intersection, and the same
    bit-packed mask-NMS kernel serves both cases."""
    is_tiled = len(predictions) > 0 and "global_bbox" in predictions[0]
    if is_tiled and shape is None:  # _infer_tiled_shape, util.py:1687-1695
        shape = [0, 0]
        for pred in predictions:
            bbox, gbb = pred["bbox"], pred["global_bbox"]
            ms = pred["segmentation"].shape
            shape[0] = max(shape[0], gbb[1] - bbox[1] + ms[0])
            shape[1] = max(shape[1], gbb[0] - bbox[0] + ms[1])
        shape = tuple(int(v) for v in shape)
    if shape is None:
        shape = tuple(predictions[0]["segmentation"].shape)
    dev = torch.device("cuda")
    if is_tiled and len(predictions) * int(shape[0]) * int(shape[1]) > _DENSE_NMS_BYTES and not perform_box_nms:
        # large tiled images: no (N, H, W) canvas / N x N matrix (1000 masks on 10k x 10k would need 100 GB)
        area_l = [int(np.asarray(p["segmentation"]).sum()) for p in predictions]
        idx_l = [k for k in range(len(predictions)) if area_l[k] > min_size and (max_size is None or area_l[k] < max_size)] \
            if min_size > 0 or max_size is not None else list(range(len(predictions)))
        if not idx_l:
            return np.zeros(shape, dtype="uint32")
        sc = [predictions[k]["predicted_iou"] * predictions[k]["stability_score"] for k in idx_l]
        keep = _tiled_mask_nms_sparse(predictions, idx_l, sc, nms_thresh, intersection_over_min, area_l, device=dev)
        mask_data = [{"segmentation": predictions[idx_l[k]]["segmentation"], "area": area_l[idx_l[k]], "bbox": list(predictions[idx_l[k]]["bbox"]),
                      "global_bbox": list(predictions[idx_l[k]]["global_bbox"])} for k in keep.tolist()]
        return mask_data_to_segmentation(mask_data, shape=shape, min_object_size=min_size)
    if is_tiled:
        masks = torch.zeros((len(predictions),) + tuple(shape), dtype=torch.uint8, device=dev)
        for k, pred in enumerate(predictions):
            m = torch.as_tensor(pred["segmentation"]).to(dev).to(torch.uint8)
            oy, ox = int(pred["global_bbox"][1] - pred["bbox"][1]), int(pred["global_bbox"][0] - pred["bbox"][0])
            y0, x0 = max(oy, 0), max(ox, 0)
            y1, x1 = min(oy + m.shape[0], shape[0]), min(ox + m.shape[1], shape[1])
            masks[k, y0:y1, x0:x1] = m[y0 - oy:y1 - oy, x0 - ox:x1 - ox]
    else:
        masks = torch.stack([torch.as_tensor(p["segmentation"]).to(dev) for p in predictions]).to(torch.uint8)
    iou = torch.tensor([p["predicted_iou"] for p in predictions], dtype=torch.float32)
    stab = torch.tensor([p["stability_score"] for p in predictions], dtype=torch.float32)
    local_boxes = torch.tensor(np.array([p["bbox"] for p in predictions]))
    boxes = torch.tensor(np.array([p["global_bbox"] for p in predictions])) if is_tiled else local_boxes
    area = masks.flatten(1).sum(1).cpu()
    idx = torch.arange(len(predictions))
    if min_size > 0:
        idx = idx[area[idx] > min_size]
    if max_size is not None:
        idx = idx[area[idx] < max_size]
    if len(idx) == 0:
        return np.zeros(shape, dtype="uint32")
    scores = (iou * stab)[idx]
    bxyxy = _xywh_to_xyxy(boxes[idx])
    if perform_box_nms:
        assert not intersection_over_min
        keep = torch.empty(len(idx), dtype=torch.int32, device=dev)
        nk = torch.zeros(1, dtype=torch.int32, device=dev)
        import ctypes
        z = (ctypes.c_int32 * 4)(0, 0, 0, 0)
        bi = bxyxy.to(dev, torch.int32).contiguous()
        sd = scores.to(dev).contiguous()
        _lib.check(_lib.lib().msam_amg_filter_nms(_lib.ptr(bi), _lib.ptr(sd), _lib.ptr(sd), len(idx), 0, 0.0, 0.0,
                                                  float(nms_thresh), z, z, _lib.ptr(keep), _lib.ptr(nk), _lib.cur_stream()))
        keep = keep[: int(nk.item())].long().cpu()
    else:
        keep = batched_mask_nms(masks[idx.to(dev)], bxyxy, scores, nms_thresh, intersection_over_min).cpu()
    sel = idx[keep]
    if is_tiled:
        mask_data = [{"segmentation": predictions[k]["segmentation"], "area": int(area[k]), "bbox": local_boxes[k].tolist(),
                      "global_bbox": boxes[k].tolist()} for k in sel.tolist()]
    else:
        mask_data = [{"segmentation": masks[k].bool(), "area": int(area[k]), "bbox": boxes[k]} for k in sel.tolist()]
    return mask_data_to_segmentation(mask_data, shape=shape, min_object_size=min_size)
