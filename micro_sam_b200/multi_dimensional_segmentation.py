"""micro-sam's `segment_mask_in_volume` (micro_sam/multi_dimensional_segmentation.py:45-233): carry an object segmented in one
or a few slices through a volume of precomputed 3-D embeddings, slice by slice, each slice prompted with the mask of its
neighbour.

The slice schedule (`_propagate`) is a plain Python driver.  Each slice step runs on the device (`_DeviceStep`): the
previous mask stays in a device uint8 working volume, csrc/volume.cu derives its box / points / mask-prompt logits there,
one decoder pass and the upsampling write the next slice, and the IoU with the previous slice is counted on the device.  At
most one small device-to-host copy is made per slice (the prompt statistics and IoU counts); tiled embeddings need a second
one, for the statistics of the tile the mask is routed to.  Only the slices the call writes are copied back into the
caller's array, once, at the end.  `_HostStep` is the same step through the host glue of `segment_from_mask`.

The tracking annotator's `track_from_prompts` (micro_sam/sam_annotator/util.py:561-675) runs the same step frame by frame
(`_track`), each frame prompted with the previous one shifted by a motion model: csrc/volume.cu's msam_shift_mask shifts the
device plane, and the centroids behind the model come from the count and coordinate sums the step reads back anyway: two
small reads per frame (the shifted plane's prompts, then the IoU counts with the new frame's sums), one more when tiled.

Out of scope: merge_instance_segmentation_3d / automatic_3d_segmentation (multicut), automatic tracking (trackastra), the
evaluation wrapper and the unused _advanced_stopping_criteria (DESIGN.md §7).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple, Union

import numpy as np
import torch
from scipy import ndimage

from . import _lib, util
from .prompt_based_segmentation import _tile_of, segment_from_mask

PROJECTION_MODES = ("box", "mask", "points", "points_and_mask", "single_point")

_MAX_POINTS = 64   # point buffer of the device step; more than 16 tokens per prompt is refused by the decoder anyway


def _validate_projection(projection):
    """projection mode -> (use_box, use_mask, use_points, use_single_point) (:48-72)."""
    modes = {"mask": (True, True, False, False), "points": (False, False, True, False), "box": (True, False, False, False),
             "points_and_mask": (False, True, True, False), "single_point": (False, False, True, True)}
    if isinstance(projection, str):
        if projection not in modes:
            raise ValueError("Choose projection method from 'mask' / 'points' / 'box' / 'points_and_mask' / 'single_point'. "
                             f"You have passed the invalid option {projection}.")
        return modes[projection]
    if isinstance(projection, dict):
        assert len(projection.keys()) == 3, "There should be three parameters assigned for the projection method."
        return projection["use_box"], projection["use_mask"], projection["use_points"], False
    raise ValueError(f"{projection} is not a supported projection method.")


def _propagate(n_slices, segmented_slices, stop_lower, stop_upper, iou_threshold, step, update_progress, verbose):
    """The slice schedule of segment_mask_in_volume (:145-233).  `step.segment(z, prev, threshold)` segments slice z from
    slice prev and writes it unless its IoU with prev is below `threshold` (returns (written, iou)); `step.segment_pair(z, a,
    b)` segments z from the union of slices a and b and writes it."""
    def segment_range(z_start, z_stop, increment, stop, threshold=None):
        z = z_start + increment
        while True:
            if verbose:
                print(f"Segment {z_start} to {z_stop}: segmenting slice {z}")
            written, iou = step.segment(z, z - increment, threshold)
            if not written:
                if verbose:
                    print(f"Segmentation stopped at slice {z} due to IOU {iou} < {threshold}.")
                break
            z += increment
            if stop(z, z_stop):
                if verbose:
                    print(f"Segment {z_start} to {z_stop}: stop at slice {z}")
                break
            update_progress(1)
        return z - increment

    z0, z1 = int(segmented_slices.min()), int(segmented_slices.max())
    z_min = segment_range(z0, 0, -1, np.less, iou_threshold) if z0 > 0 and not stop_lower else z0
    z_max = segment_range(z1, n_slices - 1, 1, np.greater, iou_threshold) if z1 < n_slices - 1 and not stop_upper else z1
    if z0 != z1:
        for z_start, z_stop in zip(segmented_slices[:-1], segmented_slices[1:]):
            diff, z_mid = z_stop - z_start, int((z_start + z_stop) // 2)
            if diff == 1:
                continue
            if z_start == z0 and stop_lower:
                segment_range(z_stop, z_start, -1, np.less_equal)
            elif z_stop == z1 and stop_upper:
                segment_range(z_start, z_stop, 1, np.greater_equal)
            elif diff == 2:
                step.segment_pair(z_start + 1, z_start, z_stop)
                update_progress(1)
            else:
                segment_range(z_start, z_mid, 1, np.greater_equal if diff % 2 == 0 else np.greater)
                segment_range(z_stop, z_mid, -1, np.less_equal)
                if diff % 2 == 0:   # the middle slice is as far from both ends: prompt it with both neighbours
                    step.segment_pair(z_mid, z_mid - 1, z_mid + 1)
                    update_progress(1)
    return z_min, z_max


class _HostStep:
    """The slice step through segment_from_mask's host glue, writing the caller's array directly."""

    def __init__(self, segmentation, predictor, image_embeddings, projection, box_extension):
        self.seg, self.predictor, self.emb, self.box_extension = segmentation, predictor, image_embeddings, box_extension
        self.use_box, self.use_mask, self.use_points, self.use_single_point = _validate_projection(projection)

    def segment(self, z, prev, threshold):
        seg_prev = self.seg[prev]
        seg_z = segment_from_mask(self.predictor, seg_prev, image_embeddings=self.emb, i=z, use_mask=self.use_mask, use_box=self.use_box,
                                  use_points=self.use_points, box_extension=self.box_extension, return_all=True,
                                  use_single_point=self.use_single_point)[0]
        if threshold is not None:
            iou = util.compute_iou(seg_prev, seg_z)
            if iou < threshold:
                return False, iou
        self.seg[z] = seg_z
        return True, None

    def segment_pair(self, z, a, b):
        # upstream prompts the middle slices without use_single_point: "single_point" derives multiple points here
        self.seg[z] = segment_from_mask(self.predictor, np.logical_or(self.seg[a] == 1, self.seg[b] == 1), image_embeddings=self.emb, i=z,
                                        use_mask=self.use_mask, use_box=self.use_box, use_points=self.use_points,
                                        box_extension=self.box_extension)

    def centroid(self, t):
        """_compute_movement's centre of frame t (sam_annotator/util.py:561-573): NaN for an empty frame."""
        ys, xs = np.where(self.seg[t] == 1)
        return np.array([np.mean(ys), np.mean(xs)])

    def track(self, t, motion, threshold):
        """Frame t from frame t - 1 shifted by `motion` (None: unshifted), as track_from_prompts does
        (sam_annotator/util.py:627-664); returns (written, iou)."""
        seg_prev = self.seg[t - 1]
        if motion is not None:   # _shift_object (:576-579)
            shifted = np.zeros_like(seg_prev)
            ndimage.shift(seg_prev, motion, output=shifted, order=0, prefilter=False)
            seg_prev = shifted
        seg_t = segment_from_mask(self.predictor, seg_prev, image_embeddings=self.emb, i=t, use_mask=self.use_mask, use_box=self.use_box,
                                  use_points=self.use_points, box_extension=self.box_extension, return_all=True,
                                  use_single_point=self.use_single_point)[0]
        if threshold is not None:
            iou = util.compute_iou(seg_prev, seg_t)
            if iou < threshold:
                return False, iou
        self.seg[t] = seg_t
        return True, None

    def finish(self):
        pass


class _DeviceStep:
    """The slice step on the device: prompts from the previous slice's device mask (msam_mask_prompts), one decoder pass
    (msam_decode_ex, or msam_mask_decode with no prompt at all), the upsampled binary mask into the working volume
    (msam_upsample_masks), the IoU counts with the previous slice (msam_mask_iou_counts).  For tracking, `track` prompts the
    frame from the previous one shifted by the motion model (msam_shift_mask) and keeps each frame's count and coordinate sums
    for the centroids."""

    def __init__(self, segmentation, predictor, image_embeddings, projection, box_extension, segmented_slices,
                 name="segment_mask_in_volume"):
        self.name = name   # the public function named in error messages
        use_box, use_mask, use_points, single = _validate_projection(projection)
        self.use_box, self.use_mask = bool(use_box), bool(use_mask)
        self.point_mode = (1 if single else 2) if use_points else 0   # slice steps of the ranges
        self.pair_point_mode = 2 if use_points else 0                  # the middle slices prompted by two neighbours (:206-230)
        self.seg, self.predictor, self.emb, self.box_extension = segmentation, predictor, image_embeddings, float(box_extension)
        dev = predictor.device
        Z, H, W = segmentation.shape
        self.H, self.W = H, W
        self.vol = torch.zeros(Z, H, W, dtype=torch.uint8, device=dev)
        seeds = np.unique(np.asarray(segmented_slices).astype(int))
        self.vol[torch.as_tensor(seeds, device=dev)] = torch.from_numpy(np.ascontiguousarray(segmentation[seeds] == 1)).to(dev, torch.uint8)
        self.pair = torch.zeros(H, W, dtype=torch.uint8, device=dev)
        L = _lib.lib()
        self.ws = torch.empty(int(L.msam_mask_prompts_workspace(H, W)), dtype=torch.uint8, device=dev)
        self.stats = torch.zeros(16, dtype=torch.int64, device=dev)   # [0:12] prompt stats, [12:14] IoU counts
        self.host = torch.zeros(16, dtype=torch.int64).pin_memory()
        self.box = torch.zeros(1, 4, dtype=torch.float32, device=dev)
        self.logits = torch.zeros(1, 256, 256, dtype=torch.float32, device=dev)
        self.points = torch.zeros(1, _MAX_POINTS, 2, dtype=torch.float32, device=dev)
        self.labels = torch.zeros(1, _MAX_POINTS, dtype=torch.float32, device=dev)
        self.low = torch.empty(1, 1, 256, 256, dtype=torch.float32, device=dev)
        self.iou_pred = torch.empty(1, 1, dtype=torch.float32, device=dev)
        self.tiled = image_embeddings is not None and image_embeddings["input_size"] is None
        self.written = set()
        self.ready = None   # slice whose prompts (or, tiled, whose full-frame statistics) are in the buffers and self.host
        self.shifted = None   # tracking: the previous frame shifted by the motion model
        self.sums = {}        # tracking: frame -> (count, sum_y, sum_x) of its pixels == 1

    def _read(self):
        self.host.copy_(self.stats)   # synchronising copy of the 16 stats words
        return self.host.numpy()

    def _derive(self, mask, h, w, ld, point_mode, logits):
        # `mask` may be a tile's view into the frame (row pitch ld), so its address is passed without the contiguity check
        _lib.check(_lib.lib().msam_mask_prompts(ctypes.c_void_p(mask.data_ptr()), h, w, ld, self.box_extension, int(logits), point_mode, _MAX_POINTS,
                                                _lib.ptr(self.ws), self.ws.numel(), _lib.ptr(self.stats), _lib.ptr(self.box),
                                                _lib.ptr(self.logits) if logits else None, _lib.ptr(self.points),
                                                _lib.ptr(self.labels), None, _lib.cur_stream()))

    def _prepare(self, mask, point_mode):
        """Prompts of `mask` (a device [H, W] uint8 plane) in the buffers; returns (stats, tile or None)."""
        if not self.tiled:
            self._derive(mask, self.H, self.W, self.W, point_mode, self.use_mask)
            return self._read(), None
        if self.ready is None:
            self._derive(mask, self.H, self.W, self.W, 0, False)
            self._read()
        st = self.host.numpy()
        if st[0] == 0:
            raise RuntimeError(f"{self.name}: an empty mask cannot be routed to a tile of tiled embeddings")
        attrs = self.emb["features"].attrs
        tile_id, tile = _tile_of([st[1] / st[0], st[2] / st[0]], tuple(attrs["shape"]), tuple(attrs["tile_shape"]), tuple(attrs["halo"]))
        view = mask[tile.begin[0]:tile.end[0], tile.begin[1]:tile.end[1]]
        self._derive(view, view.shape[0], view.shape[1], self.W, point_mode, self.use_mask)
        return self._read(), (tile_id, tile)   # the tile's own count decides whether a box and points are passed

    def _decode(self, z, st, tile, out, point_mode):
        if tile is None:
            util.set_precomputed(self.predictor, self.emb, z)
        else:
            util.set_precomputed(self.predictor, self.emb, z, tile_id=tile[0])
        p = self.predictor
        p._bind_features()
        nonempty = st[0] != 0
        n_pts = int(st[11]) if (point_mode and nonempty) else 0
        if n_pts < 0 or n_pts > _MAX_POINTS:
            raise RuntimeError(f"{self.name}: {n_pts} point prompts, more tokens per prompt than the decoder takes")
        box = self.box if (self.use_box and nonempty) else None
        logits = self.logits if self.use_mask else None
        L, h = _lib.lib(), p.model._h
        if n_pts == 0 and box is None and logits is None:   # no prompt left: decode the output tokens alone, as upstream does
            _lib.check(L.msam_mask_decode(h, None, 0, None, 1, 0, _lib.ptr(self.low), _lib.ptr(self.iou_pred), _lib.cur_stream()))
        else:
            pts = self.points[:, :n_pts].contiguous() if n_pts else None
            lbl = self.labels[:, :n_pts].contiguous() if n_pts else None
            _lib.check(L.msam_decode_ex(h, _lib.ptr(pts), _lib.ptr(lbl), n_pts, _lib.ptr(box), _lib.ptr(logits), 1, 0,
                                        _lib.ptr(self.low), _lib.ptr(self.iou_pred), _lib.cur_stream()))
        oh, ow = p.original_size
        target = out if tile is None else torch.empty(oh, ow, dtype=torch.uint8, device=out.device)
        _lib.check(L.msam_upsample_masks(_lib.ptr(self.low), None, 1, int(p.input_size[0]), int(p.input_size[1]), int(oh), int(ow),
                                         p.model.mask_threshold, None, _lib.ptr(target), _lib.cur_stream()))
        if tile is not None:
            t = tile[1]
            out.zero_()
            out[t.begin[0]:t.end[0], t.begin[1]:t.end[1]] = target

    def _after(self, z, prev_plane, threshold, prompts=True):
        """IoU counts of (prev_plane, slice z) and the statistics of slice z -- with its prompts for the next step unless tiled or
        not `prompts` -- read back together."""
        if threshold is not None:
            _lib.check(_lib.lib().msam_mask_iou_counts(_lib.ptr(prev_plane), self.W, _lib.ptr(self.vol[z]), self.W, self.H, self.W,
                                                       _lib.ptr(self.stats[12:]), _lib.cur_stream()))
        if self.tiled or not prompts:
            self._derive(self.vol[z], self.H, self.W, self.W, 0, False)
        else:
            self._derive(self.vol[z], self.H, self.W, self.W, self.point_mode, self.use_mask)
        return self._read()

    def segment(self, z, prev, threshold):
        if self.ready == prev:
            st, tile = (self.host.numpy(), None) if not self.tiled else self._prepare(self.vol[prev], self.point_mode)
        else:
            self.ready = None
            st, tile = self._prepare(self.vol[prev], self.point_mode)
        self._decode(z, st, tile, self.vol[z], self.point_mode)
        st = self._after(z, self.vol[prev], threshold)
        self.ready = z
        if threshold is not None:
            iou = float(st[12]) / (float(st[13]) + 1e-7)
            if iou < threshold:
                self.ready = None
                return False, iou
        self.written.add(z)
        return True, None

    def segment_pair(self, z, a, b):
        self.pair.copy_((self.vol[a] == 1) | (self.vol[b] == 1))
        self.ready = None
        st, tile = self._prepare(self.pair, self.pair_point_mode)
        self._decode(z, st, tile, self.vol[z], self.pair_point_mode)
        self.written.add(z)

    def centroid(self, t):
        """The centre of frame t from its count and coordinate sums; a frame the step has not segmented (a prompt frame) is
        counted once, on the device."""
        if t not in self.sums:
            self._derive(self.vol[t], self.H, self.W, self.W, 0, False)
            st = self._read()
            self.sums[t] = (int(st[0]), int(st[1]), int(st[2]))
        return _centroid(*self.sums[t])

    def track(self, t, motion, threshold):
        """Frame t from frame t - 1 shifted by `motion` (None: unshifted): the shifted plane is materialised once, prompts are
        derived from it (tiled embeddings route by its centroid), and the IoU is counted against it.  Two stats reads (one
        more when tiled): the prompts, then the IoU counts with frame t's sums."""
        plane = self.vol[t - 1]
        if motion is not None:
            if self.shifted is None:
                self.shifted = torch.empty(self.H, self.W, dtype=torch.uint8, device=self.vol.device)
            _lib.check(_lib.lib().msam_shift_mask(_lib.ptr(plane), self.W, _lib.ptr(self.shifted), self.W, self.H, self.W,
                                                  float(motion[0]), float(motion[1]), _lib.cur_stream()))
            plane = self.shifted
        self.ready = None   # the buffers hold the shifted plane's prompts, then frame t's statistics alone
        st, tile = self._prepare(plane, self.point_mode)
        self._decode(t, st, tile, self.vol[t], self.point_mode)
        st = self._after(t, plane, threshold, prompts=False)
        self.sums[t] = (int(st[0]), int(st[1]), int(st[2]))
        if threshold is not None:
            iou = float(st[12]) / (float(st[13]) + 1e-7)
            if iou < threshold:
                return False, iou
        self.written.add(t)
        return True, None

    def finish(self):
        if self.written:
            idx = sorted(self.written)
            self.seg[idx] = self.vol[torch.as_tensor(idx, device=self.vol.device)].cpu().numpy()


def _run(step, segmentation, segmented_slices, stop_lower, stop_upper, iou_threshold, update_progress, verbose):
    if update_progress is None:
        def update_progress(*args):
            pass
    z_range = _propagate(segmentation.shape[0], segmented_slices, stop_lower, stop_upper, iou_threshold, step, update_progress, verbose)
    step.finish()
    return segmentation, z_range


def segment_mask_in_volume(segmentation: np.ndarray, predictor, image_embeddings: util.ImageEmbeddings, segmented_slices: np.ndarray,
                           stop_lower: bool, stop_upper: bool, iou_threshold: float, projection: Union[str, dict],
                           update_progress: Optional[callable] = None, box_extension: float = 0.0,
                           verbose: bool = False) -> Tuple[np.ndarray, Tuple[int, int]]:
    """Segment an object through a volume (:105-233).  `segmentation` [Z, H, W] holds the object (== 1) in
    `segmented_slices` and is written in place on the slices this call segments; returns (segmentation, (z_min, z_max)).
    `image_embeddings` are 3-D embeddings (in memory, zarr or tiled) from `util.precompute_image_embeddings(..., ndim=3)`."""
    step = _DeviceStep(segmentation, predictor, image_embeddings, projection, box_extension, segmented_slices)
    return _run(step, segmentation, segmented_slices, stop_lower, stop_upper, iou_threshold, update_progress, verbose)


def _segment_mask_in_volume_host(segmentation, predictor, image_embeddings, segmented_slices, stop_lower, stop_upper, iou_threshold,
                                 projection, update_progress=None, box_extension=0.0, verbose=False):
    """The same schedule with every slice step through segment_from_mask's host glue (the parity oracle of the device step)."""
    step = _HostStep(segmentation, predictor, image_embeddings, projection, box_extension)
    return _run(step, segmentation, segmented_slices, stop_lower, stop_upper, iou_threshold, update_progress, verbose)


# ------------------------------------------------------------------------------------------------ tracking
def _centroid(count, sum_y, sum_x):
    """(mean row, mean col) in fp64 from a frame's pixel count and coordinate sums.  np.mean of np.where's indices sums them
    exactly (integers below 2**53) and divides once, so this is bit-equal to _compute_movement's centre; an empty frame gives
    NaN, as np.mean of nothing does."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.array([np.float64(sum_y) / np.float64(count), np.float64(sum_x) / np.float64(count)])


def prompt_layer_to_state(prompt_layer, i: int) -> str:
    """The track state of frame i (sam_annotator/util.py:280-305): "division" if any point of that frame has the state
    "division", else "track".  `prompt_layer` needs `.data` (N, 3) with the frame in column 0 and `.properties["state"]` (N,);
    a napari Points layer has both."""
    state = np.asarray(prompt_layer.properties["state"])
    points = np.asarray(prompt_layer.data)
    assert points.shape[1] == 3 and len(points) == len(state), f"{points.shape}, {len(state)} states"
    return "division" if any(st == "division" for st in state[points[:, 0] == i]) else "track"


def _track(seg, slices, point_prompts, stop_upper, threshold, motion_smoothing, step, update_progress):
    """The frame schedule of track_from_prompts (sam_annotator/util.py:582-675).  `step.centroid(t)` is frame t's centre,
    `step.track(t, motion, threshold)` segments frame t from frame t - 1 shifted by `motion` and writes it unless its IoU with
    that shifted plane is below `threshold` (returns (written, iou))."""
    if update_progress is None:
        def update_progress(*args):
            pass
    t0 = int(slices.min())
    if t0 + 1 >= seg.shape[0]:
        raise ValueError(f"track_from_prompts: the first prompt frame {t0} is the last of {seg.shape[0]} frames; there is nothing to track")
    motion_model, has_division = None, False
    t = t0 + 1
    while True:
        if t == t0 + 2:     # _update_motion_model: the first move initialises the model, later moves are averaged in
            motion_model = step.centroid(t - 1) - step.centroid(t - 2)
        elif t > t0 + 2:
            motion_model = motion_smoothing * motion_model + (1 - motion_smoothing) * (step.centroid(t - 1) - step.centroid(t - 2))
        if t in slices:     # a prompt frame keeps its segmentation; there is no IoU check
            if prompt_layer_to_state(point_prompts, t) == "division":
                has_division = True
                break
        else:
            # the IoU is only checked beyond the last prompt frame: before it the track must connect to a later frame
            written, iou = step.track(t, motion_model, threshold if t >= slices[-1] else None)
            update_progress(1)
            if not written:
                print(f"Segmentation stopped at frame {t} due to IOU {iou} < {threshold}.")
                break
        t += 1
        if t == slices[-1] and stop_upper:
            break
        if t == seg.shape[0]:
            break
    step.finish()
    return seg, has_division


def track_from_prompts(point_prompts, box_prompts, seg: np.ndarray, predictor, slices: np.ndarray,
                       image_embeddings: util.ImageEmbeddings, stop_upper: bool, threshold: Optional[float], projection: Union[str, dict],
                       motion_smoothing: float = 0.5, box_extension: float = 0,
                       update_progress: Optional[callable] = None) -> Tuple[np.ndarray, bool]:
    """Track an object through a timeseries (sam_annotator/util.py:582-675), the tracking annotator's "Track Object".

    `seg` [T, H, W] holds the object (== 1, background 0) in the prompt frames `slices` (sorted) and is written in place on the
    frames this call segments.  From the first prompt frame on, each other frame is segmented from the previous one, shifted by
    a motion model: the exponential moving average, with weight `motion_smoothing` on the old value, of the centroid's move
    between the two frames before.  Beyond the last prompt frame a frame whose IoU with that shifted mask is below `threshold`
    (None: no check) stops the track unwritten.  A prompt frame whose points in `point_prompts` include the state "division"
    stops it too; `stop_upper` stops it at the last prompt frame.  `point_prompts` needs `.data` (N, 3) and
    `.properties["state"]`; `box_prompts` is not read, as upstream.  `image_embeddings` are 3-D embeddings (in memory, zarr or
    tiled) of the timeseries.  Returns (seg, has_division)."""
    slices = np.asarray(slices)
    step = _DeviceStep(seg, predictor, image_embeddings, projection, box_extension, slices, name="track_from_prompts")
    return _track(seg, slices, point_prompts, stop_upper, threshold, motion_smoothing, step, update_progress)


def _track_from_prompts_host(point_prompts, box_prompts, seg, predictor, slices, image_embeddings, stop_upper, threshold, projection,
                             motion_smoothing=0.5, box_extension=0, update_progress=None):
    """The same schedule with every frame through scipy.ndimage.shift and segment_from_mask's host glue (the parity oracle of the
    device step)."""
    slices = np.asarray(slices)
    step = _HostStep(seg, predictor, image_embeddings, projection, box_extension)
    return _track(seg, slices, point_prompts, stop_upper, threshold, motion_smoothing, step, update_progress)
