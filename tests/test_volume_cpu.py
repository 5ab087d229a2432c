"""CPU tests of segment_mask_in_volume's slice schedule (micro_sam_b200.multi_dimensional_segmentation._propagate) against a
restatement of the reference's loop (micro_sam/multi_dimensional_segmentation.py:105-233) with a recording stand-in predictor,
the projection modes, the CPU arithmetic the device prompt derivation reproduces (torch's antialiased resize, scipy's distance
field), and the fill-the-crop distance field."""
import numpy as np
import pytest
import torch
from scipy import ndimage

from micro_sam_b200 import multi_dimensional_segmentation as mds
from micro_sam_b200 import prompt_based_segmentation as pbs
from micro_sam_b200 import util
from micro_sam_b200.sam import ResizeLongestSide, get_preprocess_shape


class _Rec:
    """predict() records the mask prompt and returns a mask that depends on it and on the bound slice, with a score."""

    def __init__(self, shape, vanish=()):
        self.original_size = shape
        self.transform = ResizeLongestSide(1024)
        self.device = torch.device("cpu")
        self.is_image_set = True
        self.vanish, self.calls, self.z = set(vanish), [], None

    def predict(self, point_coords=None, point_labels=None, box=None, mask_input=None, multimask_output=True, return_logits=False):
        self.calls.append((self.z, None if mask_input is None else mask_input.copy(), None if box is None else np.array(box)))
        h, w = self.original_size
        m = np.zeros((1, h, w), bool)
        if box is not None:
            m[0, box[1] + 1:box[3] - 1, box[0]:box[2]] = True     # shrinks by one row per slice
        if self.z in self.vanish:
            m[:] = False
        return m, np.array([0.5], "float32"), np.zeros((1, 256, 256), "float32")


def _patch(monkeypatch, rec):
    def fake_set_precomputed(predictor, emb, i=None, tile_id=None):
        rec.z = i
    monkeypatch.setattr(pbs.util, "set_precomputed", fake_set_precomputed)


def _reference(segmentation, predictor, image_embeddings, segmented_slices, stop_lower, stop_upper, iou_threshold, projection,
               update_progress=None, box_extension=0.0, verbose=False):
    """Restatement of the reference's segment_mask_in_volume loop."""
    use_box, use_mask, use_points, use_single_point = mds._validate_projection(projection)
    update_progress = update_progress or (lambda *a: None)

    def segment_range(z_start, z_stop, increment, stopping_criterion, threshold=None):
        z = z_start + increment
        while True:
            if verbose:
                print(f"Segment {z_start} to {z_stop}: segmenting slice {z}")
            seg_prev = segmentation[z - increment]
            seg_z, score, _ = pbs.segment_from_mask(predictor, seg_prev, image_embeddings=image_embeddings, i=z, use_mask=use_mask,
                                                    use_box=use_box, use_points=use_points, box_extension=box_extension, return_all=True,
                                                    use_single_point=use_single_point)
            if threshold is not None:
                iou = util.compute_iou(seg_prev, seg_z)
                if iou < threshold:
                    if verbose:
                        print(f"Segmentation stopped at slice {z} due to IOU {iou} < {threshold}.")
                    break
            segmentation[z] = seg_z
            z += increment
            if stopping_criterion(z, z_stop):
                if verbose:
                    print(f"Segment {z_start} to {z_stop}: stop at slice {z}")
                break
            update_progress(1)
        return z - increment

    z0, z1 = int(segmented_slices.min()), int(segmented_slices.max())
    z_min = segment_range(z0, 0, -1, np.less, iou_threshold) if z0 > 0 and not stop_lower else z0
    z_max = segment_range(z1, segmentation.shape[0] - 1, 1, np.greater, iou_threshold) \
        if z1 < segmentation.shape[0] - 1 and not stop_upper else z1
    if z0 != z1:
        for z_start, z_stop in zip(segmented_slices[:-1], segmented_slices[1:]):
            slice_diff = z_stop - z_start
            z_mid = int((z_start + z_stop) // 2)
            if slice_diff == 1:
                pass
            elif z_start == z0 and stop_lower:
                segment_range(z_stop, z_start, -1, np.less_equal)
            elif z_stop == z1 and stop_upper:
                segment_range(z_start, z_stop, 1, np.greater_equal)
            elif slice_diff == 2:
                z = z_start + 1
                seg_prompt = np.logical_or(segmentation[z_start] == 1, segmentation[z_stop] == 1)
                segmentation[z] = pbs.segment_from_mask(predictor, seg_prompt, image_embeddings=image_embeddings, i=z, use_mask=use_mask,
                                                        use_box=use_box, use_points=use_points, box_extension=box_extension)
                update_progress(1)
            else:
                segment_range(z_start, z_mid, 1, np.greater_equal if slice_diff % 2 == 0 else np.greater)
                segment_range(z_stop, z_mid, -1, np.less_equal)
                if slice_diff % 2 == 0:
                    seg_prompt = np.logical_or(segmentation[z_mid - 1] == 1, segmentation[z_mid + 1] == 1)
                    segmentation[z_mid] = pbs.segment_from_mask(predictor, seg_prompt, image_embeddings=image_embeddings, i=z_mid,
                                                                use_mask=use_mask, use_box=use_box, use_points=use_points,
                                                                box_extension=box_extension)
                    update_progress(1)
    return segmentation, (z_min, z_max)


def _seeded(Z, slices, shape=(40, 48)):
    seg = np.zeros((Z,) + shape, np.uint16)
    for k in slices:
        seg[k, 5:35, 4 + k % 5:40] = 1
    return seg


CASES = [
    (9, [4]), (9, [0]), (9, [8]), (9, [3, 4]), (12, [3, 5]), (12, [3, 6]), (12, [3, 7]), (14, [2, 6, 11]),
]


@pytest.mark.parametrize("Z,slices", CASES)
@pytest.mark.parametrize("stop_lower,stop_upper", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("thr", [0.0, 0.9])
def test_schedule_matches_reference(monkeypatch, capsys, Z, slices, stop_lower, stop_upper, thr):
    slices = np.array(slices)
    out = {}
    for name, fn in (("ref", _reference), ("lib", mds._segment_mask_in_volume_host)):
        rec = _Rec((40, 48), vanish={1})
        _patch(monkeypatch, rec)
        seg = _seeded(Z, slices)
        n = [0]
        res = fn(seg, rec, {"features": None, "input_size": (1, 1), "original_size": (40, 48)}, slices, stop_lower, stop_upper, thr, "mask",
                 lambda k: n.__setitem__(0, n[0] + k), 0.0, True)
        out[name] = (res[0], res[1], n[0], rec.calls, capsys.readouterr().out)
    r, l = out["ref"], out["lib"]
    assert np.array_equal(r[0], l[0]) and r[1] == l[1] and r[2] == l[2] and r[4] == l[4]
    assert [c[0] for c in r[3]] == [c[0] for c in l[3]]
    for a, b in zip(r[3], l[3]):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


class _RecPoints(_Rec):
    """Records the point prompts; the mask is a disk around the positive points."""

    def predict(self, point_coords=None, point_labels=None, box=None, mask_input=None, multimask_output=True, return_logits=False):
        self.calls.append((self.z, None if point_coords is None else np.array(point_coords),
                           None if point_labels is None else np.array(point_labels)))
        h, w = self.original_size
        m = np.zeros((1, h, w), bool)
        if point_coords is not None:
            pos = np.asarray(point_coords)[np.asarray(point_labels) == 1].astype(int)
            if len(pos):
                cx, cy = pos.mean(0)
                yy, xx = np.mgrid[:h, :w]
                m[0] = (yy - cy) ** 2 + (xx - cx) ** 2 < (8 + 2 * (self.z % 3)) ** 2
        return m, np.array([0.5], "float32"), np.zeros((1, 256, 256), "float32")


@pytest.mark.parametrize("proj", ["single_point", "points"])
@pytest.mark.parametrize("slices", [[2, 4, 8], [1, 3, 7, 9]])
def test_middle_slices_use_multi_point_prompts(monkeypatch, proj, slices):
    """The middle slices of gaps of 2 and of even gaps are prompted with the union of both neighbours through segment_from_mask
    WITHOUT use_single_point (:206-230), so "single_point" derives multiple points there."""
    slices = np.array(slices)
    out = {}
    for name, fn in (("ref", _reference), ("lib", mds._segment_mask_in_volume_host)):
        rec = _RecPoints((40, 48))
        _patch(monkeypatch, rec)
        seg = np.zeros((11, 40, 48), np.uint16)
        yy, xx = np.mgrid[:40, :48]
        for k in slices:
            seg[k][(yy - 20) ** 2 + (xx - 18 - k) ** 2 < (6 + k) ** 2] = 1
        res = fn(seg, rec, {"features": None, "input_size": (1, 1), "original_size": (40, 48)}, slices, False, False, 0.0, proj)
        out[name] = (res[0], res[1], rec.calls)
    r, l = out["ref"], out["lib"]
    assert np.array_equal(r[0], l[0]) and r[1] == l[1]
    assert [c[0] for c in r[2]] == [c[0] for c in l[2]]
    for a, b in zip(r[2], l[2]):
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), a[0]
    middles = [int(a + b) // 2 for a, b in zip(slices[:-1], slices[1:]) if (b - a) % 2 == 0]
    n_pts = {c[0]: len(c[1]) for c in r[2] if c[1] is not None}
    assert all(n_pts[z] > 1 for z in middles)                   # several points on the middle slices
    if proj == "single_point":
        assert all(n == 1 for z, n in n_pts.items() if z not in middles)


def test_threshold_stops_early(monkeypatch):
    rec = _Rec((40, 48))
    _patch(monkeypatch, rec)
    seg = _seeded(20, [10])
    _, (z0, z1) = mds._segment_mask_in_volume_host(seg, rec, {"features": None, "input_size": (1, 1), "original_size": (40, 48)}, np.array([10]), False, False,
                                                   0.9, "box")
    assert 0 < z0 < 10 < z1 < 19          # the mask shrinks by two rows per slice: IoU falls below 0.9 after six slices


@pytest.mark.parametrize("proj", list(mds.PROJECTION_MODES) + [{"use_box": True, "use_mask": False, "use_points": True}])
def test_projection_modes(monkeypatch, proj):
    rec = _Rec((40, 48))
    _patch(monkeypatch, rec)
    seg_r, seg_l = _seeded(7, [3]), _seeded(7, [3])
    emb = {"features": None, "input_size": (1, 1), "original_size": (40, 48)}
    calls = []
    for fn, seg in ((_reference, seg_r), (mds._segment_mask_in_volume_host, seg_l)):
        rec.calls = []
        assert fn(seg, rec, emb, np.array([3]), False, False, 0.0, proj)[1] == (0, 6)
        calls.append(rec.calls)
    assert np.array_equal(seg_r, seg_l) and len(calls[0]) == len(calls[1]) == 6


def test_invalid_projection():
    with pytest.raises(ValueError, match="invalid option"):
        mds._validate_projection("boxes")
    with pytest.raises(ValueError):
        mds._validate_projection(3)
    with pytest.raises(AssertionError):
        mds._validate_projection({"use_box": True})
    assert mds._validate_projection("single_point") == (False, False, True, True)


def test_compute_iou():
    a = np.zeros((4, 4), np.uint8); a[:2] = 1
    b = np.zeros((4, 4), bool); b[1:3] = True
    assert util.compute_iou(a, b) == 4 / (12 + 1e-7)
    assert util.compute_iou(np.zeros(3), np.zeros(3)) == 0.0


# ------------------------------------------------------------------------------------------------ the arithmetic csrc/volume.cu reproduces
def _aa_weights(insz, outsz):
    f32 = np.float32
    scale = f32(f32(insz) / f32(outsz))
    support = scale if scale >= 1 else f32(1.0)
    maxsz = int(np.ceil(support)) * 2 + 1
    invscale = f32(1.0 / np.float64(scale)) if scale >= 1 else f32(1.0)
    out = []
    for i in range(outsz):
        center = f32(np.float64(scale) * (i + 0.5))
        xmin = max(int(np.float64(f32(center - support)) + 0.5), 0)
        xsize = min(max(min(int(np.float64(f32(center + support)) + 0.5), insz) - xmin, 0), maxsz)
        w = []
        for j in range(xsize):
            x = abs(f32((np.float64(f32(f32(j + xmin) - center)) + 0.5) * np.float64(invscale)))
            w.append(f32(1.0 - np.float64(x)) if x < 1 else f32(0))
        tot = f32(0)
        for v in w:
            tot = f32(tot + v)
        out.append((xmin, [f32(v / tot) for v in w] if tot != 0 else w))
    return out


def _resize_like_volume_cu(m):
    """The logits kernels' arithmetic: horizontal pass on the 0/1 mask, then the vertical pass adding taps 1 .. 4q unfused and
    the remaining (n - 1) % 4 with one rounding each (FMA)."""
    H, W = m.shape
    th, tw = get_preprocess_shape(H, W, 256)
    x = m.astype(np.float32)
    if tw != W:
        t = np.zeros((H, tw), np.float32)
        for ox, (x0, w) in enumerate(_aa_weights(W, tw)):
            acc = (x[:, x0] * w[0]).astype(np.float32)
            for j in range(1, len(w)):
                acc = (acc + (x[:, x0 + j] * w[j]).astype(np.float32)).astype(np.float32)
            t[:, ox] = acc
        x = t
    if th != H:
        t = np.zeros((th, x.shape[1]), np.float32)
        for oy, (y0, w) in enumerate(_aa_weights(H, th)):
            n = len(w)
            unfused = ((n - 1) // 4) * 4
            acc = (x[y0] * w[0]).astype(np.float32)
            for j in range(1, n):
                if j - 1 < unfused:
                    acc = (acc + (x[y0 + j] * w[j]).astype(np.float32)).astype(np.float32)
                else:   # a*b is exact in fp64, so one fp64 add rounded to fp32 is the FMA up to double rounding (pinned below)
                    acc = (x[y0 + j].astype(np.float64) * np.float64(w[j]) + acc.astype(np.float64)).astype(np.float32)
            t[oy] = acc
        x = t
    return x


@pytest.mark.parametrize("shape", [(300, 77), (100, 140), (700, 1000), (257, 1023), (256, 100)])
def test_resize_arithmetic_matches_torch(shape):
    rng = np.random.default_rng(sum(shape))
    m = (rng.random(shape) < 0.5).astype(np.float32)
    th, tw = get_preprocess_shape(*shape, 256)
    ref = torch.nn.functional.interpolate(torch.from_numpy(m)[None, None], (th, tw), mode="bilinear", align_corners=False,
                                          antialias=True).numpy()[0, 0]
    if torch.backends.cpu.get_cpu_capability() != "AVX512":
        pytest.skip("the vertical pass's accumulation was pinned on torch's AVX512 kernels")
    assert np.array_equal(_resize_like_volume_cu(m).view(np.uint32), ref.view(np.uint32))


def test_fill_the_crop_distance_field_is_pinned():
    """No boundary pixel in the crop: scipy measures to the virtual feature (-1, 0)."""
    d = ndimage.distance_transform_edt(np.ones((3, 4), bool))
    yy, xx = np.mgrid[:3, :4]
    assert np.array_equal(d, np.sqrt((yy + 1.0) ** 2 + xx ** 2))
    m = np.zeros((12, 14), np.uint8)
    m[2:9, 3:11] = 1
    pts, lbl = pbs._compute_points_from_mask(m, None, 0, use_single_point=True)
    f = ndimage.gaussian_filter(np.sqrt((np.mgrid[:7, :8][0] + 1.0) ** 2 + np.mgrid[:7, :8][1] ** 2).astype("float32"), sigma=1.0)
    y, x = np.unravel_index(f.argmax(), f.shape)
    assert np.array_equal(pts, [[x + 3, y + 2]]) and lbl.tolist() == [1]
