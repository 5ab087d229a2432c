"""CPU tests of track_from_prompts (micro_sam_b200.multi_dimensional_segmentation): the index rule msam_shift_mask implements
against scipy.ndimage.shift(order=0, prefilter=False); the centre formed from counts and coordinate sums against np.mean; the
frame schedule `_track`, driven by a host stand-in step, against a restatement of the reference's loop
(micro_sam/sam_annotator/util.py:561-675) -- motion values bit for bit, division stops, stop_upper, the IoU checked only from
the last prompt frame on, progress calls and the return value; and `_track_from_prompts_host` through segment_from_mask with
a stand-in predictor."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import ndimage

from micro_sam_b200 import multi_dimensional_segmentation as mds
from micro_sam_b200 import prompt_based_segmentation as pbs
from micro_sam_b200 import util
from micro_sam_b200.sam import ResizeLongestSide


def _shift_rule(mask, s):
    """msam_shift_mask's rule: per axis x = o - s in fp64; 0 unless 0 <= x <= n - 1 on both axes, else mask[floor(x + 0.5)]."""
    keep, src = [], []
    for ax, n in enumerate(mask.shape):
        x = np.arange(n, dtype=np.float64) - np.float64(s[ax])
        ok = (x >= 0) & (x <= n - 1)
        keep.append(ok)
        src.append(np.floor(x[ok] + 0.5).astype(np.int64))
    out = np.zeros_like(mask)
    out[np.ix_(*keep)] = mask[np.ix_(*src)]
    return out


def _shift_grid(H, W):
    vals = [0.0, 1e-9, -1e-9, 0.5000001, -0.5000001, 12.49999999]
    for k in range(4):
        for d in (0.0, 1e-9, -1e-9):
            vals += [k + 0.5 + d, -(k + 0.5 + d)]
    vals += [H - 1, H - 0.5, H - 0.5 + 1e-9, H, -(H - 1), -(H - 0.5), -H, W - 1, W - 0.5, W, -(W - 0.5), -W, 1e300, -1e300, np.nan]
    return vals


@pytest.mark.parametrize("H,W", [(13, 17), (7, 5), (1, 9), (21, 1), (16, 16), (30, 11)])
def test_shift_rule_matches_scipy(H, W):
    rng = np.random.default_rng(H * 100 + W)
    m = (rng.random((H, W)) < 0.5).astype(np.uint8) * rng.integers(1, 4, (H, W)).astype(np.uint8)
    vals = _shift_grid(H, W)
    n = 0
    for sy in vals:
        for sx in vals[::2] + [vals[-1]]:
            ref = np.zeros_like(m)
            ndimage.shift(m, np.array([sy, sx]), output=ref, order=0, prefilter=False)
            assert np.array_equal(_shift_rule(m, (sy, sx)), ref), (sy, sx)
            n += 1
    assert n > 1000
    out = np.zeros_like(m)
    ndimage.shift(m, np.array([np.nan, 0.0]), output=out, order=0, prefilter=False)
    assert not out.any()


def test_shift_rule_examples():
    m = np.zeros((1, 8), np.uint8)
    m[0, 3] = 1
    assert _shift_rule(m, (0.0, 0.5))[0, 3] == 1 and _shift_rule(m, (0.0, 0.5000001))[0, 4] == 1
    assert not _shift_rule(np.ones((4, 4), np.uint8), (0.0, -1e-9))[:, 3].any()     # x = 3 + 1e-9 > n - 1: outside
    assert not _shift_rule(np.ones((4, 4), np.uint8), (0.0, 1e-9))[:, 0].any()      # x = -1e-9 < 0: outside


def test_centroid_from_sums_is_np_mean():
    rng = np.random.default_rng(1)
    for H, W in [(300, 380), (1, 1), (7, 1000), (1024, 1024)]:
        for p in (0.5, 0.01, 1e-5):
            m = rng.random((H, W)) < p
            ys, xs = np.where(m)
            if len(ys) == 0:
                continue
            ref = np.array([np.mean(ys), np.mean(xs)])
            got = mds._centroid(len(ys), int(ys.sum()), int(xs.sum()))
            assert got.dtype == np.float64 and np.array_equal(got.view(np.int64), ref.view(np.int64)), (H, W, p)
    assert np.isnan(mds._centroid(0, 0, 0)).all()


def test_prompt_layer_to_state():
    layer = SimpleNamespace(data=np.array([[2, 10, 10], [2, 20, 20], [5, 1, 1], [7, 3, 3]], float),
                            properties={"state": np.array(["track", "division", "track", "track"])})
    assert [mds.prompt_layer_to_state(layer, t) for t in (2, 5, 7, 3)] == ["division", "track", "track", "track"]


# ------------------------------------------------------------------------------------------------ the frame schedule
def _reference(point_prompts, seg, slices, stop_upper, threshold, motion_smoothing, segment, update_progress, motions):
    """Restatement of the reference's track_from_prompts loop with `segment(prev, t)` in place of segment_from_mask; appends
    (t, motion model) for every frame it segments."""
    def centre(t):
        ys, xs = np.where(seg[t] == 1)
        return np.array([np.mean(ys), np.mean(xs)])

    def movement(t_a, t_b):
        return (centre(t_a) - centre(t_b)).astype("float64")

    model, division = None, False
    t0 = int(slices.min())
    t = t0 + 1
    while True:
        if t == t0 + 2:
            model = movement(t - 1, t - 2)
        elif t > t0 + 2:
            model = motion_smoothing * model + (1 - motion_smoothing) * movement(t - 1, t - 2)
        if t in slices:
            prev, new = None, seg[t]
            layer_state = point_prompts.properties["state"][point_prompts.data[:, 0] == t]
            state = "division" if (layer_state == "division").any() else "track"
        else:
            prev = seg[t - 1]
            if model is not None:
                shifted = np.zeros_like(prev)
                ndimage.shift(prev, model, output=shifted, order=0, prefilter=False)
                prev = shifted
            motions.append((t, None if model is None else model.copy()))
            new, state = segment(prev, t), "track"
            if t < slices[-1]:
                prev = None
            update_progress(1)
        if threshold is not None and prev is not None:
            iou = util.compute_iou(prev, new)
            if iou < threshold:
                print(f"Segmentation stopped at frame {t} due to IOU {iou} < {threshold}.")
                break
        if state == "division":
            division = True
            break
        seg[t] = new
        t += 1
        if t == slices[-1] and stop_upper:
            break
        if t == seg.shape[0]:
            break
    return seg, division


class _FakeStep:
    """Host stand-in of the device step: frame t = segment(previous frame shifted by the motion, t) with the kernel's index
    rule, centres formed from counts and sums as the device step forms them."""

    def __init__(self, seg, segment):
        self.seg, self.segment, self.motions = seg, segment, []

    def centroid(self, t):
        ys, xs = np.nonzero(self.seg[t] == 1)
        return mds._centroid(len(ys), int(ys.sum()), int(xs.sum()))

    def track(self, t, motion, threshold):
        self.motions.append((t, None if motion is None else np.array(motion)))
        prev = self.seg[t - 1] if motion is None else _shift_rule(self.seg[t - 1], motion)
        new = self.segment(prev, t)
        if threshold is not None:
            iou = util.compute_iou(prev, new)
            if iou < threshold:
                return False, iou
        self.seg[t] = new
        return True, None

    def finish(self):
        pass


def _segmenter(H, W, vanish=(), jump=()):
    """A stand-in segmentation: a disk a non-integer step away from the prompt's centre; empty on `vanish`, far off on `jump`."""
    yy, xx = np.mgrid[:H, :W]

    def segment(prev, t):
        out = np.zeros((H, W), bool)
        if t in vanish:
            return out
        ys, xs = np.nonzero(prev == 1)
        cy, cx = (ys.mean() + 1.37, xs.mean() - 0.83) if len(ys) else (H / 2, W / 2)
        if t in jump:
            cy = (cy + H / 2) % H
        out[(yy - cy) ** 2 + (xx - cx) ** 2 < (5 + t % 3) ** 2] = True
        return out
    return segment


def _series(T, slices, H=48, W=56, empty=()):
    seg = np.zeros((T, H, W), np.uint32)
    yy, xx = np.mgrid[:H, :W]
    for k in slices:
        if k not in empty:
            seg[k][(yy - 14 - 2.3 * k) ** 2 + (xx - 30 + 1.6 * k) ** 2 < 36] = 1
    return seg


def _layer(slices, division=()):
    data = np.array([[t, 1.0, 1.0] for t in slices] + [[t, 2.0, 2.0] for t in division], float).reshape(-1, 3)
    return SimpleNamespace(data=data, properties={"state": np.array(["track"] * len(slices) + ["division"] * len(division))})


def _motion_equal(a, b):
    assert [t for t, _ in a] == [t for t, _ in b]
    for (t, m), (_, r) in zip(a, b):
        assert (m is None) == (r is None), t
        if m is not None:
            assert m.dtype == np.float64 and r.dtype == np.float64
            assert np.array_equal(np.isnan(m), np.isnan(r)), (t, m, r)
            fin = ~np.isnan(m)
            assert np.array_equal(m[fin].view(np.int64), r[fin].view(np.int64)), (t, m, r)


CASES = [
    # T, slices, division frames, empty prompt frames, vanish / jump frames of the stand-in segmentation
    (10, [2], (), (), (), ()),
    (10, [0], (), (), (), (6,)),
    (12, [1, 4, 9], (), (), (), (3, 10)),
    (12, [2, 5, 8], (5,), (), (), ()),
    (12, [2, 5, 8], (8,), (), (), ()),
    (12, [1, 3, 7], (), (3,), (), ()),       # an empty prompt frame: NaN centre, NaN motion from then on
    (12, [1, 6], (), (), (3,), ()),          # the object vanishes between prompt frames
    (9, [7], (), (), (), ()),
    (10, [3, 4], (), (), (), (7,)),
]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("stop_upper", [False, True])
@pytest.mark.parametrize("threshold", [None, 0.5, 0.9])
@pytest.mark.parametrize("alpha", [0, 0.5, 1.0])
def test_schedule_matches_reference(capsys, case, stop_upper, threshold, alpha):
    T, slices, division, empty, vanish, jump = CASES[case]
    slices = np.array(slices)
    seg0 = _series(T, slices, empty=empty)
    layer = _layer(slices, division)
    H, W = seg0.shape[1:]
    calls = {"ref": 0, "sched": 0}

    ref_motions = []
    with np.errstate(invalid="ignore"):
        ref, ref_div = _reference(layer, seg0.copy(), slices, stop_upper, threshold, alpha, _segmenter(H, W, vanish, jump),
                                  lambda n: calls.__setitem__("ref", calls["ref"] + n), ref_motions)
    ref_out = capsys.readouterr().out

    seg = seg0.copy()
    step = _FakeStep(seg, _segmenter(H, W, vanish, jump))
    out, div = mds._track(seg, slices, layer, stop_upper, threshold, alpha, step,
                          lambda n: calls.__setitem__("sched", calls["sched"] + n))
    assert out is seg and div == ref_div
    assert np.array_equal(seg, ref), [int((seg[t] != ref[t]).sum()) for t in range(T)]
    _motion_equal(step.motions, ref_motions)
    assert calls["sched"] == calls["ref"]
    assert capsys.readouterr().out == ref_out


def test_schedule_covers_its_rules():
    """The cases above reach every exit: a division, stop_upper, an IoU stop past the last prompt frame only, the last frame."""
    seg = _series(12, [2, 5, 8])
    step = _FakeStep(seg, _segmenter(48, 56))
    _, div = mds._track(seg, np.array([2, 5, 8]), _layer([2, 5, 8], (5,)), False, None, 0.5, step, None)
    assert div and [t for t, _ in step.motions] == [3, 4]
    seg = _series(12, [2, 5, 8])
    step = _FakeStep(seg, _segmenter(48, 56))
    _, div = mds._track(seg, np.array([2, 5, 8]), _layer([2, 5, 8]), True, None, 0.5, step, None)
    assert not div and [t for t, _ in step.motions] == [3, 4, 6, 7]
    # a jump before the last prompt frame is kept whatever the threshold; one after it stops the track unwritten
    seg = _series(12, [1, 4, 9])
    step = _FakeStep(seg, _segmenter(48, 56, jump=(3, 10)))
    mds._track(seg, np.array([1, 4, 9]), _layer([1, 4, 9]), False, 0.9, 0.5, step, None)
    assert seg[3].any() and not seg[10].any() and seg[11].sum() == 0 and [t for t, _ in step.motions][-1] == 10
    seg = _series(10, [2])
    step = _FakeStep(seg, _segmenter(48, 56))
    mds._track(seg, np.array([2]), _layer([2]), False, None, 0.5, step, None)
    assert [t for t, _ in step.motions] == list(range(3, 10)) and step.motions[0][1] is None and seg[9].any()
    with pytest.raises(ValueError, match="nothing to track"):
        mds._track(seg, np.array([9]), _layer([9]), False, None, 0.5, _FakeStep(seg, None), None)


# ------------------------------------------------------------------------------------------------ the host glue
class _Rec:
    """predict() returns the box prompt moved down by 2 and right by 3 pixels (empty without a box)."""

    def __init__(self, shape):
        self.original_size = shape
        self.transform = ResizeLongestSide(1024)
        self.device = torch.device("cpu")
        self.is_image_set = True

    def predict(self, point_coords=None, point_labels=None, box=None, mask_input=None, multimask_output=True, return_logits=False):
        h, w = self.original_size
        m = np.zeros((1, h, w), bool)
        if box is not None:
            m[0, box[1] + 2:box[3] + 2, box[0] + 3:box[2] + 3] = True
        return m, np.array([0.5], "float32"), np.zeros((1, 256, 256), "float32")


@pytest.mark.parametrize("proj", ["box", "mask"])
@pytest.mark.parametrize("threshold", [None, 0.3])
def test_host_glue_matches_reference(monkeypatch, capsys, proj, threshold):
    monkeypatch.setattr(pbs.util, "set_precomputed", lambda predictor, emb, i=None, tile_id=None: predictor)
    slices = np.array([1, 4])
    seg0 = _series(11, slices)
    layer = _layer(slices)
    emb = {"input_size": (1024, 1024), "original_size": seg0.shape[1:]}
    use_box, use_mask, use_points, single = mds._validate_projection(proj)

    def segment(prev, t):
        return pbs.segment_from_mask(_Rec(seg0.shape[1:]), prev, image_embeddings=emb, i=t, use_mask=use_mask, use_box=use_box,
                                     use_points=use_points, box_extension=0.05, use_single_point=single)

    with np.errstate(invalid="ignore"):
        ref, ref_div = _reference(layer, seg0.copy(), slices, False, threshold, 0.5, segment, lambda n: None, [])
    seg = seg0.copy()
    out, div = mds._track_from_prompts_host(layer, None, seg, _Rec(seg0.shape[1:]), slices, emb, False, threshold, proj,
                                            box_extension=0.05)
    assert out is seg and div == ref_div
    assert np.array_equal(seg, ref)
