"""`-m gpu`: track_from_prompts' device frame step (csrc/volume.cu's msam_shift_mask, micro_sam_b200.multi_dimensional_segmentation).

Op level: msam_shift_mask against scipy.ndimage.shift(order=0, prefilter=False) bit for bit on random masks and shifts (half-pixel
ties, +-1e-9 off them, shifts past every edge, NaN), through pitched source and destination views, and its refusals.
End to end: the device step against the same schedule driven by scipy.ndimage.shift and segment_from_mask on the same
predictor -- bit-identical series and has_division for every projection, thresholds None / 0.5 / 0.9, in-memory / zarr / tiled
embeddings, motion smoothing 0 / 0.5 / 1, prompt frames in the middle of the series, a division frame, stop_upper, an object
that vanishes (NaN motion), and a prompt of more than 16 tokens refused on both paths.
"""
import gc
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import ndimage

from micro_sam_b200 import _lib, util
from micro_sam_b200 import multi_dimensional_segmentation as mds
from micro_sam_b200.sample_data import em_volume
from oracle import sam_ref
from tests.test_gpu_volume import _EmptyPromptPredictor

pytestmark = pytest.mark.gpu
DEV = "cuda"
T, H, W = 9, 300, 380


@pytest.fixture(autouse=True)
def _free_device_memory():
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _scipy_shift(m, s):
    out = np.zeros_like(m)
    ndimage.shift(m, np.asarray(s, np.float64), output=out, order=0, prefilter=False)
    return out


def _dev_shift(m, s, pad_src=0, pad_dst=0):
    """msam_shift_mask of m through views of pitch W + pad into larger buffers; checks the padding is left alone."""
    h, w = m.shape
    src = torch.full((h + 2, w + pad_src), 7, dtype=torch.uint8, device=DEV)
    src[1:h + 1, :w] = torch.from_numpy(m).to(DEV)
    dst = torch.full((h + 2, w + pad_dst), 9, dtype=torch.uint8, device=DEV)
    sv, dv = src[1:h + 1, :w], dst[1:h + 1, :w]
    _lib.check(_lib.lib().msam_shift_mask(sv.data_ptr(), w + pad_src, dv.data_ptr(), w + pad_dst, h, w, float(s[0]), float(s[1]), None))
    out = dst.cpu().numpy()
    assert (out[0] == 9).all() and (out[-1] == 9).all() and (out[:, w:] == 9).all()
    return out[1:h + 1, :w]


def test_shift_mask_matches_scipy():
    rng = np.random.default_rng(0)
    n = 0
    for (h, w) in [(300, 380), (1024, 1024), (17, 13), (1, 9), (21, 1), (257, 1023)]:
        m = ((rng.random((h, w)) < 0.3) * rng.integers(1, 3, (h, w))).astype(np.uint8)
        shifts = [(0.0, 0.0), (np.nan, 1.0), (2.0, np.nan), (h, 0.0), (-h + 0.5, 0.0), (0.0, w - 0.5), (0.0, -w), (1e300, -1e300)]
        for k in range(4):
            for d in (0.0, 1e-9, -1e-9):
                shifts += [(k + 0.5 + d, -(k + 0.5 + d)), (-(k + 0.5 + d), k + d), (d, k + 0.5 + d)]
        shifts += [tuple(rng.uniform(-1.2, 1.2, 2) * (h, w)) for _ in range(12)]
        shifts += [tuple(np.round(rng.uniform(-20, 20, 2)) + 0.5) for _ in range(6)]
        for i, s in enumerate(shifts):
            pads = (i % 3, (i // 3) % 2 * 5)
            got = _dev_shift(m, s, *pads)
            assert np.array_equal(got, _scipy_shift(m, s)), (h, w, s, pads)
            n += 1
    assert n > 300


def test_shift_mask_rejects_bad_arguments():
    L = _lib.lib()
    x = torch.zeros(64, dtype=torch.uint8, device=DEV)
    p = _lib.ptr(x)
    for args in [(None, 4, p, 4, 4, 4), (p, 4, None, 4, 4, 4), (p, 3, p, 4, 4, 4), (p, 4, p, 3, 4, 4), (p, 4, p, 4, 0, 4),
                 (p, 4, p, 4, 4, 0), (p, 4, p, 4, -1, 4)]:
        assert L.msam_shift_mask(*args, 0.5, 0.5, None) != 0, args
        assert b"shift_mask" in L.msam_last_error()
    assert L.msam_shift_mask(p, 4, _lib.ptr(x[32:]), 4, 4, 4, 0.5, 0.5, None) == 0


# ------------------------------------------------------------------------------------------------ end to end
_CACHE = {}


def _setup(kind, tmp_path_factory):
    if kind not in _CACHE:
        if "pred" not in _CACHE:
            sd = sam_ref.seeded_state_dict("vit_test", seed=1)
            _CACHE["pred"] = util.get_sam_model("vit_test", device=DEV, state_dict=sd, max_batch=4, max_prompts=64)
        pred = _CACHE["pred"]
        series = em_volume((T, H, W), seed=4)
        kw = {}
        if kind == "zarr":
            kw = dict(save_path=str(tmp_path_factory.mktemp("emb") / "e.zarr"))
        elif kind == "tiled":
            kw = dict(tile_shape=(192, 192), halo=(48, 48))
        _CACHE[kind] = (pred, util.precompute_image_embeddings(pred, series, ndim=3, **kw))
    return _CACHE[kind]


def _series(slices, empty=()):
    """A disk that moves by (2.6, -1.9) pixels per frame, drawn in the prompt frames."""
    seg = np.zeros((T, H, W), np.uint32)
    yy, xx = np.mgrid[:H, :W]
    for k in slices:
        if k not in empty:
            seg[k][(yy - 140 - 2.6 * k) ** 2 + (xx - 170 + 1.9 * k) ** 2 < 40 ** 2] = 1
    return seg


def _layer(slices, division=()):
    """A stand-in for the annotator's point layer: one point per prompt frame, state "division" on `division`."""
    data = np.array([[t, 150.0, 160.0] for t in slices] + [[t, 151.0, 161.0] for t in division], float).reshape(-1, 3)
    return SimpleNamespace(data=data, properties={"state": np.array(["track"] * len(slices) + ["division"] * len(division))})


def _compare(pred, emb, seg, slices, layer, stop_upper, thr, proj, alpha=0.5, ext=0.05, may_refuse=True, wrapper=None):
    """Device step vs the host-glue schedule.  With may_refuse, a prompt of more than 16 tokens (the decoder's limit, reached by
    points projections of the random-weight decoder's masks) must be refused by both sides; any other error fails."""
    calls = {"host": 0, "dev": 0}
    host = seg.copy()
    err = None
    try:
        _, h_div = mds._track_from_prompts_host(layer, None, host, wrapper or _EmptyPromptPredictor(pred), slices, emb, stop_upper, thr, proj,
                                                alpha, ext, lambda n: calls.__setitem__("host", calls["host"] + n))
    except RuntimeError as e:
        if not may_refuse or "tokens per prompt" not in str(e):
            raise
        err = e
    dev = seg.copy()
    if err is not None:
        with pytest.raises(RuntimeError, match="tokens per prompt"):
            mds.track_from_prompts(layer, None, dev, pred, slices, emb, stop_upper, thr, proj, alpha, ext)
        return None
    out, d_div = mds.track_from_prompts(layer, None, dev, pred, slices, emb, stop_upper, thr, proj, alpha, ext,
                                        lambda n: calls.__setitem__("dev", calls["dev"] + n))
    assert out is dev and dev.dtype == seg.dtype
    assert d_div == h_div
    assert np.array_equal(dev, host), [int((dev[t] != host[t]).sum()) for t in range(T)]
    assert calls["dev"] == calls["host"]
    return dev, d_div


@pytest.mark.parametrize("kind,proj,thr", [("memory", p, t) for p in mds.PROJECTION_MODES for t in (None, 0.5, 0.9)] +
                         [(k, p, 0.5) for k in ("zarr", "tiled") for p in mds.PROJECTION_MODES])
def test_tracking_matches_host_glue(kind, proj, thr, tmp_path_factory):
    pred, emb = _setup(kind, tmp_path_factory)
    _compare(pred, emb, _series([2]), np.array([2]), _layer([2]), False, thr, proj)
    slices = np.array([1, 4, 6])   # prompt frames in the middle of the series
    _compare(pred, emb, _series(slices), slices, _layer(slices), False, thr, proj)


@pytest.mark.parametrize("alpha", [0, 0.5, 1])
def test_motion_smoothing(alpha, tmp_path_factory):
    pred, emb = _setup("memory", tmp_path_factory)
    slices = np.array([0, 1, 5])
    assert _compare(pred, emb, _series(slices), slices, _layer(slices), False, None, "mask", alpha=alpha, may_refuse=False) is not None


@pytest.mark.parametrize("kind", ["memory", "tiled"])
def test_division_stops(kind, tmp_path_factory):
    pred, emb = _setup(kind, tmp_path_factory)
    slices = np.array([1, 5, 7])
    seg = _series(slices)
    dev, div = _compare(pred, emb, seg, slices, _layer(slices, division=[5]), False, 0.5, "box", may_refuse=False)
    assert div and np.array_equal(dev[5:], seg[5:])


def test_stop_upper(tmp_path_factory):
    pred, emb = _setup("memory", tmp_path_factory)
    slices = np.array([1, 6])
    seg = _series(slices)
    dev, div = _compare(pred, emb, seg, slices, _layer(slices), True, 0.9, "mask", may_refuse=False)
    assert not div and np.array_equal(dev[6:], seg[6:]) and np.array_equal(dev[:2], seg[:2])


@pytest.mark.parametrize("proj", ["box", "mask", "single_point"])
def test_vanishing_object(proj, tmp_path_factory):
    """Prompt frame 3 is empty: its centre is NaN, so is the motion model from frame 4 on, and every shifted plane after it is
    empty.  Under "box" and "single_point" that leaves no prompt at all."""
    pred, emb = _setup("memory", tmp_path_factory)
    slices = np.array([1, 3, 6])
    wrapper = _EmptyPromptPredictor(pred)
    _compare(pred, emb, _series(slices, empty=(3,)), slices, _layer(slices), False, None, proj, may_refuse=False, wrapper=wrapper)
    if proj != "mask":
        assert wrapper.empty_prompts >= 3


def test_more_than_16_tokens_is_refused_on_both_paths(tmp_path_factory):
    pred, emb = _setup("memory", tmp_path_factory)
    seg = np.zeros((T, H, W), np.uint32)
    for k in range(20):   # 20 separate squares: 20 inner peaks
        y, x = 20 + (k // 5) * 60, 20 + (k % 5) * 70
        seg[2, y:y + 12, x:x + 12] = 1
    slices = np.array([2])
    assert _compare(pred, emb, seg, slices, _layer(slices), False, None, "points") is None
