"""`-m gpu`: segment_mask_in_volume's device slice step (csrc/volume.cu, micro_sam_b200.multi_dimensional_segmentation).

Op level: the box, count and coordinate sums, the mask-prompt logits (bit for bit), the smoothed distance field (<= 1 ulp) and the
derived points of msam_mask_prompts against segment_from_mask's host glue (prompt_based_segmentation.py) on random blobs, odd and
non-square sizes, 1x1 objects, objects touching every border and masks that fill their crop; msam_mask_iou_counts exactly.
End to end: the device step against the same schedule driven by segment_from_mask on the same predictor -- bit-identical volumes
and (z_min, z_max) for every projection, in-memory / zarr / tiled embeddings, IoU thresholds 0 and 0.8, and a thresholdless
range that reaches an empty slice under "box" projection.
"""
import gc

import numpy as np
import pytest
import torch
from scipy import ndimage

from micro_sam_b200 import _lib, util
from micro_sam_b200 import multi_dimensional_segmentation as mds
from micro_sam_b200 import prompt_based_segmentation as pbs
from micro_sam_b200.sam import ResizeLongestSide
from micro_sam_b200.sample_data import em_volume
from oracle import sam_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAXP = 256


@pytest.fixture(autouse=True)
def _free_device_memory():
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _dev_prompts(mask, ext, point_mode, logits=True):
    H, W = mask.shape
    L = _lib.lib()
    m = torch.from_numpy(np.ascontiguousarray(mask == 1).astype(np.uint8)).to(DEV)
    ws = torch.empty(int(L.msam_mask_prompts_workspace(H, W)), dtype=torch.uint8, device=DEV)
    st = torch.zeros(12, dtype=torch.int64, device=DEV)
    box = torch.zeros(4, device=DEV)
    lg = torch.zeros(256, 256, device=DEV)
    pts = torch.zeros(MAXP, 2, device=DEV)
    lbl = torch.zeros(MAXP, device=DEV)
    field = torch.zeros(H * W, device=DEV)
    _lib.check(L.msam_mask_prompts(_lib.ptr(m), H, W, W, float(ext), int(logits), point_mode, MAXP, _lib.ptr(ws), ws.numel(),
                                   _lib.ptr(st), _lib.ptr(box), _lib.ptr(lg), _lib.ptr(pts), _lib.ptr(lbl), _lib.ptr(field), None))
    torch.cuda.synchronize()
    return st.cpu().numpy(), box.cpu().numpy(), lg.cpu().numpy(), pts.cpu().numpy(), lbl.cpu().numpy(), field.cpu().numpy()


def _blob(H, W, rng, n=3):
    yy, xx = np.mgrid[:H, :W]
    m = np.zeros((H, W), np.uint8)
    for _ in range(n):
        cy, cx = rng.uniform(0, H), rng.uniform(0, W)
        ry, rx = rng.uniform(1, max(2, H / 4)), rng.uniform(1, max(2, W / 4))
        m[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1] = 1
    return m


def _masks():
    rng = np.random.default_rng(0)
    out = []
    for (H, W) in [(700, 1000), (257, 1023), (256, 256), (64, 96), (100, 140), (300, 77), (1024, 1024), (33, 512)]:
        for _ in range(24):
            out.append(_blob(H, W, rng, int(rng.integers(1, 4))))
    for (H, W) in [(700, 1000), (256, 256), (31, 45)]:
        m = np.zeros((H, W), np.uint8); m[H // 2, W // 3] = 1; out.append(m)                   # 1x1 object
        m = np.zeros((H, W), np.uint8); m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = 1; out.append(m)   # touches every border
        m = np.zeros((H, W), np.uint8); m[3:H // 2, 5:W // 2] = 1; out.append(m)               # fills its crop
        out.append(np.ones((H, W), np.uint8))
    return out


MASKS = _masks()


def test_box_count_sums_and_logits():
    assert len(MASKS) >= 200
    for k, m in enumerate(MASKS):
        H, W = m.shape
        for ext in (0, 0.1, 5):
            st, box, lg, *_ = _dev_prompts(m, ext, 0, logits=ext == 0)
            ys, xs = np.nonzero(m == 1)
            assert st[0] == len(ys) and st[1] == ys.sum() and st[2] == xs.sum(), k
            ref = pbs._compute_box_from_mask(m, box_extension=ext)
            assert np.array_equal(st[7:11], ref), (k, ext, st[7:11], ref)
            assert np.array_equal(st[3:7], [ys.min(), xs.min(), ys.max() + 1, xs.max() + 1])
            ref1024 = torch.as_tensor(ResizeLongestSide(1024).apply_boxes(ref, (H, W)), dtype=torch.float).numpy()[0]
            assert np.array_equal(box, ref1024), (k, ext, box, ref1024)
            if ext == 0:
                ref_lg = pbs._compute_logits_from_mask(m)[0]
                assert np.array_equal(lg.view(np.uint32), ref_lg.view(np.uint32)), (k, H, W, int((lg != ref_lg).sum()))


def _host_field(m, ext):
    box = pbs._compute_box_from_mask(m, box_extension=ext)
    crop = m[box[1]:box[3], box[0]:box[2]].astype(bool)
    bnd = ndimage.binary_dilation(crop) & ~crop
    return ndimage.gaussian_filter(ndimage.distance_transform_edt(~bnd).astype("float32"), sigma=1.0)


@pytest.mark.parametrize("single", [True, False])
def test_points_and_field(single):
    for k, m in enumerate(MASKS[::2] if not single else MASKS):
        H, W = m.shape
        ext = (0, 0.1, 5)[k % 3]
        st, _, _, pts, lbl, field = _dev_prompts(m, ext, 1 if single else 2, logits=False)
        ref_f = _host_field(m, ext)
        f = field[:ref_f.size].reshape(ref_f.shape)
        ulp = np.abs(f.view(np.int32).astype(np.int64) - ref_f.view(np.int32).astype(np.int64)).max()
        assert ulp <= 1, (k, ulp)
        coords, labels = pbs._compute_points_from_mask(m, None, ext, use_single_point=single)
        ref = torch.as_tensor(ResizeLongestSide(1024).apply_coords(coords, (H, W)), dtype=torch.float).numpy()
        assert st[11] == len(ref), (k, st[11], len(ref))
        n = min(len(ref), MAXP)
        assert np.array_equal(pts[:n], ref[:n]), k
        assert np.array_equal(lbl[:n], labels[:n].astype(np.float32)), k


def test_fill_the_crop_distance_field():
    m = np.zeros((40, 50), np.uint8)
    m[10:20, 5:30] = 1
    _, _, _, _, _, field = _dev_prompts(m, 0, 1, logits=False)
    assert np.array_equal(field[:250].reshape(10, 25), _host_field(m, 0))


def test_iou_counts():
    rng = np.random.default_rng(3)
    L = _lib.lib()
    for (H, W) in [(700, 1000), (1, 1), (257, 1023)]:
        for _ in range(5):
            a, b = _blob(H, W, rng), _blob(H, W, rng)
            b[rng.random((H, W)) < 0.01] = 2     # only pixels == 1 count
            ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
            c = torch.zeros(2, dtype=torch.int64, device=DEV)
            _lib.check(L.msam_mask_iou_counts(_lib.ptr(ta), W, _lib.ptr(tb), W, H, W, _lib.ptr(c), None))
            c = c.cpu().numpy()
            assert c[0] == np.logical_and(a == 1, b == 1).sum() and c[1] == np.logical_or(a == 1, b == 1).sum()


def test_rejects_bad_arguments():
    L = _lib.lib()
    x = torch.zeros(16, dtype=torch.int64, device=DEV)
    assert L.msam_mask_prompts(None, 4, 4, 4, 0.0, 0, 0, 1, _lib.ptr(x), 8, _lib.ptr(x), None, None, None, None, None, None) != 0
    assert L.msam_mask_prompts(_lib.ptr(x), 4, 4, 3, 0.0, 0, 0, 1, _lib.ptr(x), 8, _lib.ptr(x), None, None, None, None, None, None) != 0
    assert L.msam_mask_prompts(_lib.ptr(x), 4, 4, 4, 0.0, 0, 0, 1, _lib.ptr(x), 8, _lib.ptr(x), None, None, None, None, None, None) != 0
    assert L.msam_mask_iou_counts(_lib.ptr(x), 3, _lib.ptr(x), 4, 4, 4, _lib.ptr(x), None) != 0
    # 8192 x 111 resizes its width 111 -> 3 (scale 37): 75 taps per pixel, more than the kernel holds -> refused, not truncated
    H, W = 8192, 111
    m = torch.zeros(H, W, dtype=torch.uint8, device=DEV)
    ws = torch.empty(int(L.msam_mask_prompts_workspace(H, W)), dtype=torch.uint8, device=DEV)
    lg = torch.zeros(256, 256, device=DEV)
    assert L.msam_mask_prompts(_lib.ptr(m), H, W, W, 0.0, 1, 0, 1, _lib.ptr(ws), ws.numel(), _lib.ptr(x), None, _lib.ptr(lg), None, None,
                               None, None) != 0
    assert b"taps" in L.msam_last_error()
    assert L.msam_mask_prompts(_lib.ptr(m), H, W, W, 0.0, 0, 0, 1, _lib.ptr(ws), ws.numel(), _lib.ptr(x), None, None, None, None,
                               None, None) == 0


# ------------------------------------------------------------------------------------------------ end to end
class _EmptyPromptPredictor:
    """The predictor with predict() decoding an empty prompt (no box, points or mask) through msam_mask_decode's n_sparse = 0
    route, as upstream's predictor does."""

    def __init__(self, p):
        self.__dict__["_p"] = p
        self.__dict__["empty_prompts"] = 0

    def __getattr__(self, k):
        return getattr(self._p, k)

    def __setattr__(self, k, v):
        setattr(self._p, k, v)

    def predict(self, point_coords=None, point_labels=None, box=None, mask_input=None, multimask_output=True, return_logits=False):
        p = self._p
        if point_coords is not None or box is not None or mask_input is not None:
            return p.predict(point_coords, point_labels, box, mask_input, multimask_output, return_logits)
        self.__dict__["empty_prompts"] += 1
        p._bind_features()
        low = torch.empty(1, 1, 256, 256, device=DEV)
        iou = torch.empty(1, 1, device=DEV)
        _lib.check(_lib.lib().msam_mask_decode(p.model._h, None, 0, None, 1, 0, _lib.ptr(low), _lib.ptr(iou), _lib.cur_stream()))
        H, W = p.original_size
        m = torch.empty(1, H, W, dtype=torch.uint8, device=DEV)
        _lib.check(_lib.lib().msam_upsample_masks(_lib.ptr(low), None, 1, int(p.input_size[0]), int(p.input_size[1]), H, W,
                                                  p.model.mask_threshold, None, _lib.ptr(m), _lib.cur_stream()))
        return m.bool().cpu().numpy(), iou[0].cpu().numpy(), low[0].cpu().numpy()


_CACHE = {}


def _setup(model_type, kind, tmp_path_factory):
    key = (model_type, kind)
    if key not in _CACHE:
        if model_type not in _CACHE:
            sd = sam_ref.seeded_state_dict(model_type, seed=1)
            _CACHE[model_type] = util.get_sam_model(model_type, device=DEV, state_dict=sd, max_batch=4, max_prompts=64)
        pred = _CACHE[model_type]
        vol = em_volume((9, 300, 380), seed=4)
        kw = {}
        if kind == "zarr":
            kw = dict(save_path=str(tmp_path_factory.mktemp("emb") / "e.zarr"))
        elif kind == "tiled":
            kw = dict(tile_shape=(192, 192), halo=(48, 48))
        emb = util.precompute_image_embeddings(pred, vol, ndim=3, **kw)
        _CACHE[key] = (pred, emb)
    return _CACHE[key]


def _seed(shape, z, rng, empty_at=()):
    seg = np.zeros(shape, np.uint32)
    yy, xx = np.mgrid[:shape[1], :shape[2]]
    for k in z:
        if k not in empty_at:
            seg[k][(yy - shape[1] * 0.5) ** 2 + (xx - shape[2] * 0.45) ** 2 < (30 + 3 * k) ** 2] = 1
    return seg


def _compare(pred, emb, seg, slices, stop_lower, stop_upper, thr, proj, ext=0.0, may_refuse=True, wrapper=None):
    """Device step vs the host-glue schedule.  With may_refuse, a prompt of more than 16 tokens (the decoder's limit, reached by
    points projections of the random-weight decoder's large masks) must be refused by both sides; any other error fails."""
    host = seg.copy()
    calls = {"host": 0, "dev": 0}
    err = None
    try:
        hz = mds._segment_mask_in_volume_host(host, wrapper or _EmptyPromptPredictor(pred), emb, slices, stop_lower, stop_upper, thr, proj,
                                              lambda n: calls.__setitem__("host", calls["host"] + n), ext)
    except RuntimeError as e:
        if not may_refuse or "tokens per prompt" not in str(e):
            raise
        err = e
    dev = seg.copy()
    if err is not None:
        with pytest.raises(RuntimeError, match="tokens per prompt"):
            mds.segment_mask_in_volume(dev, pred, emb, slices, stop_lower, stop_upper, thr, proj, None, ext)
        return None
    dz = mds.segment_mask_in_volume(dev, pred, emb, slices, stop_lower, stop_upper, thr, proj,
                                    lambda n: calls.__setitem__("dev", calls["dev"] + n), ext)
    assert dz[1] == hz[1], (dz[1], hz[1])
    assert dev.dtype == seg.dtype
    assert np.array_equal(dev, host), [int((dev[z] != host[z]).sum()) for z in range(seg.shape[0])]
    assert calls["dev"] == calls["host"]
    return dev


@pytest.mark.parametrize("kind", ["memory", "zarr", "tiled"])
@pytest.mark.parametrize("proj", list(mds.PROJECTION_MODES))
@pytest.mark.parametrize("thr", [0.0, 0.8])
def test_volume_matches_host_glue(kind, proj, thr, tmp_path_factory):
    pred, emb = _setup("vit_test", kind, tmp_path_factory)
    rng = np.random.default_rng(0)
    seg = _seed((9, 300, 380), [4], rng)
    _compare(pred, emb, seg, np.array([4]), False, False, thr, proj)
    seg = _seed((9, 300, 380), [1, 5, 8], rng)
    _compare(pred, emb, seg, np.array([1, 5, 8]), False, True, thr, proj, ext=0.1)


def test_empty_slice_in_thresholdless_range_under_box(tmp_path_factory):
    """Seed 1 is empty: the thresholdless range 1 -> 3 of the gap (1, 6) starts from an empty mask, which under "box" leaves no
    prompt at all (and so does the thresholded range below slice 1, which then stops)."""
    pred, emb = _setup("vit_test", "memory", tmp_path_factory)
    seg = _seed((9, 300, 380), [1, 6], None, empty_at=(1,))
    wrapper = _EmptyPromptPredictor(pred)
    assert _compare(pred, emb, seg, np.array([1, 6]), False, True, 0.5, "box", may_refuse=False, wrapper=wrapper) is not None
    assert wrapper.empty_prompts >= 2


@pytest.mark.parametrize("kind", ["memory", "tiled"])
@pytest.mark.parametrize("proj", ["points", "points_and_mask", "single_point"])
def test_multi_point_projections_run_through(kind, proj, tmp_path_factory):
    """Every slice prompted from a seed disk (few points), the middle slice of the gap (4, 6) by the union of both seeds: the
    point projections must finish, not be refused."""
    pred, emb = _setup("vit_test", kind, tmp_path_factory)
    slices = np.array([2, 4, 6, 8])
    seg = _seed((9, 300, 380), slices, None)
    assert _compare(pred, emb, seg, slices, True, True, 0.0, proj, may_refuse=False) is not None


def test_tiled_object_outside_its_centroid_tile(tmp_path_factory):
    """Two components whose centroid lies in a tile whose outer block holds no object pixel: the tile's mask is empty, so the
    box is None upstream (mask.sum() == 0 on the tile), not the whole frame's box."""
    pred, emb = _setup("vit_test", "tiled", tmp_path_factory)
    seg = np.zeros((9, 300, 380), np.uint8)
    seg[7, 270:295, 5:30] = 1
    seg[7, 5:30, 350:375] = 1
    attrs = emb["features"].attrs
    _, _, tile_mask = pbs._mask_to_tile(seg[7], tuple(attrs["shape"]), tuple(attrs["tile_shape"]), tuple(attrs["halo"]))
    assert tile_mask.sum() == 0
    for proj in ("mask", "box"):
        assert _compare(pred, emb, seg, np.array([7]), True, False, 0.0, proj, may_refuse=False) is not None


def test_only_the_written_slices_change(tmp_path_factory):
    pred, emb = _setup("vit_test", "memory", tmp_path_factory)
    seg = _seed((9, 300, 380), [2, 6], None).astype(np.int16)
    seg[0] = 7          # a slice the schedule never writes (stop_lower)
    out = seg.copy()
    _, (z0, z1) = mds.segment_mask_in_volume(out, pred, emb, np.array([2, 6]), True, False, 0.0, "mask")
    assert out.dtype == np.int16 and np.array_equal(out[:2], seg[:2]) and np.array_equal(out[2], seg[2])


def test_vit_b_single_point_threshold():
    sd = sam_ref.seeded_state_dict("vit_b", seed=0)
    pred = util.get_sam_model("vit_b", device=DEV, state_dict=sd, max_batch=4, max_prompts=64)
    vol = em_volume((7, 256, 320), seed=5)
    emb = util.precompute_image_embeddings(pred, vol, ndim=3)
    seg = _seed((7, 256, 320), [3], None)
    _compare(pred, emb, seg, np.array([3]), False, False, 0.8, "single_point")
