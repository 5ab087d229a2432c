"""`-m gpu`: object features and their projection on the device (csrc/objfeat.cu, micro_sam_b200.object_classification)
against the fp64 oracle (oracle/objfeat_ref.py).

seg_ids and areas must match exactly, means within 1e-5 x max|E|, dtypes as the reference's (float64 for a 2-D image, float32
for slices and tiles), two runs bit-identical and the projection exact.  Cases: 2-D square, non-square both ways, S < 64,
S = 1, S > 1024; labels lost in the resize; no objects; uint32 and int64 ids above 2^24; non-default and non-square
resize_embedding_shape (r < 64 included); 3-D stacks from numpy and device tensors; tiled 2-D and 3-D embeddings of a
seeded vit_b from memory and from a lazily loaded container; a joblib-saved random forest end to end.
"""
import gc

import numpy as np
import pytest
import torch

from micro_sam_b200 import _lib, util
from micro_sam_b200 import object_classification as oc
from micro_sam_b200.sample_data import em_volume
from oracle import objfeat_ref as ref
from oracle import sam_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _free_device_memory():
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def predictor():
    return util.get_sam_model("vit_b", state_dict=sam_ref.seeded_state_dict("vit_b", seed=0), max_batch=4, max_prompts=16)


def _blobs(shape, n, rng, base=1, dtype=np.int64):
    h, w = shape
    seg = np.zeros((h, w), np.int64)
    yy, xx = np.mgrid[:h, :w]
    ids = base + rng.choice(np.arange(0, 20 * n), size=n, replace=False)
    for lab in ids:
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        r = rng.uniform(0.5, max(1.0, min(h, w) / 5))
        seg[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = lab
    return seg.astype(dtype)


def _emb2d(rng, on_device=False):
    e = (rng.standard_normal((1, 256, 64, 64)) * 3).astype(np.float32)
    return {"features": torch.from_numpy(e).to(DEV) if on_device else e, "input_size": (1024, 1024), "original_size": (1024, 1024)}


def _host(emb):
    """the same embeddings with every array on the host (numpy), for the oracle"""
    f = emb["features"]
    if isinstance(f, util._MemGroup):
        g = util._MemGroup()
        g.attrs.update(f.attrs)
        for k, ds in f.items():
            g[k] = util._MemDataset(ds.data.cpu().numpy() if torch.is_tensor(ds.data) else np.asarray(ds.data), ds.attrs)
        return {**emb, "features": g}
    return {**emb, "features": f.cpu().numpy() if torch.is_tensor(f) else f}


def _emax(emb):
    f = _host(emb)["features"]
    if isinstance(f, util._MemGroup):
        return max(float(np.abs(ds.data).max()) for ds in f.values())
    return float(np.abs(np.asarray(f[:])).max())


def _check(emb, seg, shape=(256, 256), seg_dev=False, emax=None):
    got = oc.compute_object_features(emb, torch.as_tensor(seg).to(DEV) if seg_dev else seg, shape, verbose=False)
    again = oc.compute_object_features(emb, seg, shape, verbose=False)
    want = ref.compute_object_features(_host(emb), np.asarray(seg).astype(np.int64), shape)
    ids, feats = got
    assert ids.dtype == np.int64 and feats.dtype == want[1].dtype and feats.shape == (len(ids), 257)
    np.testing.assert_array_equal(ids, want[0])
    np.testing.assert_array_equal(feats[:, 0], want[1][:, 0])
    tol = 1e-5 * (emax if emax is not None else _emax(emb))
    if len(ids):
        err = np.abs(feats[:, 1:].astype(np.float64) - want[1][:, 1:]).max()
        assert err <= tol, f"max mean error {err} > {tol}"
    np.testing.assert_array_equal(again[0], ids)
    assert again[1].tobytes() == feats.tobytes(), "two runs differ"
    return ids, feats


@pytest.mark.parametrize("shape", [(512, 512), (600, 300), (300, 600), (40, 40), (50, 17), (1, 1), (1100, 1030), (1024, 1024)])
def test_2d(shape):
    rng = np.random.default_rng(sum(shape))
    seg = _blobs(shape, 25, rng)
    ids, feats = _check(_emb2d(rng), seg)
    assert feats.dtype == np.float64


@pytest.mark.parametrize("dtype", [np.uint32, np.int64])
def test_large_ids_and_device_inputs(dtype):
    rng = np.random.default_rng(7)
    seg = _blobs((700, 500), 40, rng, base=(1 << 24) + 3 if dtype == np.uint32 else (1 << 40) + 5, dtype=dtype)
    if dtype == np.uint32:
        seg[seg != 0] += np.uint32(3 << 30)   # above 2^31: widened, not sign-extended
    _check(_emb2d(rng, on_device=True), seg, seg_dev=dtype == np.int64)


def test_labels_lost_in_the_resize():
    rng = np.random.default_rng(3)
    seg = np.zeros((1024, 1024), np.int64)
    seg[100:180, 300:420] = 5
    seg[501, 501] = 6            # 1024 -> 256 samples pixels 4 o + 2: lost
    seg[602, 602] = 7            # sampled: one pixel on the grid
    seg[603:606, 700:703] = 8    # a 3 x 3 block between sample rows: lost
    ids, feats = _check(_emb2d(rng), seg)
    assert ids.tolist() == [5, 7] and feats[1, 0] == 1
    seg3 = np.stack([seg, np.where(seg == 5, 5, 0)[::-1]])   # 6 and 8 are lost in both slices
    emb3 = {"features": rng.standard_normal((2, 1, 256, 64, 64)).astype(np.float32), "input_size": (1024, 1024),
            "original_size": (1024, 1024)}
    ids, feats = _check(emb3, seg3)
    assert ids.tolist() == [5, 6, 7, 8] and feats.dtype == np.float32
    assert not feats[1].any() and not feats[3].any()


def test_no_objects():
    rng = np.random.default_rng(4)
    ids, feats = oc.compute_object_features(_emb2d(rng), np.zeros((300, 200), np.int32), verbose=False)
    assert ids.shape == (0,) and ids.dtype == np.int64 and feats.shape == (0, 257) and feats.dtype == np.float64
    emb3 = {"features": rng.standard_normal((2, 1, 256, 64, 64)).astype(np.float32), "input_size": (1024, 1024),
            "original_size": (1024, 1024)}
    ids, feats = oc.compute_object_features(emb3, np.zeros((2, 64, 64), np.int32), verbose=False)
    assert ids.shape == (0,) and feats.shape == (0, 257) and feats.dtype == np.float32


@pytest.mark.parametrize("rshape", [(128, 200), (32, 300), (100, 64), (1, 3), (512, 512)])
def test_resize_embedding_shape(rshape):
    rng = np.random.default_rng(rshape[0] * 1000 + rshape[1])
    seg = _blobs((600, 540), 20, rng)
    _check(_emb2d(rng), seg, rshape)


@pytest.mark.parametrize("on_device", [False, True])
def test_3d_stack(on_device):
    rng = np.random.default_rng(11)
    Z = 5
    seg = np.stack([_blobs((300, 420), 12, rng) for _ in range(Z)])
    seg[1:4, 100:160, 100:200] = 99999        # one object through three slices
    e = (rng.standard_normal((Z, 1, 256, 64, 64)) * 2).astype(np.float32)
    emb = {"features": torch.from_numpy(e).to(DEV) if on_device else e, "input_size": (1024, 731), "original_size": (300, 420)}
    _check(emb, seg, seg_dev=on_device)


def test_tiled_2d_and_3d(predictor, tmp_path):
    img = em_volume((2, 700, 900), seed=1)
    rng = np.random.default_rng(12)
    seg2 = _blobs((700, 900), 30, rng)
    emb = util.precompute_image_embeddings(predictor, img[0], ndim=2, tile_shape=(512, 512), halo=(64, 64), to_numpy=False)
    assert emb["input_size"] is None
    _check(emb, seg2)
    _check(emb, seg2, (100, 300))
    seg3 = np.stack([seg2, _blobs((700, 900), 30, rng)])
    emb3 = util.precompute_image_embeddings(predictor, img, ndim=3, tile_shape=(512, 512), halo=(64, 64), to_numpy=False)
    ids, feats = _check(emb3, seg3)
    assert feats.dtype == np.float32
    saved = util.precompute_image_embeddings(predictor, img, save_path=str(tmp_path / "emb.zarr"), lazy_loading=True, ndim=3,
                                             tile_shape=(512, 512), halo=(64, 64))
    ids_z, _ = _check(saved, seg3, emax=_emax(emb3))
    np.testing.assert_array_equal(ids_z, ids)


def test_projection():
    rng = np.random.default_rng(13)
    for dtype in (np.uint32, np.int64):
        seg = _blobs((301, 257), 30, rng, base=(1 << 31) + 1 if dtype == np.uint32 else (1 << 50), dtype=dtype)
        ids = np.unique(seg)
        ids = ids[ids != 0][::2]                                  # every other object has no prediction
        for pred in (rng.integers(1, 5, len(ids)), rng.standard_normal(len(ids)).astype(np.float32)):
            want = ref.project_prediction_to_segmentation(seg, pred, ids)
            got = oc.project_prediction_to_segmentation(seg, pred, ids)
            assert got.dtype == pred.dtype and got.shape == seg.shape
            np.testing.assert_array_equal(got, want)
        if dtype == np.int64:
            got_t = oc.project_prediction_to_segmentation(torch.from_numpy(seg).to(DEV), pred, ids)
            assert got_t.is_cuda
            np.testing.assert_array_equal(got_t.cpu().numpy().astype(pred.dtype), want)
    vol = np.stack([seg, seg[::-1], seg[:, ::-1]])
    np.testing.assert_array_equal(oc.project_prediction_to_segmentation(vol, pred, ids),
                                  ref.project_prediction_to_segmentation(vol, pred, ids))


def test_run_prediction_with_object_classifier(predictor, tmp_path):
    sklearn_ensemble = pytest.importorskip("sklearn.ensemble")
    import joblib
    rng = np.random.default_rng(14)
    images = [em_volume((1, 256, 320), seed=s)[0] for s in (2, 3)]
    segs = [_blobs((256, 320), 15, rng) for _ in images]
    emb = util.precompute_image_embeddings(predictor, images[0], to_numpy=False)
    seg_ids, feats = oc.compute_object_features(emb, segs[0], verbose=False)
    rf = sklearn_ensemble.RandomForestClassifier(n_estimators=10, random_state=0)
    rf.fit(feats, (seg_ids % 3).astype(np.int64))
    path = tmp_path / "rf.joblib"
    joblib.dump(rf, path)
    preds = oc.run_prediction_with_object_classifier(images, segs, predictor, str(path))
    raw = oc.run_prediction_with_object_classifier(images, segs, predictor, str(path), project_prediction=False)
    for image, seg, pred, obj in zip(images, segs, preds, raw):
        e = util.precompute_image_embeddings(predictor, image)
        ids, f = oc.compute_object_features(e, seg, verbose=False)
        np.testing.assert_array_equal(obj, rf.predict(f))
        np.testing.assert_array_equal(pred, ref.project_prediction_to_segmentation(seg, rf.predict(f), ids))


def test_abi_refusals():
    L = _lib.lib()
    n = 3
    ws = torch.empty(int(L.msam_object_features_workspace(n)), dtype=torch.uint8, device=DEV)
    emb = torch.zeros(256, 64, 64, device=DEV)
    seg = torch.zeros(10, 12, dtype=torch.int32, device=DEV)
    sums = torch.zeros(n, 256, dtype=torch.float64, device=DEV)
    areas = torch.zeros(n, dtype=torch.int64, device=DEV)

    def call(emb_p=_lib.ptr(emb), ld=12, h=10, w=12, ry=12, rx=12, ws_bytes=ws.numel()):
        return L.msam_object_features(emb_p, _lib.ptr(seg), ld, h, w, ry, rx, n, _lib.ptr(ws), ws_bytes, _lib.ptr(sums),
                                      _lib.ptr(areas), None)

    assert call() == 0
    assert call(emb_p=None) != 0 and b"null argument" in L.msam_last_error()
    for kw in (dict(ld=11), dict(ry=13), dict(rx=0), dict(h=0), dict(ws_bytes=ws.numel() - 1)):
        assert call(**kw) != 0, kw
    assert L.msam_object_features_finish(None, _lib.ptr(areas), n, 1, _lib.ptr(sums), None) != 0
    assert L.msam_project_labels(None, 4, None, None, 0, None, None) != 0
    torch.cuda.synchronize()
    assert not sums.any() and not areas.any()
