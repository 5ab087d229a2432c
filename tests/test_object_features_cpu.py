"""Object features without a GPU (oracle/objfeat_ref.py, micro_sam_b200.object_classification's host side).

- The index and weight rules the device follows (nearest source index, bilinear taps folded at the borders, the anti-aliasing
  Gaussian) against scipy.ndimage.zoom / gaussian_filter over many sides S and grid sizes r, r < 64 included.
- A numpy form of the device algorithm -- A = Wy^T [seg == l] Wx per object, sums = E A, never the resized embedding --
  against the oracle's skimage restatement to 1e-12.
- The oracle's merge of slices (fp64 totals) against a running float32 area-weighted merge, unit by unit.
- The projection with ids missing from seg_ids, repeated ids and float predictions; the refusals that need no device.
"""
import numpy as np
import pytest
from scipy import ndimage

from micro_sam_b200 import object_classification as oc
from micro_sam_b200 import util
from oracle import objfeat_ref as ref

RS = [1, 2, 3, 5, 17, 31, 32, 63, 64, 65, 100, 127, 200, 255, 256, 300, 511, 1000]


@pytest.mark.parametrize("r", RS)
def test_nearest_rule_matches_zoom(r):
    for S in sorted({r, r + 1, r + 2, 2 * r - 1, 2 * r + 1, 3 * r + 7, 1024, 1399, 2048, 4097} - {0}):
        if S < r:
            continue
        src = np.arange(S, dtype=np.int64)
        want = ndimage.zoom(src, r / S, order=0, mode="mirror", grid_mode=True)
        assert want.shape == (r,)
        np.testing.assert_array_equal(ref.nearest_index(S, r), want, err_msg=f"S={S} r={r}")


@pytest.mark.parametrize("r", RS)
def test_linear_rule_matches_zoom(r):
    rng = np.random.default_rng(r)
    x = rng.standard_normal(64)
    want = ndimage.zoom(x, r / 64, order=1, mode="mirror", grid_mode=True)
    assert want.shape == (r,)
    t, f = ref.linear_taps(r)
    got = (1 - f) * x[ref.fold(t)] + f * x[ref.fold(t + 1)]
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-14)


@pytest.mark.parametrize("r", [1, 2, 3, 5, 17, 31, 32, 63, 64, 256])
def test_gaussian_rule_matches_gaussian_filter(r):
    rng = np.random.default_rng(r)
    x = rng.standard_normal(64)
    w = ref.gaussian_weights(r)
    sigma = max(0.0, (64 / r - 1) / 2)
    if w is None:
        assert r >= 64 and sigma == 0
        return
    R = (len(w) - 1) // 2
    got = np.array([sum(w[k] * x[ref.fold(y + k - R)] for k in range(2 * R + 1)) for y in range(64)])
    want = ndimage.gaussian_filter(x, sigma, mode="mirror")
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-14)


def _blobs(h, w, n, rng, max_r=None):
    seg = np.zeros((h, w), np.int64)
    yy, xx = np.mgrid[:h, :w]
    ids = rng.choice(np.arange(1, 10 * n + 2), size=n, replace=False)
    for lab in ids:
        cy, cx = rng.uniform(0, h), rng.uniform(0, w)
        rr = rng.uniform(0.5, max_r or max(1.0, min(h, w) / 4))
        seg[(yy - cy) ** 2 + (xx - cx) ** 2 <= rr * rr] = lab
    return seg


def algebra_unit(emb, seg, resize_embedding_shape=(256, 256)):
    """the device algorithm in numpy: per-axis nearest indices and folded tap weights, A = Wy^T M Wx per object, E A"""
    h, w = seg.shape
    S = max(h, w)
    ry, rx = ref.resize_shape(seg.shape, resize_embedding_shape)
    E = np.asarray(emb, np.float64)
    for axis, r in ((1, ry), (2, rx)):
        g = ref.gaussian_weights(r)
        if g is not None:
            R = (len(g) - 1) // 2
            E = sum(g[k] * np.take(E, ref.fold(np.arange(64) + k - R), axis=axis) for k in range(2 * R + 1))

    def weights(r):
        t, f = ref.linear_taps(r)
        W = np.zeros((r, 64))
        np.add.at(W, (np.arange(r), ref.fold(t)), 1 - f)
        np.add.at(W, (np.arange(r), ref.fold(t + 1)), f)
        return W

    Wy, Wx = weights(ry), weights(rx)
    ny, nx = ref.nearest_index(S, ry), ref.nearest_index(S, rx)
    lab = np.zeros((ry, rx), np.int64)
    vy, vx = ny < h, nx < w
    lab[np.ix_(vy, vx)] = seg[np.ix_(ny[vy], nx[vx])]
    ids = np.unique(lab)
    ids = ids[ids > 0]
    feats = np.zeros((len(ids), 257))
    for k, lbl in enumerate(ids):
        M = (lab == lbl).astype(np.float64)
        A = Wy.T @ M @ Wx
        feats[k, 0] = M.sum()
        feats[k, 1:] = E.reshape(E.shape[0], -1) @ A.ravel() / M.sum()
    return ids, feats


CASES = [((300, 300), (256, 256)), ((300, 170), (256, 256)), ((170, 300), (256, 256)), ((40, 40), (256, 256)),
         ((40, 25), (256, 256)), ((1, 1), (256, 256)), ((1, 5), (256, 256)), ((1100, 1030), (256, 256)),
         ((200, 200), (128, 200)), ((500, 90), (32, 300)), ((100, 100), (100, 64)), ((64, 64), (256, 256)),
         ((513, 513), (512, 512))]


@pytest.mark.parametrize("shape,rshape", CASES)
def test_sparse_weight_algebra_matches_oracle(shape, rshape):
    rng = np.random.default_rng(sum(shape) + sum(rshape))
    emb = rng.standard_normal((256, 64, 64)).astype(np.float32)
    seg = _blobs(*shape, n=12, rng=rng)
    ids0, f0 = ref.compute_unit(emb, seg, rshape)
    ids1, f1 = algebra_unit(emb, seg, rshape)
    np.testing.assert_array_equal(ids1, ids0)
    np.testing.assert_array_equal(f1[:, 0], f0[:, 0])
    np.testing.assert_allclose(f1[:, 1:], f0[:, 1:], rtol=0, atol=1e-12 * np.abs(emb).max())


def test_labels_lost_in_the_resize_are_absent_from_a_2d_result():
    rng = np.random.default_rng(0)
    emb = rng.standard_normal((256, 64, 64)).astype(np.float32)
    seg = np.zeros((1024, 1024), np.int64)
    seg[100:140, 100:140] = 3
    seg[501, 501] = 7       # one pixel between nearest samples (1024 -> 256 samples pixels 4 o + 2)
    seg[602, 602] = 9       # a sampled pixel
    ids, feats = ref.compute_unit(emb, seg)
    assert ids.tolist() == [3, 9]
    assert feats[:, 0].tolist() == [100, 1]


def test_merge_loop_matches_a_whole_volume_computation():
    """3-D: the oracle's totals (areas summed, means weighted by area, in fp64) against a running merge that updates a float32
    table unit by unit, as a float32 implementation of the specification would; ids that no unit keeps have an all-zero row"""
    rng = np.random.default_rng(1)
    Z, H, W = 4, 90, 130
    seg = np.stack([_blobs(H, W, 6, rng) for _ in range(Z)])
    seg[1, 2, 2] = 4242     # a single pixel the resize to r = 64 does not sample (130 -> 64 samples 1, 3, 5, ...)
    emb = rng.standard_normal((Z, 1, 256, 64, 64)).astype(np.float32)
    shape = (64, 64)
    ids, feats = ref.compute_object_features({"features": emb, "input_size": (1024, 1024)}, seg, shape)
    assert feats.dtype == np.float32 and ids.dtype == np.int64
    want_ids = np.unique(seg)
    want_ids = want_ids[want_ids != 0]
    np.testing.assert_array_equal(ids, want_ids)
    table = {int(i): np.zeros(257, np.float32) for i in ids}
    for z in range(Z):
        uid, uf = ref.compute_unit(emb[z, 0], seg[z], shape)
        for i, row in zip(uid.tolist(), uf.astype(np.float32)):
            a0, a1 = table[i][0], row[0]
            table[i][1:] = (a0 * table[i][1:] + a1 * row[1:]) / (a0 + a1)
            table[i][0] = a0 + a1
    running = np.stack([table[int(i)] for i in ids])
    assert not running[np.searchsorted(ids, 4242)].any() and not feats[np.searchsorted(ids, 4242)].any()
    np.testing.assert_array_equal(feats[:, 0], running[:, 0])
    np.testing.assert_allclose(feats[:, 1:], running[:, 1:], rtol=0, atol=2e-6 * np.abs(emb).max())


def test_tiled_units_use_outer_blocks_in_c_order():
    boxes = ref.tile_outer_boxes((300, 500), (128, 256), (16, 32))
    from micro_sam_b200._amg_utils import Blocking
    tiling = Blocking([0, 0], (300, 500), (128, 256))
    assert len(boxes) == tiling.number_of_blocks == 6
    for i, bb in enumerate(boxes):
        ob = tiling.get_block_with_halo(i, [16, 32]).outer_block
        assert bb == tuple(slice(b, e) for b, e in zip(ob.begin, ob.end))


def test_projection_with_missing_and_repeated_ids():
    seg = np.array([[0, 1, 2], [5, 5, 9], [2, 1, 0]], np.uint32)
    seg_ids = np.array([5, 1, 2, 1])             # 9 and 0 missing; 1 repeated: the last prediction wins
    pred = np.array([3, 4, 6, 8])
    out = ref.project_prediction_to_segmentation(seg, pred, seg_ids)
    np.testing.assert_array_equal(out, [[0, 8, 6], [3, 3, 0], [6, 8, 0]])
    ids, payload, dtype = oc._projection_table(seg_ids, pred)
    assert ids.tolist() == [1, 2, 5] and payload.tolist() == [8, 6, 3] and dtype == pred.dtype
    lut = dict(zip(ids.tolist(), payload.tolist()))
    np.testing.assert_array_equal(np.vectorize(lambda v: lut.get(v, 0))(seg), out)
    ids, payload, dtype = oc._projection_table([7, 3], np.array([0.25, -1.5]))
    assert ids.tolist() == [3, 7] and payload.view(np.float64).tolist() == [-1.5, 0.25] and dtype == np.float64
    with pytest.raises(TypeError):
        oc._projection_table([1], np.array(["a"]))


def test_refusals_without_a_device():
    feats = util._MemGroup()
    feats.attrs.update({"shape": (64, 64), "tile_shape": (32, 32), "halo": (4, 4), "tiles_in_mask": [0, 1]})
    with pytest.raises(ValueError, match="mask"):
        oc.compute_object_features({"features": feats, "input_size": None, "original_size": None}, np.zeros((64, 64), np.int32))
    with pytest.raises(NotImplementedError):
        oc.run_prediction_with_object_classifier(["image.tif"], [np.zeros((8, 8), np.int32)], None, "rf.joblib")
