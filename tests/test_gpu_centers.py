"""get_centers_and_bounding_boxes and segmentation_to_one_hot on the device (csrc/centers.cu) against the oracle
(oracle/centers_ref.py, itself pinned to the reference's own code by tests/test_centers_cpu.py), bit for bit: the golden cases,
seeded random label images and volumes at production sizes, the label images AMG and AIS produce, the boundary and squared-EDT
ops on their own, one-hot planes, the device-tensor extension, repeats, refusals, and the prompts fed downstream."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import ndimage
from scipy.spatial import cKDTree

from micro_sam_b200 import _lib, inference, instance_segmentation as iseg, prompt_generators, util
from micro_sam_b200.sample_data import lm_tile
from oracle import centers_ref, sam_ref, unetr_ref
from tests.test_centers_cpu import G, NAMES, ONE_HOT

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_CACHE = {}


def voronoi_labels(shape, n_seeds, seed, background=0.3, sparse=True):
    """Voronoi cells of n_seeds random points (touching objects of irregular shape), a fraction set to background, ids drawn
    from [1, 2^31) when sparse"""
    rng = np.random.default_rng(seed)
    pts = rng.uniform(0, shape, (n_seeds, len(shape)))
    grid = np.stack(np.meshgrid(*[np.arange(s, dtype=np.float32) for s in shape], indexing="ij"), -1).reshape(-1, len(shape))
    cell = cKDTree(pts).query(grid, workers=-1)[1].reshape(shape)
    ids = rng.choice(2 ** 31 - 1, n_seeds, replace=False) + 1 if sparse else np.arange(1, n_seeds + 1)
    ids = np.where(rng.random(n_seeds) < background, 0, ids)
    return ids[cell].astype(np.int64)


def _device(seg, mode):
    ids, c, b = util.get_centers_and_bounding_boxes(seg, mode, device_result=True)
    return ids.cpu().numpy(), c.cpu().numpy(), b.cpu().numpy()


def _assert_equal_oracle(seg, mode):
    ids, c, b = _device(seg, mode)
    rids, rc, rb = centers_ref.get_centers_and_bounding_boxes(seg, mode)
    assert np.array_equal(ids, rids)
    assert np.array_equal(b, rb)
    assert c.dtype == (np.int32 if mode == "v" else np.float64)
    if mode == "v":
        assert np.array_equal(c, rc)
    else:
        assert np.array_equal(c.view(np.int64), rc.view(np.int64))
    return ids, c, b


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("mode", ["v", "p"])
def test_golden_cases(name, mode):
    seg = G[f"{name}__seg"]
    _assert_equal_oracle(seg, mode)
    centers, boxes = util.get_centers_and_bounding_boxes(seg, mode)
    ids = G[f"{name}__ids"]
    assert list(centers) == list(boxes) == [int(i) for i in ids]
    want_c, want_b = G[f"{name}__centers_{mode}"], G[f"{name}__boxes"]
    for k, i in enumerate(ids):
        assert boxes[int(i)] == tuple(int(v) for v in want_b[k])
        assert centers[int(i)] == tuple(want_c[k].tolist())
        assert all(type(v) is (int if mode == "v" else float) for v in centers[int(i)])


@pytest.mark.parametrize("shape,n_seeds", [((1024, 1024), 3000), ((2048, 2048), 6000), ((32, 512, 512), 2500)])
@pytest.mark.parametrize("mode", ["v", "p"])
def test_random_label_images(shape, n_seeds, mode):
    seg = voronoi_labels(shape, n_seeds, seed=len(shape) * 10 + shape[-1] // 512)
    ids, _, _ = _assert_equal_oracle(seg, mode)
    assert len(ids) > 1000
    # the same image as uint32 numpy and as a device int32 tensor
    assert all(np.array_equal(a, b) for a, b in zip(_device(seg.astype(np.uint32), mode), _device(torch.from_numpy(seg).to(DEV).int(), mode)))


def _sam_sd():
    if "sd" not in _CACHE:
        _CACHE["sd"] = sam_ref.seeded_state_dict("vit_test", seed=1)
    return _CACHE["sd"]


def test_amg_and_ais_label_images(tmp_path):
    img = lm_tile((256, 256), 12, seed=2)
    pred = util.get_sam_model("vit_test", device=DEV, state_dict=_sam_sd(), max_batch=1, max_prompts=64)
    amg = iseg.AutomaticMaskGenerator(pred, points_per_side=8)
    amg.initialize(img)
    amg_seg = amg.generate(pred_iou_thresh=0.0, stability_score_thresh=0.0, box_nms_thresh=1.0, with_background=False)
    path = tmp_path / "ais.pt"
    torch.save({"model_state": _sam_sd(), "decoder_state": unetr_ref.seeded_state(seed=9)}, path)
    p2, dec = iseg.get_predictor_and_decoder("vit_test", str(path), device=DEV)
    ais = iseg.InstanceSegmentationWithDecoder(p2, dec)
    ais.initialize(lm_tile((300, 400), 12, seed=2))
    ais_seg = ais.generate(foreground_threshold=0.45, min_size=5)
    for seg in (amg_seg, ais_seg):
        assert seg.dtype == np.uint32 and seg.max() > 1
        for mode in ("v", "p"):
            _assert_equal_oracle(seg, mode)


def _edt_op(mask):
    dims = (ctypes.c_int * mask.ndim)(*mask.shape)
    m = torch.from_numpy(np.ascontiguousarray(mask, dtype=np.uint8)).to(DEV)
    out = torch.empty(mask.shape, dtype=torch.int32, device=DEV)
    ws = torch.empty(3 * ((4 * mask.size + 255) // 256 * 256), dtype=torch.uint8, device=DEV)
    _lib.check(_lib.lib().msam_op_edt_squared(_lib.ptr(m), mask.ndim, dims, _lib.ptr(ws), ws.numel(), _lib.ptr(out), _lib.cur_stream()))
    return out.cpu().numpy()


def test_edt_op_equals_scipy():
    rng = np.random.default_rng(7)
    for shape in ((1, 700), (700, 1), (1, 1), (513, 517), (2050, 2050), (33, 65, 129), (1, 40, 50), (40, 1, 50)):
        for p in (0.002, 0.3):
            m = rng.random(shape) > p
            m.flat[rng.integers(m.size)] = False
            want = np.rint(ndimage.distance_transform_edt(m) ** 2).astype(np.int64)
            assert np.array_equal(_edt_op(m), want), (shape, p)
    for shape in ((5, 9), (4, 6, 3)):   # all feature pixels (all boundary): zero everywhere
        assert not _edt_op(np.zeros(shape, bool)).any()


def test_boundary_op_equals_restatement():
    for seg in [G[f"{n}__seg"] for n in NAMES] + [voronoi_labels((300, 301), 400, 1), voronoi_labels((20, 70, 90), 300, 2)]:
        t = torch.from_numpy(seg.astype(np.int32)).to(DEV)
        out = torch.empty(tuple(s + 2 for s in seg.shape), dtype=torch.uint8, device=DEV)
        dims = (ctypes.c_int * seg.ndim)(*seg.shape)
        _lib.check(_lib.lib().msam_op_label_boundaries(_lib.ptr(t), seg.ndim, dims, _lib.ptr(out), _lib.cur_stream()))
        assert np.array_equal(out.cpu().numpy().astype(bool), centers_ref.inner_boundaries(np.pad(seg, 1)))


@pytest.mark.parametrize("name", ONE_HOT)
def test_one_hot_golden(name):
    ids = G[f"{name}__ids"]
    seg = G[f"{name[len('onehot_'):]}__seg"]
    out = util.segmentation_to_one_hot(seg, ids if len(ids) else None)
    assert out.is_cuda and out.dtype == torch.float32
    assert torch.equal(out.cpu(), torch.from_numpy(G[f"{name}__out"].astype(np.float32)))


def test_one_hot_random():
    seg = voronoi_labels((509, 515), 300, 3, sparse=False)      # plane size not a multiple of 4: the scalar store path
    seg2 = voronoi_labels((12, 100, 128), 150, 4, sparse=False)
    for s in (seg, seg2):
        assert torch.equal(util.segmentation_to_one_hot(s).cpu(), torch.from_numpy(centers_ref.segmentation_to_one_hot(s)))
        rng = np.random.default_rng(0)
        sel = rng.choice(np.arange(1, 400), 60, replace=False)    # a subset, some ids absent
        got = util.segmentation_to_one_hot(torch.from_numpy(s).to(DEV), sel)
        assert torch.equal(got.cpu(), torch.from_numpy(centers_ref.segmentation_to_one_hot(s, sel)))


def test_device_result_matches_dicts_and_repeats():
    seg = voronoi_labels((700, 900), 800, 5)
    for mode in ("v", "p"):
        centers, boxes = util.get_centers_and_bounding_boxes(seg, mode)
        ids, c, b = util.get_centers_and_bounding_boxes(seg, mode, device_result=True)
        assert ids.dtype == torch.int64 and b.dtype == torch.int32 and ids.is_cuda and c.is_cuda and b.is_cuda
        assert list(centers) == ids.tolist()
        assert [tuple(v) for v in c.tolist()] == list(centers.values())
        assert [tuple(v) for v in b.tolist()] == list(boxes.values())
        for _ in range(3):
            _, c2, b2 = util.get_centers_and_bounding_boxes(seg, mode, device_result=True)
            assert torch.equal(c2, c) and torch.equal(b2, b)
    dense = voronoi_labels((200, 300), 100, 5, sparse=False)
    assert torch.equal(util.segmentation_to_one_hot(dense), util.segmentation_to_one_hot(dense))
    assert util.get_centers_and_bounding_boxes(np.zeros((5, 6), np.uint8)) == ({}, {})
    assert util.segmentation_to_one_hot(np.zeros((5, 6), np.uint8)).shape == (0, 1, 5, 6)


def test_refusals():
    seg = G["touching__seg"]
    with pytest.raises(AssertionError, match="Choose either"):
        util.get_centers_and_bounding_boxes(seg, mode="x")
    for f in (lambda s: util.get_centers_and_bounding_boxes(s), lambda s: util.segmentation_to_one_hot(s)):
        with pytest.raises(ValueError, match="integer labels"):
            f(seg.astype(np.float32))
        with pytest.raises(ValueError, match="integer labels"):
            f(torch.from_numpy(seg).double())
        with pytest.raises(ValueError, match="non-negative"):
            f(-seg)
        for big in (np.full((3, 4), 2 ** 31, np.uint32), np.full((3, 4), 2 ** 31, np.int64), np.full((3, 4), 2 ** 63, np.uint64)):
            with pytest.raises(ValueError, match="below 2\\^31"):
                f(big)
        for s in (np.zeros(7, np.int32), np.zeros((2, 3, 4, 5), np.int32)):
            with pytest.raises(ValueError, match="2-D or 3-D"):
                f(s)
        for shape in ((46340, 46340), (1290, 1290, 1290), (0, 5)):   # padded sizes past int32 (broadcast views: nothing is allocated)
            with pytest.raises(ValueError, match="2\\^31"):
                f(np.broadcast_to(np.zeros(1, np.int32), shape))
    for bad in ([], [0, 1], np.array([3, 0])):
        with pytest.raises(RuntimeError, match="No foreground"):
            util.segmentation_to_one_hot(seg, bad)


def test_prompts_feed_generator_and_batched_inference():
    img = lm_tile((256, 256), 12, seed=2)
    seg = voronoi_labels((256, 256), 30, 6, sparse=False)
    ids = np.unique(seg)[1:]
    centers, boxes = util.get_centers_and_bounding_boxes(seg)
    masks = util.segmentation_to_one_hot(seg, ids)
    gen = prompt_generators.PointAndBoxPromptGenerator(2, 1, 3, get_point_prompts=True, get_box_prompts=True)
    coords, labels, bbox_list, _ = gen(masks, [boxes[i] for i in ids], [centers[i] for i in ids], seed=1)
    assert coords.shape == (len(ids), 3, 2) and bbox_list.shape == (len(ids), 4)
    want = torch.tensor([[centers[i][1], centers[i][0]] for i in ids], device=coords.device)
    assert torch.equal(coords[:, 0], want)   # the first positive point is the centre, (x, y)
    pred = util.get_sam_model("vit_test", device=DEV, state_dict=_sam_sd(), max_batch=1, max_prompts=64)
    xyxy = np.array([[b[1], b[0], b[3], b[2]] for b in (boxes[i] for i in ids)])
    pts = np.array([[[centers[i][1], centers[i][0]]] for i in ids])
    out = inference.batched_inference(pred, img, batch_size=16, boxes=xyxy, points=pts, point_labels=np.ones((len(ids), 1)))
    assert out.shape == (256, 256)
