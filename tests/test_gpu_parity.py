"""`-m gpu` parity tests: the CUDA path (through the C ABI / the reference-facing Python API) against the oracle.

Tolerances (SURVEY.md 8c; the reference states none -- its inference is fp32, ours uses bf16 MMA operands with fp32
accumulation / residual stream / softmax):  encoder rel-L2 <= 2e-2; low-res logits rel-L2 <= 3e-2; iou_pred abs <= 2e-2;
integer stages (boxes, area, stability counts, NMS keep set, painting) bit-exact GIVEN the same low-res logits.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _diag():
    spec = importlib.util.spec_from_file_location("gpu_diag", os.path.join(HERE, "gpu_diag.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("section", ["gemm", "wgrad", "ln", "attn", "encoder", "decoder", "post", "nms"])
def test_ops(section):
    d = _diag()
    d.SECTIONS[section]()
    assert d.RESULTS and all(d.RESULTS), f"{section}: {sum(d.RESULTS)}/{len(d.RESULTS)} checks ok"


def _partition_equal(a, b):
    """label images equal up to a relabelling."""
    if a.shape != b.shape or (a == 0).sum() != (b == 0).sum() or not np.array_equal(a == 0, b == 0):
        return False
    pairs = np.unique(np.stack([a.ravel(), b.ravel()], 1), axis=0)
    return len(pairs) == len(np.unique(a)) == len(np.unique(b))


@pytest.fixture(scope="module")
def models():
    from oracle import sam_ref
    from micro_sam_b200 import util
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    pred = util.get_sam_model("vit_test", state_dict=sd, max_batch=4, max_prompts=64)
    return sam_ref.SamPredictor(osam), pred


def test_to_image_and_embeddings(models):
    from oracle import amg_ref
    from micro_sam_b200 import util
    from micro_sam_b200.sample_data import lm_tile
    opred, pred = models
    img = lm_tile((512, 512), 40, seed=0)
    assert np.array_equal(util._to_image(img), amg_ref.to_image(img))
    ref = amg_ref.precompute_image_embeddings_2d(opred, img)
    got = util.precompute_image_embeddings(pred, img)
    assert got["features"].shape == (1, 256, 64, 64) and got["input_size"] == (1024, 1024) and got["original_size"] == (512, 512)
    rel = np.linalg.norm(got["features"] - ref["features"]) / np.linalg.norm(ref["features"])
    assert rel < 2e-2, rel
    # tiled: 4 tiles for 512^2 / tile 256 / halo 16 (test/test_util.py:179-208), each tile normalised on its own
    tiled = util.precompute_image_embeddings(pred, img, tile_shape=(256, 256), halo=(16, 16), batch_size=3)
    feats = tiled["features"]
    assert sorted(feats.keys()) == ["0", "1", "2", "3"] and feats.attrs["tile_shape"] == (256, 256)
    tile1 = amg_ref.precompute_image_embeddings_2d(opred, img[0:272, 240:512])
    rel = np.linalg.norm(feats["1"][:] - tile1["features"]) / np.linalg.norm(tile1["features"])
    assert feats["1"].attrs["original_size"] == (272, 272) and rel < 2e-2, rel
    # 3d
    vol = np.stack([img, img[::-1]])
    e3 = util.precompute_image_embeddings(pred, vol, batch_size=2)
    assert e3["features"].shape == (2, 1, 256, 64, 64)
    assert np.allclose(e3["features"][0], got["features"], atol=1e-5)


@pytest.mark.parametrize("shape", [(512, 512), (300, 500)])
def test_amg_against_oracle(models, shape):
    """End to end AMG.  (1) float stages within tolerance of the oracle; (2) every integer stage bit-exact when the
    oracle is fed the SAME low-res logits the GPU produced."""
    from oracle import amg_ref
    from micro_sam_b200 import instance_segmentation as iseg
    from micro_sam_b200.sample_data import lm_tile
    opred, pred = models
    img = lm_tile(shape, 30, seed=3)
    amg = iseg.AutomaticMaskGenerator(pred, points_per_side=6)
    amg.initialize(img)
    d = amg.crop_list[0]
    oamg = amg_ref.AutomaticMaskGenerator(opred, points_per_side=6, points_per_batch=12)
    oamg.initialize(img)
    od = oamg._crop_list[0]
    # (1) float stages
    assert np.abs(d["iou_preds"].cpu().numpy() - od["iou_preds"].numpy()).max() < 2e-2
    # (2) integer stages from identical logits: patch the oracle predictor to return the GPU low-res logits
    low = d["low_res"].cpu().view(-1, 3, 256, 256)
    iou = d["iou_preds"].cpu().view(-1, 3)
    state = {"i": 0}

    def fake_predict_torch(point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True,
                           return_logits=False):
        n = point_coords.shape[0]
        s = state["i"]
        state["i"] += n
        masks = opred.model.postprocess_masks(low[s:s + n], opred.input_size, opred.original_size)
        return masks, iou[s:s + n], low[s:s + n]

    orig = opred.predict_torch
    opred.predict_torch = fake_predict_torch
    try:
        oamg2 = amg_ref.AutomaticMaskGenerator(opred, points_per_side=6, points_per_batch=12)
        oamg2.initialize(img)
    finally:
        opred.predict_torch = orig
    od2 = oamg2._crop_list[0]
    assert np.array_equal(d["boxes"].cpu().numpy(), od2["boxes"].numpy())
    assert np.array_equal(d["stability_score"].cpu().numpy(), od2["stability_score"].numpy(), equal_nan=True)
    assert np.array_equal(d["area"].cpu().numpy(), np.array([amg_ref.area_from_rle(r) for r in od2["rles"]]))
    for kw in (dict(pred_iou_thresh=0.0, stability_score_thresh=0.0), dict(pred_iou_thresh=0.2, stability_score_thresh=0.6),
               dict(pred_iou_thresh=0.3, stability_score_thresh=0.8, box_nms_thresh=0.3)):
        recs = amg.generate(output_mode="binary_mask", **kw)
        orecs = oamg2.generate(output_mode="binary_mask", **kw)
        assert len(recs) == len(orecs), (kw, len(recs), len(orecs))
        for a, b in zip(recs, orecs):
            assert a["bbox"] == b["bbox"] and a["area"] == b["area"] and np.array_equal(a["segmentation"], b["segmentation"])
            assert a["point_coords"] == b["point_coords"]
        rles = amg.generate(output_mode="rle", **kw)
        orles = oamg2.generate(output_mode="rle", **kw)
        assert [r["segmentation"] for r in rles] == [r["segmentation"] for r in orles]
        seg = amg.generate(output_mode="instance_segmentation", **kw)
        oseg = oamg2.generate(output_mode="instance_segmentation", **kw)
        assert _partition_equal(seg, oseg), kw
        assert np.array_equal(seg, amg.generate(output_mode="instance_segmentation", **kw))  # deterministic


def test_errors(models):
    _, pred = models
    from micro_sam_b200 import util
    pred.reset_image()
    with pytest.raises(RuntimeError):
        pred.get_image_embedding()
    with pytest.raises(RuntimeError):
        pred.predict_torch(torch.zeros(1, 1, 2), torch.ones(1, 1))
    with pytest.raises(RuntimeError):
        util.get_sam_model("vit_b", device="cpu", state_dict={})


def test_batched_inference_against_oracle(models):
    """inference.batched_inference (boxes, cfg4 recipe): float stages within tolerance, integer stages bit-exact given the
    GPU's own low-res logits."""
    from oracle import amg_ref
    from micro_sam_b200 import inference
    from micro_sam_b200.sample_data import lm_tile, random_boxes
    opred, pred = models
    img = lm_tile((512, 512), 30, seed=5)
    boxes = random_boxes(20, (512, 512), seed=1)
    recs = inference.batched_inference(pred, img, batch_size=8, boxes=boxes, return_instance_segmentation=False)
    orecs = amg_ref.batched_inference(opred, img, batch_size=8, boxes=boxes, return_instance_segmentation=False)
    assert len(recs) == len(orecs) == 20
    iou_g = np.array([r["predicted_iou"] for r in recs]); iou_o = np.array([r["predicted_iou"] for r in orecs])
    assert np.abs(iou_g - iou_o).max() < 2e-2
    agree = np.mean([(r["segmentation"].cpu().numpy() == o["segmentation"].numpy()).mean() for r, o in zip(recs, orecs)])
    assert agree > 0.98, agree
    # integer stages: feed the oracle the GPU low-res logits
    low = torch.stack([r["logits"] for r in recs]).cpu()          # (20,1,256,256)
    iou = torch.tensor(iou_g, dtype=torch.float32)[:, None]
    state = {"i": 0}

    def fake(point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True, return_logits=False):
        n = boxes.shape[0]
        s = state["i"]; state["i"] += n
        return opred.model.postprocess_masks(low[s:s + n], opred.input_size, opred.original_size), iou[s:s + n], low[s:s + n]

    orig = opred.predict_torch
    opred.predict_torch = fake
    try:
        orecs2 = amg_ref.batched_inference(opred, img, batch_size=8, boxes=boxes, return_instance_segmentation=False)
        state["i"] = 0
        oseg = amg_ref.batched_inference(opred, img, batch_size=8, boxes=boxes, return_instance_segmentation=True)
    finally:
        opred.predict_torch = orig
    for r, o in zip(recs, orecs2):
        assert r["bbox"] == o["bbox"] and r["area"] == int(o["area"]) and r["seg_id"] == o["seg_id"]
        assert np.array_equal(r["segmentation"].cpu().numpy(), o["segmentation"].numpy())
        assert r["stability_score"] == o["stability_score"] or (np.isnan(r["stability_score"]) and np.isnan(o["stability_score"]))
    seg = inference.batched_inference(pred, img, batch_size=8, boxes=boxes)
    assert _partition_equal(seg, oseg)
    with pytest.raises(ValueError):
        inference.batched_inference(pred, img, batch_size=8)
    # mask_threshold="auto" (local Otsu per mask, a16): same low-res logits -> identical thresholds, masks, boxes, painting
    recs_a = inference.batched_inference(pred, img, batch_size=8, boxes=boxes[:6], return_instance_segmentation=False,
                                         mask_threshold="auto")
    low = torch.stack([r["logits"] for r in recs_a]).cpu()
    iou = torch.tensor([r["predicted_iou"] for r in recs_a], dtype=torch.float32)[:, None]
    state["i"] = 0
    opred.predict_torch = fake
    try:
        orecs_a = amg_ref.batched_inference(opred, img, batch_size=8, boxes=boxes[:6], return_instance_segmentation=False,
                                            mask_threshold="auto")
        state["i"] = 0
        oseg_a = amg_ref.batched_inference(opred, img, batch_size=8, boxes=boxes[:6], mask_threshold="auto")
    finally:
        opred.predict_torch = orig
    for r, o in zip(recs_a, orecs_a):
        assert r["bbox"] == o["bbox"] and r["area"] == int(o["area"])
        assert np.array_equal(r["segmentation"].cpu().numpy(), o["segmentation"].numpy())
    seg_a = inference.batched_inference(pred, img, batch_size=8, boxes=boxes[:6], mask_threshold="auto")
    assert _partition_equal(seg_a, oseg_a)


def test_device_to_image_and_finish_segmentation_bit_exact(models):
    """a1 / a20 on the device: msam_to_image == util._to_image (== oracle) bit for bit; msam_finish_segmentation ==
    util._finish_segmentation (ids included) and == the oracle up to relabelling."""
    from oracle import amg_ref
    from micro_sam_b200 import _lib, util
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 60000, (333, 517)).astype("uint16"), rng.normal(5, 3, (256, 300)).astype("float32"),
            rng.integers(0, 255, (100, 120, 3)).astype("uint8"), rng.random((64, 80, 2)), np.full((32, 32), 3, "int16"),
            rng.normal(0, 1e-3, (50, 60, 1)).astype("float32")]
    for im in imgs:
        got = util._to_image_device(im, "cuda").cpu().numpy()
        assert np.array_equal(got, amg_ref.to_image(im)), (im.dtype, im.shape)
    # finish_segmentation
    yy, xx = np.mgrid[:200, :260]
    seg = np.zeros((200, 260), np.int32)
    for k in range(40):
        cy, cx, r = rng.integers(0, 200), rng.integers(0, 260), rng.integers(3, 30)
        seg[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = k + 1
    seg[50:60, :] = 7   # a label split into several components by overpainting, and one touching itself diagonally only
    seg[100, 100] = 99; seg[101, 101] = 99
    L = _lib.lib()
    for (mn, wb) in ((0, 0), (0, 1), (25, 0), (40, 1)):
        d = torch.from_numpy(seg).cuda()
        out = torch.empty(200, 260, dtype=torch.int32, device="cuda")
        ws = torch.empty(4 * 200 * 260 + 4096 + 8, dtype=torch.int32, device="cuda")
        _lib.check(L.msam_finish_segmentation(_lib.ptr(d), 200, 260, mn, wb, _lib.ptr(out), _lib.ptr(ws), _lib.cur_stream()))
        got = out.cpu().numpy().view(np.uint32)
        ref = util._finish_segmentation(seg.astype(np.uint32), mn, True, bool(wb))
        assert np.array_equal(got, ref), (mn, wb)
    full = np.ones((64, 64), np.int32)   # no background pixel at all: the single component is the largest segment
    d = torch.from_numpy(full).cuda()
    out = torch.empty(64, 64, dtype=torch.int32, device="cuda")
    ws = torch.empty(4 * 64 * 64 + 4096 + 8, dtype=torch.int32, device="cuda")
    _lib.check(L.msam_finish_segmentation(_lib.ptr(d), 64, 64, 0, 1, _lib.ptr(out), _lib.ptr(ws), _lib.cur_stream()))
    assert np.array_equal(out.cpu().numpy().view(np.uint32), util._finish_segmentation(full.astype(np.uint32), 0, True, True))


def test_tiled_amg_against_oracle(models):
    """TiledAutomaticMaskGenerator (a13): tiles as crops, per-tile filters + NMS, cross-tile NMS, global painting.
    Integer stages bit-exact given the GPU's low-res logits; tiled embeddings within tolerance."""
    from oracle import amg_ref
    from micro_sam_b200 import instance_segmentation as iseg
    from micro_sam_b200.sample_data import lm_tile
    opred, pred = models
    img = lm_tile((300, 420), 30, seed=7)
    tile_shape, halo = (160, 224), (24, 24)
    amg = iseg.TiledAutomaticMaskGenerator(pred, points_per_side=4)
    amg.initialize(img, tile_shape=tile_shape, halo=halo, batch_size=2)
    assert len(amg.crop_list) == 4 and amg.crop_boxes[3] == [200, 136, 420, 300]
    lows = [d["low_res"].cpu().view(-1, 3, 256, 256) for d in amg.crop_list]
    ious = [d["iou_preds"].cpu().view(-1, 3) for d in amg.crop_list]
    calls = {"i": 0}

    def fake(point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True, return_logits=False):
        t = calls["i"]
        calls["i"] += 1
        return opred.model.postprocess_masks(lows[t], opred.input_size, opred.original_size), ious[t], lows[t]

    oamg_f = amg_ref.TiledAutomaticMaskGenerator(opred, points_per_side=4, points_per_batch=16)
    oamg_f.initialize(img, tile_shape=tile_shape, halo=halo)       # float path: embeddings + decoder on the oracle
    for d, od in zip(amg.crop_list, oamg_f._crop_list):
        assert np.abs(d["iou_preds"].cpu().numpy() - od["iou_preds"].numpy()).max() < 2e-2
    orig = opred.predict_torch
    opred.predict_torch = fake
    try:
        oamg = amg_ref.TiledAutomaticMaskGenerator(opred, points_per_side=4, points_per_batch=16)
        oamg.initialize(img, tile_shape=tile_shape, halo=halo)
    finally:
        opred.predict_torch = orig
    for d, od in zip(amg.crop_list, oamg._crop_list):
        assert np.array_equal(d["boxes"].cpu().numpy(), od["boxes"].numpy())
        assert np.array_equal(d["stability_score"].cpu().numpy(), od["stability_score"].numpy(), equal_nan=True)
    for kw in (dict(pred_iou_thresh=0.0, stability_score_thresh=0.0), dict(pred_iou_thresh=0.1, stability_score_thresh=0.6),
               dict(pred_iou_thresh=0.0, stability_score_thresh=0.5, crop_nms_thresh=0.2)):
        recs = amg.generate(output_mode="binary_mask", **kw)
        orecs = oamg.generate(output_mode="binary_mask", **kw)
        assert len(recs) == len(orecs), (kw, len(recs), len(orecs))
        for a, b in zip(recs, orecs):
            assert a["bbox"] == b["bbox"] and a["area"] == b["area"] and a["crop_box"] == b["crop_box"]
            assert np.array_equal(a["segmentation"], b["segmentation"])
        seg = amg.generate(output_mode="instance_segmentation", **kw)
        oseg = oamg.generate(output_mode="instance_segmentation", **kw)
        assert seg.shape == (300, 420) and _partition_equal(seg, oseg), kw
    # offloaded state (per-tile logits in pinned host memory, only the survivors travel back): identical results
    amg_off = iseg.TiledAutomaticMaskGenerator(pred, points_per_side=4)
    amg_off.initialize(img, tile_shape=tile_shape, halo=halo, batch_size=2, offload_state=True)
    assert not amg_off.crop_list[0]["low_res"].is_cuda and amg_off.crop_list[0]["boxes"].is_cuda
    kw = dict(pred_iou_thresh=0.1, stability_score_thresh=0.6)
    assert np.array_equal(amg_off.generate(**kw), amg.generate(**kw))
    for a, b in zip(amg_off.generate(output_mode="binary_mask", **kw), amg.generate(output_mode="binary_mask", **kw)):
        assert a["bbox"] == b["bbox"] and np.array_equal(a["segmentation"], b["segmentation"])
    state = amg_off.get_state()          # AMG state round trip into a fresh generator (no hidden geometry)
    fresh = iseg.TiledAutomaticMaskGenerator(pred, points_per_side=4)
    fresh.set_state(state)
    assert np.array_equal(fresh.generate(**kw), amg.generate(**kw))


def test_mask_nms_bit_exact_vs_reference_golden():
    """a19: device mask NMS == the reference's own `_batched_mask_nms` outputs (golden, IoU and IoMin) incl. the IoU matrix."""
    from micro_sam_b200 import util
    z = np.load(os.path.join(HERE, "golden", "util.npz"))
    m = torch.from_numpy(np.unpackbits(z["nms_masks"], axis=-1)[..., :64].astype(bool).reshape(24, 64, 64))
    boxes, scores = torch.from_numpy(z["nms_boxes"]).float(), torch.from_numpy(z["nms_scores"])
    keep, mat = util.batched_mask_nms(m, boxes, scores, 0.3, False, return_matrix=True)
    assert np.array_equal(mat.cpu().numpy(), z["nms_iou_matrix"])
    for thr in (0.3, 0.9):
        assert util.batched_mask_nms(m, boxes, scores, thr, False).tolist() == z[f"nms_keep_iou_{thr}"].tolist()
        assert util.batched_mask_nms(m, boxes, scores, thr, True).tolist() == z[f"nms_keep_iomin_{thr}"].tolist()
    # apply_nms end to end against the oracle restatement
    from oracle import amg_ref
    recs = [{"segmentation": m[k], "bbox": [int(boxes[k][0]), int(boxes[k][1]), int(boxes[k][2] - boxes[k][0]), int(boxes[k][3] - boxes[k][1])],
             "predicted_iou": float(scores[k]), "stability_score": 1.0} for k in range(24)]
    seg = util.apply_nms(recs, min_size=5, nms_thresh=0.3)
    area = m.flatten(1).sum(1)
    idx = torch.arange(24)[area > 5]
    keep = amg_ref.batched_mask_nms(m[idx], boxes[idx], scores[idx], 0.3, False)
    oseg = amg_ref.mask_data_to_segmentation([{"segmentation": m[k].numpy(), "area": int(area[k])} for k in idx[keep].tolist()],
                                             shape=(64, 64), min_object_size=5)
    assert _partition_equal(seg, oseg)


def test_tiled_apply_nms_vs_reference_golden():
    """a19 tiled variant: util.apply_nms on records with `global_bbox` == oracle (itself pinned on the reference's
    `_calculate_tiled_mask_overlap_matrix` / `_batched_tiled_mask_nms` outputs, tests/golden/tiled_nms.npz)."""
    from micro_sam_b200 import util
    from oracle import amg_ref
    z = np.load(os.path.join(HERE, "golden", "tiled_nms.npz"))
    n = int(z["n"])
    recs = [{"segmentation": torch.from_numpy(z[f"mask_{k}"]), "bbox": z["boxes"][k].tolist(),
             "global_bbox": z["global_boxes"][k].tolist(), "predicted_iou": float(z["scores"][k]), "stability_score": 1.0}
            for k in range(n)]
    for kw in (dict(min_size=0, nms_thresh=0.3), dict(min_size=20, nms_thresh=0.9), dict(min_size=0, nms_thresh=0.3,
                                                                                        intersection_over_min=True)):
        seg = util.apply_nms(recs, **kw)
        oseg = amg_ref.apply_nms(recs, **kw)
        assert seg.shape == tuple(z["inferred_shape"]) and _partition_equal(seg, oseg), kw


def test_batched_tiled_inference_against_oracle(models):
    """a18: prompts routed to tiles, tile-local decoding, `global_bbox` records, global painting; optimize_memory path
    (per-tile apply_nms + first-come stitching).  Integer stages bit-exact given the GPU's low-res logits."""
    from oracle import amg_ref
    from micro_sam_b200 import inference, util
    from micro_sam_b200.sample_data import lm_tile, random_boxes
    opred, pred = models
    img = lm_tile((300, 420), 30, seed=9)
    tile_shape, halo = (160, 224), (24, 24)
    boxes = random_boxes(24, (300, 420), seed=3)
    emb = util.precompute_image_embeddings(pred, img, ndim=2, tile_shape=tile_shape, halo=halo, to_numpy=False)
    recs = inference.batched_tiled_inference(pred, img, batch_size=8, image_embeddings=emb, boxes=boxes,
                                             return_instance_segmentation=False)
    assert len(recs) == 24 and all("global_bbox" in r for r in recs)
    # oracle on the GPU's low-res logits: the records come back tile by tile, in prompt order inside a tile
    low = torch.stack([r["logits"] for r in recs]).cpu()
    iou = torch.tensor([r["predicted_iou"] for r in recs], dtype=torch.float32)[:, None]
    state = {"i": 0}

    def fake(point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True, return_logits=False):
        k = boxes.shape[0]
        s0 = state["i"]; state["i"] += k
        return opred.model.postprocess_masks(low[s0:s0 + k], opred.input_size, opred.original_size), iou[s0:s0 + k], low[s0:s0 + k]

    oemb = amg_ref.precompute_tiled_embeddings_2d(opred, img, tile_shape, halo)
    orig = opred.predict_torch
    opred.predict_torch = fake
    try:
        orecs = amg_ref.batched_tiled_inference(opred, img, 8, image_embeddings=oemb, boxes=boxes, return_instance_segmentation=False)
        state["i"] = 0
        oseg = amg_ref.batched_tiled_inference(opred, img, 8, image_embeddings=oemb, boxes=boxes)
    finally:
        opred.predict_torch = orig
    assert len(orecs) == 24
    for r, o in zip(recs, orecs):
        assert r["bbox"] == o["bbox"] and r["global_bbox"] == o["global_bbox"] and r["area"] == int(o["area"])
        assert np.array_equal(r["segmentation"].cpu().numpy(), o["segmentation"].numpy())
    seg = inference.batched_tiled_inference(pred, img, batch_size=8, image_embeddings=emb, boxes=boxes)
    assert seg.shape == (300, 420) and _partition_equal(seg, oseg)
    # optimize_memory: per-tile NMS + stitching (reference semantics: earlier tiles win)
    seg2 = inference.batched_tiled_inference(pred, img, batch_size=8, image_embeddings=emb, boxes=boxes, optimize_memory=True,
                                             min_size=0)
    assert seg2.shape == (300, 420) and seg2.dtype == np.uint32 and seg2.max() > 0


def test_amg_crop_layers_against_oracle(models):
    """a13 with crop_n_layers=1: 1 + 4 crops, each embedded on its own from the globally normalised image, points of the
    down-scaled grid, crop-edge filter, cross-crop NMS preferring smaller crops.  Integer stages bit-exact given the GPU's
    low-res logits."""
    from oracle import amg_ref
    from micro_sam_b200 import instance_segmentation as iseg
    from micro_sam_b200.sample_data import lm_tile
    opred, pred = models
    img = lm_tile((240, 320), 25, seed=11)
    kw0 = dict(points_per_side=4, crop_n_layers=1, crop_n_points_downscale_factor=2)
    amg = iseg.AutomaticMaskGenerator(pred, **kw0)
    amg.initialize(img)
    assert len(amg.crop_list) == 5 and len(amg.crop_list[1]["iou_preds"]) == 2 * 2 * 3
    lows = [d["low_res"].cpu().view(-1, 3, 256, 256) for d in amg.crop_list]
    ious = [d["iou_preds"].cpu().view(-1, 3) for d in amg.crop_list]
    calls = {"i": 0}

    def fake(point_coords, point_labels, boxes=None, mask_input=None, multimask_output=True, return_logits=False):
        t = calls["i"]
        calls["i"] += 1
        return opred.model.postprocess_masks(lows[t], opred.input_size, opred.original_size), ious[t], lows[t]

    oamg_f = amg_ref.AutomaticMaskGenerator(opred, points_per_batch=64, **kw0)
    oamg_f.initialize(img)                                          # float path: per-crop embeddings + decoder on the oracle
    assert oamg_f._crop_boxes == amg.crop_boxes
    for d, od in zip(amg.crop_list, oamg_f._crop_list):
        assert np.abs(d["iou_preds"].cpu().numpy() - od["iou_preds"].numpy()).max() < 2e-2
    orig = opred.predict_torch
    opred.predict_torch = fake
    try:
        oamg = amg_ref.AutomaticMaskGenerator(opred, points_per_batch=64, **kw0)
        oamg.initialize(img)
    finally:
        opred.predict_torch = orig
    for d, od in zip(amg.crop_list, oamg._crop_list):
        assert np.array_equal(d["boxes"].cpu().numpy(), od["boxes"].numpy())
    for kw in (dict(pred_iou_thresh=0.0, stability_score_thresh=0.0), dict(pred_iou_thresh=0.0, stability_score_thresh=0.5,
                                                                            crop_nms_thresh=0.3)):
        recs = amg.generate(output_mode="binary_mask", **kw)
        orecs = oamg.generate(output_mode="binary_mask", **kw)
        assert len(recs) == len(orecs), (kw, len(recs), len(orecs))
        for a, b in zip(recs, orecs):
            assert a["bbox"] == b["bbox"] and a["area"] == b["area"] and a["crop_box"] == b["crop_box"]
            assert np.array_equal(a["segmentation"], b["segmentation"])
        seg = amg.generate(output_mode="instance_segmentation", **kw)
        oseg = oamg.generate(output_mode="instance_segmentation", **kw)
        assert _partition_equal(seg, oseg), kw
    # a15: min_mask_region_area > 0 (holes / islands removal, re-boxing, NMS preferring unchanged masks)
    kw = dict(pred_iou_thresh=0.0, stability_score_thresh=0.0, box_nms_thresh=0.95, crop_nms_thresh=0.95, min_mask_region_area=40)
    recs = amg.generate(output_mode="binary_mask", **kw)
    orecs = oamg.generate(output_mode="binary_mask", **kw)
    assert len(recs) == len(orecs) and len(recs) > 0
    for a, b in zip(recs, orecs):
        assert a["bbox"] == b["bbox"] and a["area"] == b["area"] and np.array_equal(a["segmentation"], b["segmentation"])
    assert _partition_equal(amg.generate(output_mode="instance_segmentation", **kw), oamg.generate(output_mode="instance_segmentation", **kw))



def test_model_level_prompt_encoder_and_mask_decoder(models):
    """Row (b): the `predictor.model` duck type -- `prompt_encoder(points, boxes, masks)`, `get_dense_pe()`,
    `mask_decoder(image_embeddings, image_pe, sparse, dense, multimask_output)`, `load_state_dict` -- used the way
    micro_sam/training/trainable_sam.py:88-106 uses it, against the oracle modules on the same image embedding."""
    opred, pred = models
    osam, sam = opred.model, pred.model
    from micro_sam_b200.sample_data import lm_tile
    from micro_sam_b200 import util
    img = util._to_image(lm_tile((1024, 1024), 60, seed=4))
    opred.set_image(img)
    feat = opred.features
    pe = sam.prompt_encoder.get_dense_pe()
    assert pe.shape == (1, 256, 64, 64)
    assert torch.allclose(pe.cpu(), osam.prompt_encoder.get_dense_pe(), atol=2e-5)
    g = torch.Generator().manual_seed(0)
    P = 9
    pts = torch.rand(P, 2, 2, generator=g) * 1024
    lbl = torch.tensor([[1, 0], [1, 1], [1, -1]] * 3)
    boxes = torch.sort(torch.rand(P, 2, 2, generator=g) * 1024, dim=1)[0].reshape(P, 4)
    masks = torch.randn(P, 1, 256, 256, generator=g) * 4
    cases = [dict(points=(pts, lbl), boxes=None, masks=None), dict(points=None, boxes=boxes, masks=None),
             dict(points=(pts, lbl), boxes=boxes, masks=None), dict(points=None, boxes=None, masks=masks),
             dict(points=(pts[:, :1], lbl[:, :1]), boxes=None, masks=masks)]
    for kw in cases:
        with torch.no_grad():
            osp, ode = osam.prompt_encoder(**kw)
        sp, de = sam.prompt_encoder(**kw)
        assert sp.shape == osp.shape and de.shape == ode.shape, (sp.shape, osp.shape, de.shape, ode.shape)
        assert torch.allclose(sp.cpu(), osp, atol=1e-4)
        assert torch.allclose(de.cpu(), ode, atol=2e-3, rtol=1e-3)
        for mm in (True, False):
            with torch.no_grad():
                olow, oiou = osam.mask_decoder(image_embeddings=feat, image_pe=osam.prompt_encoder.get_dense_pe(),
                                               sparse_prompt_embeddings=osp, dense_prompt_embeddings=ode, multimask_output=mm)
            low, iou = sam.mask_decoder(image_embeddings=feat.cuda(), image_pe=pe, sparse_prompt_embeddings=sp,
                                        dense_prompt_embeddings=de, multimask_output=mm)
            assert low.shape == olow.shape and iou.shape == oiou.shape
            rel = float((low.cpu() - olow).norm() / olow.norm())
            assert rel < 3e-2 and float((iou.cpu() - oiou).abs().max()) < 2e-2, (list(kw), mm, rel)
    # a dense embedding that is NOT the prompt encoder's no-mask view takes the general (per-prompt keys) path: same result
    sp, de = sam.prompt_encoder(points=(pts, lbl), boxes=None, masks=None)
    low_fast, _ = sam.mask_decoder(image_embeddings=feat.cuda(), image_pe=pe, sparse_prompt_embeddings=sp,
                                   dense_prompt_embeddings=de, multimask_output=True)
    low_gen, _ = sam.mask_decoder(image_embeddings=feat.cuda(), image_pe=pe, sparse_prompt_embeddings=sp,
                                  dense_prompt_embeddings=de.clone(), multimask_output=True)
    assert float((low_fast - low_gen).norm() / low_fast.norm()) < 2e-2
    # load_state_dict rebuilds the engine; identical weights -> identical outputs; perturbed weights -> different outputs
    sd = sam.state_dict()
    assert set(dict(sam.named_parameters())) == set(sd) and len(list(sam.parameters())) == len(sd)
    sam.load_state_dict(sd)
    low2, _ = sam.mask_decoder(image_embeddings=feat.cuda(), image_pe=sam.prompt_encoder.get_dense_pe(),
                               sparse_prompt_embeddings=sp, dense_prompt_embeddings=sam.prompt_encoder(points=(pts, lbl))[1],
                               multimask_output=True)
    assert torch.equal(low2, low_fast)
    with pytest.raises(RuntimeError):
        sam.load_state_dict({"nope": torch.zeros(1)})


def test_trainable_sam_forward_and_loss(models):
    """a21 / a22 (forward half of cfg 5): TrainableSAM.preprocess / image_embeddings_oft / forward and SamTrainer._compute_loss
    on the GPU kernels against the oracle restatement (oracle/train_ref.py): floats within the usual tolerances; the loss
    statistics kernel is additionally checked against the oracle loss evaluated on the GPU's OWN logits (tight tolerance)."""
    from oracle import train_ref
    from micro_sam_b200 import training
    from micro_sam_b200.sample_data import lm_tile
    opred, pred = models
    om, m = train_ref.TrainableSAM(opred.model), training.TrainableSAM(pred.model)
    g = torch.Generator().manual_seed(0)
    B, n_obj, H, W = 2, 5, 96, 128
    imgs = [torch.from_numpy(np.repeat(lm_tile((H, W), 12, seed=20 + b, dtype="uint8")[None], 3, 0).astype("float32")) for b in range(B)]
    pts = [torch.rand(n_obj, 1, 2, generator=g) * torch.tensor([1024.0, 768.0]) for _ in range(B)]
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    y_one_hot = [torch.stack([(((yy - 20 - 12 * k) ** 2 + (xx - 30 - 18 * k) ** 2) < (8 + 2 * k) ** 2).float()[None] for k in range(n_obj)])
                 for _ in range(B)]

    def records():
        return [{"image": im.clone(), "original_size": (H, W), "point_coords": p.clone(), "point_labels": torch.ones(n_obj, 1)}
                for im, p in zip(imgs, pts)]
    with torch.no_grad():
        oemb, orecs = om.image_embeddings_oft(records())
    emb, recs = m.image_embeddings_oft(records())
    assert tuple(recs[0]["input_size"]) == tuple(orecs[0]["input_size"]) == (768, 1024)
    assert float((emb.cpu() - oemb).norm() / oemb.norm()) < 2e-2
    for mm in (True, False):
        with torch.no_grad():
            oout = om(orecs, oemb, multimask_output=mm)
            oloss = train_ref.compute_loss(oout, y_one_hot)
        out = m(recs, emb, multimask_output=mm)
        for a, b in zip(out, oout):
            assert a["masks"].shape == b["masks"].shape == (n_obj, 3 if mm else 1, H, W)
            assert float((a["low_res_masks"].cpu() - b["low_res_masks"]).norm() / b["low_res_masks"].norm()) < 3e-2
            assert float((a["masks"].cpu() - b["masks"]).norm() / b["masks"].norm()) < 3e-2
            assert float((a["iou_predictions"].cpu() - b["iou_predictions"]).abs().max()) < 2e-2
        loss = training.compute_loss(m(recs, emb, multimask_output=mm, return_masks=False), y_one_hot)
        for got, ref in zip(loss, oloss):
            assert abs(float(got) - float(ref)) < 2e-2, (mm, [float(v) for v in loss], [float(v) for v in oloss])
        # the loss kernel itself: oracle loss on the GPU's own logits (bit-identical interpolation, fp32 sums)
        same = [{"masks": a["masks"].cpu(), "iou_predictions": a["iou_predictions"].cpu()} for a in out]
        with torch.no_grad():
            eloss = train_ref.compute_loss(same, y_one_hot)
        for got, ref in zip(loss, eloss):
            assert abs(float(got) - float(ref)) < 2e-4, (mm, [float(v) for v in loss], [float(v) for v in eloss])
    best_masks, best_logits = training.get_best_masks(out)
    assert best_masks.shape == (B, n_obj, 1, H, W) and best_logits.shape == (B, n_obj, 1, 256, 256)


def test_interactive_segmentation_against_oracle(models):
    """f1: `B200SamPredictor.predict` through micro_sam's interactive entry points (segment_from_points / _box /
    _box_and_points / _mask incl. the mask-prompt logits) against the oracle predictor fed the same prompts."""
    from micro_sam_b200 import prompt_based_segmentation as pbs, util
    from micro_sam_b200.sample_data import lm_tile
    opred, pred = models
    img = util._to_image(lm_tile((300, 420), 30, seed=21))
    opred.set_image(img)
    pred.set_image(img)
    assert pred.original_size == (300, 420) and tuple(pred.input_size) == tuple(opred.input_size)

    def check(got, ref, what):
        (m, s, l), (om, os_, ol) = got, ref
        assert m.shape == om.shape and s.shape == os_.shape and l.shape == ol.shape, what
        assert np.abs(s - os_).max() < 2e-2, (what, s, os_)
        assert np.linalg.norm(l - ol) / np.linalg.norm(ol) < 3e-2, what
        assert (m == om).mean() > 0.98, (what, (m == om).mean())

    pts, lbl = np.array([[150, 200], [40, 60]]), np.array([1, 0])
    got = pbs.segment_from_points(pred, pts, lbl, return_all=True)
    check(got, opred.predict(point_coords=pts[:, ::-1], point_labels=lbl, multimask_output=False), "points")
    got = pbs.segment_from_points(pred, pts[:1], lbl[:1], return_all=True)          # single positive point: best of 3
    om, os_, ol = opred.predict(point_coords=pts[:1, ::-1], point_labels=lbl[:1], multimask_output=True)
    assert got[0].shape == (1, 300, 420) and (got[0][0] == om[np.argmax(os_)]).mean() > 0.98
    box = np.array([50, 80, 200, 300])
    check(pbs.segment_from_box(pred, box, return_all=True), opred.predict(box=box[[1, 0, 3, 2]], multimask_output=False), "box")
    check(pbs.segment_from_box_and_points(pred, box, pts, lbl, return_all=True),
          opred.predict(point_coords=pts[:, ::-1], point_labels=lbl, box=box[[1, 0, 3, 2]], multimask_output=False), "box+points")
    mask = np.zeros((300, 420), "uint8")
    mask[60:180, 100:260] = 1
    got = pbs.segment_from_mask(pred, mask, return_all=True)
    ref = opred.predict(mask_input=pbs._compute_logits_from_mask(mask), box=pbs._compute_box_from_mask(mask), multimask_output=False)
    check(got, ref, "mask+box")


def test_large_inputs_beyond_the_former_size_caps():
    """Advisor finding (round 1): filter_nms rejected n > 8192 and finish_segmentation images above 2048 x 2048.  Both run on
    global-memory workspaces now: 12288 boxes (points_per_side 64 x 3 masks) against the oracle NMS, a 2304 x 2560 label image
    against the host assembly."""
    import ctypes
    from oracle import amg_ref
    from micro_sam_b200 import _lib, util
    g = torch.Generator().manual_seed(5)
    n = 12288
    xy = torch.rand(n, 2, generator=g) * 1800
    wh = torch.rand(n, 2, generator=g) * 200 + 8
    boxes = torch.cat([xy, xy + wh], 1).round().to(torch.int32)
    scores = torch.rand(n, generator=g)
    keep = torch.empty(n, dtype=torch.int32, device="cuda")
    nk = torch.zeros(1, dtype=torch.int32, device="cuda")
    z4 = (ctypes.c_int32 * 4)(0, 0, 0, 0)
    bd, sd = boxes.cuda().contiguous(), scores.cuda().contiguous()
    _lib.check(_lib.lib().msam_amg_filter_nms(_lib.ptr(bd), _lib.ptr(sd), _lib.ptr(sd), n, 0, 0.0, 0.0, 0.5, z4, z4, _lib.ptr(keep),
                                              _lib.ptr(nk), _lib.cur_stream()))
    got = keep[: int(nk.item())].cpu().long()
    ref = amg_ref.nms(boxes.float(), scores, 0.5)
    assert len(got) == len(ref) > 1000 and torch.equal(got, ref)
    rng = np.random.default_rng(0)
    H, W = 2304, 2560
    seg = np.zeros((H, W), np.int32)
    for k in range(300):
        cy, cx, r = rng.integers(0, H), rng.integers(0, W), rng.integers(10, 120)
        seg[max(cy - r, 0):cy + r, max(cx - r, 0):cx + r] = k + 1
    d = torch.from_numpy(seg).cuda()
    out = torch.empty(H, W, dtype=torch.int32, device="cuda")
    ws = torch.empty(util.finish_ws_size(H, W), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().msam_finish_segmentation(_lib.ptr(d), H, W, 50, 1, _lib.ptr(out), _lib.ptr(ws), _lib.cur_stream()))
    assert np.array_equal(out.cpu().numpy().view(np.uint32), util._finish_segmentation(seg.astype(np.uint32), 50, True, True))


def test_precompute_state_round_trip(models, tmp_path):
    """precompute_state.precompute_state: embeddings container + cached AMG state for a folder of images; a second generator built from
    the cache (cache_amg_state load path) segments exactly like the one that computed it."""
    from micro_sam_b200 import precompute_state as ps, util
    from micro_sam_b200.sample_data import lm_tile
    _, pred = models
    os.makedirs(tmp_path / "in")
    imgs = [lm_tile((200, 240), 12, seed=50 + k) for k in range(2)]
    for k, im in enumerate(imgs):
        np.save(tmp_path / "in" / f"im{k}.npy", im)
    ps.precompute_state(str(tmp_path / "in"), str(tmp_path / "out"), pattern="*.npy", predictor=pred, precompute_amg_state=True)
    for k, im in enumerate(imgs):
        zpath = str(tmp_path / "out" / f"im{k}.zarr")
        assert os.path.exists(os.path.join(zpath, "amg_state.pickle"))
        emb = util.precompute_image_embeddings(pred, im, zpath)                 # loads: the signature matches
        amg = ps.cache_amg_state(pred, im, emb, zpath, verbose=False)     # loads the pickle (32 x 32 grid, the default)
        kw = dict(pred_iou_thresh=0.5, stability_score_thresh=0.5, box_nms_thresh=0.7)
        seg = amg.generate(**kw)
        from micro_sam_b200 import instance_segmentation as iseg
        ref = iseg.AutomaticMaskGenerator(pred)
        ref.initialize(im, image_embeddings=emb)
        assert np.array_equal(seg, ref.generate(**kw))


def test_rank_sharded_tiled_amg_emulated_on_one_gpu(models):
    """The multi-rank tiled AMG (instance_segmentation._generate_distributed) without a second GPU: every 'rank' initialises its tile
    shard in this process, the instance tables are concatenated in rank order (= what the all-gather returns) and stitched; the result
    must equal the single-process label image bit for bit, for 1, 2 and 4 ranks.  (tests/test_gpu_multi.py runs the same over NCCL.)"""
    from micro_sam_b200 import instance_segmentation as iseg
    from micro_sam_b200.sample_data import lm_tile
    _, pred = models
    img = lm_tile((500, 700), 40, seed=13)
    # 2 x 2 tiles whose halo reaches the image border on every side: the random-init model predicts near-full-crop masks, which the
    # near-crop-edge filter (instance_segmentation.py:99-132) removes at every INTERIOR tile edge -- with ordinary halos nothing
    # survives and the comparison would be vacuous
    tile_shape, halo = (250, 350), (250, 350)
    ref_amg = iseg.TiledAutomaticMaskGenerator(pred, points_per_side=4)
    ref_amg.initialize(img, tile_shape=tile_shape, halo=halo, batch_size=2)
    ref = ref_amg.generate(pred_iou_thresh=0.0, stability_score_thresh=0.0, crop_nms_thresh=0.3, with_background=False)
    assert ref.max() > 0
    tabs1 = None
    for world in (1, 2, 4):
        gens, locs = [], []
        for r in range(world):
            a = iseg.TiledAutomaticMaskGenerator(pred, points_per_side=4)
            a.initialize(img, tile_shape=tile_shape, halo=halo, batch_size=2, rank=r, world_size=world)
            gens.append(a)
            locs.append(a._local_instance_tables(0.0, 0.0, 0.7))
        tab = {k: torch.cat([l[k] for l in locs]) for k in locs[0]}
        if tabs1 is None:
            tabs1 = tab
        same_tab = {k: bool(tab[k].shape == tabs1[k].shape and torch.equal(tab[k], tabs1[k])) for k in tab}
        seg = gens[0]._stitch_gathered(tab, 0.3, False)
        ndiff = int((seg != ref).sum())
        print(f"world {world}: {int(tab['gbox'].shape[0])} gathered instances, tables equal to world 1: {same_tab}, "
              f"{int(seg.max())} labels (single process {int(ref.max())}), {ndiff} differing pixels")
        assert all(same_tab.values()), (world, same_tab)
        assert ndiff == 0, (world, ndiff)
