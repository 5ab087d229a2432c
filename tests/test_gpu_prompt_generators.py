"""`-m gpu`: the training prompts of csrc/prompts.cu (micro_sam_b200.prompt_generators, training.ConvertToSamInputs /
IterativePromptUpdate / interactive_train_iteration) against torch and the numpy oracle (oracle/prompt_ref.py).

The draws are not numpy's, so the checks are on what must hold for every draw: targets, counts and boxes bit-exact; every point in
the set the reference would draw it from (the oracle's regions), in the reference's order and number; no repeats where the
reference draws without replacement; uniform over the set (chi-square with fixed seeds); reproducible from the seed; no host
synchronisation in a prompt update; and the reference's 8-pass training step (up to 21 tokens per prompt), replayed through the oracle with the prompts the library drew,
gives the oracle's loss and gradients.
"""
import gc
import random

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import prompt_ref as pr

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_SUB = 8               # sub-iterations of the reference trainer: its last pass has 21 tokens per prompt (training decoder)


@pytest.fixture(autouse=True)
def _free_device_memory():
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _label_image(seed, H=96, W=80):
    """disks, two touching squares, objects on the border and in the corner, 1-pixel objects, a large object"""
    rng = np.random.default_rng(seed)
    lab = np.zeros((H, W), np.int64)
    yy, xx = np.mgrid[:H, :W]
    nid = 3
    for _ in range(6):
        cy, cx, r = rng.integers(8, H - 8), rng.integers(8, W - 8), rng.integers(2, 7)
        lab[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = nid
        nid += 2
    lab[40:50, 0:10] = nid; lab[40:50, 10:20] = nid + 1          # touching, on the left border
    lab[0:4, W - 5:W] = nid + 2                                   # top-right corner
    lab[H - 1, 30] = nid + 3; lab[20, 40] = nid + 4               # 1-pixel objects
    lab[60:90, 30:75] = nid + 5                                   # large object
    lab[70:75, 40:45] = nid + 6                                   # a hole inside it
    return lab


def _ids(lab):
    return np.unique(lab)[1:]


# ---------------------------------------------------------------------------------------------------------------------------
# 1. targets, counts, boxes

@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_targets_counts_boxes_are_exact(dtype):
    from micro_sam_b200 import training
    from micro_sam_b200.sam import ResizeLongestSide
    labs = [_label_image(1), _label_image(2)]
    sampled = [_ids(labs[0]), _ids(labs[1])[::2].copy()]          # different object counts per image
    y = torch.from_numpy(np.stack(labs)[:, None]).to(dtype)
    tg, counts, boxes = training._label_targets(y, sampled, torch.device(DEV))
    tr = ResizeLongestSide(1024)
    for b in range(2):
        planes, cnt, bx = pr.one_hot_counts_boxes(labs[b], sampled[b])
        n = len(sampled[b])
        assert np.array_equal(tg[b, :n].cpu().numpy(), planes.astype(np.uint8))
        assert not tg[b, n:].any()
        assert np.array_equal(counts[b, :n].cpu().numpy(), cnt)
        assert np.array_equal(boxes[b, :n].cpu().numpy(), bx)
        ref_xyxy = torch.from_numpy(bx[:, [1, 0, 3, 2]])
        got = tr.apply_boxes_torch(boxes[b, :n][:, [1, 0, 3, 2]].long(), labs[b].shape)
        assert torch.equal(got.cpu(), tr.apply_boxes_torch(ref_xyxy, labs[b].shape))


def test_box_distortion_matches_the_reference_arithmetic():
    from micro_sam_b200 import training
    lab = _label_image(3)
    ids = _ids(lab)
    np.random.seed(11)
    seed = int(np.random.randint(0, 2 ** 64, dtype=np.uint64))
    np.random.seed(11)
    _, _, boxes = training._label_targets(torch.from_numpy(lab[None]), [ids], torch.device(DEV), box_distortion=0.25)
    _, _, bx = pr.one_hot_counts_boxes(lab, ids)
    want = [pr.distort_box(b, 0.25, lab.shape, [pr.uniform01(seed, pr.TAG_BOX, 0, k, d) for d in range(4)]) for k, b in enumerate(bx)]
    assert boxes[0].cpu().tolist() == want
    assert any(w != list(b) for w, b in zip(want, bx.tolist()))


# ---------------------------------------------------------------------------------------------------------------------------
# 2. point-and-box sampling

def _check_points(coords, labels, planes, boxes, n_pos, n_neg, ds, centers=None):
    coords, labels = coords.cpu().numpy(), labels.cpu().numpy()
    assert coords.shape == (len(planes), n_pos + n_neg, 2) and labels.shape == (len(planes), n_pos + n_neg)
    assert (labels[:, :n_pos] == 1).all() and (labels[:, n_pos:] == 0).all()
    for k, (obj, box) in enumerate(zip(planes, boxes)):
        reg = pr.point_box_regions(obj, box, ds)
        xy = coords[k]
        pts = [(int(y), int(x)) for x, y in xy]
        start = 0
        if centers is not None:
            assert pts[0] == (int(centers[k][0]), int(centers[k][1]))
            start = 1
        pos = pts[start:n_pos]
        assert all(reg["positive"][p] for p in pos), k
        n_obj = int(obj.sum())
        if n_pos - start <= n_obj:
            assert len(set(pos)) == len(pos), k                      # without replacement
        n_ring = min(n_neg, int(reg["ring"].sum()))
        ring_pts, fill_pts = pts[n_pos:n_pos + n_ring], pts[n_pos + n_ring:]
        assert all(reg["ring"][p] for p in ring_pts), k
        assert all(reg["fill"][p] for p in fill_pts), k
        assert len(set(ring_pts)) == len(ring_pts) and len(set(fill_pts)) == len(fill_pts), k


@pytest.mark.parametrize("n_pos,n_neg,ds", [(1, 0, 10), (13, 27, 4), (3, 9, 8), (2, 4, 0), (1, 3, 10), (4, 40, 2)])
def test_point_and_box_generator(n_pos, n_neg, ds):
    from micro_sam_b200.prompt_generators import PointAndBoxPromptGenerator
    lab = _label_image(4)
    ids = _ids(lab)
    planes, _, boxes = pr.one_hot_counts_boxes(lab, ids)
    gen = PointAndBoxPromptGenerator(n_pos, n_neg, ds, get_box_prompts=True)
    seg = torch.from_numpy(planes[:, None].astype(np.float32)).to(DEV)
    coords, labels, bx, none = gen(seg, [tuple(b) for b in boxes], seed=5)
    assert none is None and coords.is_cuda and coords.dtype == torch.int64
    assert torch.equal(bx.cpu(), torch.from_numpy(boxes[:, [1, 0, 3, 2]]))
    _check_points(coords, labels, planes, boxes, n_pos, n_neg, ds)
    # the reference test's point counts (R/test/test_prompt_generators.py) with centres as the first positive point
    centers = [np.argwhere(p)[len(np.argwhere(p)) // 2] + 0.7 for p in planes]
    coords, labels, _, _ = gen(seg, [tuple(b) for b in boxes], center_coordinates=centers, seed=6)
    _check_points(coords, labels, planes, boxes, n_pos, n_neg, ds, centers=[c.astype(int) for c in centers])


def test_more_positive_points_than_pixels_and_ring_smaller_than_n_neg():
    from micro_sam_b200.prompt_generators import PointAndBoxPromptGenerator
    lab = np.zeros((20, 20), np.int64)
    lab[5, 5] = 1                    # 1 pixel: 3 positives with replacement
    lab[10:20, 10:20] = 2            # corner object, ds = 1: small ring, the rest from the background
    planes, _, boxes = pr.one_hot_counts_boxes(lab, [1, 2])
    seg = torch.from_numpy(planes[:, None].astype(np.float32)).to(DEV)
    coords, labels, _, _ = PointAndBoxPromptGenerator(3, 30, 1)(seg, [tuple(b) for b in boxes], seed=1)
    c = coords.cpu().numpy()
    assert (c[0, :3] == [5, 5]).all()
    _check_points(coords, labels, planes, boxes, 3, 30, 1)
    assert pr.point_box_regions(planes[1], boxes[1], 1)["ring"].sum() < 30


def test_convert_to_sam_inputs():
    from micro_sam_b200 import training
    from micro_sam_b200.sam import ResizeLongestSide, get_preprocess_shape
    labs = np.stack([_label_image(7), _label_image(8)])[:, None].astype(np.float32)
    x = torch.rand(2, 3, 96, 80) * 255
    conv = training.ConvertToSamInputs(ResizeLongestSide(1024), dilation_strength=3)
    np.random.seed(3)
    recs, sampled = conv(x, torch.from_numpy(labs), 2, 3, get_boxes=True, n_samples=5)
    tr = ResizeLongestSide(1024)
    for b, (rec, ids) in enumerate(zip(recs, sampled)):
        assert len(ids) == 5 and np.all(np.diff(ids) > 0)
        planes, _, boxes = pr.one_hot_counts_boxes(labs[b, 0].astype(np.int64), ids)
        assert torch.equal(rec["boxes"].cpu(), tr.apply_boxes_torch(torch.from_numpy(boxes[:, [1, 0, 3, 2]]), (96, 80)))
        assert rec["point_coords"].shape == (5, 5, 2) and rec["point_labels"].tolist() == [[1, 1, 0, 0, 0]] * 5
        th, tw = get_preprocess_shape(96, 80, 1024)
        raw = torch.round(rec["point_coords"].cpu() / torch.tensor([tw / 80, th / 96]))
        _check_points(raw.long(), rec["point_labels"], planes, boxes, 2, 3, 3)
    recs2, y1h = training.preprocess_batch(recs, torch.from_numpy(labs), sampled)
    assert y1h.shape == (2, 5, 1, 96, 80) and y1h.dtype == torch.float32 and y1h.is_cuda
    ref = torch.stack([torch.stack([torch.from_numpy(labs[b, 0] == i) for i in sampled[b][:5]]) for b in range(2)]).float()[:, :, None]
    assert torch.equal(y1h.cpu(), ref)
    assert all("_one_hot" not in r for r in recs2)
    _, y1h_b = training.preprocess_batch([{k: v for k, v in r.items() if k != "_one_hot"} for r in recs], torch.from_numpy(labs), sampled)
    assert torch.equal(y1h_b, y1h)


# ---------------------------------------------------------------------------------------------------------------------------
# 3. iterative sampling

def _decoder_logits():
    """real low-res logits of the vit_test decoder: 2 images x 12 box-prompted objects x 3 masks"""
    from micro_sam_b200 import util
    from micro_sam_b200.sample_data import lm_tile
    from oracle import sam_ref
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    pred = util.get_sam_model("vit_test", device=DEV, state_dict=sd, max_batch=1, max_prompts=64)
    lows, ious = [], []
    for s in (2, 3):
        img = np.repeat(lm_tile((96, 80), 12, seed=s, dtype="uint8")[..., None], 3, -1)
        pred.set_image(img)
        bx = torch.tensor([[4 + 6 * k, 4 + 4 * k, 30 + 4 * k, 40 + 3 * k] for k in range(12)], dtype=torch.float32)
        bx = pred.transform.apply_boxes_torch(bx, (96, 80)).to(DEV)
        _, iou, low = pred.predict_torch(None, None, boxes=bx, multimask_output=True)
        lows.append(low.float())
        ious.append(iou.float())
    return pred.model, torch.cat(lows), torch.cat(ious), tuple(pred.input_size)


def _check_iterative(coords, labels, targets, preds):
    coords, labels = coords.cpu().numpy(), labels.cpu().numpy()
    assert (labels == [[1, 0]]).all()
    names = []
    for k, (t, p) in enumerate(zip(targets, preds)):
        reg = pr.iterative_regions(t, p)
        (px, py), (nx, ny) = coords[k]
        assert reg["positive"][py, px], (k, reg["positive_set"])
        assert reg["negative"][ny, nx], (k, reg["negative_set"])
        names.append((reg["positive_set"], reg["negative_set"]))
    return names


def test_iterative_points_from_decoder_logits():
    from micro_sam_b200 import prompt_generators as pg
    sam, low, iou, input_size = _decoder_logits()
    n = low.shape[0]
    H, W = 96, 80
    full = sam.postprocess_masks(low, input_size, (H, W)) > 0
    best = iou.argmax(1)
    pred = full[torch.arange(n), best].cpu().numpy()
    rng = np.random.default_rng(0)
    targets = np.zeros((n, H, W), bool)
    for k in range(n):
        ys, xs = np.nonzero(pred[k])
        if k % 4 == 0:
            targets[k] = pred[k]                               # perfect prediction: overlap + box ring
        elif k % 4 == 1:
            targets[k] = np.roll(pred[k], 3, axis=1)           # shifted: FN and FP
        elif k % 4 == 2:
            targets[k, 40:50, 30:40] = True                    # unrelated object
        else:
            targets[k] = pred[k]
            targets[k, rng.integers(0, H), rng.integers(0, W)] = True   # one false negative pixel
        if not targets[k].any():
            targets[k, 5, 5] = True
        if targets[k].all():
            targets[k, 0, 0] = False
    tg = torch.from_numpy(targets.astype(np.uint8)).to(DEV)
    names = set()
    for seed in range(4):
        coords, labels = pg.iterative_points(tg, seed, low_res=low.contiguous(), iou=iou.contiguous(), input_size=input_size)
        names |= set(_check_iterative(coords, labels, targets, pred))
        coords2, _ = pg.iterative_points(tg, seed, pred=torch.from_numpy(pred.astype(np.uint8)).to(DEV))
        assert torch.equal(coords, coords2)                    # the binary-plane path sees the same sets
    assert len(names) >= 2, names


def test_iterative_planted_edge_cases():
    from micro_sam_b200.prompt_generators import IterativePromptGenerator
    H, W = 24, 20
    t = np.zeros((5, H, W), bool)
    p = np.zeros((5, H, W), bool)
    t[0, 5:9, 5:9] = True; p[0] = t[0]                                  # overlap / ring
    t[1, 5:9, 5:9] = True                                               # empty prediction: FN / ring
    t[2] = True; t[2, 0, 0] = False; p[2] = t[2]                        # ring = the one background pixel
    t[3] = True; t[3, 0, :] = False; t[3, 12, 10] = False; p[3] = t[3]  # ring is the background inside the box
    t[4, 0:2, 0:2] = True; p[4, 10:12, 10:12] = True                    # FN and FP
    gen = IterativePromptGenerator()
    seg = torch.from_numpy(t[:, None].astype(np.float32)).to(DEV)
    prd = torch.from_numpy(p[:, None].astype(np.float32)).to(DEV)
    coords, labels, none1, none2 = gen(seg, prd, seed=3)
    assert none1 is None and none2 is None and coords.shape == (5, 2, 2)
    names = _check_iterative(coords, labels, t, p)
    assert names == [("overlap", "ring"), ("fn", "ring"), ("overlap", "ring"), ("overlap", "ring"), ("fn", "fp")]
    assert coords[2, 1].tolist() == [0, 0]
    with pytest.raises(NotImplementedError):
        gen(seg[:, :, None], prd[:, :, None])


# ---------------------------------------------------------------------------------------------------------------------------
# sampling and reproducibility

def test_draws_are_uniform():
    """>= 20k draws over small regions, fixed seeds: chi-square p > 1e-3 for positives (20-pixel object), ring negatives and the
    iterative false negatives"""
    from micro_sam_b200 import prompt_generators as pg
    H, W, N = 16, 16, 1000
    obj = np.zeros((H, W), bool)
    obj[6:10, 5:10] = True                                    # 20 pixels
    tg = torch.from_numpy(np.repeat(obj[None], N, 0).astype(np.uint8)).to(DEV)
    counts = torch.full((N,), 20, dtype=torch.int32, device=DEV)
    boxes = torch.tensor([[4, 3, 12, 12]] * N, dtype=torch.int32, device=DEV)      # a distorted box: ring of 68 pixels
    ring = pr.point_box_regions(obj, (4, 3, 12, 12), 1)["ring"]
    pos_hist, neg_hist = np.zeros((H, W)), np.zeros((H, W))
    for seed in range(20):
        c, _ = pg.sample_points(tg, counts, boxes, 1, 1, 1, seed)
        c = c.cpu().numpy()
        np.add.at(pos_hist, (c[:, 0, 1], c[:, 0, 0]), 1)
        np.add.at(neg_hist, (c[:, 1, 1], c[:, 1, 0]), 1)
    assert pos_hist[~obj].sum() == 0 and neg_hist[~ring].sum() == 0
    assert stats.chisquare(pos_hist[obj]).pvalue > 1e-3
    assert stats.chisquare(neg_hist[ring]).pvalue > 1e-3
    fn_hist = np.zeros((H, W))
    pred = torch.zeros_like(tg)
    for seed in range(20):
        c, _ = pg.iterative_points(tg, seed, pred=pred)
        c = c.cpu().numpy()
        np.add.at(fn_hist, (c[:, 0, 1], c[:, 0, 0]), 1)
    assert fn_hist[~obj].sum() == 0 and stats.chisquare(fn_hist[obj]).pvalue > 1e-3


def test_same_seed_same_points():
    from micro_sam_b200.prompt_generators import PointAndBoxPromptGenerator
    lab = _label_image(9)
    planes, _, boxes = pr.one_hot_counts_boxes(lab, _ids(lab))
    seg = torch.from_numpy(planes[:, None].astype(np.float32)).to(DEV)
    gen = PointAndBoxPromptGenerator(3, 5, 4)
    a = gen(seg, [tuple(b) for b in boxes], seed=123)[0]
    b = gen(seg, [tuple(b) for b in boxes], seed=123)[0]
    c = gen(seg, [tuple(b) for b in boxes], seed=124)[0]
    assert torch.equal(a, b) and not torch.equal(a, c)
    np.random.seed(7)
    d = gen(seg, [tuple(b) for b in boxes])[0]
    np.random.seed(7)
    e = gen(seg, [tuple(b) for b in boxes])[0]
    assert torch.equal(d, e)
    # the first objects' points do not depend on how many objects are in the launch
    f = gen(seg[:3], [tuple(b) for b in boxes[:3]], seed=123)[0]
    assert torch.equal(f, a[:3])


@pytest.mark.parametrize("mask_prob", [0.0, 1.0])
def test_prompt_update_does_not_synchronise(mask_prob):
    from micro_sam_b200 import training
    from micro_sam_b200.sam import ResizeLongestSide
    B, n, H, W = 2, 6, 64, 48
    y = torch.zeros(B, n, 1, H, W, device=DEV)
    for k in range(n):
        y[:, k, :, 5 + 8 * k:10 + 8 * k, 10:20] = 1
    logits = torch.randn(B, n, 1, 256, 256, device=DEV)
    recs = [{"input_size": (1024, 768), "original_size": (H, W), "point_coords": torch.zeros(n, 1, 2, device=DEV),
             "point_labels": torch.ones(n, 1, dtype=torch.int64, device=DEV)} for _ in range(B)]
    upd = training.IterativePromptUpdate(y, ResizeLongestSide(1024), mask_prob=mask_prob)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        recs = upd(recs, None, logits)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert recs[0]["point_coords"].shape == (n, 3, 2) and recs[0]["point_labels"][0].tolist() == [1, 1, 0]
    assert ("mask_inputs" in recs[0]) == (mask_prob == 1.0)


# ---------------------------------------------------------------------------------------------------------------------------
# end to end: interactive_train_iteration against the oracle replaying the library's prompts


def _train_setup():
    from micro_sam_b200 import training, util
    from micro_sam_b200.sample_data import lm_tile
    from oracle import sam_ref
    from tests import mask_prompt_mirror as mmirror
    sd = mmirror.perturbed_state_dict()
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    osam.to(DEV)
    for p in osam.parameters():
        p.requires_grad_(True)
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
    sam.train()
    H = W = 128
    x = torch.stack([torch.from_numpy(np.repeat(lm_tile((H, W), 12, seed=50 + b, dtype="uint8")[None], 3, 0).astype("float32"))
                     for b in range(2)])
    yy, xx = np.mgrid[:H, :W]
    labs = np.zeros((2, 1, H, W), np.float32)
    for k in range(25):
        cy, cx, r = 12 + 24 * (k // 5), 12 + 24 * (k % 5), 6 + k % 4
        labs[0, 0][(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = k + 1
    labs[1] = labs[0][..., ::-1]
    return training, osam, sam, x, torch.from_numpy(labs)


def _record_library_prompts(monkeypatch, training):
    """snapshots of the records at the start of every pass"""
    passes = []

    def snap(recs):
        passes.append([{k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in r.items() if k != "image"} for r in recs])

    orig_loss = training.compute_iterative_loss

    def loss_wrapper(model, batched_inputs, *a, **k):
        snap(batched_inputs)
        return orig_loss(model, batched_inputs, *a, **k)

    class Recording(training.IterativePromptUpdate):
        def __call__(self, batched_inputs, masks, logits):
            out = super().__call__(batched_inputs, masks, logits)
            snap(out)
            return out

    monkeypatch.setattr(training, "compute_iterative_loss", loss_wrapper)
    monkeypatch.setattr(training, "IterativePromptUpdate", Recording)
    return passes


@pytest.mark.parametrize("iteration,mask_prob", [(1, 0.0), (1, 1.0), (0, 0.0), (0, 1.0)])
def test_interactive_train_iteration_against_the_oracle(monkeypatch, iteration, mask_prob):
    """iteration 1: a box per object in pass 0, single mask; iteration 0: one point (+ SAM's padding token) and multimask output
    in pass 0, where the loss takes the best of 3 masks -- so the library and the oracle must choose the same mask per object"""
    from tests.test_gpu_backward import _compare_grads
    from tests.test_gpu_iterative_loss import _oracle_iterative_loss
    training, osam, sam, x, y = _train_setup()
    passes = _record_library_prompts(monkeypatch, training)
    np.random.seed(0)
    random.seed(0)
    sam.zero_decoder_grads()
    m = training.TrainableSAM(sam)
    loss, mask_loss, iou_loss, miou, y_one_hot = training.interactive_train_iteration(m, x, y, iteration=iteration, n_sub_iteration=N_SUB,
                                                                                       mask_prob=mask_prob)
    loss.backward()
    assert len(passes) == N_SUB and y_one_hot.shape == (2, 25, 1, 128, 128)
    n0 = 1 if iteration % 2 == 0 else 0                     # pass 0: one point (even iterations) or a box (odd)
    assert all(p[0].get("point_coords", torch.empty(1, 0, 2)).shape[1] == n0 + 2 * i for i, p in enumerate(passes))
    assert all(("mask_inputs" in p[0]) == (mask_prob == 1.0 and i > 0) for i, p in enumerate(passes))

    def records(dev):
        return [{"image": x[b].clone().to(dev), "original_size": (128, 128),
                 **{k: v.to(dev) for k, v in passes[0][b].items() if k in ("boxes", "point_coords", "point_labels")}} for b in range(2)]
    state = {"i": 0}

    def replay(recs, masks, logits):
        state["i"] += 1
        for b, rec in enumerate(recs):
            snapshot = passes[state["i"]][b]
            rec["point_coords"], rec["point_labels"] = snapshot["point_coords"].to(DEV), snapshot["point_labels"].to(DEV)
            if "mask_inputs" in snapshot:
                rec["mask_inputs"] = logits[b].to(DEV)
            else:
                rec.pop("mask_inputs", None)
        return recs
    oloss, ochoice = _oracle_iterative_loss(osam, records, y_one_hot.cpu(), replay, N_SUB, iteration % 2 == 0)
    oloss.backward()
    if iteration % 2 == 0:
        from tests.test_gpu_iterative_loss import _library_pass0_choice
        state["i"] = 0
        gchoice = _library_pass0_choice(sam, records, y_one_hot.cpu())
        assert all(torch.equal(g, o) for g, o in zip(gchoice, ochoice)), "pass-0 mask choice differs: gradients not comparable"
    ref = dict(osam.cpu().named_parameters())
    r_enc, bad_enc = _compare_grads(sam.encoder_grads(), ref, 1.5e-1, min_cos=0.99)
    r_dec, bad_dec = _compare_grads(sam.decoder_grads(), ref, 1.5e-1, min_cos=0.99)
    print(f"\ninteractive_train_iteration iteration={iteration} mask_prob={mask_prob}: loss {float(loss):.4f} (oracle {float(oloss):.4f}), encoder max "
          f"rel-L2 {max(r_enc.values()):.2e}, decoder max rel-L2 {max(r_dec.values()):.2e}", flush=True)
    assert abs(float(loss) - float(oloss)) < 2e-2
    assert not bad_enc and not bad_dec, (bad_enc, bad_dec)


def test_full_masks_false_gives_the_same_loss():
    training, _, sam, x, y = _train_setup()
    sam.eval()
    out = []
    for full in (True, False):
        np.random.seed(1)
        random.seed(1)
        conv = training.ConvertToSamInputs(training.TrainableSAM(sam).transform)
        recs, ids = conv(x, y, 1, 0, False, 25)
        recs, y1h = training.preprocess_batch(recs, y, ids)
        upd = training.IterativePromptUpdate(y1h, training.TrainableSAM(sam).transform, 0.5)
        with torch.no_grad():
            out.append(training.compute_iterative_loss(training.TrainableSAM(sam), recs, y1h, N_SUB, True, upd, full_masks=full))
    assert all(float(a) == float(b) for a, b in zip(out[0], out[1])), out
