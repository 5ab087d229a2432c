"""PerObjectDistanceTransform on the device (csrc/distance_targets.cu) against the numpy / scipy restatement
(oracle/distance_targets_ref.py), bit for bit in every channel; determinism, the numpy path, the refusals, the 8-connected
components, and the targets feeding the UNETR decoder's training step."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import ndimage

from micro_sam_b200 import _lib, training, util
from oracle import distance_targets_ref as ref
from oracle import sam_ref, unetr_ref
from tests.test_gpu_centers import voronoi_labels

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ALL = dict(instances=True, foreground=True, distances=True, boundary_distances=True)


def _oracle(lab, **kw):
    return ref.per_object_distance_transform(np.asarray(lab), **kw)


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def _assert_bits(got, want):
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    assert got.shape == want.shape and got.dtype == np.float32
    bad = _bits(got) != _bits(want)
    assert not bad.any(), f"{int(bad.sum())} values differ, first at {np.argwhere(bad)[0]}: {got[bad][0]} vs {want[bad][0]}"


def _planted():
    cases = []
    lab = np.zeros((12, 12), np.int64)
    lab[1:8, 1:8] = 1
    lab[3:6, 3:8] = 0                      # C shape
    lab[9, 1:6] = 2
    lab[8:11, 8] = 2                       # thin L: all boundary
    lab[0, 11] = 3                         # single pixel on the edge
    lab[10:12, 10:12] = 3                  # same id, apart: split
    cases.append(lab)
    yy, xx = np.mgrid[:15, :17]
    r2 = (yy - 7) ** 2 + (xx - 8) ** 2
    cases.append(((r2 <= 36) & (r2 >= 9)).astype(np.int64) * 5)   # ring
    diag = np.zeros((6, 6), np.int64)
    diag[[0, 1, 2, 3], [3, 2, 1, 0]] = 4
    diag[4:6, 4:6] = 9
    diag[3, 3] = 9                         # diagonal touch: merged with the block
    cases.append(diag)
    two = np.zeros((4, 6), np.int64)
    two[1, 2:4] = 1
    two[:, 5] = 2
    cases.append(two)
    cases.append(np.full((5, 7), 3, np.int64))   # one object covering the image
    cases.append(np.zeros((4, 4), np.int64))     # empty
    touch = np.zeros((6, 8), np.int64)
    touch[:, :3] = 7
    touch[:, 3:6] = 2
    cases.append(touch)
    return cases


@pytest.mark.parametrize("i", range(7))
@pytest.mark.parametrize("kw", [ALL, dict(), dict(instances=True, min_size=3), dict(ALL, apply_label=False),
                                dict(foreground=False, distance_fill_value=-2.5), dict(distances=False, instances=True),
                                dict(boundary_distances=False, foreground=False)])
def test_planted_cases_bit_exact(i, kw):
    lab = _planted()[i]
    want = _oracle(lab, **kw)
    t = training.PerObjectDistanceTransform(**kw)
    _assert_bits(t(torch.as_tensor(lab, device=DEV)), want)
    _assert_bits(t(lab), want)


@pytest.mark.parametrize("shape,n,seed", [((512, 512), 1200, 1), ((1024, 1024), 1500, 2), ((700, 1300), 1100, 3)])
@pytest.mark.parametrize("min_size,apply_label", [(0, True), (25, True), (0, False)])
def test_voronoi_bit_exact(shape, n, seed, min_size, apply_label):
    lab = voronoi_labels(shape, n, seed)
    if seed == 1:
        lab[:40, :40] = 2 ** 31 - 1   # the largest id
    want = _oracle(lab, min_size=min_size, apply_label=apply_label, **ALL)
    assert int(want[0].max()) > 700
    t = training.PerObjectDistanceTransform(min_size=min_size, apply_label=apply_label, **ALL)
    _assert_bits(t(torch.as_tensor(lab, device=DEV)), want)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64, torch.uint16, torch.float32, torch.float64])
@pytest.mark.parametrize("B", [1, 3])
def test_batches_and_dtypes(dtype, B):
    labs = [voronoi_labels((160, 200), 90, 10 + b, sparse=dtype in (torch.int32, torch.int64, torch.float64)) for b in range(B)]
    if dtype == torch.float32:
        labs = [np.minimum(lab, 2 ** 24) for lab in labs]
    want = np.stack([_oracle(lab, instances=True, min_size=4) for lab in labs])
    x = torch.as_tensor(np.stack(labs), device=DEV).to(dtype)
    t = training.PerObjectDistanceTransform(instances=True, min_size=4)
    got = t(x)
    assert got.shape == (B, 4, 160, 200)
    _assert_bits(got, want)


def test_odd_width_takes_the_scalar_stores():
    lab = voronoi_labels((37, 51), 20, 5)
    t = training.PerObjectDistanceTransform(**ALL)
    _assert_bits(t(torch.as_tensor(np.stack([lab, lab[::-1].copy()]), device=DEV)),
                 np.stack([_oracle(lab, **ALL), _oracle(lab[::-1].copy(), **ALL)]))


def test_repeats_are_bit_identical_and_numpy_matches():
    lab = voronoi_labels((512, 512), 1200, 7)
    t = training.PerObjectDistanceTransform(**ALL)
    x = torch.as_tensor(lab, device=DEV)
    a, b = t(x), t(x)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert np.array_equal(_bits(t(lab)), _bits(a.cpu().numpy()))


def test_components_with_8_connectivity():
    rng = np.random.default_rng(3)
    fg = rng.random((300, 400)) < 0.45
    want, n = ndimage.label(fg, structure=np.ones((3, 3)))
    t = training.PerObjectDistanceTransform(instances=True, foreground=False, distances=False, boundary_distances=False)
    got = t(torch.as_tensor(fg.astype(np.int32), device=DEV))[0].cpu().numpy()
    assert n > 500 and np.array_equal(got, want.astype(np.float32))


def test_refusals():
    t = training.PerObjectDistanceTransform()
    with pytest.raises(ValueError, match="non-negative"):
        t(torch.tensor([[0, -1]], device=DEV))
    with pytest.raises(ValueError, match="2\\^31"):
        t(torch.tensor([[0, 2 ** 31]], device=DEV))
    with pytest.raises(ValueError, match="whole numbers"):
        t(torch.tensor([[0.0, 1.5]], device=DEV))
    with pytest.raises(ValueError, match="\\(H, W\\) or \\(B, H, W\\)"):
        t(torch.zeros(1, 1, 4, 4, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="32768"):
        t(torch.zeros(1, 32769, dtype=torch.int32, device=DEV))
    with pytest.raises(NotImplementedError):
        t(np.zeros((2, 3, 3), np.int32))
    L = _lib.lib()
    lab = torch.zeros(4, 4, dtype=torch.int32, device=DEV)
    out = torch.zeros(3, 4, 4, device=DEV)
    nb = int(L.msam_distance_targets_workspace(1, 4, 4, 1))
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st = _lib.cur_stream()
    assert L.msam_distance_targets_workspace(1, 32769, 4, 1) == -1
    assert L.msam_distance_targets_workspace(2, 32768, 32768, 1) == -1
    call = lambda lab_p, dt, ch, wsb, out_p: L.msam_distance_targets(lab_p, dt, 1, 4, 4, 1, 0, ch, 1.0, _lib.ptr(ws), wsb,  # noqa
                                                                      out_p, st)
    assert call(None, 0, 14, nb, _lib.ptr(out)) != 0
    assert call(_lib.ptr(lab), 0, 14, nb, None) != 0
    assert call(_lib.ptr(lab), 2, 14, nb, _lib.ptr(out)) != 0
    assert call(_lib.ptr(lab), 0, 16, nb, _lib.ptr(out)) != 0
    assert call(_lib.ptr(lab), 0, 0, nb, _lib.ptr(out)) != 0
    assert call(_lib.ptr(lab), 0, 14, nb - 1, _lib.ptr(out)) != 0
    assert L.msam_distance_targets(_lib.ptr(lab), 0, 1, 32769, 1, 1, 0, 14, 1.0, _lib.ptr(ws), nb, _lib.ptr(out), st) != 0
    assert "msam_distance_targets" in L.msam_last_error().decode()
    assert call(_lib.ptr(lab), 0, 14, nb, _lib.ptr(out)) == 0


def test_resize_label_trafo():
    lab = voronoi_labels((50, 61), 30, 4)
    r = training.ResizeLabelTrafo((64, 64), min_size=3)
    got = r(lab)
    want = np.pad(_oracle(lab, instances=True, min_size=3), ((0, 0), (7, 7), (2, 1)))
    _assert_bits(got, want)
    dev = r(torch.as_tensor(np.stack([lab, lab]), device=DEV))
    assert dev.shape == (2, 4, 64, 64)
    _assert_bits(dev[1], want)
    with pytest.raises(AssertionError):
        training.ResizeLabelTrafo((64, 80))(lab)


def _cells(B, H, W, seed):
    rng = np.random.default_rng(seed)
    labs = np.stack([voronoi_labels((H, W), 40, seed + b, background=0.4) for b in range(B)])
    img = np.repeat((labs[:, None] > 0) * 170.0 + rng.normal(40, 8, (B, 1, H, W)), 3, 1).clip(0, 255).astype(np.float32)
    return torch.from_numpy(img), labs


def test_targets_train_the_decoder_as_the_oracle_targets_do():
    sam = util.get_sam_model("vit_test", device=DEV, state_dict=sam_ref.seeded_state_dict("vit_test", seed=1), max_batch=2,
                             max_prompts=64).model
    state = unetr_ref.seeded_state(seed=23, emb=256, feats=(128, 64, 64, 64), deconv=(64, 64, 64, 64), head_in=64)
    net_a, net_b = training.get_unetr(sam, state), training.get_unetr(sam, state)
    x, labs = _cells(2, 128, 128, 30)
    yy = training.PerObjectDistanceTransform(instances=True)(torch.as_tensor(labs, device=DEV))
    want = torch.from_numpy(np.stack([_oracle(lab, instances=True) for lab in labs]))
    _assert_bits(yy, want.numpy())
    la = training.instance_train_iteration(net_a, x, yy[:, 1:], lr=1e-4)
    lb = training.instance_train_iteration(net_b, x, want[:, 1:], lr=1e-4)
    assert torch.equal(la, lb)
    sa, sb = net_a.decoder_state_dict(), net_b.decoder_state_dict()
    assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)
    model = training.TrainableSAM(sam)
    np.random.seed(0)
    li, lu = training.joint_train_iteration(model, net_a, x, yy[:, :1].cpu(), yy[:, 1:].cpu(), iteration=1, n_objects_per_batch=4,
                                            n_sub_iteration=2, lr=1e-4)
    assert torch.isfinite(li) and torch.isfinite(lu)
