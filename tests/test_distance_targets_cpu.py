"""PerObjectDistanceTransform's restatement (oracle/distance_targets_ref.py) on planted cases, the crop-EDT = whole-image-EDT
identity the device relies on, a numpy form of the device algorithm against the oracle, and the host-side refusals."""
import os
import re

import numpy as np
import pytest
from scipy import ndimage
from scipy.spatial import cKDTree

from oracle import distance_targets_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = np.float32(1e-7)


def pod(labels, **kw):
    return ref.per_object_distance_transform(np.asarray(labels), **kw)


def norm(v):
    v = np.asarray(v, dtype=np.float32)
    return v / (v.max() + EPS)


# ------------------------------------------------------------------------------------------------------------ planted cases
def test_empty_image_holds_fill_values():
    out = pod(np.zeros((5, 7), np.int64), instances=True, distance_fill_value=0.25)
    assert out.shape == (4, 5, 7) and out.dtype == np.float32
    assert np.all(out[0] == 0) and np.all(out[1] == 0) and np.all(out[2:] == np.float32(0.25))


def test_single_pixel_object():
    lab = np.zeros((5, 5), np.int64)
    lab[2, 3] = 9
    out = pod(lab, instances=True)
    assert out[0, 2, 3] == 1 and out[1, 2, 3] == 1
    assert out[2, 2, 3] == 0 and out[3, 2, 3] == 0   # 0 / (0 + eps)
    assert np.all(out[2:, lab == 0] == 1)


def test_two_pixel_object_rounds_half_to_even():
    lab = np.zeros((4, 6), np.int64)
    lab[1, 2:4] = 1   # centroid x = 2.5 -> 2
    out = pod(lab, boundary_distances=False, foreground=False)
    assert out[0, 1, 2] == 0 and out[0, 1, 3] == np.float32(1) / (np.float32(1) + EPS)
    lab = np.zeros((4, 6), np.int64)
    lab[1, 3:5] = 1   # centroid x = 3.5 -> 4
    out = pod(lab, boundary_distances=False, foreground=False)
    assert out[0, 1, 4] == 0 and out[0, 1, 3] > 0


def test_c_shape_corrects_the_centre():
    lab = np.zeros((9, 9), np.int64)
    lab[1:8, 1:8] = 1
    lab[3:6, 3:8] = 0   # C open to the right; the centroid (4, ~3.7) -> (4, 4) lies in the gap
    mask = lab == 1
    bnd = ref.find_boundaries_inner(lab)
    e = np.where(mask, ndimage.distance_transform_edt(~bnd).astype(np.float32), 0)
    c = np.unravel_index(np.argmax(e), e.shape)
    assert not mask[4, 4] and mask[c]
    out = pod(lab, foreground=False)
    yy, xx = np.nonzero(mask)
    cd = np.linalg.norm(np.stack([yy - c[0], xx - c[1]]).astype(np.float32), axis=0)
    assert np.array_equal(out[0][mask], norm(cd))
    assert np.array_equal(out[1][mask], norm(e[mask]))


def test_ring_corrects_the_centre():
    yy, xx = np.mgrid[:15, :15]
    r2 = (yy - 7) ** 2 + (xx - 7) ** 2
    lab = ((r2 <= 36) & (r2 >= 9)).astype(np.int64)
    out = pod(lab, foreground=False, boundary_distances=False)
    assert out[0][7, 7] == 1   # background: fill
    mask = lab == 1
    assert np.count_nonzero(out[0][mask] == 0) == 1   # the corrected centre is an object pixel


def test_thin_line_takes_the_crop_origin():
    # every pixel of an L is a boundary pixel: E = 0 on the object, the argmax is the crop's first pixel (0, 0) of the box,
    # which is not in the object; centre distances are measured from there
    lab = np.zeros((6, 6), np.int64)
    lab[1, 1:5] = 1
    lab[1:5, 4] = 1
    # centroid (1.86, 3.29) -> (2, 3) is not in the L
    out = pod(lab, foreground=False)
    mask = lab == 1
    yy, xx = np.nonzero(mask)
    cd = np.linalg.norm(np.stack([yy - 1, xx - 1]).astype(np.float32), axis=0)
    assert np.array_equal(out[0][mask], norm(cd))
    assert np.all(out[1][mask] == 0)
    diag = np.zeros((5, 5), np.int64)
    diag[[0, 1, 2, 3], [3, 2, 1, 0]] = 4   # anti-diagonal, 8-connected: one object, box origin (0, 0) outside it
    out = pod(diag, foreground=False)
    m = diag == 4
    yy, xx = np.nonzero(m)
    cd = np.linalg.norm(np.stack([yy, xx]).astype(np.float32), axis=0)   # centroid (1.5, 1.5) -> (2, 2) is not in it either
    assert np.array_equal(out[0][m], norm(cd))


def test_no_boundary_on_the_image_edge():
    lab = np.zeros((6, 8), np.int64)
    lab[:, :3] = 1   # touches top, bottom and left edges; boundary only at column 2
    out = pod(lab, foreground=False, distances=False)
    e = np.broadcast_to(np.float32([2, 1, 0]), (6, 3))
    assert np.array_equal(out[0][:, :3], norm(e))


def test_one_id_merged_across_a_diagonal_and_split_when_apart():
    lab = np.zeros((6, 6), np.int64)
    lab[0:2, 0:2] = 5
    lab[2:4, 2:4] = 5   # touches the first block diagonally: one object
    lab[5, 5] = 5       # apart: a second object
    out = pod(lab, instances=True, foreground=False, distances=False, boundary_distances=False)[0]
    assert set(np.unique(out[lab == 5])) == {1, 2}
    assert np.all(out[0:4, 0:4][lab[0:4, 0:4] == 5] == 1) and out[5, 5] == 2
    out = pod(lab, instances=True, apply_label=False, foreground=False, distances=False, boundary_distances=False)[0]
    assert np.all(out[lab == 5] == 1)


def test_touching_ids_stay_apart():
    lab = np.zeros((4, 6), np.int64)
    lab[:, :3] = 7
    lab[:, 3:] = 2
    out = pod(lab, instances=True, foreground=False, distances=False, boundary_distances=False)[0]
    assert np.all(out[:, :3] == 1) and np.all(out[:, 3:] == 2)
    out = pod(lab, instances=True, apply_label=False, foreground=False, distances=False, boundary_distances=False)[0]
    assert np.all(out[:, :3] == 2) and np.all(out[:, 3:] == 1)   # ascending ids: 2 -> 1, 7 -> 2


def test_min_size_removes_and_renumbers():
    lab = np.zeros((8, 8), np.int64)
    lab[0, 0] = 3            # 1 pixel
    lab[2:4, 2:4] = 8        # 4 pixels
    lab[5:8, 5:8] = 1        # 9 pixels
    out = pod(lab, instances=True, min_size=4)
    assert out[0, 0, 0] == 0 and out[1, 0, 0] == 0 and out[2, 0, 0] == 1
    assert np.all(out[0][2:4, 2:4] == 1) and np.all(out[0][5:8, 5:8] == 2)


def test_object_covering_the_image():
    out = pod(np.full((4, 5), 3, np.int64), instances=True)
    assert np.all(out[0] == 1) and np.all(out[1] == 1)
    assert np.all(out[3] == 0)   # no boundary anywhere: defined as 0
    assert out[2][2, 2] == 0 and out[2][0, 0] == out[2].max()   # centroid (1.5, 2) -> (2, 2)


@pytest.mark.parametrize("sel", range(1, 16))
def test_channel_selection(sel):
    names = ["instances", "foreground", "distances", "boundary_distances"]
    kw = {n: bool(sel >> i & 1) for i, n in enumerate(names)}
    lab = np.zeros((6, 6), np.int64)
    lab[1:5, 1:4] = 2
    full = pod(lab, instances=True)
    out = pod(lab, **kw)
    assert np.array_equal(out, full[[i for i in range(4) if sel >> i & 1]])


def test_default_channels_and_fill():
    lab = np.zeros((6, 6), np.int64)
    lab[1:5, 1:4] = 2
    out = pod(lab, distance_fill_value=-3.0)
    assert out.shape == (3, 6, 6)
    assert np.all(out[1:, lab == 0] == np.float32(-3))


# ------------------------------------------------------------------------------------------------ the device's shortcut
def voronoi(shape, n, seed, background=0.3):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(0, shape, (n, 2))
    grid = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, 2)
    cell = cKDTree(pts).query(grid)[1].reshape(shape)
    ids = rng.choice(2 ** 31 - 1, n, replace=False) + 1
    return np.where(rng.random(n) < background, 0, ids)[cell].astype(np.int64)


def noisy(shape, seed, smooth):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, 6, shape)
    if smooth:
        lab = ndimage.median_filter(lab, 5)
    return lab.astype(np.int64)


CASES = [("voronoi", s) for s in range(4)] + [("noisy", s) for s in range(3)] + [("smooth", s) for s in range(3)]


def make(kind, seed):
    if kind == "voronoi":
        return voronoi((70, 90), 60, seed)
    return noisy((48, 64), seed, kind == "smooth")


@pytest.mark.parametrize("kind,seed", CASES)
def test_crop_edt_equals_whole_image_edt(kind, seed):
    lab = ref.label_components(make(kind, seed))
    bnd = ref.find_boundaries_inner(lab)
    whole = ndimage.distance_transform_edt(~bnd)
    for k, bb in enumerate(ndimage.find_objects(lab)):
        if bb is None:
            continue
        mask = lab[bb] == k + 1
        crop = ndimage.distance_transform_edt(~bnd[bb])
        assert np.array_equal(crop[mask], whole[bb][mask]), k


def squared_edt(feature: np.ndarray) -> np.ndarray:
    """Exact integer squared distance to the nearest True pixel (from scipy's nearest-feature indices)."""
    idx = ndimage.distance_transform_edt(~feature, return_distances=False, return_indices=True)
    yy, xx = np.indices(feature.shape)
    return (idx[0] - yy).astype(np.int64) ** 2 + (idx[1] - xx).astype(np.int64) ** 2


def device_algorithm(labels, min_size=0, apply_label=True, fill=1.0):
    """The device's algorithm in numpy: one whole-image integer EDT, integer per-object maxima, the packed argmax key,
    rint centroids; every float is one rounding of an integer expression."""
    lab = ref.label_components(labels) if apply_label else ref.relabel_consecutive(labels)
    if min_size:
        lab = ref.size_filter(lab, min_size)
    H, W = lab.shape
    n = int(lab.max())
    bnd = ref.find_boundaries_inner(lab)
    d2 = squared_edt(bnd) if bnd.any() else np.zeros(lab.shape, np.int64)
    fgm = lab > 0
    k = lab[fgm] - 1
    yy, xx = np.nonzero(fgm)
    i = yy * W + xx
    key = (d2[fgm] << 32) | (0xFFFFFFFF - i)
    best = np.zeros(n, np.int64)
    np.maximum.at(best, k, key)
    cnt = np.bincount(k, minlength=n)
    cy = np.rint(np.bincount(k, yy, n) / cnt).astype(np.int64)
    cx = np.rint(np.bincount(k, xx, n) / cnt).astype(np.int64)
    y0 = np.full(n, H); x0 = np.full(n, W)
    np.minimum.at(y0, k, yy); np.minimum.at(x0, k, xx)
    bmax = best >> 32
    inside = lab[cy, cx] == np.arange(1, n + 1)
    bi = 0xFFFFFFFF - (best & 0xFFFFFFFF)
    cy = np.where(inside, cy, np.where(bmax > 0, bi // W, y0))
    cx = np.where(inside, cx, np.where(bmax > 0, bi % W, x0))
    c2 = (yy - cy[k]) ** 2 + (xx - cx[k]) ** 2
    cmax = np.zeros(n, np.int64)
    np.maximum.at(cmax, k, c2)
    csq = lambda v: np.sqrt(np.asarray(v, np.float32))
    bsq = lambda v: np.sqrt(np.asarray(v, np.float64)).astype(np.float32)
    cd = np.full(lab.shape, np.float32(fill), np.float32)
    bd = cd.copy()
    cd[fgm] = csq(c2) / (csq(cmax[k]) + EPS)
    bd[fgm] = bsq(d2[fgm]) / (bsq(bmax[k]) + EPS)
    return np.stack([lab.astype(np.float32), fgm.astype(np.float32), cd, bd])


@pytest.mark.parametrize("kind,seed", CASES)
@pytest.mark.parametrize("min_size,apply_label", [(0, True), (25, True), (0, False)])
def test_device_algorithm_equals_oracle(kind, seed, min_size, apply_label):
    lab = make(kind, seed)
    want = pod(lab, instances=True, min_size=min_size, apply_label=apply_label)
    got = device_algorithm(lab, min_size, apply_label)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_device_algorithm_on_planted_shapes():
    lab = np.zeros((12, 12), np.int64)
    lab[1:8, 1:8] = 1
    lab[3:6, 3:8] = 0
    lab[9, 1:6] = 2
    lab[8:11, 8] = 2
    lab[0, 11] = 3
    assert np.array_equal(device_algorithm(lab).view(np.uint32), pod(lab, instances=True).view(np.uint32))
    full = np.full((5, 7), 4, np.int64)
    assert np.array_equal(device_algorithm(full).view(np.uint32), pod(full, instances=True).view(np.uint32))


# ------------------------------------------------------------------------------------------------------------ host side
def test_refusals_before_the_device():
    from micro_sam_b200 import training
    with pytest.raises(NotImplementedError, match="directed"):
        training.PerObjectDistanceTransform(directed_distances=True)
    with pytest.raises(NotImplementedError, match="sampling"):
        training.PerObjectDistanceTransform(sampling=(1.0, 2.0))
    with pytest.raises(ValueError, match="min_size"):
        training.PerObjectDistanceTransform(min_size=-1)
    with pytest.raises(ValueError, match="no output channel"):
        training.PerObjectDistanceTransform(distances=False, boundary_distances=False, foreground=False)
    t = training.PerObjectDistanceTransform()
    with pytest.raises(NotImplementedError, match="3-D"):
        t(np.zeros((2, 4, 4), np.int32))
    with pytest.raises(ValueError, match="2-D"):
        t(np.zeros(4, np.int32))
    with pytest.raises(ValueError, match="integers"):
        t(np.zeros((4, 4), np.complex64))
    with pytest.raises(NotImplementedError, match="constant"):
        training.ResizeLabelTrafo((8, 8), padding="reflect")


def test_header_declares_the_entry_points():
    with open(os.path.join(ROOT, "include", "msam_b200.h")) as f:
        h = f.read()
    assert re.search(r"int64_t msam_distance_targets_workspace\(int B, int H, int W, int apply_label\);", h)
    assert re.search(r"int msam_distance_targets\(const void\* labels, int label_dtype, int B, int H, int W, int apply_label, "
                     r"int min_size, int channels,\s+float fill, void\* ws, int64_t ws_bytes, float\* out, void\* stream\);", h)
