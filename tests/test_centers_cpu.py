"""The oracle of get_centers_and_bounding_boxes / segmentation_to_one_hot (oracle/centers_ref.py) against the reference's own
code (tests/golden/centers.npz, written by make_centers_golden.py), the inner-boundary rule on planted cases, and the fp64
centroid identity the device relies on (int64 sums divided once equal numpy's float64 mean while the sums stay below 2^53)."""
import os

import numpy as np
import pytest

from oracle import centers_ref

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "centers.npz"))
NAMES = sorted({k.split("__")[0] for k in G.files if k.endswith("__seg")})
ONE_HOT = sorted({k.split("__")[0] for k in G.files if k.startswith("onehot_") and k.endswith("__out")})


def test_golden_covers_the_cases():
    assert {"touching", "concave", "borders", "thin", "sparse_ids", "stack3d"} <= set(NAMES)
    assert G["stack3d__seg"].ndim == 3
    assert int(G["sparse_ids__ids"].max()) == 2 ** 31 - 1
    # a selected id absent from the image leaves an empty last plane
    assert not G["onehot_borders__out"][-1].any() and G["onehot_borders__out"][:-1].reshape(3, -1).any(1).all()


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("mode", ["v", "p"])
def test_oracle_equals_reference(name, mode):
    seg = G[f"{name}__seg"]
    ids, centers, boxes = centers_ref.get_centers_and_bounding_boxes(seg, mode)
    assert np.array_equal(ids, G[f"{name}__ids"])
    assert np.array_equal(boxes, G[f"{name}__boxes"])
    want = G[f"{name}__centers_{mode}"]
    assert centers.dtype == want.dtype
    assert np.array_equal(centers.view(np.int64), want.view(np.int64))   # bit for bit, fp64 included


def test_concave_centres_lie_inside_and_centroids_outside():
    seg = G["concave__seg"]
    for k, c in zip(G["concave__ids"], G["concave__centers_v"]):
        assert seg[tuple(c)] == k
    cy, cx = (int(round(v)) for v in G["concave__centers_p"][1])   # the ring's centroid is its hole
    assert seg[cy, cx] != 2


@pytest.mark.parametrize("name", ONE_HOT)
def test_one_hot_oracle_equals_reference(name):
    ids = G[f"{name}__ids"]
    seg = G[f"{name[len('onehot_'):]}__seg"]
    out = centers_ref.segmentation_to_one_hot(seg, ids if len(ids) else None)
    assert out.dtype == np.float32
    assert np.array_equal(out, G[f"{name}__out"].astype(np.float32))


def test_one_hot_refusals():
    seg = G["thin__seg"]
    for bad in ([], [0, 2]):
        with pytest.raises(RuntimeError, match="No foreground"):
            centers_ref.segmentation_to_one_hot(seg, np.array(bad, np.int64))


def _cross_boundaries_loop(lab):
    """rule 2 by a loop over pixels and their in-grid cross neighbours"""
    out = np.zeros(lab.shape, bool)
    for p in np.ndindex(lab.shape):
        if lab[p] == 0:
            continue
        for ax in range(lab.ndim):
            for d in (-1, 1):
                q = list(p)
                q[ax] += d
                if 0 <= q[ax] < lab.shape[ax] and lab[tuple(q)] != lab[p]:
                    out[p] = True
    return out


def test_inner_boundaries_planted():
    # a 3 x 3 block: only its centre is interior; background is never a boundary
    lab = np.zeros((5, 5), np.int64)
    lab[1:4, 1:4] = 7
    want = np.zeros((5, 5), bool)
    want[1:4, 1:4] = True
    want[2, 2] = False
    assert np.array_equal(centers_ref.inner_boundaries(lab), want)
    # two touching objects: both sides of the shared edge are boundary; the array edge is not a boundary by itself (a label
    # filling the whole array has no boundary: neighbours outside are ignored)
    lab = np.array([[1, 1, 2, 2]] * 3)
    assert np.array_equal(centers_ref.inner_boundaries(lab), np.array([[0, 1, 1, 0]] * 3, bool))
    assert not centers_ref.inner_boundaries(np.full((4, 4), 3)).any()
    # diagonal contact is not a boundary (connectivity 1)
    lab = np.zeros((4, 4), np.int64)
    lab[:2, :2], lab[2:, 2:] = 1, 2
    lab[0, 0] = lab[3, 3] = 0
    b = centers_ref.inner_boundaries(np.pad(lab, 1))[1:-1, 1:-1]
    assert b[1, 1] and b[2, 2]   # border of the padded objects
    lab2 = np.full((6, 6), 5)
    lab2[3, 3] = 4
    assert not centers_ref.inner_boundaries(lab2)[2, 2]   # only diagonal to the other label
    # 3-D: the six face neighbours count, edges and corners do not
    v = np.full((3, 3, 3), 1)
    v[0, 0, 0] = 2
    b = centers_ref.inner_boundaries(v)
    assert b[0, 0, 1] and b[0, 1, 0] and b[1, 0, 0] and not b[0, 1, 1] and not b[1, 1, 1]
    rng = np.random.default_rng(3)
    for shape in ((9, 11), (5, 6, 7)):
        lab = rng.integers(0, 3, shape)
        assert np.array_equal(centers_ref.inner_boundaries(lab), _cross_boundaries_loop(lab))


def test_edt_squared_brute_force():
    rng = np.random.default_rng(4)
    for shape in ((1, 13), (13, 1), (12, 17), (5, 6, 7)):
        m = rng.random(shape) > 0.15
        m.flat[0] = False
        zeros = np.stack(np.nonzero(~m), 1)
        pts = np.stack(np.unravel_index(np.arange(m.size), shape), 1)
        want = ((pts[:, None, :] - zeros[None]) ** 2).sum(-1).min(1).reshape(shape)
        assert np.array_equal(centers_ref.edt_squared(m), want)


def test_centroid_identity():
    """int64 coordinate sums divided once in fp64 equal numpy's float64 mean (what skimage's regionprops computes) while the sums
    stay below 2^53: pairwise summation of integers below 2^53 is exact, and both sides round one quotient."""
    rng = np.random.default_rng(5)
    for n, hi in ((1, 10), (7, 2 ** 15), (1000, 2 ** 20), (100_000, 2 ** 31 - 1), (3_000_000, 2 ** 31 - 1)):
        coords = rng.integers(0, hi, (n, 3), dtype=np.int64)
        assert coords.sum(0).max() < 2 ** 53
        ours = coords.sum(0).astype(np.float64) / np.float64(n)
        ref = coords.astype(np.float64).mean(axis=0)
        assert np.array_equal(ours.view(np.int64), ref.view(np.int64))
