"""CPU: the prompt oracle (oracle/prompt_ref.py) -- the square dilation the kernels compute equals the iterated 3 x 3 dilation the
reference applies, also at the image borders; the numpy Philox4x32-10 matches the published known-answer vectors; the regions
behave as the reference's generators on hand-made cases."""
import numpy as np
import pytest

from oracle import prompt_ref as pr


@pytest.mark.parametrize("ds", [0, 1, 2, 3, 5, 10])
def test_square_dilation_is_the_iterated_3x3_dilation(ds):
    rng = np.random.default_rng(ds)
    for shape in [(1, 1), (1, 7), (9, 1), (17, 23), (40, 31)]:
        for density in (0.002, 0.02, 0.2):
            m = rng.random(shape) < density
            m[0, 0] = m[-1, -1] = rng.random() < 0.5          # objects touching the corners and borders
            m[:, 0] |= rng.random(shape[0]) < 0.1
            assert np.array_equal(pr.square_dilation(m, ds), pr.iterated_dilation(m, ds)), (shape, density, ds)


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10"""
    assert pr.philox4x32_10((0, 0, 0, 0), 0) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert pr.philox4x32_10((0xFFFFFFFF,) * 4, 0xFFFFFFFFFFFFFFFF) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def test_point_box_regions_by_hand():
    obj = np.zeros((12, 12), bool)
    obj[5:7, 5:7] = True
    r = pr.point_box_regions(obj, (5, 5, 7, 7), 2)
    assert r["positive"].sum() == 4 and r["fill"].sum() == 140
    # box widened by 2 = [3, 9)^2, dilated object = [3, 9)^2 as well: no ring
    assert r["ring"].sum() == 0
    r = pr.point_box_regions(obj, (2, 2, 10, 10), 1)      # a larger (distorted) box: the ring is box+1 minus the 4 x 4 dilation
    assert r["ring"].sum() == 10 * 10 - 4 * 4
    # a box smaller than the dilated object: the symmetric difference also keeps the dilated pixels outside the box
    r = pr.point_box_regions(obj, (5, 5, 7, 7), 0)
    assert r["ring"].sum() == 0
    r = pr.point_box_regions(obj, (6, 6, 7, 7), 1)
    assert r["ring"].sum() == 16 - 9 + 0


def test_iterative_regions_fallbacks():
    t = np.zeros((10, 10), bool)
    t[4:6, 4:6] = True
    r = pr.iterative_regions(t, t)                        # perfect prediction: overlap / box ring
    assert r["positive_set"] == "overlap" and r["negative_set"] == "ring" and r["negative"].sum() == 64 - 4
    p = np.zeros_like(t)
    r = pr.iterative_regions(t, p)
    assert r["positive_set"] == "fn" and r["positive"].sum() == 4 and r["negative_set"] == "ring"
    p = t.copy()
    p[0, 0] = True
    assert pr.iterative_regions(t, p)["negative_set"] == "fp"
    full = np.ones((10, 10), bool)                        # no background at all: the chain ends in an empty set
    assert pr.iterative_regions(full, full)["negative"].sum() == 0
    t2 = np.zeros((4, 4), bool)
    t2[1:3, 1:3] = True
    t2[:, :] = True
    t2[0, 0] = False                                      # box ring empty (box = whole image, only (0, 0) outside the target)
    r = pr.iterative_regions(t2, t2)
    assert r["negative_set"] == "ring" and r["negative"].sum() == 1


def test_distort_box_rounds_half_to_even():
    assert pr.distort_box((10, 10, 20, 20), 0.5, (100, 100), [0.1, 0.1, 0.1, 0.1]) == [round(9.5), round(9.5), round(20.5), round(20.5)]
    assert pr.distort_box((10, 10, 20, 20), 0.5, (100, 100), [0.1] * 4) == [10, 10, 20, 20]
    assert pr.distort_box((0, 0, 20, 20), 1.0, (25, 25), [0.9] * 4) == [0, 0, 25, 25]
