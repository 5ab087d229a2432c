"""CPU: pin the prompt oracle's candidate regions (oracle/prompt_ref.py) on the sets the reference's own prompt_generators.py samples
from, recorded by tests/golden/make_prompt_golden.py (its single-argument torch.where calls).  The reference's kornia dilation is
stood in for there by a -inf-padded 3 x 3 max-pool, so the dilation inside the ring is unpinned; the box arithmetic, the symmetric
difference and the order of the fallbacks are the reference's."""
import os

import numpy as np
import pytest

from oracle import prompt_ref as pr

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "prompt_regions.npz"))


@pytest.mark.parametrize("ds", [0, 1, 3, 10])
@pytest.mark.parametrize("which", ["box", "bigbox"])
def test_point_and_box_regions_match_the_reference(ds, which):
    lab, ids = G["label"], G["ids"]
    boxes = G["boxes" if which == "box" else "boxes_big"]
    for k, (i, b) in enumerate(zip(ids, boxes)):
        reg = pr.point_box_regions(lab == i, b, ds)
        for name in ("positive", "ring", "fill"):
            assert np.array_equal(reg[name], G[f"pb_{which}_ds{ds}_{name}"][k]), (k, name)


def test_iterative_regions_match_the_reference():
    names = set()
    for k, (t, p) in enumerate(zip(G["it_targets"], G["it_preds"])):
        reg = pr.iterative_regions(t, p)
        assert np.array_equal(reg["positive"], G["it_positive"][k]), k
        assert np.array_equal(reg["negative"], G["it_negative"][k]), k
        names |= {reg["positive_set"], reg["negative_set"]}
    # the background fallback cannot be reached in 2-D: an empty box ring means the target's box widened by 3 (clipped) lies inside
    # the target, so the box is the whole image and so is the target
    assert names == {"fn", "overlap", "fp", "ring"}, names
