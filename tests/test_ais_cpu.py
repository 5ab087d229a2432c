"""CPU checks of the AIS restatements (DESIGN.md section 2): the smoothing against scipy, the two implementations of the
watershed rule against each other, the rule's distance from a skimage-style priority flood, the decoder's plan inference and
the conv1x1 / bilinear x2 commutation the interpolation upsampler relies on."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import ndimage

from micro_sam_b200 import unetr
from oracle import ais_ref, unetr_ref


@pytest.mark.parametrize("sigma", [0.5, 1.0, 1.6, 3.3])
@pytest.mark.parametrize("shape", [(37, 53), (8, 5), (1, 9)])
def test_smoothing_equals_scipy_mirror(sigma, shape):
    x = np.random.default_rng(0).random(shape)
    ours = ais_ref._smooth_axis(ais_ref._smooth_axis(x, ais_ref.gaussian_taps(sigma), 0), ais_ref.gaussian_taps(sigma), 1)
    ref = ndimage.gaussian_filter1d(ndimage.gaussian_filter1d(x, sigma, axis=0, mode="mirror", truncate=3.0), sigma, axis=1,
                                    mode="mirror", truncate=3.0)
    assert np.abs(ours - ref).max() < 1e-12
    assert np.array_equal(unetr.gaussian_taps(sigma), ais_ref.gaussian_taps(sigma))   # the device gets the oracle's taps


def test_smoothing_zero_sigma_is_identity():
    x = np.random.default_rng(1).random((9, 7)).astype(np.float32)
    assert np.array_equal(ais_ref.smooth(x, 0), x)


def _random_case(rng, H, W, density):
    h = rng.random((H, W)).astype(np.float32)
    h[rng.random((H, W)) < 0.2] = np.float32(0.5)   # plateaus: exact ties of B
    fmask = rng.random((H, W)) < density
    seeds = np.zeros((H, W), np.int64)
    idx = rng.choice(H * W, size=max(1, H * W // 40), replace=False)
    seeds.flat[idx] = rng.permutation(len(idx)) + 1
    seeds[~fmask] = 0
    return h, fmask, seeds


@pytest.mark.parametrize("seed", range(6))
def test_watershed_rule_two_implementations_agree(seed):
    rng = np.random.default_rng(seed)
    h, fmask, seeds = _random_case(rng, 29 + seed, 41, [0.6, 0.8, 1.0][seed % 3])
    l1, b1 = ais_ref.watershed_relax(h, fmask, seeds)
    l2, b2 = ais_ref.watershed_dijkstra(h, fmask, seeds)
    assert np.array_equal(b1, b2) and np.array_equal(l1, l2)


def test_watershed_rule_planted():
    """Two seeds in a valley split at the ridge; an island no seed reaches stays 0; a tie goes to the smaller id."""
    h = np.array([[0, 1, 2, 5, 2, 1, 0, 9, 3]], np.float32)
    fmask = np.array([[1, 1, 1, 1, 1, 1, 1, 0, 1]], bool)
    seeds = np.array([[2, 0, 0, 0, 0, 0, 1, 0, 0]], np.int64)
    for ws in (ais_ref.watershed_relax, ais_ref.watershed_dijkstra):
        lab, _ = ws(h, fmask, seeds)
        assert lab.tolist() == [[2, 2, 2, 1, 1, 1, 1, 0, 0]]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_watershed_rule_on_touching_disks(seed):
    fg, cd, bd = ais_ref.touching_disks(96, 128, 30, seed=seed)
    seeds, _, fmask, bd_s = ais_ref.markers_and_mask(fg, cd, bd, 0.5, 0.5, 0.5, 1.0, 1.6)
    l1, _ = ais_ref.watershed_relax(bd_s, fmask, seeds)
    l2, _ = ais_ref.watershed_dijkstra(bd_s, fmask, seeds)
    assert np.array_equal(l1, l2)
    flood = ais_ref.heap_flood(bd_s, fmask, seeds)
    reached = l1 > 0
    frac = float((flood[reached] != l1[reached]).mean())
    print(f"seed {seed}: {frac:.2e} of the reached pixels differ from the priority flood")
    assert frac <= 2e-3   # DESIGN.md section 2 states the measured fractions


def test_size_filter_renumbers_in_id_order():
    lab = np.array([[1, 1, 2, 3, 3, 3, 0, 4]])
    assert ais_ref.size_filter(lab, 2).tolist() == [[1, 1, 0, 2, 2, 2, 0, 0]]


def _state(**kw):
    return unetr_ref.seeded_state(**kw)


def test_plan_production_and_reduced():
    p = unetr.infer_plan(_state())
    assert p["deconv"] == [(256, 256), (256, 128), (128, 64), (64, 64)]
    assert p["base"][:2] == (256, 512) and p["samplers"] == [(512, 256), (256, 128), (128, 64)]
    assert [b[:2] for b in p["blocks"]] == [(512, 256), (256, 128), (128, 64)]
    assert p["deconv_out"] == (64, 64) and p["head"][:2] == (128, 64) and not p["transposed"]
    r = unetr.infer_plan(_state(emb=64, feats=(128, 64, 64, 64), deconv=(64, 64, 64, 64), transposed=True, affine=True))
    assert r["transposed"] and r["base"] == (64, 128, True) and r["head"][:2] == (128, 64)


def test_plan_rejections_name_the_key():
    sd = _state()
    bad = dict(sd)
    del bad["decoder.blocks.1.block.4.bias"]
    with pytest.raises(ValueError, match="decoder.blocks.1.block.4.bias"):
        unetr.infer_plan(bad)
    bad = dict(sd, **{"decoder.blocks.0.extra.weight": torch.zeros(1)})
    with pytest.raises(ValueError, match="decoder.blocks.0.extra.weight"):
        unetr.infer_plan(bad)
    bad = dict(sd)
    bad["decoder.blocks.2.block.1.weight"] = torch.zeros(64, 96, 3, 3)
    with pytest.raises(ValueError, match="decoder.blocks.2.block.1.weight"):
        unetr.infer_plan(bad)
    bad = dict(sd, **{"base.block.0.running_mean": torch.zeros(256)})
    with pytest.raises(ValueError, match="base.block.0.running_mean"):
        unetr.infer_plan(bad)


def test_conv1x1_commutes_with_bilinear_x2():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 32, 9, 13, generator=g, dtype=torch.float64)
    w, b = torch.randn(16, 32, 1, 1, generator=g, dtype=torch.float64), torch.randn(16, generator=g, dtype=torch.float64)
    up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
    assert (F.conv2d(up(x), w, b) - up(F.conv2d(x, w, b))).abs().max() < 1e-12
