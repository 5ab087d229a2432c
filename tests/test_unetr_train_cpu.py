"""CPU checks of the UNETR decoder's training references: the float64 training-mode restatement against the numpy-style
oracle, the loss and its gradient, and the default init."""
import math

import pytest
import torch

from oracle import unetr_ref
from micro_sam_b200 import unetr
from tests import unetr_train_ref as ref

REDUCED = dict(emb=64, feats=(128, 64, 64, 64), deconv=(64, 64, 64, 64), head_in=64)


@pytest.mark.parametrize("transposed,affine", [(False, False), (True, False), (False, True)])
def test_train_reference_matches_oracle_in_eval_mode(transposed, affine):
    sd = unetr_ref.seeded_state(transposed=transposed, affine=affine, seed=3, **REDUCED)
    z = torch.randn(2, 64, 2, 2, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    want = unetr_ref.forward_maps(sd, z)
    got = ref.forward_maps(ref.leaves(sd), z, train=False)
    assert float((got - want).abs().max()) < 1e-12


def test_train_mode_batchnorm_updates_running_statistics_as_torch():
    sd = unetr_ref.seeded_state(seed=4, **REDUCED)
    z = torch.randn(2, 64, 2, 2, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    lv = ref.leaves(sd)
    rm0 = lv["deconv1.block.2.running_mean"].clone()
    ref.forward_maps(lv, z, train=True)
    bn = torch.nn.BatchNorm2d(64).double()
    bn.load_state_dict({k.split(".", 3)[-1]: v.double() if v.is_floating_point() else v
                        for k, v in sd.items() if k.startswith("deconv1.block.2.")})
    x = unetr_ref.upsampler({k: v.double() for k, v in sd.items()}, "deconv1.block.0", z)
    x = torch.nn.functional.conv2d(x, sd["deconv1.block.1.block.weight"].double(), sd["deconv1.block.1.block.bias"].double(), padding=1)
    bn.train()
    bn(x)
    assert not torch.equal(rm0, lv["deconv1.block.2.running_mean"])
    assert torch.allclose(lv["deconv1.block.2.running_mean"], bn.running_mean, atol=1e-12)
    assert torch.allclose(lv["deconv1.block.2.running_var"], bn.running_var, atol=1e-12)


@pytest.mark.parametrize("mask", [True, False])
def test_loss_gradcheck(mask):
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 3, 5, 7, generator=g, dtype=torch.float64).requires_grad_(True)
    y = torch.rand(2, 3, 5, 7, generator=g, dtype=torch.float64)
    y[:, 0] = (y[:, 0] > 0.5).double()
    assert torch.autograd.gradcheck(lambda t: ref.dice_based_distance_loss(t, y, mask), (x,))


def test_loss_from_stats_matches_restatement():
    from micro_sam_b200.training import dice_from_stats
    g = torch.Generator().manual_seed(6)
    x = torch.rand(2, 3, 9, 4, generator=g, dtype=torch.float64)
    y = torch.rand(2, 3, 9, 4, generator=g, dtype=torch.float64)
    y[:, 0] = (y[:, 0] > 0.3).double()
    m = torch.ones_like(y)
    m[:, 1:] = y[:, :1]
    st = torch.stack([torch.stack([(x * y * m * m)[:, k].sum(), ((x * m) ** 2)[:, k].sum(), ((y * m) ** 2)[:, k].sum()])
                      for k in range(3)])
    assert abs(float(dice_from_stats(st)) - float(ref.dice_based_distance_loss(x, y))) < 1e-12


def test_default_init_is_torch_default():
    sd = unetr.default_decoder_state()
    plan = unetr.infer_plan(sd)
    assert plan["base"] == (256, 512, False) and not plan["transposed"]
    w = sd["decoder_head.block.1.weight"]
    bound = 1 / math.sqrt(w.shape[1] * 9)
    assert float(w.abs().max()) <= bound and float(w.abs().max()) > 0.9 * bound
    assert torch.equal(sd["deconv2.block.2.weight"], torch.ones(128)) and torch.equal(sd["deconv2.block.2.running_var"], torch.ones(128))
    assert torch.equal(unetr.default_decoder_state()["out_conv.weight"], sd["out_conv.weight"])   # seeded
    t = unetr.default_decoder_state(transposed=True)
    assert unetr.infer_plan(t)["transposed"] and float(t["deconv1.block.0.block.weight"].abs().max()) <= 1 / math.sqrt(256 * 4)
