"""CPU tests of the semantic fine-tuning loss: the float64 oracle (oracle/semantic_ref.py) against a direct numpy formula,
ConvertToSemanticSamInputs, the host-side refusals and the C-ABI declarations."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import semantic_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _numpy_loss(z, lab, C, dice_weight):
    """z (B, C, H, W) float64 logits, lab (B, H, W) int labels (-100 ignored)"""
    e = np.exp(z - z.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True)
    dice = 0.0
    for c in range(C):
        t = (lab == c).astype(np.float64)
        dice += 1.0 - 2.0 * (p[:, c] * t).sum() / max((p[:, c] ** 2).sum() + (t ** 2).sum(), 1e-7)
    valid = lab != -100
    lse = np.log(np.exp(z - z.max(1, keepdims=True)).sum(1)) + z.max(1)
    zl = np.take_along_axis(z, np.where(valid, lab, 0)[:, None], 1)[:, 0]
    ce = (lse - zl)[valid].mean()
    return dice + ce if dice_weight is None else dice_weight * dice + (1 - dice_weight) * ce


@pytest.mark.parametrize("C", [2, 3, 8])
@pytest.mark.parametrize("dice_weight", [None, 0.3])
def test_oracle_loss_matches_numpy(C, dice_weight):
    g = torch.Generator().manual_seed(C)
    B, H, W = 2, 24, 20
    z = torch.randn(B, C, H, W, generator=g, dtype=torch.float64) * 3
    lab = torch.randint(0, C, (B, 1, H, W), generator=g)
    lab[lab == C - 1] = 0                                  # an empty class
    lab[0, 0, :3] = -100                                   # ignored by the cross entropy, in no class for Dice
    got = semantic_ref.semantic_loss(z, lab, C, dice_weight)
    want = _numpy_loss(z.numpy(), lab[:, 0].numpy(), C, dice_weight)
    assert abs(float(got) - want) <= 1e-12 * abs(want)


def test_oracle_low_res_chain_and_refusal():
    g = torch.Generator().manual_seed(0)
    low = torch.randn(1, 3, 256, 256, generator=g, dtype=torch.float64)
    lab = torch.randint(0, 3, (1, 1, 40, 30), generator=g)
    masks = torch.nn.functional.interpolate(low, (1024, 1024), mode="bilinear", align_corners=False)[..., :1024, :768]
    masks = torch.nn.functional.interpolate(masks, (40, 30), mode="bilinear", align_corners=False)
    want = semantic_ref.semantic_loss(masks, lab, 3)
    assert torch.equal(semantic_ref.semantic_loss_from_low_res(low, lab[:, 0], (1024, 768), (40, 30), 3), want)
    with pytest.raises(ValueError):
        semantic_ref.semantic_loss(masks, lab, 3, dice_weight=1.5)


def test_convert_to_semantic_sam_inputs():
    from micro_sam_b200.training import ConvertToSemanticSamInputs
    x = torch.zeros(2, 3, 50, 70)
    recs = ConvertToSemanticSamInputs()(x, torch.zeros(2, 1, 50, 70))
    assert len(recs) == 2
    for rec, image in zip(recs, x):
        assert set(rec) == {"image", "original_size"}
        assert rec["image"] is not None and torch.equal(rec["image"], image)
        assert tuple(rec["original_size"]) == (50, 70)


def test_host_side_refusals():
    from micro_sam_b200 import training
    low = torch.zeros(1, 3, 256, 256)
    y = torch.zeros(1, 1, 32, 32, dtype=torch.int64)
    for w in (-0.1, 1.1):
        with pytest.raises(ValueError, match="between 0 and 1"):
            training.compute_semantic_loss(low, y, 3, dice_weight=w)
    with pytest.raises(NotImplementedError):
        training.CustomDiceLoss(3, softmax=False)
    with pytest.raises(ValueError, match="logit channels"):
        training.compute_semantic_loss(low, y, 4)
    with pytest.raises(ValueError, match="1..15"):
        training.compute_semantic_loss(torch.zeros(1, 16, 256, 256), y, 16)
    with pytest.raises(ValueError, match="low-res"):
        training.compute_semantic_loss(torch.zeros(1, 3, 32, 32), y, 3)
    with pytest.raises(ValueError, match="labels"):
        training.compute_semantic_loss(low, torch.zeros(2, 1, 32, 32), 3)


def test_header_declares_semantic_loss():
    hdr = open(os.path.join(ROOT, "include", "msam_b200.h")).read()
    names = set(re.findall(r"\b(msam_[a-z0-9_]+)\s*\(", hdr))
    assert {"msam_semantic_loss_workspace", "msam_semantic_loss_stats", "msam_semantic_loss_backward"} <= names


def test_semantic_model_options_are_refused_not_ignored():
    from micro_sam_b200 import util
    sd = {"mask_decoder.mask_tokens.weight": torch.zeros(4, 256)}
    for kw in ({"num_multimask_outputs": 5}, {"num_multimask_outputs": 1}, {"flexible_load_checkpoint": True}):
        with pytest.raises(NotImplementedError, match="num_multimask_outputs|flexible_load_checkpoint"):
            util.get_sam_model("vit_b", state_dict=sd, **kw)
    util.check_mask_token_count(sd)                                     # the standard model: 4 mask tokens
    util.check_mask_token_count({"x": torch.zeros(1)})
    for n in (2, 6, 16):
        with pytest.raises(NotImplementedError, match=f"{n} mask tokens"):
            util.check_mask_token_count({"mask_decoder.mask_tokens.weight": torch.zeros(n, 256)})
