"""ORACLE (test infrastructure, NOT product code) -- float64 PyTorch restatement of the loss of micro-sam's semantic fine-tuning:
`CustomDiceLoss` and `SemanticSamTrainer._compute_loss` (micro_sam/training/semantic_sam_trainer.py:11-86) on the full-resolution
logits that `Sam.postprocess_masks` makes from the low-res ones (`_get_model_outputs`, semantic_sam_trainer.py:88-104).

The Dice term is torch_em's `DiceLoss()` (third party, not under the reference, not installed), restated as DESIGN.md section 2
does for `DiceBasedDistanceLoss`: per channel `1 - 2 sum(p t) / max(sum p^2 + sum t^2, 1e-7)` with each sum over the whole batch
and all pixels, summed over the channels.  PARITY UNPINNED for that formula.  The cross entropy is torch's own
`nn.CrossEntropyLoss()` (mean over the pixels whose label is not -100).  Everything is differentiable (autograd).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .unetr_ref import postprocess_masks


def one_hot(target: torch.Tensor, num_classes: int) -> torch.Tensor:
    """CustomDiceLoss._one_hot_encoder: (B, 1, H, W) labels -> (B, C, H, W) float, channel c = (label == c)"""
    return torch.cat([target == i for i in range(num_classes)], dim=1).to(torch.float64)


def dice_loss(pred: torch.Tensor, target: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    """torch_em DiceLoss(): channels first, every other axis flattened, 1 - 2 sum(x y) / max(sum x^2 + sum y^2, eps) per channel,
    summed over the channels"""
    C = pred.shape[1]
    x = pred.transpose(0, 1).reshape(C, -1)
    y = target.transpose(0, 1).reshape(C, -1)
    return (1.0 - 2.0 * (x * y).sum(-1) / ((x * x).sum(-1) + (y * y).sum(-1)).clamp(min=eps)).sum()


def custom_dice_loss(masks: torch.Tensor, target: torch.Tensor, num_classes: int) -> torch.Tensor:
    """CustomDiceLoss(num_classes, softmax=True)(masks (B, C, H, W) logits, target (B, 1, H, W) labels)"""
    return dice_loss(torch.softmax(masks, dim=1), one_hot(target, num_classes))


def semantic_loss(masks: torch.Tensor, y: torch.Tensor, num_classes: int, dice_weight: Optional[float] = None) -> torch.Tensor:
    """SemanticSamTrainer._compute_loss(y (B, 1, H, W), masks (B, C, H, W))"""
    if dice_weight is not None and (dice_weight < 0 or dice_weight > 1):
        raise ValueError("The weight factor should lie between 0 and 1.")
    dice = custom_dice_loss(masks, y, num_classes)
    ce = F.cross_entropy(masks, y.squeeze(1).long())
    return dice + ce if dice_weight is None else dice_weight * dice + (1 - dice_weight) * ce


def semantic_loss_from_low_res(low_res: torch.Tensor, y: torch.Tensor, input_size, original_size, num_classes: int,
                               dice_weight: Optional[float] = None) -> torch.Tensor:
    """The same loss of low-res logits (B, C, 256, 256): postprocess_masks (bilinear to 1024, crop to input_size, bilinear to
    original_size), then `semantic_loss`, in the dtype of `low_res` (float64 for the reference)."""
    masks = postprocess_masks(low_res, tuple(input_size), tuple(original_size))
    y = y if y.dim() == 4 else y[:, None]
    return semantic_loss(masks, y, num_classes, dice_weight)
