"""Forward half of micro-sam's fine-tuning step on the H100 core (cfg 5; micro_sam/training/trainable_sam.py:24-114,
micro_sam/training/sam_trainer.py:122-172).

`TrainableSAM` keeps the reference's protocol -- `preprocess` (torch resize with antialias, normalise, pad),
`image_embeddings_oft` (ONE encoder pass for the batch), `forward` (per image: prompt encoder -> mask decoder ->
postprocess_masks) -- on the engine's kernels; `compute_loss` evaluates `_compute_loss` (dice of sigmoid(masks) per object,
minimum over the 1 / 3 predicted masks, + MSE between predicted and true IoU) from five per-mask sums that
`msam_mask_loss_stats` accumulates straight from the low-res logits, so the (n_obj, M, H, W) logits are only materialised
when the caller asks for `masks`.

Backward: with `sam.train()` and grad mode on, every stage is differentiable.  The embeddings returned by `image_embeddings_oft`
are part of the autograd graph (encoder backward: csrc/encoder_train.cu); `forward` runs the prompt encoder and mask decoder of
image i in decoder slot i (csrc/decoder_train.cu; point, box and mask prompts) and `compute_loss` has an adjoint, so
`loss.backward()` fills `sam.encoder_grads()` and `sam.decoder_grads()` (fp32, upstream keys / shapes).

`compute_iterative_loss` restates `SamTrainer._compute_iterative_loss` (sam_trainer.py:243-289): several decoder passes per step,
the later ones prompted with the previous predictions (points and / or mask logits).  Each pass is back-propagated as soon as its
loss exists, so any number of passes fits in the one decoder slot per image.

The prompts of the reference trainer come from the GPU (csrc/prompts.cu): `ConvertToSamInputs` makes the targets, boxes and points
of pass 0 from the label images, `IterativePromptUpdate` the corrective point of every later pass from the best low-res logits, and
`interactive_train_iteration` is SamTrainer._interactive_train_iteration on top of them.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import math
import random

import numpy as np
import torch

from . import _lib
from . import prompt_generators as pg
from .sam import B200Sam, ResizeLongestSide


# The inference decoder (csrc/decoder.cu) takes at most 16 tokens per prompt, 5 of them output tokens; the training decoder
# (csrc/decoder_train.cu) takes up to 64.  Iterative prompting adds 2 points per pass, so the reference's 8 passes end with 16 or 17
# sparse tokens: the training decoder runs those passes, also in eval() mode.
MAX_INFERENCE_SPARSE_TOKENS = 11


def _sparse_tokens(points, boxes) -> int:
    n_points = 0 if points is None else int(points[0].shape[1])
    return (n_points + (0 if boxes is not None else 1) if n_points else 0) + (2 if boxes is not None else 0)


_PROMPT_KEYS = ("point_coords", "boxes", "mask_inputs")


def decoder_slots(batched_inputs: List[Dict[str, Any]]) -> List[Optional[int]]:
    """The training decoder slot of each record: the prompted records (points, boxes or mask inputs) take slots 0, 1, ... in batch
    order; a record with no prompt gets None, and all of those are decoded together in the next slot.  A slot holds its
    activations until its backward pass has run, and there are 8."""
    slots, n = [], 0
    for rec in batched_inputs:
        if any(k in rec for k in _PROMPT_KEYS):
            slots.append(n)
            n += 1
        else:
            slots.append(None)
    used = n + (1 if n < len(slots) else 0)
    if used > 8:
        raise ValueError(f"training forward: {n} prompted images need {used} decoder slots, and there are 8 (one slot per prompted "
                         "image, one for all images without prompts, each held until its backward pass has run)")
    return slots


class TrainableSAM:
    """micro_sam.training.TrainableSAM on a `B200Sam` (trainable_sam.py:12-114)."""

    def __init__(self, sam: B200Sam) -> None:
        self.sam = sam
        self.transform = ResizeLongestSide(sam.image_encoder.img_size)

    def preprocess(self, x: torch.Tensor) -> Tuple[torch.Tensor, Tuple[int, int]]:
        """(B, 3, H, W) in [0, 255] -> resized (antialiased bilinear), normalised, zero-padded (B, 3, S, S) + the resized shape."""
        x = self.transform.apply_image_torch(x.to(self.sam.device, torch.float32))
        input_size = tuple(x.shape[-2:])
        x = (x - self.sam.pixel_mean.unsqueeze(0)) / self.sam.pixel_std.unsqueeze(0)
        s = self.sam.image_encoder.img_size
        return torch.nn.functional.pad(x, (0, s - x.shape[-1], 0, s - x.shape[-2])), input_size

    def image_embeddings_oft(self, batched_inputs: List[Dict[str, Any]]):
        with torch.set_grad_enabled(bool(getattr(self.sam, "training", False)) and torch.is_grad_enabled()):
            images, input_size = self.preprocess(torch.stack([x["image"] for x in batched_inputs], dim=0))
            for rec in batched_inputs:
                rec["input_size"] = input_size
            return self.sam.image_encoder(images), batched_inputs

    def forward(self, batched_inputs: List[Dict[str, Any]], image_embeddings: torch.Tensor, multimask_output: bool = False,
                return_masks: bool = True) -> List[Dict[str, Any]]:
        """trainable_sam.py:62-114.  `return_masks=False` skips the (n_obj, M, H, W) up-sampled logits (the loss does not need
        them: `compute_loss` works from `low_res_masks`).  In train() mode with grad enabled the outputs are part of the autograd
        graph (point, box and `mask_inputs` prompts; the mask inputs get no gradient): each prompted image uses a decoder slot of
        its own, and the images without prompts (semantic training) are decoded together in one more slot (`decoder_slots`); a
        slot holds its activations until its backward pass has run."""
        if getattr(self.sam, "training", False) and torch.is_grad_enabled():
            return self._forward_train(batched_inputs, image_embeddings, multimask_output, return_masks)
        with torch.no_grad():
            return self._forward_eval(batched_inputs, image_embeddings, multimask_output, return_masks)

    def _forward_train(self, batched_inputs, image_embeddings, multimask_output, return_masks):
        sam, dev = self.sam, self.sam.device
        slots = decoder_slots(batched_inputs)
        free = [i for i, s in enumerate(slots) if s is None]
        decoded = {}
        if free:   # every prompt-free image in one call and one slot, after the prompted ones
            low, iou = sam.decoder_train_images(image_embeddings[free], multimask_output, slot=len(batched_inputs) - len(free))
            decoded = {i: (low[b:b + 1], iou[b:b + 1]) for b, i in enumerate(free)}
        outputs = []
        for i, (rec, emb) in enumerate(zip(batched_inputs, image_embeddings)):
            if slots[i] is None:
                low, iou = decoded[i]
            else:
                points = (rec["point_coords"].to(dev), rec["point_labels"].to(dev)) if "point_coords" in rec else None
                boxes = rec["boxes"].to(dev) if "boxes" in rec else None
                masks = rec["mask_inputs"].to(dev) if "mask_inputs" in rec else None
                low, iou = sam.decoder_train(emb, points, boxes, multimask_output, slot=slots[i], masks=masks)
            out = {"low_res_masks": low, "iou_predictions": iou, "input_size": tuple(rec["input_size"]),
                   "original_size": tuple(rec["original_size"])}
            if return_masks:
                with torch.no_grad():
                    out["masks"] = sam.postprocess_masks(low.detach(), input_size=rec["input_size"], original_size=rec["original_size"])
            outputs.append(out)
        return outputs

    def _forward_eval(self, batched_inputs, image_embeddings, multimask_output, return_masks):
        sam, dev = self.sam, self.sam.device
        outputs = []
        for rec, emb in zip(batched_inputs, image_embeddings):
            points = (rec["point_coords"].to(dev), rec["point_labels"].to(dev)) if "point_coords" in rec else None
            boxes = rec["boxes"].to(dev) if "boxes" in rec else None
            masks_in = rec["mask_inputs"].to(dev) if "mask_inputs" in rec else None
            if _sparse_tokens(points, boxes) > MAX_INFERENCE_SPARSE_TOKENS:   # more tokens than the inference decoder takes
                low, iou = sam.decode_with_training_decoder(emb, points, boxes, multimask_output, slot=len(outputs) % 8, masks=masks_in)
                out = {"low_res_masks": low, "iou_predictions": iou, "input_size": tuple(rec["input_size"]),
                       "original_size": tuple(rec["original_size"])}
                if return_masks:
                    out["masks"] = sam.postprocess_masks(low, input_size=rec["input_size"], original_size=rec["original_size"])
                outputs.append(out)
                continue
            sparse, dense = sam.prompt_encoder(points=points, boxes=boxes, masks=masks_in)
            low, iou = sam.mask_decoder(image_embeddings=emb.unsqueeze(0), image_pe=sam.prompt_encoder.get_dense_pe(),
                                        sparse_prompt_embeddings=sparse, dense_prompt_embeddings=dense,
                                        multimask_output=multimask_output)
            out = {"low_res_masks": low, "iou_predictions": iou, "input_size": tuple(rec["input_size"]),
                   "original_size": tuple(rec["original_size"])}
            if return_masks:
                out["masks"] = sam.postprocess_masks(low, input_size=rec["input_size"], original_size=rec["original_size"])
            outputs.append(out)
        return outputs

    __call__ = forward


class _LossStatsFn(torch.autograd.Function):
    """msam_mask_loss_stats with its adjoint (msam_mask_loss_backward): the loss depends on the logits only through the first two
    sums (sum p t, sum p^2); the three counts are piecewise constant."""

    @staticmethod
    def forward(ctx, lr, tg, in_h, in_w, H, W):
        n_obj, M = lr.shape[:2]
        out = torch.empty(n_obj, M, 5, device=lr.device, dtype=torch.float32)
        _lib.check(_lib.lib().msam_mask_loss_stats(_lib.ptr(lr), _lib.ptr(tg), n_obj, M, in_h, in_w, H, W, _lib.ptr(out), _lib.cur_stream()))
        ctx.save_for_backward(lr, tg)
        ctx.geom = (in_h, in_w, H, W)
        return out

    @staticmethod
    def backward(ctx, d_stats):
        lr, tg = ctx.saved_tensors
        n_obj, M = lr.shape[:2]
        d_lr = torch.zeros_like(lr)
        ds = d_stats.to(torch.float32).contiguous()
        _lib.check(_lib.lib().msam_mask_loss_backward(_lib.ptr(lr), _lib.ptr(tg), _lib.ptr(ds), n_obj, M, *ctx.geom, _lib.ptr(d_lr),
                                                      _lib.cur_stream()))
        return d_lr, None, None, None, None, None


def mask_loss_stats(low_res: torch.Tensor, targets: torch.Tensor, input_size, original_size) -> torch.Tensor:
    """`msam_mask_loss_stats`: low_res (n_obj, M, 256, 256) logits + targets (n_obj, 1, H, W) {0,1} -> (n_obj, M, 5); differentiable
    w.r.t. `low_res` when it requires grad."""
    n_obj, M = low_res.shape[:2]
    H, W = int(original_size[0]), int(original_size[1])
    lr = low_res.to(torch.float32).contiguous()
    tg = (targets.reshape(n_obj, H, W).to(lr.device) != 0).to(torch.uint8).contiguous()
    return _LossStatsFn.apply(lr, tg, int(input_size[0]), int(input_size[1]), H, W)


def compute_loss(batched_outputs: List[Dict[str, Any]], y_one_hot, eps_dice: float = 1e-7, eps_iou: float = 1e-7):
    """SamTrainer._compute_loss (sam_trainer.py:131-172): per image, dice loss per object (torch_em DiceLoss(reduce_channel=
    None): 1 - 2 sum(p t) / max(sum p^2 + sum t^2, eps)) minimised over the predicted masks, averaged over objects, plus
    MSE(true IoU, predicted IoU); both averaged over the batch.  `y_one_hot[b]`: (n_obj, 1, H, W) binary targets."""
    mask_loss = iou_loss = 0.0
    for out, targets in zip(batched_outputs, y_one_hot):
        st = mask_loss_stats(out["low_res_masks"], targets, out["input_size"], out["original_size"])
        pt, pp, t, n_and, n_or = st.unbind(-1)                       # (n_obj, M) each
        dice = 1.0 - 2.0 * pt / (pp + t).clamp(min=eps_dice)         # t in {0,1}: sum t^2 = sum t
        true_iou = n_and / (n_or + eps_iou)
        mask_loss = mask_loss + dice.min(dim=1).values.mean()
        iou_loss = iou_loss + torch.mean((true_iou - out["iou_predictions"]) ** 2)
    n = len(batched_outputs)
    mask_loss, iou_loss = mask_loss / n, iou_loss / n
    return mask_loss + iou_loss, mask_loss, iou_loss


def get_best_masks(batched_outputs: List[Dict[str, Any]]):
    """SamTrainer._get_best_masks (sam_trainer.py:178-205): per object the mask with the highest predicted IoU, as binary
    (logit > 0) full-size masks (B, n_obj, 1, H, W) and low-res logits (B, n_obj, 1, 256, 256)."""
    masks, logits = [], []
    for out in batched_outputs:
        best = out["iou_predictions"].argmax(dim=1)
        sel = torch.arange(best.shape[0], device=best.device)
        low = out["low_res_masks"][sel, best][:, None]
        full = out["masks"][sel, best][:, None] if "masks" in out else None
        logits.append(low)
        masks.append(None if full is None else (full > 0.0).float())
    return (None if masks[0] is None else torch.stack(masks)), torch.stack(logits)


class _IterativeLossFn(torch.autograd.Function):
    """Ties the loss of `compute_iterative_loss` to the image embeddings: its backward hands the dL/d embeddings accumulated over the
    sub-iterations to the encoder's backward pass once.  The decoder gradients were accumulated at scale 1 while the passes ran, so
    only an upstream gradient of 1 (`loss.backward()`) keeps the two consistent, and zeroing them in between would lose them."""

    @staticmethod
    def forward(ctx, loss, image_embeddings, d_embeddings, sam, zeroings):
        ctx.save_for_backward(d_embeddings)
        ctx.sam, ctx.zeroings = sam, zeroings
        return loss.clone()

    @staticmethod
    def backward(ctx, grad):
        if float(grad) != 1.0:
            raise ValueError(f"compute_iterative_loss: upstream gradient {float(grad)} != 1; the decoder gradients were already "
                             "accumulated for the loss itself (scale the learning rate instead)")
        if getattr(ctx.sam, "_decoder_zeroings", 0) != ctx.zeroings:
            raise RuntimeError("compute_iterative_loss: zero_decoder_grads() ran after the passes and discarded their decoder "
                               "gradients; zero them before compute_iterative_loss, not between it and loss.backward()")
        d_emb, = ctx.saved_tensors
        return None, d_emb, None, None, None


def compute_iterative_loss(model: TrainableSAM, batched_inputs: List[Dict[str, Any]], y_one_hot, num_subiter: int,
                           multimask_output: bool, update_prompts, full_masks: bool = True):
    """SamTrainer._compute_iterative_loss (sam_trainer.py:243-289) -> (loss, mask_loss, iou_regression_loss, mean_model_iou),
    each averaged over the `num_subiter` passes.  Pass 0 uses `multimask_output`, the later ones a single mask.  Between passes
    `update_prompts(batched_inputs, masks, logits)` runs under no_grad with the best mask per object (binary full-size (B, n_obj,
    1, H, W) and low-res logits (B, n_obj, 1, 256, 256), `get_best_masks`) and returns the records of the next pass, e.g. with
    more points and the logits as "mask_inputs".  With `full_masks=False` no pass materialises the (n_obj, M, H, W) up-sampled
    logits and `update_prompts` gets `masks=None` (enough for `IterativePromptUpdate`, which reads the low-res logits).

    Training (`sam.train()` and grad mode): every pass runs the decoder on a detached copy of the embeddings and back-propagates
    its loss / num_subiter at once, which accumulates the decoder gradients and dL/d embeddings and frees the image's decoder slot.
    So the decoder gradients exist when this returns: call `sam.zero_decoder_grads()` BEFORE it (where the reference trainer calls
    `optimizer.zero_grad()`), never between it and `loss.backward()` -- that backward raises if it happened.  `loss.backward()`
    carries the summed dL/d embeddings into the encoder's backward pass, once.  The passes share nothing but the embeddings, so
    these are the gradients of the reference's single backward through all passes.

    Otherwise (validation: eval() mode or no_grad) the passes only run forward and the returned values carry no graph."""
    sam = model.sam
    train = bool(getattr(sam, "training", False)) and torch.is_grad_enabled()
    image_embeddings, batched_inputs = model.image_embeddings_oft(batched_inputs)
    d_emb = torch.zeros_like(image_embeddings, dtype=torch.float32) if train else None
    loss = mask_loss = iou_loss = mean_iou = 0.0
    for i in range(num_subiter):
        last = i == num_subiter - 1
        multimask = multimask_output if i == 0 else False
        if train:
            emb = image_embeddings.detach().requires_grad_(True)
            outputs = model(batched_inputs, emb, multimask_output=multimask, return_masks=full_masks and not last)
            net_loss, net_mask_loss, net_iou_loss = compute_loss(outputs, y_one_hot)
            (net_loss / num_subiter).backward()
            d_emb += emb.grad
        else:
            with torch.no_grad():
                outputs = model(batched_inputs, image_embeddings, multimask_output=multimask, return_masks=full_masks and not last)
                net_loss, net_mask_loss, net_iou_loss = compute_loss(outputs, y_one_hot)
        with torch.no_grad():
            loss = loss + net_loss.detach()
            mask_loss = mask_loss + net_mask_loss.detach()
            iou_loss = iou_loss + net_iou_loss.detach()
            mean_iou = mean_iou + torch.stack([o["iou_predictions"] for o in outputs]).mean()
            if not last:
                masks, logits = get_best_masks(outputs)
                batched_inputs = update_prompts(batched_inputs, masks, logits)
    loss = loss / num_subiter
    if train:
        loss = _IterativeLossFn.apply(loss, image_embeddings, d_emb, sam, getattr(sam, "_decoder_zeroings", 0))
    return loss, mask_loss / num_subiter, iou_loss / num_subiter, mean_iou / num_subiter


# ---------------------------------------------------------------------------------------------------------------------------------
# Prompt generation of the reference trainer (micro_sam/training/util.py:153-265, sam_trainer.py:70-120, 291-371)

def _label_targets(y, sampled_ids, dev, box_distortion: Optional[float] = None):
    """`msam_prompt_targets`: label images (B, [1,] H, W) and per-image sorted ids -> uint8 one-hot targets (B, n_max, H, W), int32
    pixel counts (B, n_max) and int32 boxes (B, n_max, 4) (min_row, min_col, max_row + 1, max_col + 1), optionally distorted"""
    B = len(sampled_ids)
    lab = torch.as_tensor(y).to(dev)
    lab = lab.reshape(B, lab.shape[-2], lab.shape[-1])
    if lab.dtype not in (torch.int32, torch.int64):
        lab = lab.to(torch.int64)
    lab = lab.contiguous()
    H, W = lab.shape[-2:]
    n_max = max(1, max(len(ids) for ids in sampled_ids))
    ids = np.full((B, n_max), np.iinfo(np.int64).max, dtype=np.int64)
    for b, v in enumerate(sampled_ids):
        ids[b, :len(v)] = np.asarray(v, dtype=np.int64)
    ids_d = torch.from_numpy(ids).to(dev)
    n_ids = torch.tensor([len(v) for v in sampled_ids], dtype=torch.int32).to(dev)
    targets = torch.empty(B, n_max, H, W, device=dev, dtype=torch.uint8)
    counts = torch.empty(B, n_max, device=dev, dtype=torch.int32)
    boxes = torch.empty(B, n_max, 4, device=dev, dtype=torch.int32)
    _lib.check(_lib.lib().msam_prompt_targets(
        _lib.ptr(lab), 0 if lab.dtype == torch.int32 else 1, B, H, W, _lib.ptr(ids_d), _lib.ptr(n_ids), n_max,
        -1.0 if box_distortion is None else float(box_distortion), pg.draw_seed(), _lib.ptr(targets), _lib.ptr(counts), _lib.ptr(boxes),
        _lib.cur_stream()))
    return targets, counts, boxes


class SampledIds(list):
    """The per-image sampled ids that `ConvertToSamInputs` returns (a list, as in the reference), plus the one-hot targets it made
    from them, so that `preprocess_batch` does not make them again."""

    def __init__(self, ids, targets: Optional[torch.Tensor] = None):
        super().__init__(ids)
        self.targets = targets


class ConvertToSamInputs:
    """micro_sam.training.util.ConvertToSamInputs (training/util.py:153-265).  `__call__(x, y, n_pos, n_neg, get_boxes=False,
    n_samples=None)` -> (batched_inputs, sampled_ids) with the reference's records: "image", "original_size", and "boxes"
    (n_obj, 4) xyxy / "point_coords" (n_obj, n_pos + n_neg, 2) xy / "point_labels" (n_obj, n_pos + n_neg), resized by
    `transform`.  The ids are enumerated and sub-sampled on the host (np.unique, np.random.choice without replacement, sorted --
    one copy of the label images per batch); targets, boxes, `_distort_boxes` and the points come from csrc/prompts.cu and are
    device tensors.  The returned id list also carries the one-hot targets (`sampled_ids.targets`, uint8 (B, n_max, H, W)) for
    `preprocess_batch`.  Neither points nor boxes requested raises ValueError, as the reference's generator does."""

    def __init__(self, transform: Optional[ResizeLongestSide], dilation_strength: int = 10, box_distortion_factor: Optional[float] = None):
        self.dilation_strength = dilation_strength
        self.transform = transform
        self.box_distortion_factor = box_distortion_factor

    def __call__(self, x, y, n_pos, n_neg, get_boxes=False, n_samples=None):
        get_points = not (n_pos == 0 and n_neg == 0)
        if not get_points and not get_boxes:
            raise ValueError("You need to request box prompts, point prompts or both.")
        dev = y.device if isinstance(y, torch.Tensor) and y.is_cuda else torch.device("cuda", torch.cuda.current_device())
        y_host = y.detach().cpu().numpy() if isinstance(y, torch.Tensor) else np.asarray(y)
        sampled = []
        for gt in y_host:
            cell_ids = np.unique(gt.squeeze().astype(np.int64))[1:]
            if n_samples is not None:
                cell_ids = np.sort(np.random.choice(cell_ids, size=min(n_samples, len(cell_ids)), replace=False))
            sampled.append(cell_ids)
        targets, counts, boxes = _label_targets(y if isinstance(y, torch.Tensor) else torch.from_numpy(y_host), sampled, dev,
                                                self.box_distortion_factor)
        B, n_max, H, W = targets.shape
        if get_points:
            coords, labels = pg.sample_points(targets.view(B * n_max, H, W), counts.view(-1), boxes.view(-1, 4), n_pos, n_neg,
                                              self.dilation_strength, pg.draw_seed(), n_per_img=n_max)
            coords, labels = coords.view(B, n_max, -1, 2).long(), labels.view(B, n_max, -1).long()
        batched_inputs = []
        for b, (image, ids) in enumerate(zip(x, sampled)):
            n = len(ids)
            rec = {"image": image, "original_size": image.shape[1:]}
            if get_boxes:
                bx = boxes[b, :n][:, [1, 0, 3, 2]].long()
                rec["boxes"] = self.transform.apply_boxes_torch(bx, original_size=(H, W)) if self.transform is not None else bx
            if get_points:
                pc = coords[b, :n]
                rec["point_coords"] = self.transform.apply_coords_torch(pc, original_size=(H, W)) if self.transform is not None else pc
                rec["point_labels"] = labels[b, :n]
            batched_inputs.append(rec)
        return batched_inputs, SampledIds(sampled, targets)


def get_prompt_and_multimasking_choices(iteration: int, validation: bool = False):
    """SamTrainer._get_prompt_and_multimasking_choices / _for_val (sam_trainer.py:70-120) -> (n_pos, n_neg, get_boxes,
    multimask_output)"""
    if not validation:
        return (1, 0, False, True) if iteration % 2 == 0 else (0, 0, True, False)
    k = iteration % 4
    if k == 0:
        return 1, 0, False, True
    if k == 1:
        return 0, 0, True, False
    if k == 2:
        n_pos = np.random.randint(1, 4 + 1)
        n_neg = np.random.randint(1, 4 + 1) if n_pos == 1 else np.random.randint(0, 4 + 1)
        return n_pos, n_neg, False, False
    n_pos = np.random.randint(1, 4 + 1)
    n_neg = np.random.randint(0, 4 + 1)
    return n_pos, n_neg, True, False


def preprocess_batch(batched_inputs: List[Dict[str, Any]], y, sampled_ids):
    """SamTrainer._preprocess_batch (sam_trainer.py:333-357): restricts every image to the batch's smallest object count and
    returns (batched_inputs, y_one_hot (B, n_obj, 1, H, W) float on the device).  Reuses the targets `ConvertToSamInputs` made,
    otherwise makes them from `y` with the same kernel."""
    assert len(y) == len(sampled_ids)
    n_objects = min(len(ids) for ids in sampled_ids)
    if isinstance(sampled_ids, SampledIds) and sampled_ids.targets is not None:
        planes = sampled_ids.targets[:, :n_objects]
    else:
        dev = y.device if isinstance(y, torch.Tensor) and y.is_cuda else torch.device("cuda", torch.cuda.current_device())
        planes = _label_targets(y, [np.asarray(ids)[:n_objects] for ids in sampled_ids], dev)[0][:, :n_objects]
    y_one_hot = planes[:, :, None].float()
    batched_inputs = [
        {k: (v[:n_objects] if k in ("point_coords", "point_labels", "boxes") else v) for k, v in inp.items()}
        for inp in batched_inputs
    ]
    return batched_inputs, y_one_hot


class IterativePromptUpdate:
    """`update_prompts` for `compute_iterative_loss`: SamTrainer._update_prompts (sam_trainer.py:291-327) with the
    IterativePromptGenerator of csrc/prompts.cu.  Per object one positive and one negative point, sampled from the best low-res
    logits evaluated at full resolution per pixel (the full-size masks are not needed: pass `full_masks=False`), appended to
    "point_coords" / "point_labels"; "mask_inputs" = the best logits when this pass uses mask inputs, else removed.

    The mask-input policy is the reference's (`_use_mask_inputs`, sam_trainer.py:206-241): one `random.random() < mask_prob` per
    image and pass on one process; under torch.distributed one draw per step made by rank 0 and broadcast, and then pass 0 gets
    zero mask inputs -- add them with `initial_inputs(batched_inputs)` before `compute_iterative_loss`."""

    def __init__(self, y_one_hot: torch.Tensor, transform: ResizeLongestSide, mask_prob: float = 0.5):
        self.targets = (y_one_hot[:, :, 0] != 0).to(torch.uint8).contiguous()
        self.transform = transform
        self.mask_prob = mask_prob
        self.is_data_parallel = torch.distributed.is_available() and torch.distributed.is_initialized()
        self.use_mask_inputs, self.use_zero_mask = False, False
        if self.mask_prob == 1:
            self.use_mask_inputs, self.use_zero_mask = True, self.is_data_parallel
        elif self.mask_prob > 0 and self.is_data_parallel:
            dev = self.targets.device
            if torch.distributed.get_rank() == 0:
                t = torch.tensor(random.random() < self.mask_prob, dtype=torch.uint8, device=dev)
            else:
                t = torch.tensor(0, dtype=torch.uint8, device=dev)
            torch.distributed.broadcast(t, src=0)
            self.use_mask_inputs = bool(t.item())
            self.use_zero_mask = self.use_mask_inputs

    def initial_inputs(self, batched_inputs: List[Dict[str, Any]]) -> List[Dict[str, Any]]:
        if self.use_zero_mask:
            B, n = self.targets.shape[:2]
            for rec in batched_inputs:
                rec["mask_inputs"] = torch.zeros(n, 1, 256, 256, device=self.targets.device)
        return batched_inputs

    def __call__(self, batched_inputs: List[Dict[str, Any]], masks, logits: torch.Tensor) -> List[Dict[str, Any]]:
        B, n, H, W = self.targets.shape
        lr = logits.reshape(B * n, 1, logits.shape[-2], logits.shape[-1]).to(torch.float32).contiguous()
        coords, labels = pg.iterative_points(self.targets.view(B * n, H, W), pg.draw_seed(), low_res=lr,
                                             input_size=batched_inputs[0]["input_size"], n_per_img=n)
        coords, labels = coords.view(B, n, 2, 2), labels.view(B, n, 2).long()
        for b, rec in enumerate(batched_inputs):
            net_coords = self.transform.apply_coords_torch(coords[b], (H, W))
            if "point_coords" in rec:
                rec["point_coords"] = torch.cat([rec["point_coords"].to(net_coords.device), net_coords], dim=1)
            else:
                rec["point_coords"] = net_coords
            if "point_labels" in rec:
                rec["point_labels"] = torch.cat([rec["point_labels"].to(labels.device).long(), labels[b]], dim=1)
            else:
                rec["point_labels"] = labels[b]
            if self.is_data_parallel:
                use = self.use_mask_inputs
            else:
                use = random.random() < self.mask_prob if self.mask_prob > 0 else False
            if use:
                rec["mask_inputs"] = logits[b]
            else:
                rec.pop("mask_inputs", None)
        return batched_inputs


def interactive_train_iteration(model: TrainableSAM, x, y, iteration: int, n_objects_per_batch: int = 25, n_sub_iteration: int = 8,
                                mask_prob: float = 0.5, convert_inputs: Optional[ConvertToSamInputs] = None):
    """SamTrainer._interactive_train_iteration (sam_trainer.py:359-371): prompts for `iteration` (a point on even, a box on odd
    iterations), targets and prompts from the label images `y` on the GPU, then `compute_iterative_loss` over `n_sub_iteration`
    passes with `IterativePromptUpdate` and no full-size masks.  Returns (loss, mask_loss, iou_regression_loss, model_iou,
    y_one_hot); in training mode call `sam.zero_decoder_grads()` before it and `loss.backward()` after it."""
    convert_inputs = ConvertToSamInputs(model.transform) if convert_inputs is None else convert_inputs
    n_pos, n_neg, get_boxes, multimask_output = get_prompt_and_multimasking_choices(iteration)
    batched_inputs, sampled_ids = convert_inputs(x, y, n_pos, n_neg, get_boxes, n_objects_per_batch)
    batched_inputs, y_one_hot = preprocess_batch(batched_inputs, y, sampled_ids)
    update = IterativePromptUpdate(y_one_hot, model.transform, mask_prob)
    batched_inputs = update.initial_inputs(batched_inputs)
    loss, mask_loss, iou_loss, model_iou = compute_iterative_loss(model, batched_inputs, y_one_hot, n_sub_iteration, multimask_output,
                                                                  update, full_masks=False)
    return loss, mask_loss, iou_loss, model_iou, y_one_hot


# ---------------------------------------------------------------------------------------------------------------------------------
# Instance-segmentation (UNETR decoder) training: micro_sam/training/training.py:train_instance_segmentation with the image encoder
# frozen, JointSamTrainer._instance_iteration (joint_sam_trainer.py:73-131) and export_instance_segmentation_model (training.py:378)

class _UNETRDecoderFn(torch.autograd.Function):
    """TrainableUNETRDecoder.forward, then crop + resize to the original size (postprocess_masks); backward fills the decoder's
    gradients and returns d embedding."""

    @staticmethod
    def forward(ctx, emb, anchor, dec, input_size, original_size):
        from .unetr import resize_maps
        maps = dec.forward(emb)
        ctx.dec, ctx.geom = dec, (tuple(maps.shape), tuple(input_size), tuple(original_size))
        if tuple(maps.shape[-2:]) == tuple(original_size) and tuple(input_size) == tuple(original_size):
            return maps
        return resize_maps(maps, input_size, original_size)

    @staticmethod
    def backward(ctx, d_out):
        (B, P, Hs, Ws), (ih, iw), (oh, ow) = ctx.geom
        d = d_out.to(torch.float32).contiguous()
        if (Hs, Ws) != (oh, ow) or (ih, iw) != (oh, ow):
            tmp = torch.empty(B * P * oh * iw, device=d.device, dtype=torch.float32)
            dm = torch.empty(B, P, Hs, Ws, device=d.device, dtype=torch.float32)
            _lib.check(_lib.lib().msam_op_ais_resize_backward(_lib.ptr(d), B * P, Hs, Ws, ih, iw, oh, ow, _lib.ptr(tmp), _lib.ptr(dm),
                                                              _lib.cur_stream()))
            d = dm
        return ctx.dec.backward(d), torch.zeros((), device=d.device), None, None, None


class UNETR:
    """micro-sam's get_unetr model (torch_em UNETR with use_skip_connection=False, resize_input=True, Sigmoid) on the device:
    `__call__(x)` takes images (B, 3, H, W) in [0, 255] and returns the foreground / center distance / boundary distance maps
    (B, 3, H, W).  preprocess (TrainableSAM.preprocess) -> image encoder (frozen) -> decoder -> crop and resize back; the result
    is differentiable with respect to the decoder's parameters."""

    def __init__(self, sam: B200Sam, decoder):
        self.sam = sam
        self.decoder = decoder
        self._trainable = TrainableSAM(sam)
        self._anchor = torch.zeros((), device=decoder.device, requires_grad=True)

    def embed(self, x: torch.Tensor, train_encoder: bool = False):
        """(embeddings (B, 256, 64, 64), input_size).  With `train_encoder` (and grad mode) the embeddings come from the encoder's
        training forward (`_EncoderFn`) and are part of the autograd graph: a backward pass fills the encoder's gradients.
        Otherwise the frozen encoder runs in eval mode without a graph."""
        with torch.no_grad():
            images, input_size = self._trainable.preprocess(x)
        was = self.sam.training
        if train_encoder and torch.is_grad_enabled():
            self.sam.train()
            try:
                return self.sam.image_encoder(images), input_size
            finally:
                if not was:
                    self.sam.eval()
        with torch.no_grad():
            self.sam.eval()
            try:
                emb = self.sam.image_encoder(images)
            finally:
                if was:
                    self.sam.train()
        return emb, input_size

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """preprocess -> image encoder -> decoder -> crop and resize back.  In train() mode of the SAM model and grad mode the
        encoder runs its training forward, so the result is differentiable w.r.t. the encoder and the decoder."""
        emb, input_size = self.embed(x, train_encoder=bool(self.sam.training))
        return self.decode(emb, input_size, tuple(x.shape[-2:]))

    def decode(self, emb: torch.Tensor, input_size, original_size) -> torch.Tensor:
        if torch.is_grad_enabled():
            return _UNETRDecoderFn.apply(emb, self._anchor, self.decoder, tuple(input_size), tuple(original_size))
        with torch.no_grad():
            return _UNETRDecoderFn.forward(_Ctx(), emb, None, self.decoder, tuple(input_size), tuple(original_size))

    def decoder_grads(self) -> Dict[str, torch.Tensor]:
        return dict(self.decoder.grads)

    def optimizer_step(self, lr: float = 1e-5, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01) -> None:
        self.decoder.optimizer_step(lr, betas, eps, weight_decay)

    def decoder_state_dict(self) -> Dict[str, torch.Tensor]:
        return self.decoder.state_dict()


class _Ctx:
    pass


def _sam_of(image_encoder) -> B200Sam:
    for cand in (image_encoder, getattr(image_encoder, "_sam", None), getattr(image_encoder, "model", None)):
        if isinstance(cand, B200Sam):
            return cand
    raise TypeError("get_unetr takes a B200Sam, its image_encoder or a predictor built on one")


def get_unetr(image_encoder, decoder_state=None, device=None, out_channels: int = 3, flexible_load_checkpoint: bool = False,
              final_activation: str = "Sigmoid") -> UNETR:
    """get_unetr (instance_segmentation.py:765): a trainable UNETR on `image_encoder`'s model.  Without `decoder_state` the
    decoder is the production plan with the bilinear upsampler, freshly initialised (`unetr.default_decoder_state`, seed 0)."""
    from .unetr import TrainableUNETRDecoder, default_decoder_state
    if out_channels != 3:
        raise NotImplementedError(f"out_channels={out_channels}: the decoder head has 3 output channels")
    if final_activation != "Sigmoid":
        raise NotImplementedError(f"final_activation={final_activation!r}: only 'Sigmoid' is implemented")
    if flexible_load_checkpoint:
        raise NotImplementedError("flexible_load_checkpoint=True is not implemented")
    sam = _sam_of(image_encoder)
    if sam.image_size != 1024:
        raise NotImplementedError(f"image_size {sam.image_size}: the UNETR decoder is built for 1024")
    state = default_decoder_state() if decoder_state is None else decoder_state
    return UNETR(sam, TrainableUNETRDecoder(state, device=device if device is not None else sam.device))


class _DistLossStatsFn(torch.autograd.Function):
    """msam_op_ais_dist_loss_stats with its adjoint: per channel (sum x y, sum x^2, sum y^2), fp64 [3, 3]"""

    @staticmethod
    def forward(ctx, x, y, mask):
        B, _, H, W = x.shape
        L = _lib.lib()
        ws = torch.empty(int(L.msam_ais_dist_loss_workspace(B, H * W)), device=x.device, dtype=torch.uint8)
        st = torch.empty(3, 3, device=x.device, dtype=torch.float64)
        _lib.check(L.msam_op_ais_dist_loss_stats(_lib.ptr(x), _lib.ptr(y), B, H * W, int(mask), _lib.ptr(ws), ws.numel(), _lib.ptr(st),
                                                 _lib.cur_stream()))
        ctx.save_for_backward(x, y)
        ctx.mask = mask
        return st

    @staticmethod
    def backward(ctx, d_st):
        x, y = ctx.saved_tensors
        B, _, H, W = x.shape
        coef = d_st[:, :2].to(torch.float32).contiguous()
        dx = torch.empty_like(x)
        _lib.check(_lib.lib().msam_op_ais_dist_loss_backward(_lib.ptr(x), _lib.ptr(y), B, H * W, int(ctx.mask), _lib.ptr(coef),
                                                             _lib.ptr(dx), _lib.cur_stream()))
        return dx, None, None


def dice_from_stats(st: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    """sum over the channels of 1 - 2 sum(x y) / max(sum x^2 + sum y^2, eps) (compute_loss's Dice convention)"""
    return (1.0 - 2.0 * st[:, 0] / (st[:, 1] + st[:, 2]).clamp(min=eps)).sum()


class DiceBasedDistanceLoss:
    """torch_em's DiceBasedDistanceLoss as DESIGN.md section 2 restates it (unpinned): prediction and target (B, 3, H, W) =
    foreground, center distances, boundary distances; the loss is the Dice loss of each channel, each reduced over the whole
    batch, summed.  With `mask_distances_in_bg` the two distance channels of both are multiplied by the foreground target."""

    def __init__(self, mask_distances_in_bg: bool = True):
        self.mask_distances_in_bg = mask_distances_in_bg

    def __call__(self, input_: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        if input_.shape != target.shape or input_.dim() != 4 or input_.shape[1] != 3:
            raise ValueError(f"DiceBasedDistanceLoss takes (B, 3, H, W) prediction and target, got {tuple(input_.shape)} and "
                             f"{tuple(target.shape)}")
        x = input_.to(torch.float32).contiguous()
        y = target.to(x.device, torch.float32).contiguous()
        return dice_from_stats(_DistLossStatsFn.apply(x, y, self.mask_distances_in_bg)).to(torch.float32)


_DT_CHANNELS = (("instances", 1), ("foreground", 2), ("distances", 4), ("boundary_distances", 8))


class PerObjectDistanceTransform:
    """torch_em's PerObjectDistanceTransform (the UNETR decoder's targets) on the device (csrc/distance_targets.cu), as DESIGN.md
    section 2 restates it (unpinned): float32 channels instances, foreground, centre distances and boundary distances (the
    selected ones, in that order), each distance normalised within its object, `distance_fill_value` on the background.

    A numpy (H, W) label image gives numpy (C, H, W), as torch_em does.  A CUDA tensor (H, W) or (B, H, W) gives a device tensor
    (C, H, W) or (B, C, H, W): the batched form, meant for the batch a DataLoader returns (forked loader workers cannot use CUDA).
    Labels are integers in [0, 2^31) (whole-number floats accepted), 0 background; sides up to 32768.  3-D labels, directed
    distances and `sampling` are not supported.
    """

    def __init__(self, distances: bool = True, boundary_distances: bool = True, directed_distances: bool = False,
                 foreground: bool = True, instances: bool = False, apply_label: bool = True, min_size: int = 0,
                 distance_fill_value: float = 1.0, sampling=None):
        if directed_distances:
            raise NotImplementedError("PerObjectDistanceTransform: directed distances are not supported (vigra's vector sign "
                                      "convention is not restated)")
        if sampling is not None:
            raise NotImplementedError("PerObjectDistanceTransform: sampling is not supported (isotropic pixels only)")
        if min_size < 0:
            raise ValueError(f"PerObjectDistanceTransform: min_size must be >= 0, got {min_size}")
        self.distances, self.boundary_distances, self.directed_distances = distances, boundary_distances, directed_distances
        self.foreground, self.instances, self.apply_label = foreground, instances, apply_label
        self.min_size, self.distance_fill_value, self.sampling = int(min_size), float(distance_fill_value), sampling
        self._channels = sum(bit for name, bit in _DT_CHANNELS if getattr(self, name))
        if self._channels == 0:
            raise ValueError("PerObjectDistanceTransform: no output channel selected")

    def _device_labels(self, t: torch.Tensor) -> torch.Tensor:
        if t.is_complex():
            raise ValueError(f"PerObjectDistanceTransform: labels must be integers, got {t.dtype}")
        if t.numel() == 0:
            raise ValueError(f"PerObjectDistanceTransform: empty labels of shape {tuple(t.shape)}")
        if t.dtype in (torch.bool, torch.uint8, torch.int8, torch.uint16, torch.int16):
            t = t.to(torch.int32)
        elif t.dtype in (torch.uint32, torch.uint64):
            t = t.to(torch.float64 if t.dtype == torch.uint64 else torch.int64)
        lo, hi = (v.item() for v in torch.aminmax(t))
        if t.is_floating_point():
            if not bool(torch.all(t == torch.floor(t))):
                raise ValueError("PerObjectDistanceTransform: float labels must hold whole numbers")
        if lo < 0:
            raise ValueError(f"PerObjectDistanceTransform: labels must be non-negative, got {lo}")
        if hi >= 2 ** 31:
            raise ValueError(f"PerObjectDistanceTransform: label ids must be below 2^31, got {hi}")
        if t.dtype not in (torch.int32, torch.int64):
            t = t.to(torch.int32)
        return t.contiguous()

    def _run(self, t: torch.Tensor) -> torch.Tensor:
        batched = t.dim() == 3
        lab = self._device_labels(t if batched else t.unsqueeze(0))
        B, H, W = lab.shape
        L = _lib.lib()
        nbytes = int(L.msam_distance_targets_workspace(B, H, W, int(self.apply_label)))
        if nbytes < 0:
            raise ValueError(f"PerObjectDistanceTransform: {B} label images of {H} x {W} (sides up to 32768, fewer than "
                             f"2^31 - 1024 pixels in all)")
        dev = lab.device
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty((B, bin(self._channels).count("1"), H, W), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.msam_distance_targets(_lib.ptr(lab), 1 if lab.dtype == torch.int64 else 0, B, H, W, int(self.apply_label),
                                               self.min_size, self._channels, self.distance_fill_value, _lib.ptr(ws), nbytes,
                                               _lib.ptr(out), _lib.cur_stream()))
        return out if batched else out[0]

    def __call__(self, labels):
        if torch.is_tensor(labels):
            if not labels.is_cuda:
                raise ValueError("PerObjectDistanceTransform: pass a CUDA tensor (H, W) / (B, H, W) or a numpy (H, W) array")
            if labels.dim() not in (2, 3):
                raise ValueError(f"PerObjectDistanceTransform: a label tensor is (H, W) or (B, H, W), got {tuple(labels.shape)}")
            return self._run(labels)
        a = np.asarray(labels)
        if a.ndim == 3:
            raise NotImplementedError("PerObjectDistanceTransform: 3-D label volumes (26-connectivity) are not supported; pass "
                                      "2-D images, or a CUDA tensor (B, H, W) for a batch")
        if a.ndim != 2:
            raise ValueError(f"PerObjectDistanceTransform: labels must be 2-D, got shape {a.shape}")
        if a.dtype.kind not in "biuf":
            raise ValueError(f"PerObjectDistanceTransform: labels must be integers, got {a.dtype}")
        if a.dtype == np.uint32:
            a = a.astype(np.int64)
        elif a.dtype == np.uint64:
            a = a.astype(np.float64)
        t = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", torch.cuda.current_device()))
        return self._run(t).cpu().numpy()


class ResizeLabelTrafo:
    """micro_sam.training.util.ResizeLabelTrafo: PerObjectDistanceTransform with instances (4 channels: instances, foreground,
    centre and boundary distances), then a centred zero pad of H and W to desired_shape[0] (ceil before, floor after).  As in
    micro-sam both axes are padded to desired_shape[0], so a non-square desired_shape fails the final shape check.  Takes what
    PerObjectDistanceTransform takes; a batch (B, H, W) on the device comes back as (B, 4, H', W')."""

    def __init__(self, desired_shape: Tuple[int, ...], min_size: int = 0, padding: str = "constant"):
        if padding != "constant":
            raise NotImplementedError(f"ResizeLabelTrafo: padding mode {padding!r} is not supported (only 'constant')")
        self.desired_shape, self.min_size, self.padding = desired_shape, min_size, padding

    def __call__(self, labels):
        trafo = PerObjectDistanceTransform(distances=True, boundary_distances=True, directed_distances=False, foreground=True,
                                           instances=True, min_size=self.min_size)
        out = trafo(labels)
        dy, dx = (self.desired_shape[0] - out.shape[-2]) / 2, (self.desired_shape[0] - out.shape[-1]) / 2
        if min(dy, dx) < 0:
            raise ValueError(f"ResizeLabelTrafo: labels of {tuple(out.shape[-2:])} exceed the desired shape {self.desired_shape}")
        pads = (math.ceil(dy), math.floor(dy), math.ceil(dx), math.floor(dx))
        if torch.is_tensor(out):
            out = torch.nn.functional.pad(out, (pads[2], pads[3], pads[0], pads[1]))
        else:
            out = np.pad(out, ((0, 0), pads[:2], pads[2:]), mode="constant")
        assert tuple(out.shape[-2:]) == tuple(self.desired_shape), out.shape
        return out


def instance_train_iteration(unetr: UNETR, x, y, freeze_encoder: bool = True, loss=None, lr: float = 1e-5, betas=(0.9, 0.999),
                             eps: float = 1e-8, weight_decay: float = 0.01) -> torch.Tensor:
    """JointSamTrainer._instance_iteration (joint_sam_trainer.py:73-89) + its backward and AdamW step: x images (B, 3, H, W) in
    [0, 255], y targets (B, 3, H, W) (foreground, center and boundary distances).  Returns the loss (detached).
    `freeze_encoder=True` is train_instance_segmentation(freeze=["image_encoder"]): no encoder backward, the encoder untouched.
    Otherwise the loss is back-propagated through the encoder too and the step updates the encoder's tensors and the decoder's;
    the optimizer's other parameters (prompt encoder, mask decoder) have no gradient in this step and are skipped, as
    torch.optim.AdamW skips them after zero_grad()."""
    loss_fn = DiceBasedDistanceLoss() if loss is None else loss
    emb, input_size = unetr.embed(x, train_encoder=not freeze_encoder)
    pred = unetr.decode(emb, input_size, tuple(x.shape[-2:]))
    value = loss_fn(pred, y.to(pred.device))
    value.backward()
    if not freeze_encoder:
        unetr.sam.optimizer_step_prefix("image_encoder.", lr, betas, eps, weight_decay)
    unetr.optimizer_step(lr, betas, eps, weight_decay)
    return value.detach()


def joint_train_iteration(model: TrainableSAM, unetr: UNETR, x, y, y_instance, iteration: int, n_objects_per_batch: int = 25,
                          n_sub_iteration: int = 8, mask_prob: float = 0.5, convert_inputs: Optional[ConvertToSamInputs] = None,
                          lr: float = 1e-5, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01):
    """One iteration of JointSamTrainer._train_epoch_impl (joint_sam_trainer.py:99-114): the interactive iteration on the label
    images `y` (`interactive_train_iteration`), its backward and AdamW step over the SAM model; then the instance iteration on
    the UNETR targets `y_instance` through the encoder, its backward and a step over the encoder and the UNETR decoder.  `unetr`
    must be built on `model.sam`.  Returns (interactive loss, instance loss), detached."""
    if unetr.sam is not model.sam:
        raise ValueError("joint training: the UNETR must share the SAM model's image encoder")
    sam = model.sam
    sam.train()
    sam.zero_decoder_grads()
    loss = interactive_train_iteration(model, x, y, iteration, n_objects_per_batch, n_sub_iteration, mask_prob, convert_inputs)[0]
    loss.backward()
    sam.optimizer_step(lr, betas, eps, weight_decay)
    sam.zero_decoder_grads()   # optimizer.zero_grad(): the prompt encoder and mask decoder get no gradient in the instance step
    unetr_loss = instance_train_iteration(unetr, x, y_instance, freeze_encoder=False, lr=lr, betas=betas, eps=eps,
                                          weight_decay=weight_decay)
    return loss.detach(), unetr_loss


# ---------------------------------------------------------------------------------------------------------------------------------
# Semantic segmentation loss: micro_sam/training/semantic_sam_trainer.py:11-86 (CustomDiceLoss, SemanticSamTrainer._compute_loss)
# and micro_sam/training/util.py:268-280 (ConvertToSemanticSamInputs)

MAX_SEMANTIC_CLASSES = 15


class ConvertToSemanticSamInputs:
    """micro_sam.training.util.ConvertToSemanticSamInputs: one record {"image", "original_size"} per image, with no prompts."""

    def __call__(self, x, y):
        return [{"image": image, "original_size": image.shape[-2:]} for image in x]


class _SemanticStatsFn(torch.autograd.Function):
    """msam_semantic_loss_stats with its adjoint (msam_semantic_loss_backward): the loss depends on the logits only through the
    per-class sums (sum p t, sum p^2) and the cross-entropy sum; the counts are piecewise constant."""

    @staticmethod
    def forward(ctx, lr, labels, in_h, in_w):
        B, C = lr.shape[:2]
        H, W = labels.shape[-2:]
        L = _lib.lib()
        label64 = int(labels.dtype == torch.int64)
        ws = torch.empty(int(L.msam_semantic_loss_workspace(B, C, in_h, in_w, H, W, 0)), device=lr.device, dtype=torch.uint8)
        st = torch.empty(3 * C + 3, device=lr.device, dtype=torch.float64)
        _lib.check(L.msam_semantic_loss_stats(_lib.ptr(lr), _lib.ptr(labels), label64, B, C, in_h, in_w, H, W, _lib.ptr(ws), ws.numel(),
                                              _lib.ptr(st), _lib.cur_stream()))
        ctx.save_for_backward(lr, labels)
        ctx.geom = (in_h, in_w)
        return st

    @staticmethod
    def backward(ctx, d_st):
        lr, labels = ctx.saved_tensors
        B, C = lr.shape[:2]
        H, W = labels.shape[-2:]
        in_h, in_w = ctx.geom
        L = _lib.lib()
        ws = torch.empty(int(L.msam_semantic_loss_workspace(B, C, in_h, in_w, H, W, 1)), device=lr.device, dtype=torch.uint8)
        ds = d_st.to(torch.float64).contiguous()
        d_lr = torch.empty_like(lr)
        _lib.check(L.msam_semantic_loss_backward(_lib.ptr(lr), _lib.ptr(labels), int(labels.dtype == torch.int64), _lib.ptr(ds), B, C,
                                                 in_h, in_w, H, W, _lib.ptr(ws), ws.numel(), _lib.ptr(d_lr), _lib.cur_stream()))
        return d_lr, None, None, None


def _semantic_inputs(pred, y, num_classes: int, input_size=None, original_size=None):
    """(low-res logits fp32 (B, C, 256, 256), labels int32 / int64 (B, H, W), input_size) from either the batched outputs of
    `TrainableSAM.forward` (records with "low_res_masks" (1, C, 256, 256) or (C, 256, 256), "input_size", "original_size") or the
    low-res logits themselves; `input_size` defaults to the resized shape of the original size (ResizeLongestSide(1024))."""
    from .sam import get_preprocess_shape
    if isinstance(pred, (list, tuple)):
        if not pred:
            raise ValueError("semantic loss: no outputs")
        lows = [o["low_res_masks"] for o in pred]
        lows = [lo.squeeze(0) if lo.dim() == 4 else lo for lo in lows]
        low = torch.stack(lows)
        sizes = {tuple(int(s) for s in o["input_size"]) for o in pred}
        origs = {tuple(int(s) for s in o["original_size"]) for o in pred}
        if len(sizes) != 1 or len(origs) != 1:
            raise ValueError("semantic loss: every image of the batch needs the same input_size and original_size")
        input_size, original_size = sizes.pop(), origs.pop()
    else:
        low = pred
    if low.dim() != 4 or tuple(low.shape[-2:]) != (256, 256):
        raise ValueError(f"semantic loss: takes the low-res logits (B, C, 256, 256), got {tuple(low.shape)}; the full-resolution "
                         "logits are evaluated per pixel from them and never materialised")
    B, C = int(low.shape[0]), int(low.shape[1])
    if C != num_classes:
        raise ValueError(f"semantic loss: {C} logit channels for num_classes={num_classes}")
    if not 1 <= C <= MAX_SEMANTIC_CLASSES:
        raise ValueError(f"semantic loss: num_classes={C}; the loss kernels take 1..{MAX_SEMANTIC_CLASSES} classes")
    lab = torch.as_tensor(y)
    if lab.dim() == 4 and lab.shape[1] == 1:
        lab = lab[:, 0]
    if lab.dim() != 3 or lab.shape[0] != B:
        raise ValueError(f"semantic loss: labels (B, 1, H, W) or (B, H, W) with B={B}, got {tuple(lab.shape)}")
    H, W = int(lab.shape[-2]), int(lab.shape[-1])
    if original_size is not None and tuple(int(s) for s in original_size) != (H, W):
        raise ValueError(f"semantic loss: original_size {tuple(original_size)} but labels of size {(H, W)}")
    if input_size is None:
        input_size = get_preprocess_shape(H, W, 1024)
    lab = lab.to(low.device)
    if lab.dtype not in (torch.int32, torch.int64):
        lab = lab.long()            # nn.CrossEntropyLoss takes target.long()
    return low.to(torch.float32).contiguous(), lab.contiguous(), (int(input_size[0]), int(input_size[1]))


def semantic_loss_stats(pred, y, num_classes: int, input_size=None, original_size=None) -> torch.Tensor:
    """`msam_semantic_loss_stats` (fp64 (3 C + 3,)), differentiable w.r.t. the low-res logits; raises ValueError when a label lies
    outside [0, num_classes) and is not -100 (nn.CrossEntropyLoss's ignore_index), as torch refuses such a target."""
    low, lab, (in_h, in_w) = _semantic_inputs(pred, y, num_classes, input_size, original_size)
    st = _SemanticStatsFn.apply(low, lab, in_h, in_w)
    n_bad = int(st[3 * num_classes + 2].item())
    if n_bad:
        raise ValueError(f"semantic loss: {n_bad} labels outside [0, {num_classes}) (only -100, the ignore index, is allowed)")
    return st


def _semantic_dice(st: torch.Tensor, C: int, eps: float = 1e-7) -> torch.Tensor:
    pt, pp, t = st[:3 * C].view(C, 3).unbind(-1)
    return (1.0 - 2.0 * pt / (pp + t).clamp(min=eps)).sum()       # one-hot targets: sum t^2 = sum t


class CustomDiceLoss:
    """micro_sam.training.semantic_sam_trainer.CustomDiceLoss: softmax over the classes, one-hot targets (label == c; -100 in no
    class), torch_em's DiceLoss() = sum over the classes of 1 - 2 sum(p t) / max(sum p^2 + sum t^2, 1e-7), each sum over the whole
    batch.  `__call__(pred, target)` takes the batched outputs of `TrainableSAM.forward` or the low-res logits (B, C, 256, 256)
    (with `input_size` / `original_size` keywords); the full-resolution logits are evaluated per pixel and never materialised."""

    def __init__(self, num_classes: int, softmax: bool = True) -> None:
        if not softmax:
            raise NotImplementedError("CustomDiceLoss(softmax=False): the loss kernels take the softmax of the logits")
        self.num_classes = num_classes
        self.softmax = softmax

    def __call__(self, pred, target, input_size=None, original_size=None) -> torch.Tensor:
        st = semantic_loss_stats(pred, target, self.num_classes, input_size, original_size)
        return _semantic_dice(st, self.num_classes).to(torch.float32)


def _check_dice_weight(dice_weight) -> None:
    if dice_weight is not None and (dice_weight < 0 or dice_weight > 1):
        raise ValueError("The weight factor should lie between 0 and 1.")


def compute_semantic_loss(pred, y, num_classes: int, dice_weight: Optional[float] = None, input_size=None,
                          original_size=None) -> torch.Tensor:
    """SemanticSamTrainer._compute_loss: CustomDiceLoss + nn.CrossEntropyLoss() (the mean over the pixels whose label is not -100)
    of the full-resolution logits, or w * dice + (1 - w) * CE for `dice_weight` w in [0, 1].  `pred`: the batched outputs of
    `TrainableSAM.forward` or the low-res logits (B, C, 256, 256); `y`: labels (B, 1, H, W) or (B, H, W).  Both terms come from one
    pass of msam_semantic_loss_stats and are combined in fp64; the result is fp32 and differentiable w.r.t. the low-res logits."""
    _check_dice_weight(dice_weight)
    st = semantic_loss_stats(pred, y, num_classes, input_size, original_size)
    dice = _semantic_dice(st, num_classes)
    ce = st[3 * num_classes] / st[3 * num_classes + 1]
    loss = dice + ce if dice_weight is None else dice_weight * dice + (1 - dice_weight) * ce
    return loss.to(torch.float32)


def get_trainable_sam_model(model_type: str = "vit_b", device=None, checkpoint_path=None, freeze=None, return_state: bool = False,
                            peft_kwargs=None, flexible_load_checkpoint: bool = False, **model_kwargs):
    """micro_sam.training.util.get_trainable_sam_model (util.py:77): a `TrainableSAM` in train() mode (and the checkpoint state
    with `return_state`).  `model_kwargs` go to `util.get_sam_model` (e.g. `state_dict=`, `max_batch=`), which refuses
    `num_multimask_outputs` other than 3 and `flexible_load_checkpoint`.  A semantic model with 3 classes is this model with
    `multimask_output=True`."""
    from . import util
    if freeze is not None:
        raise NotImplementedError("get_trainable_sam_model(freeze=...): frozen parameter groups are not implemented; every "
                                  "parameter of the model is trained")
    if peft_kwargs:
        raise NotImplementedError("get_trainable_sam_model(peft_kwargs=...): parameter-efficient fine-tuning (LoRA and the other "
                                  "PEFT wrappers) is not implemented")
    _, sam, state = util.get_sam_model(model_type=model_type, device=device, checkpoint_path=checkpoint_path, return_sam=True,
                                       return_state=True, flexible_load_checkpoint=flexible_load_checkpoint, **model_kwargs)
    sam.train()
    model = TrainableSAM(sam)
    return (model, state) if return_state else model


def semantic_train_iteration(model: TrainableSAM, x, y, num_classes: int, dice_weight: Optional[float] = None,
                             convert_inputs=None) -> torch.Tensor:
    """The body of SemanticSamTrainer._train_epoch_impl (semantic_sam_trainer.py:113-140): records without prompts
    (`ConvertToSemanticSamInputs`), one encoder pass, one prompt-free decode of the whole batch with `multimask_output=True`, and
    `compute_semantic_loss` from the low-res logits.  Returns the loss; the caller zeroes the gradients
    (`sam.zero_decoder_grads()`), calls `loss.backward()` and then `sam.optimizer_step()` (after `sam.allreduce_grads(...)` when
    training on several GPUs).  The decoder gives 3 channels, so `num_classes` must be 3."""
    convert_inputs = ConvertToSemanticSamInputs() if convert_inputs is None else convert_inputs
    batched_inputs = convert_inputs(x, y)
    image_embeddings, batched_inputs = model.image_embeddings_oft(batched_inputs)
    outputs = model(batched_inputs, image_embeddings, multimask_output=True, return_masks=False)
    return compute_semantic_loss(outputs, y, num_classes, dice_weight)


def semantic_validation(model: TrainableSAM, loader, num_classes: int, dice_weight: Optional[float] = None,
                        convert_inputs=None) -> Tuple[float, float]:
    """SemanticSamTrainer._validate_impl (semantic_sam_trainer.py:143-170): eval() mode and no_grad, the mean loss over `loader`
    (an iterable of (x, y) batches with a length) as both metric and loss.  The model's previous mode is restored afterwards.
    The batch is decoded by the training decoder's forward pass (`decode_images_with_training_decoder`, slot 0), so that
    validation between optimizer steps sees the weights trained so far.  Returns (metric, loss)."""
    convert_inputs = ConvertToSemanticSamInputs() if convert_inputs is None else convert_inputs
    was_training = bool(model.sam.training)
    model.sam.eval()
    try:
        total = 0.0
        with torch.no_grad():
            for x, y in loader:
                batched_inputs = convert_inputs(x, y)
                image_embeddings, batched_inputs = model.image_embeddings_oft(batched_inputs)
                low, _ = model.sam.decode_images_with_training_decoder(image_embeddings, True)
                outputs = [{"low_res_masks": low[b:b + 1], "input_size": tuple(rec["input_size"]),
                            "original_size": tuple(rec["original_size"])} for b, rec in enumerate(batched_inputs)]
                total += float(compute_semantic_loss(outputs, y, num_classes, dice_weight).item())
    finally:
        model.sam.train(was_training)
    loss = total / len(loader)
    return loss, loss


def export_instance_segmentation_model(unetr: UNETR, output_path) -> None:
    """export_instance_segmentation_model (training.py:378) with a different signature: the reference reads a trainer checkpoint
    (trained_model_path, output_path, model_type, initial_checkpoint_path); this writes the in-memory model.  The file is the same:
    {"model_state": the SAM weights ("sam."-prefixed; the optimizer's masters where it trained them), "decoder_state": the UNETR
    decoder}, loadable by get_predictor_and_decoder."""
    model_state = {"sam." + k: v.detach().cpu() for k, v in unetr.sam.trained_state_dict().items()}
    torch.save({"model_state": model_state, "decoder_state": unetr.decoder_state_dict()}, output_path)
