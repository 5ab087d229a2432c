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
        graph (point, box and `mask_inputs` prompts; the mask inputs get no gradient): image i of the batch uses decoder slot i,
        which holds its activations until its backward pass has run."""
        if getattr(self.sam, "training", False) and torch.is_grad_enabled():
            return self._forward_train(batched_inputs, image_embeddings, multimask_output, return_masks)
        with torch.no_grad():
            return self._forward_eval(batched_inputs, image_embeddings, multimask_output, return_masks)

    def _forward_train(self, batched_inputs, image_embeddings, multimask_output, return_masks):
        sam, dev = self.sam, self.sam.device
        if len(batched_inputs) > 8:
            raise ValueError("training forward: at most 8 images per call (one decoder slot per image until its backward pass has run)")
        outputs = []
        for i, (rec, emb) in enumerate(zip(batched_inputs, image_embeddings)):
            points = (rec["point_coords"].to(dev), rec["point_labels"].to(dev)) if "point_coords" in rec else None
            boxes = rec["boxes"].to(dev) if "boxes" in rec else None
            masks = rec["mask_inputs"].to(dev) if "mask_inputs" in rec else None
            low, iou = sam.decoder_train(emb, points, boxes, multimask_output, slot=i % 8, masks=masks)
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
