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
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple

import torch

from . import _lib
from .sam import B200Sam, ResizeLongestSide


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
                           multimask_output: bool, update_prompts):
    """SamTrainer._compute_iterative_loss (sam_trainer.py:243-289) -> (loss, mask_loss, iou_regression_loss, mean_model_iou),
    each averaged over the `num_subiter` passes.  Pass 0 uses `multimask_output`, the later ones a single mask.  Between passes
    `update_prompts(batched_inputs, masks, logits)` runs under no_grad with the best mask per object (binary full-size (B, n_obj,
    1, H, W) and low-res logits (B, n_obj, 1, 256, 256), `get_best_masks`) and returns the records of the next pass, e.g. with
    more points and the logits as "mask_inputs".

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
            outputs = model(batched_inputs, emb, multimask_output=multimask, return_masks=not last)
            net_loss, net_mask_loss, net_iou_loss = compute_loss(outputs, y_one_hot)
            (net_loss / num_subiter).backward()
            d_emb += emb.grad
        else:
            with torch.no_grad():
                outputs = model(batched_inputs, image_embeddings, multimask_output=multimask, return_masks=not last)
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
