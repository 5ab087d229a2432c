"""`-m gpu`: `training.compute_iterative_loss` (micro-sam's SamTrainer._compute_iterative_loss) against the oracle TrainableSAM running
the reference loop under fp32 autograd: B = 2 images, 25 box-prompted objects each, 8 passes, multimask output in pass 0 and mask
prompts (the previous best logits) plus one more point per object in passes 1..7.  Every pass of the library runs on a detached
embedding and is back-propagated at once; the encoder sees the summed embedding gradient once.

Which mask token an object's gradient reaches in pass 0 is chosen by the minimum of its 3 dice losses.  With the seeded weights the
3 candidate masks are close (the smallest margin between best and second-best dice is 5.8e-5), so the test first checks that the
library and the oracle make the same choice for every object; the gradients are only comparable if they do.  The choice leaves a
mask token that 1 or 2 objects select (here token 3, 1 of 50): the gradient of its hyper-network MLP is that one object's dice term,
270x smaller in norm than token 0's, so the bf16 noise is not averaged over objects as in every other tensor.  Tensors of such a
token are bounded by twice their measured value; tokens no object selects must get a zero gradient.

Measured on one H100 80GB HBM3 at a 700 W power limit (two runs, identical results): loss 1.0955 against the oracle's 1.0950;
encoder gradients rel-L2 <= 2.7e-2; decoder and prompt-encoder gradients rel-L2 <= 3.5e-2 (layers.*.self_attn.q_proj.weight),
cosine >= 0.9994, mask_downscaling <= 2.1e-2 -- bounds 1.5e-1 / 0.99, the end-to-end bounds of tests/test_gpu_backward.py; the
MLP of the one-object token 3: rel-L2 1.61e-1, cosine 0.98696 -- bound 3.3e-1 / 0.974.
"""
import gc

import numpy as np
import pytest
import torch

from tests import mask_prompt_mirror as mmirror

pytestmark = pytest.mark.gpu
DEV = "cuda"
FEW = 2                 # a mask token selected by at most this many objects in pass 0 gets the single-object bound
FEW_BOUND = (3.3e-1, 0.974)


@pytest.fixture(autouse=True)
def _free_device_memory():
    """Models of earlier tests hold decoder-slot arenas of several GB until they are collected."""
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _setup(n_obj=25):
    from oracle import sam_ref
    from micro_sam_b200 import util
    from micro_sam_b200.sample_data import lm_tile
    sd = mmirror.perturbed_state_dict()
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    osam.to(DEV)
    for p in osam.parameters():
        p.requires_grad_(True)
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
    sam.train()
    B, H, W = 2, 128, 128
    imgs = [torch.from_numpy(np.repeat(lm_tile((H, W), 12, seed=50 + b, dtype="uint8")[None], 3, 0).astype("float32")) for b in range(B)]
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    cen = [(12 + 24 * (k // 5), 12 + 24 * (k % 5), 6 + k % 4) for k in range(n_obj)]
    y1 = torch.stack([(((yy - cy) ** 2 + (xx - cx) ** 2) < r * r).float()[None] for cy, cx, r in cen])
    y_one_hot = torch.stack([y1, y1.flip(-1)])
    boxes = [torch.tensor([[cx - r, cy - r, cx + r, cy + r] for cy, cx, r in cen], dtype=torch.float32) * (1024.0 / W)]
    boxes.append(boxes[0].clone())
    boxes[1][:, [0, 2]] = 1024.0 - boxes[1][:, [2, 0]]

    def records(dev):
        return [{"image": im.clone().to(dev), "original_size": (H, W), "boxes": bx.clone().to(dev)} for im, bx in zip(imgs, boxes)]

    def update_prompts(batched_inputs, masks, logits):
        """deterministic stand-in for the prompt generator: one more positive point per object at the centre of its box, and the
        best logits as mask prompts"""
        for b, (rec, lg) in enumerate(zip(batched_inputs, logits)):
            dev = rec["boxes"].device
            c = ((boxes[b][:, :2] + boxes[b][:, 2:]) / 2)[:, None].to(dev)
            rec["point_coords"] = torch.cat([rec["point_coords"], c], 1) if "point_coords" in rec else c
            lab = torch.ones(c.shape[0], 1, device=dev)
            rec["point_labels"] = torch.cat([rec["point_labels"], lab], 1) if "point_labels" in rec else lab
            rec["mask_inputs"] = lg.to(dev)
        return batched_inputs
    return osam, sam, records, update_prompts, y_one_hot


def _dice_choice(outputs, y_one_hot):
    """per image, the candidate mask each object's loss takes (argmin of its dice losses, SamTrainer._compute_loss)"""
    from oracle import train_ref
    out = []
    for o, y in zip(outputs, y_one_hot):
        y = y.to(o["masks"].device)
        pred = torch.sigmoid(o["masks"].float())
        d = torch.stack([train_ref.dice_loss_per_channel(pred[:, i:i + 1].swapaxes(0, 1), y.swapaxes(0, 1)) for i in range(pred.shape[1])])
        out.append(d.argmin(0).cpu())
    return out


def _oracle_iterative_loss(osam, records, y_one_hot, update_prompts, num_subiter, multimask):
    """SamTrainer._compute_iterative_loss on the oracle (one graph, one backward) + the pass-0 dice choices"""
    from oracle import train_ref
    om = train_ref.TrainableSAM(osam)
    emb, recs = om.image_embeddings_oft(records(DEV))
    yo = [y.to(DEV) for y in y_one_hot]
    loss, choice = 0.0, None
    for i in range(num_subiter):
        outs = om(recs, emb, multimask_output=multimask if i == 0 else False)
        loss = loss + train_ref.compute_loss(outs, yo)[0]
        with torch.no_grad():
            if i == 0:
                choice = _dice_choice(outs, yo)
            if i < num_subiter - 1:
                logits = [o["low_res_masks"][torch.arange(o["iou_predictions"].shape[0]), o["iou_predictions"].argmax(1)][:, None]
                          for o in outs]
                recs = update_prompts(recs, None, logits)
    return loss / num_subiter, choice


def _library_pass0_choice(sam, records, y_one_hot):
    from micro_sam_b200 import training
    m = training.TrainableSAM(sam)
    emb, recs = m.image_embeddings_oft(records("cpu"))
    outs = m(recs, emb.detach(), multimask_output=True)     # the training decoder, as in compute_iterative_loss's pass 0
    with torch.no_grad():
        return _dice_choice(outs, y_one_hot)


def test_iterative_loss_against_the_oracle():
    from micro_sam_b200 import training
    from tests.test_gpu_backward import _compare_grads
    osam, sam, records, update_prompts, y_one_hot = _setup()
    oloss, ochoice = _oracle_iterative_loss(osam, records, y_one_hot, update_prompts, 8, True)
    oloss.backward()
    gchoice = _library_pass0_choice(sam, records, y_one_hot)
    differ = [(b, int(k)) for b in range(2) for k in torch.nonzero(gchoice[b] != ochoice[b]).flatten()]
    assert not differ, f"pass-0 mask choice differs from the oracle for (image, object) {differ}: gradients not comparable"
    counts = torch.bincount(torch.cat(ochoice), minlength=3)            # candidate i = mask token i + 1
    few = [f"mask_decoder.output_hypernetworks_mlps.{i + 1}." for i in range(3) if 0 < int(counts[i]) <= FEW]
    sam.zero_decoder_grads()
    m = training.TrainableSAM(sam)
    loss, mask_loss, iou_loss, miou = training.compute_iterative_loss(m, records("cpu"), list(y_one_hot), 8, True, update_prompts)
    loss.backward()
    ref = dict(osam.cpu().named_parameters())      # Module.cpu() moves the gradients too
    r_enc, bad_enc = _compare_grads(sam.encoder_grads(), ref, 1.5e-1, min_cos=0.99)
    dec = sam.decoder_grads()
    is_few = lambda k: any(k.startswith(f) for f in few)   # noqa: E731
    r_dec, bad_dec = _compare_grads({k: v for k, v in dec.items() if not is_few(k)}, ref, 1.5e-1, min_cos=0.99)
    r_few, bad_few = _compare_grads({k: v for k, v in dec.items() if is_few(k)}, ref, FEW_BOUND[0], min_cos=FEW_BOUND[1])
    md = {k.split("mask_downscaling.")[1]: f"{v:.2e}" for k, v in r_dec.items() if "mask_downscaling" in k}
    worst = sorted(r_dec.items(), key=lambda kv: -kv[1])[:3]
    print(f"\niterative loss (8 passes): {float(loss):.4f} (oracle {float(oloss):.4f}), mask {float(mask_loss):.4f}, iou "
          f"{float(iou_loss):.4f}, mean iou {float(miou):.4f}; pass-0 choices per mask token {counts.tolist()}; encoder max rel-L2 "
          f"{max(r_enc.values()):.2e}; decoder worst " + ", ".join(f"{k.split('.', 1)[1]} {v:.2e}" for k, v in worst)
          + f"; few-object tokens {few}: " + ", ".join(f"{k.split('.', 1)[1]} {v:.2e}" for k, v in r_few.items())
          + f"; mask_downscaling {md}", flush=True)
    assert abs(float(loss) - float(oloss)) < 2e-2
    assert len(md) == 10
    assert not bad_enc and not bad_dec and not bad_few, (bad_enc, bad_dec, bad_few)


def test_iterative_loss_refuses_a_scaled_backward():
    from micro_sam_b200 import training
    _, sam, records, update_prompts, y_one_hot = _setup(n_obj=3)
    sam.zero_decoder_grads()
    loss = training.compute_iterative_loss(training.TrainableSAM(sam), records("cpu"), list(y_one_hot), 2, False, update_prompts)[0]
    with pytest.raises(ValueError, match="upstream gradient"):
        (2 * loss).backward()


def test_iterative_loss_refuses_zeroing_between_passes_and_backward():
    """the decoder gradients of the passes exist when compute_iterative_loss returns; zero_decoder_grads() after it loses them"""
    from micro_sam_b200 import training
    _, sam, records, update_prompts, y_one_hot = _setup(n_obj=3)
    sam.zero_decoder_grads()
    loss = training.compute_iterative_loss(training.TrainableSAM(sam), records("cpu"), list(y_one_hot), 2, False, update_prompts)[0]
    assert any(bool(v.any()) for v in sam.decoder_grads().values())
    sam.zero_decoder_grads()
    with pytest.raises(RuntimeError, match="zero_decoder_grads"):
        loss.backward()


def test_iterative_loss_forward_only_in_eval_mode():
    """the reference's validation loop (eval() and no_grad): forward passes only, no gradient touched, the oracle's loss"""
    from micro_sam_b200 import training
    osam, sam, records, update_prompts, y_one_hot = _setup(n_obj=3)
    with torch.no_grad():
        oloss, _ = _oracle_iterative_loss(osam, records, y_one_hot, update_prompts, 3, True)
    sam.eval()
    with torch.no_grad():
        loss, mask_loss, iou_loss, miou = training.compute_iterative_loss(training.TrainableSAM(sam), records("cpu"), list(y_one_hot),
                                                                          3, True, update_prompts)
    assert not loss.requires_grad
    assert abs(float(loss) - float(oloss)) < 2e-2, (float(loss), float(oloss))
