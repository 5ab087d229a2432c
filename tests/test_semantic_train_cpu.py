"""CPU tests of semantic training (records without prompts, micro_sam/training/semantic_sam_trainer.py):

* the float64 decoder mirror (tests/decoder_train_mirror.py) with empty sparse prompts, summed over the images of a batch, is the
  oracle's TrainableSAM (oracle/train_ref.py on oracle/sam_ref.py) under the float64 semantic loss (oracle/semantic_ref.py) with
  torch autograd: the prompt-free GPU decode is checked against that mirror in tests/test_gpu_semantic_train.py;
* which parameters such a loss reaches: torch leaves `.grad` None for the IoU head, the point embeddings, not_a_point_embed and
  mask_downscaling, and gives output_hypernetworks_mlps.0 an all-zero gradient (the [:, 1:] slice), which is the rule the
  optimizer's skip follows;
* the host-side refusals of `get_trainable_sam_model`, the decoder-slot grouping of `TrainableSAM.forward` in training mode, and
  the C-ABI declaration."""
import os
import re

import pytest
import torch

from oracle import semantic_ref
from tests import decoder_train_mirror as mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORIG = (60, 90)                      # original size of the labels; input_size = (683, 1024)
SKIPPED = ("mask_decoder.iou_prediction_head.", "prompt_encoder.point_embeddings.", "prompt_encoder.not_a_point_embed.",
           "prompt_encoder.mask_downscaling.")


@pytest.fixture(scope="module")
def sd():
    from oracle import sam_ref
    return sam_ref.seeded_state_dict("vit_test", seed=1)


def _oracle64(sd):
    from oracle import sam_ref, train_ref
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    osam.double()
    pe = osam.prompt_encoder.pe_layer      # the dense positional encoding (no parameters) in float32, as the oracle computes it
    pe.positional_encoding_gaussian_matrix = pe.positional_encoding_gaussian_matrix.float()
    for p in osam.parameters():
        p.requires_grad_(True)
    return train_ref.TrainableSAM(osam)


def _batch(B, C, seed):
    from oracle.sam_ref import get_preprocess_shape
    gen = torch.Generator().manual_seed(seed)
    emb = torch.randn(B, 256, 64, 64, generator=gen, dtype=torch.float64)
    y = torch.randint(0, C, (B, 1) + ORIG, generator=gen)
    recs = [{"original_size": ORIG, "input_size": get_preprocess_shape(*ORIG, 1024)} for _ in range(B)]
    return emb, y, recs


def _oracle_step(sd, B, dice_weight, seed=5):
    """oracle TrainableSAM with prompt-free records, multimask_output=True, semantic loss of its low-res logits, autograd."""
    model = _oracle64(sd)
    emb, y, recs = _batch(B, 3, seed)
    emb.requires_grad_(True)
    outs = model(recs, emb, multimask_output=True)
    lows = [o["low_res_masks"] for o in outs]
    for lo in lows:
        lo.retain_grad()
    low = torch.cat(lows)
    loss = semantic_ref.semantic_loss_from_low_res(low, y, recs[0]["input_size"], ORIG, 3, dice_weight)
    loss.backward()
    params = {k: p for k, p in model.sam.named_parameters() if k.startswith(("mask_decoder.", "prompt_encoder."))}
    return model, emb, lows, params


@pytest.mark.parametrize("dice_weight", [None, 0.3])
def test_mirror_without_rounding_is_the_prompt_free_oracle(sd, dice_weight, monkeypatch):
    """Per image: the mirror with sparse (1, 0, 256) and emb_index (1, 0), fed the oracle's dL/d low-res, gives the oracle's
    low-res logits and dL/d embedding; its parameter gradients summed over the images are the oracle's."""
    monkeypatch.setattr(mirror, "ROUND", False)
    B = 2
    model, emb, lows, params = _oracle_step(sd, B, dice_weight)
    with torch.no_grad():
        dense_pe = model.sam.prompt_encoder.get_dense_pe()[0].double()
    total = None
    for b in range(B):
        r = mirror.run(sd, emb[b].detach(), torch.zeros(1, 0, 256, dtype=torch.float64), torch.zeros(1, 0, dtype=torch.int64),
                       dense_pe, True, lows[b].grad, None)
        assert float((r["low_res"] - lows[b].detach()).abs().max()) <= 1e-10 * float(lows[b].detach().abs().max())
        assert float((r["d_emb"] - emb.grad[b]).norm()) <= 1e-10 * float(emb.grad[b].norm())
        total = r["grads"] if total is None else {k: total[k] + v for k, v in r["grads"].items()}
    scale = max(float(v.norm()) for v in total.values())
    for k, g in total.items():
        want = params[k].grad
        want = torch.zeros_like(g) if want is None else want
        assert float((g - want).norm()) <= 1e-10 * max(float(want.norm()), 1e-6 * scale), k


def test_prompt_free_loss_reaches_these_parameters(sd):
    """The optimizer skip rule: after a semantic backward, exactly the IoU head, the point embeddings, not_a_point_embed and
    mask_downscaling have grad None; output_hypernetworks_mlps.0 has a gradient of zeros; every other tensor a nonzero one."""
    _, _, _, params = _oracle_step(sd, 2, None)
    none = sorted(k for k, p in params.items() if p.grad is None)
    assert none == sorted(k for k in params if k.startswith(SKIPPED))
    assert {k.split(".")[1] for k in none} == {"iou_prediction_head", "point_embeddings", "not_a_point_embed", "mask_downscaling"}
    hyper0 = [k for k in params if k.startswith("mask_decoder.output_hypernetworks_mlps.0.")]
    assert hyper0 and all(params[k].grad is not None and not params[k].grad.any() for k in hyper0)
    rest = [k for k in params if k not in none and k not in hyper0 and not k.endswith("k_proj.bias")]
    assert all(params[k].grad.abs().max() > 0 for k in rest), [k for k in rest if not params[k].grad.abs().max() > 0]
    assert params["prompt_encoder.no_mask_embed.weight"].grad.abs().max() > 0


def test_get_trainable_sam_model_refusals():
    from micro_sam_b200 import training
    sd = {"mask_decoder.mask_tokens.weight": torch.zeros(4, 256)}
    with pytest.raises(NotImplementedError, match="freeze"):
        training.get_trainable_sam_model("vit_b", state_dict=sd, freeze=["image_encoder"])
    with pytest.raises(NotImplementedError, match="peft"):
        training.get_trainable_sam_model("vit_b", state_dict=sd, peft_kwargs={"rank": 2})
    for kw in ({"num_multimask_outputs": 4}, {"flexible_load_checkpoint": True}):
        with pytest.raises(NotImplementedError, match="num_multimask_outputs|flexible_load_checkpoint"):
            training.get_trainable_sam_model("vit_b", state_dict=sd, **kw)


def test_decoder_slots():
    """Prompted records take slots 0, 1, ... in batch order (a batch with prompts only keeps slot i for record i); the records
    without prompts share the next slot; more than 8 slots are refused, any number of prompt-free records is not."""
    from micro_sam_b200.training import decoder_slots
    P, F = {"boxes": 0}, {"image": 0}
    assert decoder_slots([P] * 8) == list(range(8))
    assert decoder_slots([F] * 16) == [None] * 16
    assert decoder_slots([F, P, F, {"point_coords": 0}, {"mask_inputs": 0}]) == [None, 0, None, 1, 2]
    assert decoder_slots([P] * 7 + [F] * 9) == list(range(7)) + [None] * 9
    with pytest.raises(ValueError, match="8"):
        decoder_slots([P] * 8 + [F])
    with pytest.raises(ValueError, match="8"):
        decoder_slots([P] * 9)


def test_header_declares_prompt_free_training_decode():
    hdr = open(os.path.join(ROOT, "include", "msam_b200.h")).read()
    decl = re.search(r"int msam_decoder_train_forward_images\(([^)]*)\);", hdr)
    assert decl, "msam_decoder_train_forward_images is not declared"
    args = [a.split()[-1].lstrip("*") for a in decl.group(1).replace("\n", " ").split(",")]
    assert args == ["h", "slot", "emb_nchw", "B", "multimask", "low_res", "iou", "stream"]
    assert "[B, 256, 64, 64]" in hdr
