"""`-m gpu`: the registry of trainable tensors (`msam_train_tensor_count / _info`, `B200Sam.grad_views()`) after one training step
on vit_test: an encoder backward fed by one unmasked and one masked training-decoder pass.

* every registered tensor is an upstream tensor: the keys (without "@gemm") are the trained state-dict keys, the element counts
  the upstream ones, and exactly three convolution weights are held in their GEMM layout;
* the views are the gradients: unpacked, they equal `encoder_grads()` and `decoder_grads()`, and their squared norms add up to
  those of the upstream gradients (the global norm a trainer clips over `grad_views()`);
* `optimizer_step()` writes no gradient buffer, so two steps on one backward are two `torch.optim.AdamW` steps on the same gradients;
* the gradient read-outs are copies.
"""
import pytest
import torch

from tests import mask_prompt_mirror as mmirror

pytestmark = pytest.mark.gpu
DEV = "cuda"
GEMM_KEYS = {"mask_decoder.output_upscaling.0.weight", "mask_decoder.output_upscaling.3.weight", "image_encoder.neck.2.weight"}


def _model():
    from micro_sam_b200 import util
    sd = mmirror.perturbed_state_dict()
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=1, max_prompts=64).model
    sam.train()
    return sd, sam


def _backward(sam, seed):
    """zero_decoder_grads(), then the encoder forward, an unmasked (multimask, points + box) and a masked (single mask, box) training
    decoder pass on its embedding, and one backward through all three."""
    from tests.test_gpu_decoder_train import make_inputs, to_dev
    from tests.test_gpu_mask_prompt_train import _masks
    gen = torch.Generator().manual_seed(seed)
    sam.zero_decoder_grads()
    emb = sam.image_encoder(torch.randn(1, 3, 1024, 1024, generator=gen).to(DEV))[0]
    outs, d_outs = [], []
    for slot, (P, labels, mm, masked) in enumerate(((3, [[1, 0]] * 3, True, False), (4, None, False, True))):
        _, pts, boxes, d_low, d_iou = make_inputs(P, labels, True, mm, seed + slot)
        p, b = to_dev(pts, boxes)
        masks = _masks("logits", P, seed + slot).to(DEV) if masked else None
        outs += sam.decoder_train(emb, p, b, mm, slot=slot, masks=masks)
        d_outs += [d_low.to(DEV), d_iou.to(DEV)]
    torch.autograd.backward(outs, d_outs)
    torch.cuda.synchronize()


def _unpack(key, v, shape):
    """A registry view under its upstream key and shape, written out here rather than taken from the library."""
    if not key.endswith("@gemm"):
        return v.view(shape)
    if shape[2] == 2:    # ConvTranspose2d [ci, co, 2, 2] held as [(dy, dx, co), ci]
        return v.view(2, 2, shape[1], shape[0]).permute(3, 2, 0, 1)
    return v.view(shape[0], 3, 3, shape[1]).permute(0, 3, 1, 2)    # Conv2d [o, c, 3, 3] held as [o, (ky, kx), c]


@pytest.fixture(scope="module")
def stepped():
    sd, sam = _model()
    _backward(sam, seed=3)
    return sd, sam


def test_every_registered_tensor_is_an_upstream_tensor(stepped):
    sd, sam = stepped
    views = sam.grad_views()
    keys = [k.removesuffix("@gemm") for k, _ in views]
    want = {k for k in sd if k.startswith(("image_encoder.", "prompt_encoder.", "mask_decoder."))
            and not k.endswith("positional_encoding_gaussian_matrix")}
    assert len(keys) == len(set(keys)) and set(keys) == want, (set(keys) ^ want)
    assert {k.removesuffix("@gemm") for k, _ in views if k.endswith("@gemm")} == GEMM_KEYS
    bad = {k: (v.numel(), sd[k.removesuffix("@gemm")].numel()) for k, v in views if v.numel() != sd[k.removesuffix("@gemm")].numel()}
    assert not bad, bad


def test_the_views_are_the_gradients(stepped):
    sd, sam = stepped
    views = sam.grad_views()
    grads = dict(sam.encoder_grads())
    grads.update(sam.decoder_grads())
    sq_views = sum(float(v.double().square().sum()) for _, v in views)
    sq_grads = sum(float(g.double().square().sum()) for g in grads.values())
    assert abs(sq_views - sq_grads) <= 1e-6 * sq_grads, (sq_views, sq_grads)
    unpacked = {k.removesuffix("@gemm"): _unpack(k, v, sd[k.removesuffix("@gemm")].shape) for k, v in views}
    assert set(unpacked) == set(grads)
    assert all(torch.equal(unpacked[k], grads[k]) for k in grads), [k for k in grads if not torch.equal(unpacked[k], grads[k])]


def test_optimizer_step_writes_no_gradient_buffer():
    _, sam = _model()
    _backward(sam, seed=5)
    before = [(k, v.clone()) for k, v in sam.grad_views()]
    sam.optimizer_step(lr=1e-3)
    torch.cuda.synchronize()
    after = dict(sam.grad_views())
    changed = [k for k, v in before if not torch.equal(after[k], v)]
    assert not changed, changed


def test_two_steps_on_one_backward_are_two_torch_adamw_steps():
    sd, sam = _model()
    _backward(sam, seed=7)
    grads = dict(sam.encoder_grads())
    grads.update(sam.decoder_grads())
    kw = dict(lr=2e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    sam.optimizer_step(**kw)
    sam.optimizer_step(**kw)
    after = sam.trained_state_dict()
    keys = ["mask_decoder.output_upscaling.0.bias", "mask_decoder.output_upscaling.3.bias",   # one master tiled for the GEMM epilogue
            "mask_decoder.output_upscaling.0.weight", "image_encoder.neck.2.weight",           # held in the GEMM layout
            "image_encoder.blocks.0.norm1.weight",                                            # fp32 parameter, its own master
            "image_encoder.blocks.1.attn.qkv.weight", "mask_decoder.transformer.layers.0.mlp.lin1.weight",  # bf16 operand + W^T
            "image_encoder.blocks.0.attn.rel_pos_h",                                          # rows of a rel-pos table
            "mask_decoder.iou_prediction_head.layers.2.weight",                               # padded GEMM operand
            "prompt_encoder.point_embeddings.1.weight", "mask_decoder.mask_tokens.weight",    # rows of a shared table
            "prompt_encoder.mask_downscaling.0.weight"]                                       # registered at the first masked pass
    worst = {}
    for k in keys:
        p = torch.nn.Parameter(sd[k].float().clone().to(DEV))
        opt = torch.optim.AdamW([p], **kw)
        for _ in range(2):
            p.grad = grads[k].reshape(p.shape).clone()
            opt.step()
        d_ref, d_got = (p.detach().cpu() - sd[k]).double(), (after[k] - sd[k]).double()
        worst[k] = float((d_got - d_ref).norm() / d_ref.norm())
    print("\ntwo AdamW steps on one backward, rel-L2 of the update: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    bad = {k: v for k, v in worst.items() if not v < 1e-3}
    assert not bad, bad


def test_gradient_read_outs_are_copies(stepped):
    _, sam = stepped
    first = sam.decoder_grads()
    kept = {k: v.clone() for k, v in first.items()}
    _backward(sam, seed=11)
    changed = [k for k in kept if not torch.equal(first[k], kept[k])]
    assert not changed, changed
    later = sam.decoder_grads()
    assert any(not torch.equal(later[k], kept[k]) for k in kept)
