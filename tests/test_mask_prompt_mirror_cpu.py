"""The mask-prompt extension of the float64 training-decoder mirror (tests/mask_prompt_mirror.py) pinned on the CPU: with rounding
off it reproduces the oracle's prompt encoder (mask_downscaling) + mask decoder under torch autograd in float64, outputs, dL/d
embedding and every parameter gradient including the ten mask_downscaling tensors; no_mask_embed gets none.  The weights have
non-trivial LayerNorm2d gamma / beta in mask_downscaling, as in the GPU tests."""
import pytest
import torch

from tests import decoder_train_mirror as mirror
from tests import mask_prompt_mirror as mmirror
from tests.test_decoder_mirror_cpu import _inputs, _oracle64, _rel, P


@pytest.fixture(scope="module")
def sd():
    return mmirror.perturbed_state_dict()


def _masks(kind, seed=5):
    gen = torch.Generator().manual_seed(seed)
    if kind == "zero":
        return torch.zeros(P, 1, 256, 256, dtype=torch.float64)
    m = torch.nn.functional.avg_pool2d(torch.randn(P, 1, 256, 256, generator=gen, dtype=torch.float64) * 8, 9, 1, 4)
    return m.clamp(-20, 20) if kind == "logits" else torch.where(m > 0, 20.0, -20.0).double()


@pytest.mark.parametrize("multimask", [True, False])
@pytest.mark.parametrize("prompt,kind", [("points", "logits"), ("boxes", "pm20"), ("points+boxes", "zero")])
def test_masked_mirror_without_rounding_is_the_oracle(sd, prompt, kind, multimask, monkeypatch):
    monkeypatch.setattr(mirror, "ROUND", False)
    x = _inputs(sd, prompt, multimask)
    masks = _masks(kind)
    osam = _oracle64(sd)
    oemb = x["emb"].clone()[None].requires_grad_(True)
    sparse, dense = osam.prompt_encoder(points=x["pts"], boxes=x["boxes"], masks=masks)
    low, iou = osam.mask_decoder(image_embeddings=oemb, image_pe=osam.prompt_encoder.get_dense_pe(), sparse_prompt_embeddings=sparse,
                                 dense_prompt_embeddings=dense, multimask_output=multimask)
    ((low * x["d_low"]).sum() + (iou * x["d_iou"]).sum()).backward()
    got = mmirror.run(sd, x["emb"], x["sparse"], x["idx"], x["dense_pe"], masks, multimask, x["d_low"], x["d_iou"])
    assert _rel(got["low_res"], low.detach()) < 1e-12 and _rel(got["iou"], iou.detach()) < 1e-12
    assert _rel(got["d_emb"], oemb.grad[0]) < 1e-10
    ref = dict(osam.named_parameters())
    scale = max(float(p.grad.norm()) for p in ref.values() if p.grad is not None)
    checked = 0
    for k, g in got["grads"].items():
        r = ref[k].grad if ref[k].grad is not None else torch.zeros_like(ref[k])
        assert tuple(g.shape) == tuple(r.shape), k
        if k.endswith("k_proj.bias") or float(r.norm()) < 1e-9 * scale:
            assert float((g - r).norm()) < 1e-10 * scale, k
        else:
            assert _rel(g, r) < 1e-10, (k, _rel(g, r))
            checked += 1
    assert set(mmirror.MD_KEYS) <= set(got["grads"])
    assert float(got["grads"][mmirror.NO_MASK].abs().max()) == 0.0 and ref[mmirror.NO_MASK].grad is None
    assert checked > 95
