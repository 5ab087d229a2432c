"""`-m gpu`: the image encoder after an optimizer step.  AdamW (csrc/train_opt.cu) refreshes the bf16 weights that the forward GEMMs
read and the W^T operands that the dgrad GEMMs of the backward pass read.  After forward, backward and one step, a second forward and
backward must match torch autograd over the oracle encoder loaded with the updated weights, to the tolerances of
tests/test_gpu_backward.py (forward rel-L2 < 2e-2, every gradient rel-L2 < 3e-2), and so must the inference forward."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("model_type", ["vit_test", "vit_test80"])
def test_encoder_gradients_after_an_optimizer_step(model_type):
    from oracle import sam_ref
    from micro_sam_b200.sam import B200Sam
    from micro_sam_b200.sample_data import lm_tile
    from micro_sam_b200 import util
    torch.set_num_threads(min(64, os.cpu_count() or 8))
    B = 2
    sd = sam_ref.seeded_state_dict(model_type, seed=0)
    enc_sd = {k: v for k, v in sd.items() if k.startswith("image_encoder.")}
    osam = sam_ref.build_sam(model_type)
    osam.load_state_dict(sd)
    sam = B200Sam(model_type, enc_sd, max_batch=B, max_prompts=1).train()
    imgs = np.stack([util._to_image(lm_tile((1024, 1024), 150, seed=s)) for s in range(B)])
    x_pre = torch.stack([osam.preprocess(torch.from_numpy(i).permute(2, 0, 1)[None].float())[0] for i in imgs])
    gen = torch.Generator().manual_seed(7)

    sam.image_encoder(x_pre.to(DEV)).backward(torch.randn(B, 256, 64, 64, generator=gen).to(DEV))
    sam.optimizer_step(lr=5e-3)
    new_sd = {k: v for k, v in sam.trained_state_dict().items() if k.startswith("image_encoder.")}
    # the step moves every weight with a W^T operand by more than the gradient tolerance, so a stale W^T would show below
    moved = {k: _rel(new_sd[k] - enc_sd[k], enc_sd[k]) for k in enc_sd
             if k.endswith(("qkv.weight", "proj.weight", "lin1.weight", "lin2.weight", "neck.0.weight", "neck.2.weight"))}
    assert min(moved.values()) > 3e-2, moved
    osam.load_state_dict({**sd, **new_sd})

    d_out = torch.randn(B, 256, 64, 64, generator=gen)
    enc = osam.image_encoder
    for p in enc.parameters():
        p.requires_grad_(True)
    ref_out = enc(x_pre)
    ref_out.backward(d_out)
    got_out = sam.image_encoder(x_pre.to(DEV))
    rel_f = _rel(got_out.detach(), ref_out.detach())
    got_out.backward(d_out.to(DEV))
    ref_grads = dict(enc.named_parameters())
    rels = {k: _rel(g, ref_grads[k[len("image_encoder."):]].grad) for k, g in sam.encoder_grads().items()}
    worst = sorted(rels.items(), key=lambda kv: -kv[1])[:6]
    print(f"{model_type} after one step: forward rel-L2 {rel_f:.2e}; {len(rels)} gradients, worst: "
          + ", ".join(f"{k.replace('image_encoder.', '')} {v:.2e}" for k, v in worst))
    assert len(rels) == len(ref_grads)
    assert rel_f < 2e-2
    bad = {k: v for k, v in rels.items() if not v < 3e-2}
    assert not bad, bad
    with torch.no_grad():
        assert _rel(sam.eval().image_encoder(x_pre.to(DEV)), ref_out.detach()) < 2e-2
    del sam
    torch.cuda.empty_cache()
