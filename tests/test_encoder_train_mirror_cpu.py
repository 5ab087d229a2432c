"""The float64 bf16-rounding mirror of the encoder's training step (tests/encoder_train_mirror.py) pinned on the CPU:

* with rounding off it reproduces the oracle's ImageEncoderViT under float64 autograd (embedding and every parameter gradient),
  on a windowed and a global block with head_dim 64 and 80 at batch 2, so its structure (window padding, decomposed rel-pos,
  neck, positional embedding over the batch) is the oracle's and not a copy of the CUDA code;
* with rounding on it moves away from exact math, so the rounding is live;
* planted faults of 2 % and lost terms move the rounded mirror outside the bounds that tests/test_gpu_encoder_train_mirror.py
  applies to the device, in the tensors the fault touches.
"""
import pytest
import torch

from tests import encoder_train_mirror as mirror

B = 2


def _inputs(seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, 1024, 1024, generator=g, dtype=torch.float64)
    d_out = torch.randn(B, 256, 64, 64, generator=g, dtype=torch.float64)
    return x, d_out


def _state(model_type):
    from oracle import sam_ref
    return {k: v for k, v in sam_ref.seeded_state_dict(model_type, seed=0).items() if k.startswith("image_encoder.")}


@pytest.mark.parametrize("model_type", ["vit_test", "vit_test80"])
def test_mirror_without_rounding_is_the_oracle(model_type, monkeypatch):
    from oracle import sam_ref
    monkeypatch.setattr(mirror, "ROUND", False)
    torch.manual_seed(0)
    sd = _state(model_type)
    x, d_out = _inputs()
    enc = sam_ref.build_sam(model_type).image_encoder.double()
    enc.load_state_dict({k[len(mirror.E):]: v for k, v in sd.items()})
    for p in enc.parameters():
        p.requires_grad_(True)
    ref = enc(x)
    ref.backward(d_out)
    out, grads = mirror.run({k: v.double() for k, v in sd.items()}, sam_ref.ARCH[model_type], x, d_out)
    assert mirror.rel_l2(out, ref.detach()) < 1e-12
    named = dict(enc.named_parameters())
    assert set(grads) == {mirror.E + k for k in named}
    scale = max(float(p.grad.norm()) for p in named.values())
    for k, g in grads.items():
        r = named[k[len(mirror.E):]].grad
        assert tuple(g.shape) == tuple(r.shape), k
        if k.endswith("attn.qkv.bias"):   # the k third is zero in exact arithmetic
            D = r.numel() // 3
            assert float((g[D:2 * D] - r[D:2 * D]).norm()) < 1e-10 * scale, k
            assert float(r[D:2 * D].norm()) < 1e-10 * scale, k
            g, r = torch.cat([g[:D], g[2 * D:]]), torch.cat([r[:D], r[2 * D:]])
        assert mirror.rel_l2(g, r) < 1e-10, (k, mirror.rel_l2(g, r))


@pytest.fixture(scope="module")
def rounded():
    """(arch, device weights, inputs, rounded mirror's step) on vit_test"""
    from oracle import sam_ref
    w = mirror.device_weights(_state("vit_test"))
    x, d_out = _inputs()
    x = x.float()
    return sam_ref.ARCH["vit_test"], w, (x, d_out), mirror.run(w, sam_ref.ARCH["vit_test"], x, d_out)


def test_rounding_is_live(rounded, monkeypatch):
    arch, w, (x, d_out), (out, grads) = rounded
    monkeypatch.setattr(mirror, "ROUND", False)
    out0, grads0 = mirror.run(w, arch, x, d_out)
    got, exact = mirror.split_qkv_bias(grads), mirror.split_qkv_bias(grads0)
    rels = sorted(mirror.rel_l2(got[k], g) for k, g in exact.items() if not k.endswith("[k]"))
    e = mirror.rel_l2(out, out0)
    print(f"rounded mirror vs exact: embedding {e:.2e}, gradients median rel-L2 {rels[len(rels) // 2]:.2e}, max {rels[-1]:.2e}")
    assert 1e-4 < e < 5e-2
    assert rels[len(rels) // 2] > 1e-3


FAULTS = {   # fault -> keys that must be outside the bounds (a prefix ends with ".")
    "rel_window": ({"rel_window": 1.02}, {"image_encoder.blocks.0.attn.rel_pos_h", "image_encoder.blocks.0.attn.rel_pos_w"}),
    "rel_global": ({"rel_global": 1.02}, {"image_encoder.blocks.1.attn.rel_pos_h", "image_encoder.blocks.1.attn.rel_pos_w"}),
    "dk_no_pad": ({"dk_no_pad": True}, {"zero"}),
    "ln2_dgamma": ({"ln2_dgamma": 1.02}, {"image_encoder.blocks.0.norm2.weight", "image_encoder.blocks.1.norm2.weight"}),
    "pos_first_image": ({"pos_first_image": True}, {"image_encoder.pos_embed"}),
    "col2im_drop_tap": ({"col2im_drop_tap": 4}, {"image_encoder.neck.1.weight"}),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_gpu_bounds_catch_a_planted_fault(rounded, fault, monkeypatch):
    """The rounded mirror with one planted fault against the rounded mirror, under the GPU test's bounds."""
    arch, w, (x, d_out), (out, grads) = rounded
    _, clean_bad = mirror.compare(out, grads, out, grads, arch)
    assert not clean_bad
    plant, expect = FAULTS[fault]
    for k, v in plant.items():
        monkeypatch.setitem(mirror.FAULT, k, v)
    fout, fgrads = mirror.run(w, arch, x, d_out)
    res, bad = mirror.compare(fout, fgrads, out, grads, arch)
    names = {b[0] for b in bad}
    print(f"{fault}: outside the GPU bounds: {sorted(names)}; zero {res['zero']:.2e}")
    assert expect <= names, (expect, bad)
