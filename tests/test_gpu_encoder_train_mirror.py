"""`-m gpu`: the ViT encoder's training step on the device (B200Sam.train(), image_encoder(x), backward, encoder_grads();
csrc/encoder_train.cu) against the float64 mirror of tests/encoder_train_mirror.py, which rounds to bf16 exactly where the device
does, run on the GPU from the same preprocessed images and the same bf16 weights.

test_gpu_backward.py::test_encoder_backward_* compares the same gradients with fp32 autograd on the CPU at rel-L2 <= 3e-2, on
vit_test / vit_test80 at B = 2 and vit_b at B = 1 only: a gradient that is uniformly 2 % off passes it.  Against the mirror the
projection slope <device, mirror> / <mirror, mirror> of each gradient tensor is 1 to within 1e-4 .. 6e-3 (the rounding flips
between fp32 and fp64 accumulation are nearly orthogonal to the gradient), so a 2 % scaling stands out.  rel-L2 tightens too
(bf16 rounding alone moves vit_test's gradients by a median 7.6e-3 from exact math; the device sits at 5e-3 from the mirror).

Cases: vit_test and vit_test80 at B = 2; vit_b, vit_l and vit_h widths with depth 2 (block 0 windowed, block 1 global;
registered for the test only) at B = 2, where windows of two images share a batched GEMM, global attention runs over two images
and the pos_embed and weight gradients sum over them; full-depth vit_b at B = 2 (the fine-tuning benchmark's architecture);
full-depth vit_h at B = 1 (32 blocks, head_dim 80).  Metrics (encoder_train_mirror.compare): embedding rel-L2; rel-L2 and
|slope - 1| per gradient tensor, bounded per family (encoder_train_mirror.GRAD_BOUNDS); the k third of every attn.qkv.bias
gradient, zero in exact arithmetic (softmax is invariant to a constant added to every key's logit), absolutely as |device| / the
largest gradient norm.  And with one engine at max_batch = 2, the B = 2 gradients against the sums of the two B = 1 passes'.

Measured on an H100 80GB HBM3 at 700 W, worst over the seven cases (rel-L2, |slope - 1|):
  block GEMM weights (9.0e-3, 8.1e-4)      biases (8.7e-3, 8.3e-4)         block LayerNorms (8.8e-3, 1.3e-3)
  rel-pos, windowed (2.5e-2, 6.0e-3)      rel-pos, global (2.3e-2, 6.1e-3)   pos_embed (1.2e-2, 6.1e-5)
  patch embedding (8.2e-3, 7.1e-4)        neck convolutions (4.8e-3, 4.4e-4) neck LayerNorms (4.9e-3, 6.4e-4)
  embedding rel-L2 4.7e-3; k third of qkv.bias 1.1e-5 of the largest gradient norm; batch composition 1.7e-6
  the float64 mirror peaks at 8.1 GiB of device memory (vit_h, B = 1); the file runs in about 45 s (setup included)
Each bound is about twice the worst measured value.

Mutations of encoder_train.cu / backward.cu on scratch builds (arithmetic only), each run once against this file and
test_gpu_backward.py::test_encoder_backward_{small_archs,vit_b}:
  rel-pos gradient x 1.02 (sum_batch of dR): every case here fails on the rel-pos slope (1.9e-2 .. 2.6e-2 against 1.2e-2);
    of the old tests only vit_b fails, by a hair (rel-L2 3.3e-2 against 3e-2).
  dS x 1.02 (attn_ds, the dT half untouched): every case here fails on the pos_embed slope (3.6e-4 .. 1.4e-3 against 1.3e-4;
    vit_test80 also on the qkv weight slope, 2.4e-3); every old test passes.
  pad rows of dqkv zeroed before the qkv-bias column sum: every case here fails (k third of qkv.bias 6e-4 .. 1e-3 against
    2.3e-5, qkv bias slope 8e-2 .. 1.4e-1); the old tests fail too (qkv.bias rel-L2 0.23 .. 0.37).
  LayerNorm dgamma x 1.02 (layernorm_bwd): every case here fails on the block and neck LayerNorm slopes (2.0e-2 against 2.6e-3
    and 1.3e-3); every old test passes.
  pos_embed summed over B - 1 images: every case here fails (pos_embed slope 0.46, 1.0 at B = 1) and so does the batch
    composition test; the old tests fail too (pos_embed rel-L2 0.68 .. 1.0).
"""
import json
import time

import pytest
import torch

from micro_sam_b200 import sam as msam
from oracle import sam_ref
from tests import encoder_train_mirror as mirror

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# production widths with depth 2: block 0 windowed, block 1 global
DEPTH2 = {f"{t}_d2": dict(sam_ref.ARCH[t], depth=2, global_attn_indexes=(1,)) for t in ("vit_b", "vit_l", "vit_h")}
CASES = {"vit_test_b2": ("vit_test", 2), "vit_test80_b2": ("vit_test80", 2), "vit_b_d2_b2": ("vit_b_d2", 2),
         "vit_l_d2_b2": ("vit_l_d2", 2), "vit_h_d2_b2": ("vit_h_d2", 2), "vit_b_b2": ("vit_b", 2), "vit_h_b1": ("vit_h", 1)}
TOL_BATCH = 3.3e-6  # B = 2 against the sum of two B = 1 passes: |diff|_1 / (|part 1|_1 + |part 2|_1) per tensor


@pytest.fixture
def archs(monkeypatch):
    for k, v in DEPTH2.items():
        monkeypatch.setitem(msam.ARCH, k, v)
        monkeypatch.setitem(sam_ref.ARCH, k, v)
    return sam_ref.ARCH


def _inputs(model_type, B, seed=5):
    """(encoder state dict, preprocessed images [B, 3, 1024, 1024] fp32, dL/d embedding), on the CPU"""
    from micro_sam_b200 import util
    from micro_sam_b200.sample_data import lm_tile
    sd = {k: v for k, v in sam_ref.seeded_state_dict(model_type, seed=0).items() if k.startswith(mirror.E)}
    mean = torch.tensor([123.675, 116.28, 103.53]).view(3, 1, 1)
    std = torch.tensor([58.395, 57.12, 57.375]).view(3, 1, 1)
    x = torch.stack([(torch.from_numpy(util._to_image(lm_tile((1024, 1024), 150, seed=s))).permute(2, 0, 1).float() - mean) / std
                     for s in range(B)])
    d_out = torch.randn(B, 256, 64, 64, generator=torch.Generator().manual_seed(seed))
    return sd, x, d_out


def _device_step(sam, x, d_out):
    out = sam.image_encoder(x.to(DEV))
    out.backward(d_out.to(DEV))
    return out.detach(), sam.encoder_grads()


@pytest.mark.parametrize("case", list(CASES))
def test_encoder_step_against_mirror(archs, case):
    model_type, B = CASES[case]
    t0 = time.time()
    sd, x, d_out = _inputs(model_type, B)
    sam = msam.B200Sam(model_type, sd, max_batch=B, max_prompts=1).train()
    out, got = _device_step(sam, x, d_out)
    del sam
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    w = mirror.device_weights(sd, DEV)
    del sd
    want_out, want = mirror.run(w, archs[model_type], x.to(DEV), d_out.to(DEV))
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    res, bad = mirror.compare(out, got, want_out, want, archs[model_type])
    res.update(case=case, mirror_peak_GiB=round(peak, 2), seconds=round(time.time() - t0, 1))
    print(json.dumps(res))
    assert not bad, bad


def test_batch_of_two_is_the_sum_of_two_single_images(archs):
    """One engine at max_batch = 2: the gradients of a B = 2 step equal the sums of the two B = 1 steps' (same images, same
    upstream gradients), to the fp32 reordering of the split-K and column-sum atomics."""
    sd, x, d_out = _inputs("vit_b_d2", 2)
    sam = msam.B200Sam("vit_b_d2", sd, max_batch=2, max_prompts=1).train()
    _, both = _device_step(sam, x, d_out)
    _, g0 = _device_step(sam, x[:1], d_out[:1])
    _, g1 = _device_step(sam, x[1:], d_out[1:])
    worst = {}
    for k in both:
        d = float((both[k].double() - g0[k].double() - g1[k].double()).abs().sum())
        worst[k] = d / float(g0[k].double().abs().sum() + g1[k].double().abs().sum())
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    print(json.dumps({"batch_composition": top}))
    assert all(not torch.equal(g0[k], g1[k]) for k in both)
    assert top[0][1] <= TOL_BATCH, top
