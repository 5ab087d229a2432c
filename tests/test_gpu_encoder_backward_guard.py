"""`-m gpu`: the encoder's backward pass runs on the activations of the forward pass that produced its output, or refuses.

The engine keeps one training forward's activations, and an inference encode reuses the workspace that the backward pass reads
(the patches and the neck's activations).  A backward after another encoder forward would mix two images' activations, and a
second training forward would have its gradients overwritten by the first one's backward; both raise instead.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def model():
    from micro_sam_b200.sam import B200Sam
    from oracle import sam_ref
    sd = {k: v for k, v in sam_ref.seeded_state_dict("vit_test", seed=0).items() if k.startswith("image_encoder.")}
    sam = B200Sam("vit_test", sd, max_batch=2, max_prompts=1)
    g = torch.Generator().manual_seed(7)
    xs = [torch.randn(1, 3, 1024, 1024, generator=g).to(DEV) for _ in range(2)]
    d_out = torch.randn(1, 256, 64, 64, generator=g).to(DEV)
    return sam, xs, d_out


def test_backward_after_an_inference_encode_raises(model):
    sam, (a, b), d_out = model
    out = sam.train().image_encoder(a)
    with torch.no_grad():
        sam.eval().image_encoder(b)
    with pytest.raises(RuntimeError, match="another encoder forward"):
        out.backward(d_out)


def test_backward_of_an_older_training_forward_raises(model):
    sam, (a, b), d_out = model
    sam.train()
    first = sam.image_encoder(a)
    second = sam.image_encoder(b)
    with pytest.raises(RuntimeError, match="another encoder forward"):
        first.backward(d_out)
    second.backward(d_out)   # the latest one still has its activations


def test_engine_refuses_a_backward_after_an_inference_encode(model):
    """the engine's own check, below the Python one: msam_encode_f32 discards the saved training forward"""
    from micro_sam_b200 import _lib
    sam, (a, b), d_out = model
    L = _lib.lib()
    out = torch.empty(1, 256, 64, 64, device=DEV)
    _lib.check(L.msam_encode_train(sam._h, _lib.ptr(a), 1, _lib.ptr(out), _lib.cur_stream()))
    _lib.check(L.msam_encode_f32(sam._h, _lib.ptr(b), 1, _lib.ptr(out), _lib.cur_stream()))
    with pytest.raises(RuntimeError, match="no saved forward pass"):
        _lib.check(L.msam_encode_backward(sam._h, _lib.ptr(d_out), _lib.cur_stream()))


def test_inference_encode_after_a_backward_is_unaffected(model):
    sam, (a, b), d_out = model
    with torch.no_grad():
        ref = sam.eval().image_encoder(b).clone()
    out = sam.train().image_encoder(a)
    out.backward(d_out)
    grads = sam.encoder_grads()
    with torch.no_grad():
        again = sam.eval().image_encoder(b)
    assert torch.equal(again, ref)
    # the gradients are the backward pass's, whatever ran after it
    assert all(torch.equal(v, sam.encoder_grads()[k]) for k, v in grads.items())
