"""`-m gpu`: the training-mode mask decoder (csrc/decoder_train.cu) against a float64 mirror that rounds to bf16 exactly where
the CUDA tape does (tests/decoder_train_mirror.py, pinned to the oracle and torch autograd in tests/test_decoder_mirror_cpu.py).

test_gpu_backward.py::test_decoder_train_against_autograd compares the same path with exact fp32 math, where the bf16 noise floor
forces a bound of 1.5e-1 rel-L2 per gradient tensor.  Against the mirror, rel-L2 does not get much tighter: once a value lands on
the other side of a bf16 rounding boundary, the difference reaches the next roundings and flips more of them, so fp32 against
fp64 accumulation alone moves outputs and gradients by about the whole floor.  The same mirror in float32 differs from itself
in float64 by low_res 7.0e-3, d_emb 8.2e-3, gradients median 2.1e-2 (tests/test_decoder_mirror_cpu.py), and the GPU sits at that
distance.  The tight metric is the projection slope <GPU, mirror> / <mirror, mirror> of each gradient tensor: the flip noise is
nearly orthogonal to the gradient and averages out of it, while a scaled or partly lost gradient moves it.  Its noise differs by
tensor, so the bounds are per family of tensors (decoder_train_mirror.GRAD_BOUNDS).

Each case goes through `B200Sam.decoder_train` (prompt encoder on the GPU; T = 5 + n_sparse) and compares low_res, iou,
dL/d embedding and every tensor of `decoder_grads()` (which also checks the unpacking of the `@gemm` layouts) with
the mirror fed the GPU's own sparse prompt embeddings and dense positional encoding.  Metrics: rel-L2 and the worst per-row error
for the outputs (rows: prompts x masks x logit rows, prompts, embedding channels); rel-L2 and |slope - 1| for a gradient.
Gradients that are analytically zero (k_proj biases; tensors the prompts do not reach) are compared absolutely, against the
norm of the largest gradient.  The case grid covers P = 1 and odd P, T = 7 .. 16 on both sides of the attention's 8-column
pitch step, both multimask settings and the d_low_res = NULL and d_iou = NULL backward paths.

Measured on one H100 80GB HBM3 at a 400 W power limit (seeded vit_test decoder), worst over the grid:
  low_res  rel-L2 8.1e-3, worst row 2.1e-2
  iou      rel-L2 9.3e-3, worst prompt 2.2e-2
  d_emb    rel-L2 5.3e-2, worst channel 8.6e-2 (P = 13 with only the IoU gradient, where d_emb is small; 1.0e-2 elsewhere)
  gradients: |slope - 1| median 6e-4 .. 4.5e-3 per case; worst per family from 2.3e-3 (output_upscaling biases) and 3.9e-3
    (image-to-token k_proj weights) to 4.2e-2 (IoU head with P = 1); rel-L2 from 1.0e-2 (output_upscaling) to 2.1e-1 (IoU head)
  analytically zero gradients, |GPU - mirror| / largest gradient norm: 4.4e-5
Each bound is about twice the worst measured value of its family.

Mutations of decoder_train.cu / backward.cu on scratch builds (the GPU results are deterministic, so these are exact):
  dK x 1.02 in op_attention (all seven attentions): fails all 6 cases, 2 .. 6 tensors each, e.g. the image-to-token
    k_proj.weight at |slope - 1| 1.6e-2 .. 2.3e-2 against a bound of 7.8e-3.  test_decoder_train_against_autograd passes.
  token_grads_kernel summing prompts 0 .. P-2: fails all 6 cases (P = 13: point_embeddings.1 slope - 1 = -2.0e-2 against
    1.5e-2; P <= 6: rel-L2 0.3 .. 1.0 on the token tables).  test_decoder_train_against_autograd fails as well.
  masks_grad_kernel writing the single-mask gradient to column m0 + 1: fails both multimask-off cases (d_emb rel-L2 1.7 .. 1.8,
    94 gradients); the other cases do not use that path.  test_decoder_train_against_autograd fails only for points without
    multimask.
  gelu_bwd_kernel with the tanh-approximation derivative, and the final attention's op_add_cast without the query-PE gradient:
    pass every case, as test_decoder_train_against_autograd does.  They move the gradients by less than the flip noise (slope
    shift <= 1.1e-3; the lost query-PE term moves mask_tokens by 1.4e-2 rel-L2, orthogonal to it, against 5e-2 noise), so
    end to end they are out of reach; each needs an op-level test of its kernel.
"""
import numpy as np
import pytest
import torch

from tests import decoder_train_mirror as mirror

pytestmark = pytest.mark.gpu
DEV = "cuda"

# ------------------------------------------------------------------------------------------------ model and runs
@pytest.fixture(scope="module")
def model():
    from oracle import sam_ref
    from micro_sam_b200 import util
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
    sam.train()
    return sd, sam


def make_inputs(P, labels, box, multimask, seed):
    """Embedding, prompts and a random linear functional of (low_res, iou).  labels: one row per prompt or None (no points)."""
    gen = torch.Generator().manual_seed(seed)
    emb = torch.randn(256, 64, 64, generator=gen)
    pts = boxes = None
    if labels is not None:
        lab = torch.tensor(labels, dtype=torch.float32).reshape(P, -1)
        pts = (torch.rand(P, lab.shape[1], 2, generator=gen) * 1000, lab)
    if box:
        xy = torch.rand(P, 2, generator=gen) * 600 + 50
        boxes = torch.cat([xy, xy + torch.rand(P, 2, generator=gen) * 300 + 20], 1)
    M = 3 if multimask else 1
    d_low = torch.randn(P, M, 256, 256, generator=gen) / 256
    d_iou = torch.randn(P, M, generator=gen)
    return emb, pts, boxes, d_low, d_iou


def backward_raw(sam, slot, d_low, d_iou):
    """msam_decoder_train_backward called directly, so that d_low_res / d_iou can be NULL (autograd would pass zeros)."""
    from micro_sam_b200 import _lib
    d_emb = torch.empty(256, 64, 64, device=DEV)
    d_low = None if d_low is None else d_low.to(DEV, torch.float32).contiguous()
    d_iou = None if d_iou is None else d_iou.to(DEV, torch.float32).contiguous()
    _lib.check(_lib.lib().msam_decoder_train_backward(sam._h, slot, _lib.ptr(d_low), _lib.ptr(d_iou), _lib.ptr(d_emb),
                                                      _lib.cur_stream()))
    sam._decoder_grads_valid = True
    return d_emb


def to_dev(pts, boxes):
    return (None if pts is None else (pts[0].to(DEV), pts[1].to(DEV))), (None if boxes is None else boxes.to(DEV))


def forward(sam, emb, pts, boxes, multimask, slot):
    gemb = emb.to(DEV).requires_grad_(True)
    p, b = to_dev(pts, boxes)
    low, iou = sam.decoder_train(gemb, p, b, multimask, slot=slot)
    return gemb, low, iou


def gpu_run(sam, emb, pts, boxes, multimask, d_low, d_iou, slot=0):
    """zero the gradients, forward on `slot`, backward (through autograd when both upstream gradients are given, as training
    does; otherwise through the C API with NULL for the missing one)."""
    sam.zero_decoder_grads()
    gemb, low, iou = forward(sam, emb, pts, boxes, multimask, slot)
    if d_low is not None and d_iou is not None:
        torch.autograd.backward([low, iou], [d_low.to(DEV), d_iou.to(DEV)])
        d_emb = gemb.grad
    else:
        d_emb = backward_raw(sam, slot, d_low, d_iou)
    torch.cuda.synchronize()
    return {"low_res": low.detach().cpu(), "iou": iou.detach().cpu(), "d_emb": d_emb.detach().cpu(),
            "grads": {k: v.detach().cpu() for k, v in sam.decoder_grads().items()}}


def mirror_run(sd, sam, emb, pts, boxes, multimask, d_low, d_iou):
    from micro_sam_b200.sam import prompt_table_index
    p, b = to_dev(pts, boxes)
    sparse, _ = sam.prompt_encoder(points=p, boxes=b, masks=None)
    idx = prompt_table_index(None if pts is None else pts[1], boxes is not None, sparse.shape[0])
    dense_pe = sam.prompt_encoder.get_dense_pe()
    return mirror.run(sd, emb, sparse.cpu(), idx, dense_pe.cpu(), multimask, d_low, d_iou)


# ------------------------------------------------------------------------------------------------ the case grid
# id: (P, point labels per prompt or None, box, multimask, upstream gradients); T = 5 + n_points (+1 pad without a box) (+2 box)
_MIX = [[1, 0, -1, 1, 1, 0, -1, 0, 1, 1], [0, 1, 1, -1, 0, 1, 0, 1, -1, 1], [1, 1, 0, 0, -1, -1, 1, 0, 1, 0]]
CASES = {
    "P1-point-T7": (1, [[1]], False, True, "low+iou"),
    "P6-boxes-T7": (6, None, True, True, "low+iou"),
    "P5-3pts+box-T10": (5, [[1, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 0], [1, 1, 1]], True, False, "low"),
    "P13-10pts-T16": (13, [_MIX[p % 3][p % 10:] + _MIX[p % 3][:p % 10] for p in range(13)], False, True, "iou"),
    "P3-2pts+box-T9": (3, [[1, 0], [0, 1], [1, 1]], True, False, "low+iou"),
    "P4-2pts-T8": (4, [[1, 0], [1, 1], [0, 1], [1, -1]], False, True, "low+iou"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_decoder_train_against_bf16_mirror(model, case):
    sd, sam = model
    P, labels, box, multimask, upstream = CASES[case]
    emb, pts, boxes, d_low, d_iou = make_inputs(P, labels, box, multimask, seed=len(case) + 17 * P)
    d_low = d_low if "low" in upstream else None
    d_iou = d_iou if "iou" in upstream else None
    got = gpu_run(sam, emb, pts, boxes, multimask, d_low, d_iou)
    ref = mirror_run(sd, sam, emb, pts, boxes, multimask, d_low, d_iou)
    out, zero, bad = mirror.compare(got, ref, P, 3 if multimask else 1)
    grads = {k: v for k, v in out.items() if k not in ("low_res", "iou", "d_emb")}
    worst = sorted(grads.items(), key=lambda kv: -kv[1][0])[:3]
    worst_slope = sorted(grads.items(), key=lambda kv: -kv[1][1])[:3]
    print(f"\n{case}: " + ", ".join(f"{n} {out[n][0]:.2e}/{out[n][1]:.2e}" for n in ("low_res", "iou", "d_emb"))
          + f"; {len(grads)} gradients median rel-L2 {np.median([v[0] for v in grads.values()]):.2e}, worst "
          + ", ".join(f"{k.split('.', 1)[1]} {v[0]:.2e}" for k, v in worst)
          + f"; median |slope - 1| {np.median([v[1] for v in grads.values()]):.2e}, worst "
          + ", ".join(f"{k.split('.', 1)[1]} {v[1]:.2e}" for k, v in worst_slope)
          + f"; {len(zero)} zero tensors max {max(zero.values()):.2e}", flush=True)
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ semantics
def _grads(sam):
    torch.cuda.synchronize()
    return {k: v.detach().cpu().clone() for k, v in sam.decoder_grads().items()}


def test_gradients_accumulate_across_slots(model):
    """Two images in two slots, backward in the reverse order, sum to the two images run alone (TrainableSAM.forward puts image i
    in slot i and training backpropagates the whole batch at once).  Parameter gradients are reduced with atomics, so the sums
    agree to rounding; each image's dL/d embedding is the same bits as its run alone."""
    sd, sam = model
    A = make_inputs(6, None, True, True, seed=101)
    Bi = make_inputs(5, [[1, 0, 1]] * 5, True, False, seed=102)   # different P and T (7 and 10)

    def alone(inp, mm):
        emb, pts, boxes, d_low, d_iou = inp
        return gpu_run(sam, emb, pts, boxes, mm, d_low, d_iou, slot=0)
    ga, gb = alone(A, True), alone(Bi, False)
    sam.zero_decoder_grads()
    ea, la, ia = forward(sam, A[0], A[1], A[2], True, slot=0)
    eb, lb, ib = forward(sam, Bi[0], Bi[1], Bi[2], False, slot=1)
    torch.autograd.backward([lb, ib], [Bi[3].to(DEV), Bi[4].to(DEV)])
    torch.autograd.backward([la, ia], [A[3].to(DEV), A[4].to(DEV)])
    both = _grads(sam)
    assert torch.equal(ea.grad.cpu(), ga["d_emb"]) and torch.equal(eb.grad.cpu(), gb["d_emb"])
    assert torch.equal(la.detach().cpu(), ga["low_res"]) and torch.equal(lb.detach().cpu(), gb["low_res"])
    scale = max(float((ga["grads"][k] + gb["grads"][k]).norm()) for k in both)
    bad = {}
    for k, g in both.items():
        s = ga["grads"][k] + gb["grads"][k]
        err = float((g - s).norm())
        if not err <= 1e-5 * max(float(s.norm()), 1e-3 * scale):
            bad[k] = (err, float(s.norm()))
    assert not bad, bad
    # zero_decoder_grads clears every gradient
    sam.zero_decoder_grads()
    nonzero = [k for k, v in _grads(sam).items() if bool(v.any())]
    assert not nonzero, nonzero


def test_repeat_is_bit_identical(model):
    """low_res, iou and dL/d embedding depend on no atomic: the same case twice gives the same bits.  (Parameter gradients are
    reduced with atomics: column sums, LayerNorm weight / bias, the token tables.)"""
    sd, sam = model
    inp = make_inputs(13, CASES["P13-10pts-T16"][1], False, True, seed=7)
    r1 = gpu_run(sam, *inp[:3], True, inp[3], inp[4], slot=2)
    r2 = gpu_run(sam, *inp[:3], True, inp[3], inp[4], slot=3)
    for name in ("low_res", "iou", "d_emb"):
        assert torch.equal(r1[name], r2[name]), name


def test_backward_error_paths(model):
    """A second backward on the same slot, a backward on a slot that never ran forward, and slots outside [0, 8) raise; the
    failed calls leave the accumulated gradients alone."""
    sd, sam = model
    emb, pts, boxes, d_low, d_iou = make_inputs(2, None, True, True, seed=9)
    gpu_run(sam, emb, pts, boxes, True, d_low, d_iou, slot=4)
    before = _grads(sam)
    with pytest.raises(RuntimeError, match="no saved forward pass"):
        backward_raw(sam, 4, d_low, d_iou)
    with pytest.raises(RuntimeError, match="no saved forward pass"):
        backward_raw(sam, 7, d_low, d_iou)
    for slot in (8, -1):
        with pytest.raises(RuntimeError, match="slot"):
            backward_raw(sam, slot, d_low, d_iou)
        with pytest.raises(RuntimeError, match="slot"):
            forward(sam, emb, pts, boxes, True, slot)
    after = _grads(sam)
    assert all(torch.equal(before[k], after[k]) for k in before)
