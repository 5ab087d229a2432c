"""`-m gpu`: training with mask prompts -- mask_downscaling's forward and backward (csrc/decoder_train.cu, md_* kernels), the
training decoder with mask prompts, the lazily registered optimizer tensors, and `training.compute_iterative_loss`.

* op level: `msam_op_mask_downscaling_train` against float64 autograd of the oracle's own mask_downscaling module (fp32 block:
  tight bounds);
* decoder: `B200Sam.decoder_train(..., masks=...)` against the float64 bf16-rounding mirror extended with the mask path
  (tests/mask_prompt_mirror.py, pinned to the oracle on the CPU), metrics as in tests/test_gpu_decoder_train.py;
* semantics: runs without mask prompts keep the parent's key set / tensor count and never move the mask tensors; masked and
  unmasked slots accumulate in either order; repeats are bit-identical; AdamW on the mask tensors matches torch.optim.AdamW;
* the iterative loss: tests/test_gpu_iterative_loss.py.

Measured on one H100 80GB HBM3 at a 700 W power limit (seeded vit_test decoder), worst over each case grid:
  op level (fp32 block): dense_out 1.5e-7, gradients 5.4e-6 (zero masks, P = 25, LayerNorm2d(4) weight); bound 1e-5.
    Mutations of the kernels on scratch builds, each against this test: the tanh-approximation GELU' fails all 9 cases (gradient
    errors 1.5e-4 .. 3.7e-3); LayerNorm rstd x 1.01 in the backward fails all 9 (1e-2 on the eight tensors before the 1x1 conv);
    swapped sub-pixel phases in the transposed k2s2 conv fail the 6 non-zero mask cases (conv 0 weight 1.0 .. 1.9) -- with zero
    masks the first conv's weight gradient is zero whatever the phase.
  decoder against the mirror: low_res 8.1e-3 / 2.7e-2 (rel-L2 / worst row), iou 1.1e-2 / 5.4e-2, d_emb 1.4e-2 / 2.7e-2;
    mask_downscaling gradients rel-L2 <= 1.9e-1, |slope - 1| <= 7.9e-2 (weights) and 1.3e-1 / 4.1e-2 (biases); every family's
    bound is about twice its worst (tests/mask_prompt_mirror.GRAD_BOUNDS).
  AdamW on the mask tensors against torch.optim.AdamW: 3.4e-4 of the update.
Without mask prompts the results are those of the build before mask prompts existed: on a box-only training step the gradient keys
and the 159 trainable tensors are the same; the decoder gradients differ from that build's by at most 2.3e-4 relative, as two runs
of that build differ from each other (1.8e-4: the decoder's parameter-gradient reductions use float atomics); `bench.py
--dump-outputs` is bit-identical; `bench.py --config cfg5` ran at 112.6 / 113.4 ms per step against 117.0 / 122.5 ms before
(alternating runs in one session).
Timing (tests/time_mask_prompt_train.py, H100 80GB HBM3 at a 400 W power limit): a training-decoder pass + backward at P = 25
takes 20.51 ms with mask prompts and 19.92 ms without (+3.0 %); the md_* kernels take 0.24 (forward) + 0.21 + 0.065 + 0.008 ms.
"""
import numpy as np
import pytest
import torch

from tests import mask_prompt_mirror as mmirror

pytestmark = pytest.mark.gpu
DEV = "cuda"
MD_SHAPES = [(4, 1, 2, 2), (4,), (4,), (4,), (16, 4, 2, 2), (16,), (16,), (16,), (256, 16, 1, 1), (256,)]

# op level: rel-L2 of dense_out and of each of the ten gradients against float64 autograd, bound = about twice the worst measured
OP_TOL = 1e-5


@pytest.fixture(scope="module")
def model():
    from micro_sam_b200 import util
    sd = mmirror.perturbed_state_dict()
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
    sam.train()
    return sd, sam


def _masks(kind, P, seed):
    gen = torch.Generator().manual_seed(seed)
    if kind == "zero":
        return torch.zeros(P, 1, 256, 256)
    m = torch.nn.functional.avg_pool2d(torch.randn(P, 1, 256, 256, generator=gen) * 8, 9, 1, 4)
    return m.clamp(-20, 20) if kind == "logits" else torch.where(m > 0, 20.0, -20.0)


# ------------------------------------------------------------------------------------------------ op level
def op_run(sam, masks, d_dense):
    from micro_sam_b200 import _lib
    P = masks.shape[0]
    mk = masks.to(DEV, torch.float32).contiguous()
    dd = d_dense.to(DEV, torch.float32).contiguous()
    dense = torch.empty(P, 4096, 256, device=DEV)
    grads = torch.empty(4684, device=DEV)
    _lib.check(_lib.lib().msam_op_mask_downscaling_train(sam._h, _lib.ptr(mk), P, _lib.ptr(dd), _lib.ptr(dense), _lib.ptr(grads),
                                                         _lib.cur_stream()))
    torch.cuda.synchronize()
    return dense.cpu(), list(torch.split(grads.cpu(), [int(np.prod(s)) for s in MD_SHAPES]))


def op_errors(sd, sam, kind, P, seed=0):
    masks = _masks(kind, P, seed=100 + P)
    gen = torch.Generator().manual_seed(200 + P)
    d_dense = torch.randn(P, 4096, 256, generator=gen)
    dense, grads = op_run(sam, masks, d_dense)
    from oracle import sam_ref
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    md = osam.prompt_encoder.mask_downscaling.double()
    ref = md(masks.double()).reshape(P, 256, 4096).transpose(1, 2)
    ref.backward(d_dense.double())
    params = dict(md.named_parameters())
    errs = {"dense": float((dense.double() - ref.detach()).norm() / ref.detach().norm())}
    for k, g, shp in zip(mmirror.MD_KEYS, grads, MD_SHAPES):
        r = params[k.split("mask_downscaling.")[1]].grad
        errs[k.split("mask_downscaling.")[1]] = float((g.double().reshape(shp) - r).norm() / r.norm().clamp_min(1e-300)) \
            if float(r.norm()) > 0 else float(g.double().norm())
    return errs


@pytest.mark.parametrize("P", [1, 5, 25])
@pytest.mark.parametrize("kind", ["logits", "zero", "pm20"])
def test_op_mask_downscaling_against_float64_autograd(model, kind, P):
    sd, sam = model
    errs = op_errors(sd, sam, kind, P)
    print(f"\nmask_downscaling {kind} P={P}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()), flush=True)
    bad = {k: v for k, v in errs.items() if not v <= OP_TOL}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ decoder with masks
def _inputs(P, labels, box, multimask, kind, seed):
    from tests.test_gpu_decoder_train import make_inputs
    emb, pts, boxes, d_low, d_iou = make_inputs(P, labels, box, multimask, seed)
    return emb, pts, boxes, _masks(kind, P, seed), d_low, d_iou


def gpu_run(sam, emb, pts, boxes, masks, multimask, d_low, d_iou, slot=0, zero=True):
    from tests.test_gpu_decoder_train import to_dev
    if zero:
        sam.zero_decoder_grads()
    gemb = emb.to(DEV).requires_grad_(True)
    p, b = to_dev(pts, boxes)
    low, iou = sam.decoder_train(gemb, p, b, multimask, slot=slot, masks=None if masks is None else masks.to(DEV))
    torch.autograd.backward([low, iou], [d_low.to(DEV), d_iou.to(DEV)])
    torch.cuda.synchronize()
    return {"low_res": low.detach().cpu(), "iou": iou.detach().cpu(), "d_emb": gemb.grad.detach().cpu(),
            "grads": {k: v.detach().cpu().clone() for k, v in sam.decoder_grads().items()}}


CASES = {   # (P, point labels per prompt or None, box, multimask, mask kind)
    "P1-point+mask": (1, [[1]], False, True, "logits"),
    "P5-box+mask": (5, None, True, False, "pm20"),
    "P5-2pts+box+mask": (5, [[1, 0], [0, 1], [1, 1], [1, 0], [0, 0]], True, True, "logits"),
    "P25-box+zero-mask": (25, None, True, True, "zero"),
    "P25-point+mask": (25, [[1]] * 25, False, False, "logits"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_decoder_with_masks_against_bf16_mirror(model, case):
    from micro_sam_b200.sam import prompt_table_index
    from tests.test_gpu_decoder_train import to_dev
    sd, sam = model
    P, labels, box, multimask, kind = CASES[case]
    emb, pts, boxes, masks, d_low, d_iou = _inputs(P, labels, box, multimask, kind, seed=len(case) + 31 * P)
    got = gpu_run(sam, emb, pts, boxes, masks, multimask, d_low, d_iou)
    p, b = to_dev(pts, boxes)
    sparse, _ = sam.prompt_encoder(points=p, boxes=b, masks=None)
    idx = prompt_table_index(None if pts is None else pts[1], boxes is not None, P)
    ref = mmirror.run(sd, emb, sparse.cpu(), idx, sam.prompt_encoder.get_dense_pe().cpu(), masks, multimask, d_low, d_iou)
    out, zero, bad = mmirror.compare(got, ref, P, 3 if multimask else 1)
    md = {k.split("mask_downscaling.")[1]: v for k, v in out.items() if "mask_downscaling" in k}
    grads = {k: v for k, v in out.items() if k not in ("low_res", "iou", "d_emb")}
    worst = sorted(grads.items(), key=lambda kv: -kv[1][1])[:3]
    print(f"\n{case}: " + ", ".join(f"{n} {out[n][0]:.2e}/{out[n][1]:.2e}" for n in ("low_res", "iou", "d_emb"))
          + "; mask_downscaling rel-L2/|slope-1| " + ", ".join(f"{k} {v[0]:.2e}/{v[1]:.2e}" for k, v in md.items())
          + f"; worst |slope - 1| " + ", ".join(f"{k.split('.', 1)[1]} {v[1]:.2e}" for k, v in worst)
          + f"; {len(zero)} zero tensors max {max(zero.values()):.2e}", flush=True)
    assert len(md) == (9 if kind == "zero" else 10)     # zero masks: conv 0's weight gradient is exactly zero
    assert not bad, bad


def test_masks_that_require_grad_are_refused(model):
    sd, sam = model
    emb, pts, boxes, masks, d_low, d_iou = _inputs(2, None, True, True, "logits", seed=3)
    with pytest.raises(ValueError, match="require grad"):
        sam.decoder_train(emb.to(DEV), None, boxes.to(DEV), True, masks=masks.to(DEV).requires_grad_(True))


# ------------------------------------------------------------------------------------------------ semantics
def test_unmasked_runs_keep_todays_tensors_and_leave_the_mask_tensors_alone():
    """A fresh model trained with box prompts only: no mask_downscaling key in decoder_grads(), grad_views() or the trained
    state; after a masked step registered them, an unmasked step + optimizer step leaves their masters and moments bit-identical."""
    from micro_sam_b200 import util
    sd = mmirror.perturbed_state_dict()
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
    sam.train()
    emb, pts, boxes, masks, d_low, d_iou = _inputs(3, None, True, True, "logits", seed=21)
    gpu_run(sam, emb, pts, boxes, None, True, d_low, d_iou)
    keys0, views0 = set(sam.decoder_grads()), [k for k, _ in sam.grad_views()]
    assert not any("mask_downscaling" in k for k in keys0) and not any("mask_downscaling" in k for k in views0)
    sam.optimizer_step(lr=1e-3)
    st0 = sam.trained_state_dict()
    assert all(torch.equal(st0[k], sd[k].float()) for k in mmirror.MD_KEYS)
    # a masked step registers the ten tensors after every tensor registered before
    gpu_run(sam, emb, pts, boxes, masks, True, d_low, d_iou)
    views1 = [k for k, _ in sam.grad_views()]
    assert views1[:len(views0)] == views0 and sorted(views1[len(views0):]) == sorted(mmirror.MD_KEYS)
    assert set(sam.decoder_grads()) == keys0 | set(mmirror.MD_KEYS)
    sam.optimizer_step(lr=1e-3)
    st1 = sam.trained_state_dict()
    assert all(not torch.equal(st1[k], sd[k].float()) for k in mmirror.MD_KEYS)
    # unmasked step: zero_decoder_grads forgets the masked gradient, AdamW skips the tensors (torch: grad None after zero_grad)
    gpu_run(sam, emb, pts, boxes, None, True, d_low, d_iou)
    views = dict(sam.grad_views())
    assert all(not bool(views[k].any()) for k in mmirror.MD_KEYS)
    sam.optimizer_step(lr=1e-3)
    st2 = sam.trained_state_dict()
    assert all(torch.equal(st2[k], st1[k]) for k in mmirror.MD_KEYS)
    assert not all(torch.equal(st2[k], st1[k]) for k in st1 if k.startswith("mask_decoder."))


def test_masked_and_unmasked_slots_accumulate_in_either_order(model):
    sd, sam = model
    A = _inputs(6, None, True, True, "logits", seed=101)
    B = _inputs(5, [[1, 0, 1]] * 5, True, False, "logits", seed=102)
    ga = gpu_run(sam, *A[:3], A[3], True, A[4], A[5])
    gb = gpu_run(sam, *B[:3], None, False, B[4], B[5])
    for order in ((0, 1), (1, 0)):
        from tests.test_gpu_decoder_train import to_dev
        sam.zero_decoder_grads()
        outs = []
        for slot, (inp, masked, mm) in enumerate(((A, True, True), (B, False, False))):
            gemb = inp[0].to(DEV).requires_grad_(True)
            p, b = to_dev(inp[1], inp[2])
            low, iou = sam.decoder_train(gemb, p, b, mm, slot=slot, masks=inp[3].to(DEV) if masked else None)
            outs.append((gemb, low, iou, inp))
        for i in order:
            gemb, low, iou, inp = outs[i]
            torch.autograd.backward([low, iou], [inp[4].to(DEV), inp[5].to(DEV)])
        torch.cuda.synchronize()
        assert torch.equal(outs[0][0].grad.cpu(), ga["d_emb"]) and torch.equal(outs[1][0].grad.cpu(), gb["d_emb"])
        both = {k: v.cpu() for k, v in sam.decoder_grads().items()}
        for k in mmirror.MD_KEYS:    # only the masked slot reaches them; deterministic reduction: the same bits
            assert torch.equal(both[k], ga["grads"][k]), k
        assert float(both[mmirror.NO_MASK].sub(gb["grads"][mmirror.NO_MASK]).abs().max()) <= 1e-5 * float(gb["grads"][mmirror.NO_MASK].norm())
        scale = max(float((ga["grads"][k] + gb["grads"].get(k, 0)).norm()) for k in both)
        bad = {}
        for k, g in both.items():
            s = ga["grads"][k] + gb["grads"].get(k, torch.zeros_like(g))
            err = float((g - s).norm())
            if not err <= 1e-5 * max(float(s.norm()), 1e-3 * scale):
                bad[k] = (err, float(s.norm()))
        assert not bad, (order, bad)


def test_masked_repeat_is_bit_identical(model):
    sd, sam = model
    inp = _inputs(13, [[1, 0]] * 13, True, True, "logits", seed=7)
    r1 = gpu_run(sam, *inp[:4], True, inp[4], inp[5], slot=2)
    r2 = gpu_run(sam, *inp[:4], True, inp[4], inp[5], slot=3)
    for name in ("low_res", "iou", "d_emb"):
        assert torch.equal(r1[name], r2[name]), name
    for k in mmirror.MD_KEYS:
        assert torch.equal(r1["grads"][k], r2["grads"][k]), k


def test_adamw_step_on_the_mask_tensors_matches_torch():
    from micro_sam_b200 import util
    sd = mmirror.perturbed_state_dict()
    sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
    sam.train()
    emb, pts, boxes, masks, d_low, d_iou = _inputs(4, None, True, True, "logits", seed=5)
    gpu_run(sam, emb, pts, boxes, None, True, d_low, d_iou)     # the other tensors take a step first: the step counts differ
    sam.optimizer_step(lr=2e-4)
    r = gpu_run(sam, emb, pts, boxes, masks, True, d_low, d_iou)
    kw = dict(lr=2e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    sam.optimizer_step(**kw)
    after = sam.trained_state_dict()
    worst = 0.0
    for k in mmirror.MD_KEYS:
        p = torch.nn.Parameter(sd[k].float().clone())
        p.grad = r["grads"][k].reshape(p.shape).clone()
        torch.optim.AdamW([p], **kw).step()
        d_ref, d_got = (p.detach() - sd[k]).double(), (after[k] - sd[k]).double()
        worst = max(worst, float((d_got - d_ref).norm() / d_ref.norm()))
    print(f"\nAdamW on mask_downscaling: worst rel-L2 of the update {worst:.2e}")
    assert worst < 1e-3
