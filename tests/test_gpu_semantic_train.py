"""`-m gpu`: semantic training on the GPU -- the prompt-free training decode of a whole batch in one slot
(msam_decoder_train_forward_images, `B200Sam.decoder_train_images`), the optimizer's skip of the tensors such a loss cannot reach,
and the drivers `get_trainable_sam_model`, `semantic_train_iteration` and `semantic_validation`.

The decode is compared with the float64 mirror that rounds to bf16 where the tape does (tests/decoder_train_mirror.py; pinned to
the oracle with empty sparse prompts in tests/test_semantic_train_cpu.py) over the batch.  The bounds are twice the bf16 noise
floor the mirror measures on the CPU for prompt-free batches (the mirror in float32 against itself in float64), or those of
tests/test_gpu_decoder_train.py where they are larger; DESIGN.md section 7 lists the floors and the measured GPU distances.  The mask decoder has the same width (transformer_dim 256) in every model type; the vit_b case
differs from vit_test only in its seeded weights and its encoder.
"""
import numpy as np
import pytest
import torch

from oracle import semantic_ref
from tests import decoder_train_mirror as mirror

pytestmark = pytest.mark.gpu
DEV = "cuda"
SKIPPED = ("mask_decoder.iou_prediction_head.", "prompt_encoder.point_embeddings.", "prompt_encoder.not_a_point_embed.",
           "prompt_encoder.mask_downscaling.")

# Twice the distance between the mirror in float32 and in float64 (the bf16 flip floor, measured on the CPU over B = 1, 2, 5,
# both multimask settings, seeded vit_test decoder), rounded up to two digits: (rel-L2, |slope - 1|) per family of gradients.
# A prompt-free batch has one prompt per image and 5 tokens per prompt, so its floor is above the prompted one for most
# families; the bound used is the larger of this and decoder_train_mirror.GRAD_BOUNDS.
PROMPT_FREE_GRAD_BOUNDS = {
    "mask_decoder.iou_token.weight": (0.15, 0.045),
    "mask_decoder.mask_tokens.weight": (0.15, 0.052),
    "mask_decoder.output_hypernetworks_mlps.*.layers.*.bias": (0.34, 0.042),
    "mask_decoder.output_hypernetworks_mlps.*.layers.*.weight": (0.34, 0.042),
    "mask_decoder.output_upscaling.*.bias": (0.019, 0.006),
    "mask_decoder.output_upscaling.*.weight": (0.02, 0.0047),
    "mask_decoder.transformer.final_attn_token_to_image.k_proj.weight": (0.25, 0.053),
    "mask_decoder.transformer.final_attn_token_to_image.out_proj.bias": (0.26, 0.038),
    "mask_decoder.transformer.final_attn_token_to_image.out_proj.weight": (0.26, 0.038),
    "mask_decoder.transformer.final_attn_token_to_image.q_proj.bias": (0.24, 0.051),
    "mask_decoder.transformer.final_attn_token_to_image.q_proj.weight": (0.24, 0.051),
    "mask_decoder.transformer.final_attn_token_to_image.v_proj.bias": (0.24, 0.058),
    "mask_decoder.transformer.final_attn_token_to_image.v_proj.weight": (0.24, 0.058),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.k_proj.weight": (0.15, 0.02),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.out_proj.bias": (0.15, 0.032),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.out_proj.weight": (0.15, 0.032),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.q_proj.bias": (0.2, 0.062),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.q_proj.weight": (0.15, 0.023),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.v_proj.bias": (0.16, 0.062),
    "mask_decoder.transformer.layers.*.cross_attn_image_to_token.v_proj.weight": (0.16, 0.062),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.k_proj.weight": (0.17, 0.021),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.out_proj.bias": (0.16, 0.04),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.out_proj.weight": (0.17, 0.04),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.q_proj.bias": (0.15, 0.037),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.q_proj.weight": (0.16, 0.037),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.v_proj.bias": (0.16, 0.027),
    "mask_decoder.transformer.layers.*.cross_attn_token_to_image.v_proj.weight": (0.16, 0.026),
    "mask_decoder.transformer.layers.*.mlp.lin1.bias": (0.17, 0.045),
    "mask_decoder.transformer.layers.*.mlp.lin1.weight": (0.17, 0.045),
    "mask_decoder.transformer.layers.*.mlp.lin2.bias": (0.17, 0.039),
    "mask_decoder.transformer.layers.*.mlp.lin2.weight": (0.17, 0.039),
    "mask_decoder.transformer.layers.*.norm1.bias": (0.16, 0.041),
    "mask_decoder.transformer.layers.*.norm1.weight": (0.17, 0.064),
    "mask_decoder.transformer.layers.*.norm2.bias": (0.16, 0.045),
    "mask_decoder.transformer.layers.*.norm2.weight": (0.16, 0.069),
    "mask_decoder.transformer.layers.*.norm3.bias": (0.16, 0.037),
    "mask_decoder.transformer.layers.*.norm3.weight": (0.15, 0.027),
    "mask_decoder.transformer.layers.*.norm4.bias": (0.15, 0.03),
    "mask_decoder.transformer.layers.*.norm4.weight": (0.12, 0.022),
    "mask_decoder.transformer.layers.*.self_attn.k_proj.weight": (0.18, 0.073),
    "mask_decoder.transformer.layers.*.self_attn.out_proj.bias": (0.17, 0.04),
    "mask_decoder.transformer.layers.*.self_attn.out_proj.weight": (0.17, 0.04),
    "mask_decoder.transformer.layers.*.self_attn.q_proj.bias": (0.17, 0.084),
    "mask_decoder.transformer.layers.*.self_attn.q_proj.weight": (0.18, 0.057),
    "mask_decoder.transformer.layers.*.self_attn.v_proj.bias": (0.17, 0.048),
    "mask_decoder.transformer.layers.*.self_attn.v_proj.weight": (0.17, 0.048),
    "mask_decoder.transformer.norm_final_attn.bias": (0.25, 0.042),
    "mask_decoder.transformer.norm_final_attn.weight": (0.26, 0.076),
    "prompt_encoder.no_mask_embed.weight": (0.17, 0.022),
}
# Outputs, the same measurement extended to B = 8 and 16 without multimask (one IoU scalar per image, so the worst row grows with
# B): low_res 7.6e-03 / 1.5e-02, iou 5.7e-02 / 1.5e-01, d_emb 1.2e-02 / 4.5e-02 (rel-L2 / worst row)
PROMPT_FREE_TOL = {"low_res": (0.016, 0.031), "iou": (0.12, 0.31), "d_emb": (0.024, 0.09)}
GRAD_BOUNDS = {k: tuple(max(a, b) for a, b in zip(v, PROMPT_FREE_GRAD_BOUNDS.get(k, v))) for k, v in mirror.GRAD_BOUNDS.items()}
TOL = {"low_res": mirror.TOL_LOW, "iou": mirror.TOL_IOU, "d_emb": mirror.TOL_DEMB}
TOL = {k: tuple(max(a, b) for a, b in zip(v, PROMPT_FREE_TOL[k])) for k, v in TOL.items()}


def _model(model_type="vit_test", max_batch=16, seed=1):
    from oracle import sam_ref
    from micro_sam_b200 import training
    sd = sam_ref.seeded_state_dict(model_type, seed=seed)
    model = training.get_trainable_sam_model(model_type, state_dict=sd, max_batch=max_batch, max_prompts=64)
    return sd, model


@pytest.fixture(scope="module")
def small():
    return _model()


def _inputs(B, multimask, seed):
    gen = torch.Generator().manual_seed(seed)
    emb = torch.randn(B, 256, 64, 64, generator=gen)
    d_low = torch.randn(B, 3 if multimask else 1, 256, 256, generator=gen) / 256
    return emb, d_low


def _gpu(sam, emb, d_low, multimask, slot=0):
    sam.zero_decoder_grads()
    e = emb.to(DEV).requires_grad_(True)
    low, iou = sam.decoder_train_images(e, multimask, slot=slot)
    low.backward(d_low.to(DEV))
    torch.cuda.synchronize()
    return {"low_res": low.detach().cpu(), "iou": iou.detach().cpu(), "d_emb": e.grad.detach().cpu(),
            "grads": {k: v.detach().cpu() for k, v in sam.decoder_grads().items()}}


def _mirror(sd, sam, emb, d_low, multimask):
    """the mirror image by image (one prompt with no sparse token each); parameter gradients summed over the images"""
    dense_pe = sam.prompt_encoder.get_dense_pe().cpu()
    runs = [mirror.run(sd, emb[b], torch.zeros(1, 0, 256), torch.zeros(1, 0, dtype=torch.int64), dense_pe, multimask,
                       d_low[b:b + 1], None) for b in range(emb.shape[0])]
    grads = {k: sum(r["grads"][k] for r in runs) for k in runs[0]["grads"]}
    return runs, grads


def _check_against_mirror(got, runs, grads, M, monkeypatch):
    """outputs and dL/d embedding over the batch (rows: images x masks x logit rows, images, images x channels; each row's
    error against a floor of a quarter of the RMS row norm, as mirror.errors does), then every gradient with mirror.compare under
    the prompt-free bounds.  Returns (output errors, gradient errors, zero-gradient errors, violations)."""
    B = len(runs)
    ref = {n: torch.cat([r[n].reshape(1, -1) for r in runs]) for n in ("low_res", "iou", "d_emb")}
    worst, bad = {}, []
    for name, rows in (("low_res", B * M * 256), ("iou", B), ("d_emb", B * 256)):
        worst[name] = mirror.errors(got[name], ref[name], rows)
        if not (worst[name][0] <= TOL[name][0] and worst[name][1] <= TOL[name][1]):
            bad.append((name, worst[name], TOL[name]))
    monkeypatch.setattr(mirror, "GRAD_BOUNDS", GRAD_BOUNDS)
    first = {n: runs[0][n] for n in ("low_res", "iou", "d_emb")}
    out, zero, bad_g = mirror.compare({**first, "grads": got["grads"]}, {**first, "grads": grads}, 1, M)
    return worst, out, zero, bad + bad_g


@pytest.mark.parametrize("multimask", [True, False])
@pytest.mark.parametrize("B", [1, 2, 5, 8, 16])
def test_prompt_free_decode_against_bf16_mirror(small, B, multimask, monkeypatch):
    """B images in one slot: P * T = 5 B token rows (5 and 25 are multiples of no tile size)."""
    sd, model = small
    emb, d_low = _inputs(B, multimask, seed=31 * B + multimask)
    got = _gpu(model.sam, emb, d_low, multimask)
    runs, grads = _mirror(sd, model.sam, emb, d_low, multimask)
    worst, out, zero, bad = _check_against_mirror(got, runs, grads, 3 if multimask else 1, monkeypatch)
    g = {k: v for k, v in out.items() if k not in ("low_res", "iou", "d_emb")}
    print(f"\nB={B} multimask={multimask}: " + ", ".join(f"{n} {worst[n][0]:.2e}/{worst[n][1]:.2e}" for n in worst)
          + f"; {len(g)} gradients median rel-L2 {np.median([v[0] for v in g.values()]):.2e} max {max(v[0] for v in g.values()):.2e}"
          + f", |slope - 1| median {np.median([v[1] for v in g.values()]):.2e} max {max(v[1] for v in g.values()):.2e}"
          + f"; {len(zero)} zero tensors max {max(zero.values()):.2e}", flush=True)
    assert not bad, bad
    # what the loss cannot reach gets no gradient: the IoU head and the sparse-prompt tables
    for k, v in got["grads"].items():
        if k.startswith(SKIPPED):
            assert not v.any(), k
    assert got["grads"]["prompt_encoder.no_mask_embed.weight"].abs().max() > 0


def test_batch_is_independent_per_image(small):
    """Image b of a batch of 5 gives the same low_res, iou and dL/d embedding bits as a batch of one; parameter gradients are
    the sum over the single runs to atomic rounding."""
    sd, model = small
    emb, d_low = _inputs(5, True, seed=3)
    both = _gpu(model.sam, emb, d_low, True, slot=3)
    singles = [_gpu(model.sam, emb[b:b + 1], d_low[b:b + 1], True, slot=b) for b in range(5)]
    for b, s in enumerate(singles):
        for name in ("low_res", "iou", "d_emb"):
            assert torch.equal(both[name][b:b + 1], s[name]), (b, name)
    scale = max(float(sum(s["grads"][k] for s in singles).norm()) for k in both["grads"])
    bad = {}
    for k, g in both["grads"].items():
        want = sum(s["grads"][k] for s in singles)
        err = float((g - want).norm())
        if not err <= 1e-5 * max(float(want.norm()), 1e-3 * scale):
            bad[k] = (err, float(want.norm()))
    assert not bad, bad


def test_eval_mode_prompt_free_matches_oracle(small):
    """TrainableSAM in eval mode on records without prompts decodes on the inference decoder (T = 5) within the inference
    bounds of tests/test_gpu_parity.py (low-res rel-L2 <= 3e-2, IoU abs <= 2e-2)."""
    from oracle import sam_ref, train_ref
    sd, model = small
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    oracle = train_ref.TrainableSAM(osam.eval())
    emb, _ = _inputs(3, True, seed=11)
    recs = [{"original_size": (300, 400), "input_size": (768, 1024)} for _ in range(3)]
    model.sam.eval()
    try:
        outs = model([dict(r) for r in recs], emb.to(DEV), multimask_output=True, return_masks=False)
    finally:
        model.sam.train()
    with torch.no_grad():
        want = oracle([dict(r) for r in recs], emb, multimask_output=True)
    for o, w in zip(outs, want):
        lo, wl = o["low_res_masks"].cpu().double(), w["low_res_masks"].double()
        assert float((lo - wl).norm() / wl.norm()) <= 3e-2
        assert float((o["iou_predictions"].cpu() - w["iou_predictions"]).abs().max()) <= 2e-2


def _labels(B, H, W, C, seed):
    """piecewise-constant class maps (blocks of 16 x 16), with a strip of ignored pixels"""
    gen = torch.Generator().manual_seed(seed)
    y = torch.randint(0, C, (B, 1, (H + 15) // 16, (W + 15) // 16), generator=gen)
    y = y.repeat_interleave(16, 2).repeat_interleave(16, 3)[..., :H, :W].contiguous()
    y[:, :, :4] = -100
    return y


def _registry(sam):
    torch.cuda.synchronize()
    return {k: (g.clone(), w.clone()) for k, g, w in sam._registry()}


def _adamw_expected(before, grads_of, lr, wd):
    """torch.optim.AdamW, one step, on fp32 copies of the masters; grads_of(key) -> gradient or None (skipped)"""
    params, expect = {}, {}
    for k, (_, w) in before.items():
        p = torch.nn.Parameter(w.clone())
        p.grad = grads_of(k)
        params[k] = p
    opt = torch.optim.AdamW(list(params.values()), lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
    opt.step()
    return {k: p.detach() for k, p in params.items()}


@pytest.mark.parametrize("dice_weight", [None, 0.3])
@pytest.mark.parametrize("size", [(512, 512), (700, 1100)])
def test_semantic_step_vit_b(size, dice_weight, monkeypatch):
    """One semantic step at vit_b widths (seeded weights), B = 2, C = 3: the loss against the float64 oracle of the GPU's own
    low-res logits; dL/d embedding handed to the encoder and the decoder gradients against the mirror fed the oracle's dL/d
    low-res; one optimizer_step against torch.optim.AdamW with grad None for the tensors the loss cannot reach (their masters
    stay bit-identical) and output_hypernetworks_mlps.0 decayed."""
    from micro_sam_b200 import training
    sd, model = _model("vit_b", max_batch=2, seed=4)
    sam = model.sam
    H, W = size
    gen = torch.Generator().manual_seed(H + W)
    x = torch.rand(2, 3, H, W, generator=gen) * 255
    y = _labels(2, H, W, 3, seed=H)
    sam.zero_decoder_grads()
    batched = training.ConvertToSemanticSamInputs()(x, y)
    emb, batched = model.image_embeddings_oft(batched)
    emb.retain_grad()
    outs = model(batched, emb, multimask_output=True, return_masks=False)
    loss = training.compute_semantic_loss(outs, y, 3, dice_weight)
    loss.backward()
    torch.cuda.synchronize()
    input_size = batched[0]["input_size"]
    low = torch.cat([o["low_res_masks"].detach() for o in outs]).cpu().double().requires_grad_(True)
    want = semantic_ref.semantic_loss_from_low_res(low, y, input_size, (H, W), 3, dice_weight)
    want.backward()
    assert abs(float(loss.detach()) - float(want.detach())) <= 1e-5 * abs(float(want.detach()))
    # the decoder against the mirror fed the oracle's dL/d low-res
    runs, grads = _mirror(sd, sam, emb.detach().cpu(), low.grad.float(), True)
    got = {"low_res": low.detach().float(), "iou": torch.cat([o["iou_predictions"].detach() for o in outs]).cpu(),
           "d_emb": emb.grad.detach().cpu(), "grads": {k: v.cpu() for k, v in sam.decoder_grads().items()}}
    worst, out, zero, bad = _check_against_mirror(got, runs, grads, 3, monkeypatch)
    print(f"\nvit_b {size} dice_weight={dice_weight}: loss {float(loss.detach()):.6f} (oracle {float(want.detach()):.6f}), "
          + ", ".join(f"{n} {worst[n][0]:.2e}/{worst[n][1]:.2e}" for n in worst), flush=True)
    assert not bad, bad
    # one AdamW step: skipped groups untouched, everything else as torch.optim.AdamW
    lr, wd = 1e-3, 0.01
    before = _registry(sam)
    sam.optimizer_step(lr=lr, weight_decay=wd)
    after = _registry(sam)
    expect = _adamw_expected(before, lambda k: None if k.startswith(SKIPPED) else before[k][0].clone(), lr, wd)
    for k, (_, w) in after.items():
        if k.startswith(SKIPPED):
            assert torch.equal(w, before[k][1]), k
        else:
            assert torch.allclose(w, expect[k], rtol=1e-6, atol=1e-7), k
    h0 = [k for k in after if k.startswith("mask_decoder.output_hypernetworks_mlps.0.")]
    assert h0 and all(not before[k][0].any() and torch.allclose(after[k][1], before[k][1] * (1 - lr * wd), rtol=1e-6) for k in h0)


def test_prompted_backward_restores_todays_step():
    """A prompt-free and a prompted backward in one zeroing window: the step updates every tensor with its gradient, the IoU
    head and the sparse-prompt tables included, exactly as torch.optim.AdamW does."""
    sd, model = _model(max_batch=2)
    sam = model.sam
    emb, d_low = _inputs(2, True, seed=8)
    sam.zero_decoder_grads()
    e = emb.to(DEV).requires_grad_(True)
    low, _ = sam.decoder_train_images(e, True, slot=1)
    low.backward(d_low.to(DEV))
    gen = torch.Generator().manual_seed(2)
    xy = torch.rand(3, 2, generator=gen) * 600 + 50
    boxes = torch.cat([xy, xy + 200], 1).to(DEV)
    low_p, iou_p = sam.decoder_train(emb[0].to(DEV).requires_grad_(True), None, boxes, True, slot=0)
    torch.autograd.backward([low_p, iou_p], [torch.randn(3, 3, 256, 256, generator=gen).to(DEV) / 256,
                                             torch.randn(3, 3, generator=gen).to(DEV)])
    before = _registry(sam)
    sam.optimizer_step(lr=1e-3, weight_decay=0.01)
    after = _registry(sam)
    dec = {k: v for k, v in before.items() if k.startswith(("mask_decoder.", "prompt_encoder."))}
    expect = _adamw_expected(dec, lambda k: dec[k][0].clone(), 1e-3, 0.01)
    for k in dec:
        assert torch.allclose(after[k][1], expect[k], rtol=1e-6, atol=1e-7), k
    assert any(k.startswith("mask_decoder.iou_prediction_head.") and not torch.equal(after[k][1], before[k][1]) for k in dec)


def test_sixteen_images_and_mixed_batches():
    """16 prompt-free images in one training forward (more than the 8 slots), a mixed batch of 7 prompted and 9 prompt-free
    records (8 slots), and repeats of both that give the same low_res and dL/d embedding bits."""
    from micro_sam_b200 import training
    sd, model = _model(max_batch=16)
    gen = torch.Generator().manual_seed(16)
    x = torch.rand(16, 3, 96, 128, generator=gen) * 255
    y = _labels(16, 96, 128, 3, seed=16)

    def step(records):
        model.sam.zero_decoder_grads()
        emb, batched = model.image_embeddings_oft(records)
        emb.retain_grad()
        outs = model(batched, emb, multimask_output=True, return_masks=False)
        free = [i for i, r in enumerate(batched) if "boxes" not in r]
        loss = training.compute_semantic_loss([outs[i] for i in free], y[free], 3)
        prompted = [outs[i]["low_res_masks"].sum() * 1e-3 for i in range(len(outs)) if i not in free]
        (loss + sum(prompted)).backward()
        torch.cuda.synchronize()
        return torch.cat([o["low_res_masks"].detach() for o in outs]).cpu(), emb.grad.cpu()

    recs = training.ConvertToSemanticSamInputs()(x, y)
    a, b = step([dict(r) for r in recs]), step([dict(r) for r in recs])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.isfinite(a[0]).all() and a[1].abs().amax(dim=(1, 2, 3)).min() > 0
    mixed = [dict(r) for r in recs]
    for i in range(7):
        mixed[2 * i]["boxes"] = torch.tensor([[10.0 + i, 20.0, 300.0, 400.0]])
    assert training.decoder_slots(mixed).count(None) == 9
    c, d = step([dict(r) for r in mixed]), step([dict(r) for r in mixed])
    assert torch.equal(c[0], d[0]) and torch.equal(c[1], d[1])
    with pytest.raises(ValueError, match="8"):
        model([dict(r, boxes=torch.tensor([[10.0, 20.0, 300.0, 400.0]])) for r in recs[:9]], torch.zeros(9, 256, 64, 64, device=DEV))


def test_drivers_end_to_end():
    """semantic_train_iteration + optimizer_step and semantic_validation on vit_test.  allreduce_grads(1) leaves every gradient
    bit-identical, so the step that reads them is unchanged.  Validation restores train() mode and decodes with the trained
    weights (the training decoder's forward pass)."""
    from micro_sam_b200 import training
    gen = torch.Generator().manual_seed(5)
    x = torch.rand(2, 3, 200, 300, generator=gen) * 255
    y = _labels(2, 200, 300, 3, seed=5)
    _, model = _model(max_batch=2)
    model.sam.zero_decoder_grads()
    loss = training.semantic_train_iteration(model, x, y, 3, dice_weight=0.5)
    loss.backward()
    before = _registry(model.sam)
    assert model.sam.allreduce_grads(1) > 0
    after = _registry(model.sam)
    assert before.keys() == after.keys() and all(torch.equal(before[k][0], after[k][0]) for k in before)
    model.sam.optimizer_step(lr=1e-4)
    stepped = _registry(model.sam)
    assert np.isfinite(float(loss.detach()))
    assert any(not torch.equal(stepped[k][1], before[k][1]) for k in before if k.startswith("mask_decoder.transformer."))
    assert all(torch.equal(stepped[k][1], before[k][1]) for k in before if k.startswith(SKIPPED))
    loader = [(x, y), (x[:1], y[:1])]
    metric, vloss = training.semantic_validation(model, loader, 3, dice_weight=0.5)
    assert model.sam.training and metric == vloss and np.isfinite(metric)
    # the validation loss is the mean of the per-batch losses under the trained weights
    per = []
    model.sam.eval()
    with torch.no_grad():
        for xb, yb in loader:
            batched = training.ConvertToSemanticSamInputs()(xb, yb)
            emb, batched = model.image_embeddings_oft(batched)
            low, _ = model.sam.decode_images_with_training_decoder(emb, True)
            per.append(float(training.compute_semantic_loss(low, yb, 3, 0.5, input_size=batched[0]["input_size"])))
    model.sam.train()
    assert abs(metric - sum(per) / len(per)) <= 1e-6 * abs(metric)
