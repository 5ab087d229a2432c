"""`-m gpu` parity of the encoder backward pass (BASELINE.json configs[4], csrc/encoder_train.cu) against torch autograd over the
fp32 oracle encoder (oracle/sam_ref.py): op level (batched attention-backward GEMM in its four operand layouts, LayerNorm
backward) and model level (every parameter gradient of the image encoder for a random upstream gradient dL/d embedding).
Tolerance: encoder alone (random upstream gradient) rel-L2 <= 3e-2 per gradient tensor (bf16 operands, fp32 accumulation; the forward
tolerance is 2e-2); decoder and whole step: rel-L2 <= 1.5e-1 and cosine >= 0.99 per tensor = the measured bf16 noise floor of the
decoder (see test_decoder_train_against_autograd); the loss-statistics adjoint is exact to 1e-6.  The decoder is also compared with
a float64 mirror that rounds to bf16 where the kernels do, over more prompt counts, token counts and backward paths, in
tests/test_gpu_decoder_train.py."""
import os
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("hd,Tq", [(64, 196), (80, 196), (64, 512)])
def test_bgemm_layouts_against_torch(hd, Tq):
    """C[w,h] = op(A[w,h]) op(B[w,h]) on head / window slices of packed buffers, incl. the zero-filled tails (head_dim 80: the
    second 64-column box; 196-row windows in 64-row boxes)."""
    from micro_sam_b200 import _lib
    L = _lib.lib()
    H, W = 3, 2
    D = H * hd
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(W * Tq, 3 * D, generator=g).to(DEV).bfloat16()
    q = qkv[:, :D].float().view(W, Tq, H, hd).permute(0, 2, 1, 3)            # [W,H,Tq,hd]
    k = qkv[:, D:2 * D].float().view(W, Tq, H, hd).permute(0, 2, 1, 3)
    pitch = (Tq + 7) // 8 * 8
    # NT: S = Q K^T
    S = torch.full((W, H, Tq, pitch), 7.0, device=DEV)
    _lib.check(L.msam_op_bgemm(_lib.ptr(qkv), ctypes_off(qkv, D), 0, 0, Tq, Tq, hd, 3 * D, 3 * D, hd, Tq * 3 * D, hd, Tq * 3 * D, H, W,
                               _lib.ptr(S), pitch, Tq * pitch, H * Tq * pitch, 0.5, 0, _lib.cur_stream()))
    torch.cuda.synchronize()
    assert _rel(S[..., :Tq], 0.5 * q @ k.transpose(-1, -2)) < 1e-5
    assert bool((S[..., Tq:] == 7.0).all())                                     # columns beyond N untouched
    # TN: dV = P^T dO  (P [Tq, pitch] per batch entry, dO as a head slice of a [rows, D] buffer), then accumulate
    P = torch.randn(W, H, Tq, pitch, generator=g).to(DEV).bfloat16()
    dO = torch.randn(W * Tq, D, generator=g).to(DEV).bfloat16()
    do = dO.float().view(W, Tq, H, hd).permute(0, 2, 1, 3)
    dV = torch.zeros(W, H, Tq, hd, device=DEV)
    for acc in (0, 1):
        _lib.check(L.msam_op_bgemm(_lib.ptr(P), _lib.ptr(dO), 1, 1, Tq, hd, Tq, pitch, D, Tq * pitch, H * Tq * pitch, hd, Tq * D, H, W,
                                   _lib.ptr(dV), hd, Tq * hd, H * Tq * hd, 1.0, acc, _lib.cur_stream()))
    torch.cuda.synchronize()
    assert _rel(dV, 2 * P.float()[..., :Tq].transpose(-1, -2) @ do) < 1e-5
    # NN: dQ = dS K  (A K-major [Tq, Tk], B = the K slice consumed MN-major)
    dQ = torch.empty(W, H, Tq, hd, device=DEV)
    _lib.check(L.msam_op_bgemm(_lib.ptr(P), ctypes_off(qkv, D), 0, 1, Tq, hd, Tq, pitch, 3 * D, Tq * pitch, H * Tq * pitch, hd,
                               Tq * 3 * D, H, W, _lib.ptr(dQ), hd, Tq * hd, H * Tq * hd, 1.0, 0, _lib.cur_stream()))
    torch.cuda.synchronize()
    assert _rel(dQ, P.float()[..., :Tq] @ k) < 1e-5
    # NT against a table shared by every batch entry: T = Q R^T
    R = torch.zeros(64, (hd + 63) // 64 * 64, device=DEV, dtype=torch.bfloat16)
    R[:27, :hd] = torch.randn(27, hd, generator=g).to(DEV).bfloat16()
    T = torch.empty(W, H, Tq, 64, device=DEV)
    _lib.check(L.msam_op_bgemm(_lib.ptr(qkv), _lib.ptr(R), 0, 0, Tq, 64, hd, 3 * D, R.shape[1], hd, Tq * 3 * D, 0, 0, H, W,
                               _lib.ptr(T), 64, Tq * 64, H * Tq * 64, 1.0, 0, _lib.cur_stream()))
    torch.cuda.synchronize()
    assert _rel(T, q @ R.float()[:, :hd].t()) < 1e-5


def ctypes_off(t, elems):
    import ctypes
    return ctypes.c_void_p(t.data_ptr() + elems * t.element_size())


@pytest.mark.parametrize("D,window", [(768, 0), (1280, 0), (128, 1)])
def test_layernorm_backward_against_autograd(D, window):
    from micro_sam_b200 import _lib
    L = _lib.lib()
    B, g = 2, 64
    rows = B * g * g
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(rows, D, generator=gen) * 2 + 0.5).to(DEV).requires_grad_(True)
    gamma = (1 + 0.1 * torch.randn(D, generator=gen)).to(DEV).requires_grad_(True)
    beta = (0.1 * torch.randn(D, generator=gen)).to(DEV).requires_grad_(True)
    dy = torch.randn(rows, D, generator=gen).to(DEV)
    y = torch.nn.functional.layer_norm(x, (D,), gamma, beta, 1e-6)
    y.backward(dy)
    dy_in = dy
    if window:   # dy handed over in the window-partitioned row order (pad rows hold garbage that must be ignored)
        pad = torch.nn.functional.pad(dy.view(B, g, g, D), (0, 0, 0, 6, 0, 6), value=123.0)
        dy_in = pad.view(B, 5, 14, 5, 14, D).permute(0, 1, 3, 2, 4, 5).reshape(-1, D).contiguous()
    dx = torch.ones(rows, D, device=DEV)
    dg, db = torch.zeros(D, device=DEV), torch.zeros(D, device=DEV)
    _lib.check(L.msam_op_layernorm_bwd(_lib.ptr(x.detach()), rows, D, _lib.ptr(gamma.detach()), 1e-6, _lib.ptr(dy_in), window, 1,
                                       _lib.ptr(dx), _lib.ptr(dg), _lib.ptr(db), _lib.cur_stream()))
    torch.cuda.synchronize()
    assert _rel(dx - 1.0, x.grad) < 1e-4 and _rel(dg, gamma.grad) < 1e-4 and _rel(db, beta.grad) < 1e-4


def _encoder_grad_case(model_type, B, names=None, tol=3e-2):
    from oracle import sam_ref
    from micro_sam_b200.sam import B200Sam
    from micro_sam_b200.sample_data import lm_tile
    from micro_sam_b200 import util
    torch.set_num_threads(min(64, os.cpu_count() or 8))
    sd = sam_ref.seeded_state_dict(model_type, seed=0)
    osam = sam_ref.build_sam(model_type)
    osam.load_state_dict(sd)
    enc_sd = {k: v for k, v in sd.items() if k.startswith("image_encoder.")}
    sam = B200Sam(model_type, enc_sd, max_batch=B, max_prompts=1).train()
    imgs = np.stack([util._to_image(lm_tile((1024, 1024), 150, seed=s)) for s in range(B)])
    x_pre = torch.stack([osam.preprocess(torch.from_numpy(i).permute(2, 0, 1)[None].float())[0] for i in imgs])
    gen = torch.Generator().manual_seed(5)
    d_out = torch.randn(B, 256, 64, 64, generator=gen)
    enc = osam.image_encoder
    for p in enc.parameters():
        p.requires_grad_(True)
    ref_out = enc(x_pre)
    ref_out.backward(d_out)
    got_out = sam.image_encoder(x_pre.to(DEV))
    assert got_out.requires_grad
    rel_f = _rel(got_out.detach(), ref_out.detach())
    got_out.backward(d_out.to(DEV))
    grads = sam.encoder_grads(names)
    rels = {}
    for k, gten in grads.items():
        ref = dict(enc.named_parameters())[k[len("image_encoder."):]].grad
        assert ref is not None and tuple(ref.shape) == tuple(gten.shape), k
        rels[k] = _rel(gten, ref)
    worst = sorted(rels.items(), key=lambda kv: -kv[1])[:6]
    print(f"{model_type} B={B}: forward rel-L2 {rel_f:.2e}; {len(rels)} gradients, median rel-L2 {np.median(list(rels.values())):.2e}, worst: "
          + ", ".join(f"{k.replace('image_encoder.', '')} {v:.2e}" for k, v in worst))
    assert rel_f < 2e-2
    bad = {k: v for k, v in rels.items() if not v < tol}
    assert not bad, bad
    # the inference path of the same engine is untouched by training mode
    with torch.no_grad():
        assert _rel(sam.eval().image_encoder(x_pre.to(DEV)), ref_out.detach()) < 2e-2
    del sam
    torch.cuda.empty_cache()


@pytest.mark.parametrize("model_type", ["vit_test", "vit_test80"])
def test_encoder_backward_small_archs(model_type):
    """One windowed + one global block, head_dim 64 / 80, batch 2: every parameter gradient."""
    _encoder_grad_case(model_type, B=2)


def test_encoder_backward_vit_b():
    """The architecture cfg 5 names, one image (the fp32 autograd reference needs ~30 GB of host memory for the global blocks)."""
    _encoder_grad_case("vit_b", B=1)


# ------------------------------------------------------------------------------------------------ decoder + loss + full step
def _small_models(max_batch=2):
    from oracle import sam_ref
    from micro_sam_b200 import util
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    osam = sam_ref.build_sam("vit_test")
    osam.load_state_dict(sd)
    pred = util.get_sam_model("vit_test", state_dict=sd, max_batch=max_batch, max_prompts=64)
    return osam, pred.model


def _compare_grads(got, ref_named, tol, min_cos=0.0, dump=None):
    """rel-L2 per gradient tensor.  Gradients that are analytically zero (k_proj biases: softmax is invariant to a constant added to
    every key's logit; parameters the prompt type does not touch) are compared absolutely against the scale of the largest
    reference gradient instead."""
    scale = max(float(p.grad.double().norm()) for p in ref_named.values() if p.grad is not None)
    rels, bad = {}, {}
    for k, g in got.items():
        ref = ref_named[k].grad
        if ref is None or float(ref.double().norm()) < 1e-6 * scale:
            if not float(g.double().norm()) < 1e-3 * scale:
                bad[k] = ("expected ~0", float(g.double().norm()), scale)
            continue
        assert tuple(ref.shape) == tuple(g.shape), (k, ref.shape, g.shape)
        r = _rel(g, ref)
        cos = float(torch.nn.functional.cosine_similarity(g.double().cpu().flatten(), ref.double().flatten(), dim=0))
        rels[k] = r
        if not (r < tol and cos > min_cos):
            bad[k] = (r, cos)
    if dump:
        with open(dump, "w") as f:
            for k, v in sorted(rels.items(), key=lambda kv: -kv[1]):
                f.write(f"{v:.3e}  {k}\n")
    return rels, bad


@pytest.mark.parametrize("prompt,multimask", [("boxes", True), ("points", False), ("points+boxes", True)])
def test_decoder_train_against_autograd(prompt, multimask):
    """Training-mode mask decoder + prompt encoder (csrc/decoder_train.cu) for one image: forward against the oracle modules, then
    dL/d embedding and every parameter gradient for a random linear functional of (low_res, iou) against torch autograd."""
    osam, sam = _small_models()
    sam.train()
    gen = torch.Generator().manual_seed(3)
    P = 6
    emb = torch.randn(1, 256, 64, 64, generator=gen)
    boxes = pts = None
    if "boxes" in prompt:
        xy = torch.rand(P, 2, generator=gen) * 600 + 50
        boxes = torch.cat([xy, xy + torch.rand(P, 2, generator=gen) * 300 + 20], 1)
    if "points" in prompt:
        coords = torch.rand(P, 3, 2, generator=gen) * 1000
        labels = torch.tensor([[1, 0, 1]] * (P - 1) + [[1, 1, -1]], dtype=torch.float32)
        pts = (coords, labels)
    M = 3 if multimask else 1
    w_low = torch.randn(P, M, 256, 256, generator=gen) / 256
    w_iou = torch.randn(P, M, generator=gen)
    # oracle
    for p in osam.parameters():
        p.requires_grad_(True)
    oemb = emb.clone().requires_grad_(True)
    sp, de = osam.prompt_encoder(points=pts, boxes=boxes, masks=None)
    olow, oiou = osam.mask_decoder(image_embeddings=oemb, image_pe=osam.prompt_encoder.get_dense_pe(), sparse_prompt_embeddings=sp,
                                   dense_prompt_embeddings=de, multimask_output=multimask)
    ((olow * w_low).sum() + (oiou * w_iou).sum()).backward()
    # ours
    gemb = emb.clone().to(DEV).requires_grad_(True)
    gp = None if pts is None else (pts[0].to(DEV), pts[1].to(DEV))
    sam.zero_decoder_grads()
    low, iou = sam.decoder_train(gemb[0], gp, None if boxes is None else boxes.to(DEV), multimask, slot=1)
    rl, ri = _rel(low.detach(), olow.detach()), float((iou.detach().cpu() - oiou.detach()).abs().max())
    torch.autograd.backward([low, iou], [w_low.to(DEV), w_iou.to(DEV)])
    re = _rel(gemb.grad, oemb.grad)
    # Tolerance = the bf16 noise floor of this decoder, measured with torch itself (tests/bf16_noise_floor.py: the oracle under
    # autocast(bfloat16) against its own fp32 autograd gives forward 1.5e-2, d emb 1.8e-2, parameter gradients median 8.2e-2, worst
    # 1.3e-1 -- on the SAME tensors that are worst here: hyper-network MLP 1, norm_final_attn, final attention): the token side is
    # 42 rows through ~25 bf16 ops and with random weights the attention is near uniform, so dS = P (dP - sum P dP) is a small
    # difference of bf16-rounded products.  The image side (d emb) sits at 1e-2.
    rels, bad = _compare_grads(sam.decoder_grads(), dict(osam.named_parameters()), 1.5e-1, min_cos=0.99,
                               dump=os.path.join(tempfile.gettempdir(), f"decoder_grads_{prompt}.txt"))
    worst = sorted(rels.items(), key=lambda kv: -kv[1])[:5]
    print(f"decoder_train {prompt} M={M}: low-res rel-L2 {rl:.2e}, iou err {ri:.2e}, d emb rel-L2 {re:.2e}; {len(rels)} parameter gradients, "
          f"median {np.median(list(rels.values())):.2e}, worst " + ", ".join(f"{k.split('.', 1)[1]} {v:.2e}" for k, v in worst))
    assert rl < 3e-2 and ri < 2e-2 and re < 4e-2
    assert not bad, bad


@pytest.mark.parametrize("input_size,original_size", [((768, 1024), (96, 128)), ((1024, 1024), (1024, 1024)), ((1024, 1024), (512, 512))])
def test_loss_backward_against_autograd(input_size, original_size):
    """d loss / d low-res logits of compute_loss (dice of sigmoid(postprocess_masks(low_res)) minimised over the candidate masks + IoU
    MSE): the fused statistics kernel + its adjoint against autograd through the oracle's interpolate / sigmoid / dice."""
    from oracle import sam_ref, train_ref
    from micro_sam_b200 import training
    H, W = original_size
    gen = torch.Generator().manual_seed(4)
    n_obj, M = 3, 3
    low = (torch.randn(n_obj, M, 256, 256, generator=gen) * 2)
    low = torch.nn.functional.avg_pool2d(low, 9, 1, 4)        # smooth logits: masks with structure
    iou = torch.rand(n_obj, M, generator=gen)
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    tg = torch.stack([(((yy - H * (0.3 + 0.2 * k)) ** 2 + (xx - W * (0.3 + 0.2 * k)) ** 2) < (min(H, W) * 0.15) ** 2).float()[None] for k in range(n_obj)])
    osam = sam_ref.build_sam("vit_test")
    olow = low.clone().requires_grad_(True)
    oiou = iou.clone().requires_grad_(True)
    omasks = osam.postprocess_masks(olow, input_size, original_size)
    oloss = train_ref.compute_loss([{"masks": omasks, "iou_predictions": oiou}], [tg])
    oloss[0].backward()
    glow = low.clone().to(DEV).requires_grad_(True)
    giou = iou.clone().to(DEV).requires_grad_(True)
    loss = training.compute_loss([{"low_res_masks": glow, "iou_predictions": giou, "input_size": input_size, "original_size": original_size}], [tg])
    loss[0].backward()
    assert abs(float(loss[0]) - float(oloss[0])) < 1e-4
    r1, r2 = _rel(glow.grad, olow.grad), _rel(giou.grad, oiou.grad)
    print(f"loss backward {input_size}->{original_size}: loss {float(loss[0]):.4f}, d low-res rel-L2 {r1:.2e}, d iou rel-L2 {r2:.2e}")
    assert r1 < 1e-3 and r2 < 1e-4


def test_training_step_end_to_end():
    """The whole fine-tuning step of cfg 5 on the tiny architecture: TrainableSAM.image_embeddings_oft -> forward (box prompts) ->
    _compute_loss -> loss.backward(): the loss and every encoder / decoder / prompt-encoder gradient against the oracle TrainableSAM
    under torch autograd (micro_sam/training/sam_trainer.py:131-172, :393)."""
    from oracle import train_ref
    from micro_sam_b200 import training
    from micro_sam_b200.sample_data import lm_tile
    osam, sam = _small_models()
    sam.train()
    for p in osam.parameters():
        p.requires_grad_(True)
    om, m = train_ref.TrainableSAM(osam), training.TrainableSAM(sam)
    B, n_obj, H, W = 2, 4, 128, 128
    imgs = [torch.from_numpy(np.repeat(lm_tile((H, W), 12, seed=30 + b, dtype="uint8")[None], 3, 0).astype("float32")) for b in range(B)]
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    cen = [(30 + 22 * k, 28 + 24 * k, 9 + 2 * k) for k in range(n_obj)]
    y_one_hot = [torch.stack([(((yy - cy) ** 2 + (xx - cx) ** 2) < r * r).float()[None] for cy, cx, r in cen]) for _ in range(B)]
    boxes = torch.tensor([[cx - r, cy - r, cx + r, cy + r] for cy, cx, r in cen], dtype=torch.float32) * (1024.0 / W)

    def records():
        return [{"image": im.clone(), "original_size": (H, W), "boxes": boxes.clone()} for im in imgs]
    oemb, orecs = om.image_embeddings_oft(records())
    oloss = train_ref.compute_loss(om(orecs, oemb, multimask_output=True), y_one_hot)
    oloss[0].backward()
    sam.zero_decoder_grads()
    emb, recs = m.image_embeddings_oft(records())
    assert emb.requires_grad
    loss = training.compute_loss(m(recs, emb, multimask_output=True, return_masks=False), y_one_hot)
    loss[0].backward()
    ref = dict(osam.named_parameters())
    r_enc, bad_enc = _compare_grads(sam.encoder_grads(), ref, 1.5e-1, min_cos=0.99)
    r_dec, bad_dec = _compare_grads(sam.decoder_grads(), ref, 1.5e-1, min_cos=0.99)
    print(f"training step: loss {float(loss[0]):.4f} (oracle {float(oloss[0]):.4f}); encoder gradients median rel-L2 {np.median(list(r_enc.values())):.2e} "
          f"max {max(r_enc.values()):.2e}; decoder gradients median {np.median(list(r_dec.values())):.2e} max {max(r_dec.values()):.2e}")
    assert abs(float(loss[0]) - float(oloss[0])) < 2e-2
    assert not bad_enc and not bad_dec, (bad_enc, bad_dec)


def test_optimizer_steps_reduce_the_loss_and_match_torch_adamw():
    """AdamW on the device (csrc/train_opt.cu): (1) one step from zero moments equals torch.optim.AdamW applied to the same gradients,
    tensor by tensor (fp32 masters, incl. the packed conv-transpose / table layouts folded back); (2) repeated steps on a fixed batch
    reduce the loss, i.e. forward, backward, update and operand refresh work together."""
    from micro_sam_b200 import training
    from micro_sam_b200.sample_data import lm_tile
    _, sam = _small_models()
    sam.train()
    m = training.TrainableSAM(sam)
    B, n_obj, H, W = 2, 4, 128, 128
    imgs = [torch.from_numpy(np.repeat(lm_tile((H, W), 12, seed=40 + b, dtype="uint8")[None], 3, 0).astype("float32")) for b in range(B)]
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    cen = [(30 + 22 * k, 28 + 24 * k, 9 + 2 * k) for k in range(n_obj)]
    y_one_hot = [torch.stack([(((yy - cy) ** 2 + (xx - cx) ** 2) < r * r).float()[None] for cy, cx, r in cen]) for _ in range(B)]
    boxes = torch.tensor([[cx - r, cy - r, cx + r, cy + r] for cy, cx, r in cen], dtype=torch.float32) * (1024.0 / W)

    def step():
        sam.zero_decoder_grads()
        emb, recs = m.image_embeddings_oft([{"image": im.clone(), "original_size": (H, W), "boxes": boxes.clone()} for im in imgs])
        loss = training.compute_loss(m(recs, emb, multimask_output=True, return_masks=False), y_one_hot)
        loss[0].backward()
        return float(loss[0])

    kw = dict(lr=2e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    l0 = step()
    grads = dict(sam.encoder_grads())
    grads.update(sam.decoder_grads())
    before = {k: v.to(DEV) for k, v in sam.state_dict().items() if k in grads}
    sam.optimizer_step(**kw)
    after = sam.trained_state_dict()
    worst, per = 0.0, {}
    for k, g in grads.items():
        p = torch.nn.Parameter(before[k].clone())
        p.grad = g.reshape(p.shape).clone()
        torch.optim.AdamW([p], **kw).step()
        d_ref, d_got = (p.detach() - before[k]).double().cpu(), (after[k].to(torch.float64) - before[k].double().cpu())
        if float(d_ref.norm()) > 0:
            # tensors without gradient (unused mask token 0, unused point embeddings) only see the weight decay: an update of 2e-6 |w|,
            # i.e. ~30 fp32 ulps of w -- compare against a floor of 1e-4 |w| so that its rounding does not count
            per[k] = float((d_got - d_ref).norm() / max(float(d_ref.norm()), 1e-4 * float(before[k].double().norm())))
            worst = max(worst, per[k])
    print("AdamW worst tensors: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:8]))
    losses = [l0] + [0.0] * 6
    for i in range(1, 7):
        losses[i] = step()
        sam.optimizer_step(**kw)
    print(f"AdamW: update vs torch.optim.AdamW worst rel-L2 {worst:.2e} over {len(grads)} tensors; losses " + " ".join(f"{v:.4f}" for v in losses))
    assert worst < 1e-3
    assert losses[-1] < losses[0] - 0.02, losses
    # the inference engine can be rebuilt from the trained weights
    sam.load_state_dict(sam.trained_state_dict())
