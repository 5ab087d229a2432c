"""GPU tests of the semantic fine-tuning loss (csrc/semantic_loss.cu, training.compute_semantic_loss / CustomDiceLoss) against
float64 autograd through the oracle's postprocess_masks + softmax Dice + cross entropy (oracle/semantic_ref.py).

Bounds: the loss within 1e-6 relative and d low_res within 1e-5 rel-L2 of the float64 reference.  The device evaluates the
interpolation and the softmax in fp32 and sums in fp64; DESIGN.md section 5 lists the values measured on an H100."""
import math

import pytest
import torch

from oracle import semantic_ref

pytestmark = pytest.mark.gpu

LOSS_RTOL = 1e-6
GRAD_RL2 = 1e-5


def _case(B, C, H, W, seed, ignore=True):
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(B, C, 256, 256, generator=g) * 4
    # blocky labels (classes in regions, as a segmentation has them) with an ignored stripe
    coarse = torch.randint(0, C, (B, 1, max(1, H // 16), max(1, W // 16)), generator=g).float()
    lab = torch.nn.functional.interpolate(coarse, (H, W), mode="nearest")[:, 0].long()
    if ignore:
        lab[:, H // 3: H // 3 + 3, :] = -100
    return low.cuda(), lab.cuda()


def _reference(low, lab, input_size, original_size, C, dice_weight=None):
    low64 = low.double().detach().requires_grad_(True)
    loss = semantic_ref.semantic_loss_from_low_res(low64, lab, input_size, original_size, C, dice_weight)
    loss.backward()
    return loss.detach(), low64.grad


def _rel_l2(a, b):
    return float((a.double() - b).norm() / b.norm().clamp(min=1e-300))


CASES = [   # (B, C, original, input_size or None = ResizeLongestSide)
    (1, 2, (256, 256), None),
    (2, 3, (512, 512), None),
    (1, 15, (700, 500), None),
    (2, 3, (700, 500), None),
    (1, 3, (1024, 1024), None),
    (2, 15, (1024, 1024), None),
    (1, 2, (512, 512), (1024, 800)),     # non-square input_size of a square original
    (2, 3, (256, 256), (600, 1024)),
    (1, 3, (1500, 2000), None),          # original larger than the model input
]


@pytest.mark.parametrize("B,C,orig,insz", CASES)
@pytest.mark.parametrize("dice_weight", [None, 0.3])
def test_loss_and_adjoint_match_float64_autograd(B, C, orig, insz, dice_weight):
    from micro_sam_b200 import training
    from micro_sam_b200.sam import get_preprocess_shape
    H, W = orig
    low, lab = _case(B, C, H, W, seed=B * 100 + C + H)
    input_size = insz if insz is not None else get_preprocess_shape(H, W, 1024)
    ref_loss, ref_grad = _reference(low, lab, input_size, orig, C, dice_weight)
    x = low.clone().requires_grad_(True)
    loss = training.compute_semantic_loss(x, lab, C, dice_weight, input_size=insz)
    loss.backward()
    rel = abs(float(loss.detach()) - float(ref_loss)) / abs(float(ref_loss))
    rl2 = _rel_l2(x.grad, ref_grad)
    print(f"B={B} C={C} orig={orig} input={input_size} w={dice_weight}: loss rel {rel:.2e}, grad rel-L2 {rl2:.2e}")
    assert loss.dtype == torch.float32
    assert rel <= LOSS_RTOL, rel
    assert rl2 <= GRAD_RL2, rl2


def test_dice_alone_and_batched_outputs():
    from micro_sam_b200 import training
    B, C, H, W = 2, 3, 700, 500
    low, lab = _case(B, C, H, W, seed=7)
    input_size = (1024, 731)
    masks = semantic_ref.postprocess_masks(low.double(), input_size, (H, W))
    want = semantic_ref.custom_dice_loss(masks, lab[:, None], C)
    outs = [{"low_res_masks": low[b:b + 1], "input_size": input_size, "original_size": (H, W)} for b in range(B)]
    got = training.CustomDiceLoss(C)(outs, lab[:, None].float())
    assert abs(float(got) - float(want)) <= LOSS_RTOL * abs(float(want))
    full = training.compute_semantic_loss(outs, lab[:, None].to(torch.int32), C)
    assert abs(float(full) - float(semantic_ref.semantic_loss(masks, lab[:, None], C))) <= LOSS_RTOL * float(full)


def test_repeats_are_bit_identical():
    from micro_sam_b200 import training
    low, lab = _case(2, 15, 1024, 1024, seed=3)
    res = []
    for _ in range(3):
        x = low.clone().requires_grad_(True)
        loss = training.compute_semantic_loss(x, lab, 15, 0.3)
        loss.backward()
        res.append((training.semantic_loss_stats(low, lab, 15).detach().clone(), loss.detach().clone(), x.grad.clone()))
    for r in res[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, res[0]))


def test_ignore_index_and_out_of_range_labels():
    from micro_sam_b200 import training
    C, H, W = 3, 300, 200
    low, lab = _case(1, C, H, W, seed=11, ignore=False)
    lab[0, :50] = -100
    st = training.semantic_loss_stats(low, lab, C)
    n_valid = int((lab != -100).sum())
    assert int(st[3 * C + 1]) == n_valid and int(st[3 * C + 2]) == 0
    assert int(st[2::3][:C].sum()) == n_valid           # -100 is in no class
    ref, _ = _reference(low, lab, (1024, 683), (H, W), C)
    assert abs(float(training.compute_semantic_loss(low, lab, C)) - float(ref)) <= LOSS_RTOL * float(ref)
    for bad in (C, -1, 255):
        b = lab.clone()
        b[0, 100, 7] = bad
        with pytest.raises(ValueError, match="outside"):
            training.compute_semantic_loss(low, b, C)
        with pytest.raises(ValueError, match="outside"):
            training.compute_semantic_loss(low, b.to(torch.int32), C)
    b = lab.clone()
    b[0, 0, 0] = 2 ** 40                                  # int64 label beyond int32
    with pytest.raises(ValueError, match="outside"):
        training.compute_semantic_loss(low, b, C)


def test_kernel_refusals():
    from micro_sam_b200 import _lib
    L = _lib.lib()
    low = torch.zeros(1, 3, 256, 256, device="cuda")
    lab = torch.zeros(1, 64, 64, device="cuda", dtype=torch.int32)
    st = torch.zeros(12, device="cuda", dtype=torch.float64)
    n = int(L.msam_semantic_loss_workspace(1, 3, 1024, 1024, 64, 64, 1))
    ws = torch.empty(n, device="cuda", dtype=torch.uint8)
    d = torch.empty_like(low)
    p, s = _lib.ptr, _lib.cur_stream()
    ok = (p(low), p(lab), 0, 1, 3, 1024, 1024, 64, 64, p(ws), n, p(st), s)
    assert L.msam_semantic_loss_stats(*ok) == 0
    for i, v in [(0, None), (1, None), (11, None), (9, None), (4, 16), (4, 0), (3, 0), (2, 2), (5, 2000), (10, 256)]:
        args = list(ok)
        args[i] = v
        assert L.msam_semantic_loss_stats(*args) != 0, (i, v)
    assert L.msam_semantic_loss_workspace(1, 16, 1024, 1024, 64, 64, 0) < 0
    okb = (p(low), p(lab), 0, p(st), 1, 3, 1024, 1024, 64, 64, p(ws), n, p(d), s)
    assert L.msam_semantic_loss_backward(*okb) == 0
    for i, v in [(3, None), (12, None), (5, 16), (11, n - 1)]:
        args = list(okb)
        args[i] = v
        assert L.msam_semantic_loss_backward(*args) != 0, (i, v)
    torch.cuda.synchronize()
    assert math.isfinite(float(st[0]))


@pytest.mark.parametrize("clamped", [False, True])
def test_absent_class(clamped):
    """A class no pixel carries.  With `clamped` its logits are so low that sum p^2 + sum t^2 < 1e-7, so Dice takes the clamp
    branch (the term is 1 and passes no gradient)."""
    from micro_sam_b200 import training
    B, C, H, W = 2, 4, 512, 384
    low, lab = _case(B, C, H, W, seed=21)
    lab[lab == C - 1] = 0
    if clamped:
        low[:, C - 1] = -40.0
    input_size = (1024, 768)
    st = training.semantic_loss_stats(low, lab, C)
    assert float(st[3 * (C - 1) + 2]) == 0.0
    assert (float(st[3 * (C - 1) + 1]) < 1e-7) == clamped
    for w in (None, 0.3):
        ref_loss, ref_grad = _reference(low, lab, input_size, (H, W), C, w)
        x = low.clone().requires_grad_(True)
        loss = training.compute_semantic_loss(x, lab, C, w)
        loss.backward()
        rel = abs(float(loss.detach()) - float(ref_loss)) / abs(float(ref_loss))
        rl2 = _rel_l2(x.grad, ref_grad)
        print(f"absent class, clamped={clamped} w={w}: loss rel {rel:.2e}, grad rel-L2 {rl2:.2e}")
        assert rel <= LOSS_RTOL and rl2 <= GRAD_RL2, (rel, rl2)


def test_semantic_checkpoint_is_refused_with_the_limit():
    from micro_sam_b200 import util
    from oracle import sam_ref
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    sd["mask_decoder.mask_tokens.weight"] = torch.zeros(6, 256)     # num_multimask_outputs = 5
    with pytest.raises(NotImplementedError, match="6 mask tokens"):
        util.get_sam_model("vit_test", device="cuda", state_dict=sd)
