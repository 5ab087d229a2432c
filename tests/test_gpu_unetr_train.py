"""Training of the UNETR (AIS) decoder on the GPU: each csrc/ais_train.cu op against float64, the whole decoder backward against
the float64 training-mode restatement (tests/unetr_train_ref.py), determinism, the AdamW step, a short training run with export
and reload through get_predictor_and_decoder, and the argument checks."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from micro_sam_b200 import _lib, instance_segmentation as iseg, training, unetr, util
from oracle import sam_ref, unetr_ref
from tests import unetr_train_ref as ref
from tests import unetr_train_noise_floor as nf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REDUCED = dict(emb=64, feats=(128, 64, 64, 64), deconv=(64, 64, 64, 64), head_in=64)
WIDE_EMB = dict(REDUCED, emb=256)   # takes SAM's 256-channel embeddings


def _bf(t):
    return t.to(DEV, torch.bfloat16).contiguous()


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


@pytest.mark.parametrize("C0,C1,cout,H,W,B,ks", [(64, 0, 64, 16, 64, 1, 3), (64, 64, 64, 7, 50, 1, 3), (128, 64, 128, 9, 70, 2, 3),
                                                 (192, 64, 128, 32, 96, 2, 3), (256, 0, 512, 8, 8, 1, 3), (64, 0, 256, 12, 20, 2, 1)])
def test_wgrad_against_float64(C0, C1, cout, H, W, B, ks):
    g = torch.Generator().manual_seed(C0 + C1 + cout + H)
    x = torch.randn(B, C0 + C1, H, W, generator=g).to(torch.bfloat16).double()
    dy = torch.randn(B, cout, H, W, generator=g).to(torch.bfloat16).double()
    w = torch.zeros(cout, C0 + C1, ks, ks, dtype=torch.float64, requires_grad=True)
    (F.conv2d(x, w, padding=ks // 2) * dy).sum().backward()
    want = w.grad.permute(0, 2, 3, 1).reshape(cout, -1)
    xh = _bf(_nhwc(x))
    x0, x1 = xh[..., :C0].contiguous(), (xh[..., C0:].contiguous() if C1 else None)
    L = _lib.lib()
    ws = torch.empty(int(L.msam_ais_wgrad_workspace(cout, C0, C1, B, H, W, ks)), device=DEV, dtype=torch.uint8)
    dw = torch.empty(cout, ks * ks * (C0 + C1), device=DEV)
    _lib.check(L.msam_op_ais_wgrad(_lib.ptr(_bf(_nhwc(dy))), cout, _lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(ws),
                                   ws.numel(), _lib.ptr(dw), _lib.cur_stream()))
    assert ref.rel_l2(dw, want) < 1e-5
    dw2 = torch.empty_like(dw)
    _lib.check(L.msam_op_ais_wgrad(_lib.ptr(_bf(_nhwc(dy))), cout, _lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(ws),
                                   ws.numel(), _lib.ptr(dw2), _lib.cur_stream()))
    assert torch.equal(dw, dw2)


def _dec(sd):
    return unetr.TrainableUNETRDecoder(sd, device=DEV)


def wgrad_plan(cout, cin, B, H, W, ks):
    """(splits, k-blocks per split, k-blocks in all) of msam_op_ais_wgrad (wgrad_plan in csrc/ais_train.cu)"""
    mh, nb = (2 if cout % 128 == 0 else 1), (2 if cin % 128 == 0 else 1)
    kb_total = B * ((W + 63) // 64) * ((H + 1) // 2)
    ctas = (cout // (64 * mh)) * ks * ks * (cin // (64 * nb))
    splits = max(min(-(-264 // ctas), -(-kb_total // 8)), 1)
    per = -(-kb_total // splits)
    return -(-kb_total // per), per, kb_total


def production_wgrad_cases():
    """every (Cout, C0, C1, B, H, W, ks) the production decoder's backward passes to _wgrad, both samplers, B = 1 and 2, on a
    64 x 64 embedding (1024^2 maps)"""
    cases = set()
    for transposed in (False, True):
        d = _dec(unetr.default_decoder_state(transposed=transposed))
        real = d._wgrad

        def record(dy, x0, x1, ks):
            cases.add((dy.shape[3], x0.shape[3], 0 if x1 is None else x1.shape[3], *dy.shape[:3], ks))
            return real(dy, x0, x1, ks)

        d._wgrad = record
        for B in (1, 2):
            d.forward(torch.zeros(B, 256, 64, 64, device=DEV))
            d.backward(torch.zeros(B, 3, 1024, 1024, device=DEV))
        del d
    return sorted(cases)


def test_wgrad_at_production_shapes():
    """the weight gradient of every convolution the production decoder trains, at its own shape, against a float64 conv2d
    weight gradient on the GPU: long k-loops per split, short last splits, and single-split grids.  The fp32 accumulation
    error grows with the k-blocks per split: 1e-6 .. 1e-5 up to 70 of them, and about 1.5e-7 per k-block beyond (8.1e-5 at
    547 k-blocks of 128 pixels, the head block's 3x3 convolutions at B = 2, H100); bound max(1e-5, 3e-7 per k-block)."""
    L = _lib.lib()
    g = torch.Generator(device=DEV).manual_seed(17)
    bad = []
    for cout, C0, C1, B, H, W, ks in production_wgrad_cases():
        splits, per, kb_total = wgrad_plan(cout, C0 + C1, B, H, W, ks)
        nbytes = int(L.msam_ais_wgrad_workspace(cout, C0, C1, B, H, W, ks))
        assert nbytes == splits * cout * ks * ks * (C0 + C1) * 4
        x = torch.randn(B, H, W, C0 + C1, generator=g, device=DEV).to(torch.bfloat16)
        dy = torch.randn(B, H, W, cout, generator=g, device=DEV).to(torch.bfloat16)
        x0, x1 = x[..., :C0].contiguous(), (x[..., C0:].contiguous() if C1 else None)
        ws = torch.empty(nbytes, device=DEV, dtype=torch.uint8)
        dw = torch.empty(cout, ks * ks * (C0 + C1), device=DEV)
        _lib.check(L.msam_op_ais_wgrad(_lib.ptr(dy), cout, _lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(ws), ws.numel(),
                                       _lib.ptr(dw), _lib.cur_stream()))
        del x0, x1, ws
        want = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2).double(), (cout, C0 + C1, ks, ks), dy.permute(0, 3, 1, 2).double(),
                                           padding=ks // 2).permute(0, 2, 3, 1).reshape(cout, -1)
        err = ref.rel_l2(dw, want)
        print(f"wgrad Cout={cout} C0={C0} C1={C1} B={B} {H}x{W} ks={ks}: splits={splits} per={per} "
              f"last={kb_total - (splits - 1) * per} rel-L2 {err:.2e}")
        if not err < max(1e-5, 3e-7 * per):
            bad.append(((cout, C0, C1, B, H, W, ks), err))
        del x, dy, dw, want
    assert not bad, bad




def test_dgrad_through_rotated_weights():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(64, 128, 3, 3, generator=g) * 0.05
    dy = torch.randn(2, 64, 9, 70, generator=g).to(torch.bfloat16).double()
    x = torch.zeros(2, 128, 9, 70, dtype=torch.float64, requires_grad=True)
    (F.conv2d(x, w.double(), padding=1) * dy).sum().backward()
    d = _dec(unetr_ref.seeded_state(seed=1, **REDUCED))
    d.masters["decoder.blocks.0.block.1.weight"].copy_(w.to(DEV))
    d.refresh()
    got = d._conv(_bf(_nhwc(dy)), None, d.ops["decoder.blocks.0.block.1.weight"][1], None, 3, False)
    assert ref.rel_l2(got.permute(0, 3, 1, 2).float(), x.grad) < 8e-3


def _check_norm(per_image, affine, B, C, H, W, g, dev="cpu"):
    """training-mode norm forward (with BatchNorm's running statistics) and backward against float64 autograd on `dev`"""
    x = torch.relu(torch.randn(B, C, H, W, generator=g, device=dev) + 0.3).to(torch.bfloat16).double().requires_grad_(True)
    gam = (1 + 0.2 * torch.randn(C, generator=g, device=dev)).double().requires_grad_(True) if affine else None
    bet = (0.2 * torch.randn(C, generator=g, device=dev)).double().requires_grad_(True) if affine else None
    rm, rv = torch.zeros(C, dtype=torch.float64, device=dev), torch.ones(C, dtype=torch.float64, device=dev)
    if per_image:
        y = F.instance_norm(x, weight=gam, bias=bet, eps=1e-5)
    else:
        y = torch.relu(F.batch_norm(x, rm, rv, gam, bet, training=True, momentum=0.1, eps=1e-5))
    dy = torch.randn(B, C, H, W, generator=g, device=dev).to(torch.bfloat16).double()
    (y * dy).sum().backward()
    d = _dec(unetr_ref.seeded_state(seed=1, **REDUCED))
    xd = _bf(_nhwc(x.detach()))
    gd = None if gam is None else gam.detach().float().to(DEV)
    bd = None if bet is None else bet.detach().float().to(DEV)
    run = None if per_image else (torch.zeros(C, device=DEV), torch.ones(C, device=DEV))
    out, mean, rstd = d._norm_fwd(xd, per_image, gd, bd, relu=not per_image, run=run)
    assert ref.rel_l2(out.permute(0, 3, 1, 2).float(), y.detach()) < 5e-3
    if run is not None:
        assert ref.rel_l2(run[0], rm) < 1e-5 and ref.rel_l2(run[1], rv) < 1e-5
    dyd = _bf(_nhwc(dy)) if per_image else _nhwc(dy).float().to(DEV).contiguous()
    dx, dg, db = d._norm_bwd(xd, dyd, 0, C, mean, rstd, per_image, gd, relu_out=None if per_image else out, out_mode=1, dgb=True)
    assert ref.rel_l2(dx.permute(0, 3, 1, 2), x.grad) < 1e-2
    if affine:
        assert ref.rel_l2(dg, gam.grad) < 1e-3 and ref.rel_l2(db, bet.grad) < 1e-3


@pytest.mark.parametrize("per_image,affine", [(True, False), (True, True), (False, True)])
def test_norm_forward_backward_against_float64(per_image, affine):
    _check_norm(per_image, affine, 2, 64, 33, 40, torch.Generator().manual_seed(4))


@pytest.mark.parametrize("per_image", [True, False])
def test_norm_forward_backward_at_1024(per_image):
    """the head block's InstanceNorm and deconv4's BatchNorm at their production size: 1024 chunks of NT_CHUNK pixels per
    image, and BatchNorm's statistics over two images"""
    _check_norm(per_image, True, 2, 64, 1024, 1024, torch.Generator(device=DEV).manual_seed(4), dev=DEV)


def test_upsample_space_to_depth_head_resize_and_loss_backward():
    g = torch.Generator().manual_seed(5)
    L = _lib.lib()
    B, C, H, W = 2, 64, 9, 14
    dy = torch.randn(B, C, 2 * H, 2 * W, generator=g).to(torch.bfloat16).double()
    x = torch.zeros(B, C, H, W, dtype=torch.float64, requires_grad=True)
    (F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False) * dy).sum().backward()
    dx = torch.empty(B, H, W, C, device=DEV, dtype=torch.bfloat16)
    _lib.check(L.msam_op_ais_upsample2_backward(_lib.ptr(_bf(_nhwc(dy))), B, H, W, C, _lib.ptr(dx), _lib.cur_stream()))
    assert ref.rel_l2(dx.permute(0, 3, 1, 2).float(), x.grad) < 5e-3
    s2d = torch.empty(B, H, W, 4 * C, device=DEV, dtype=torch.bfloat16)
    _lib.check(L.msam_op_ais_space_to_depth(_lib.ptr(_bf(_nhwc(dy))), B, H, W, C, _lib.ptr(s2d), _lib.cur_stream()))
    want = _nhwc(dy).reshape(B, H, 2, W, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, 4 * C)
    assert torch.equal(s2d.cpu().double(), want)
    # head: out_conv + sigmoid
    h = torch.relu(torch.randn(B, C, 16, 16, generator=g)).to(torch.bfloat16).double().requires_grad_(True)
    w = (torch.randn(3, C, generator=g) * 0.1).double().requires_grad_(True)
    b = torch.randn(3, generator=g).double().requires_grad_(True)
    s = torch.sigmoid(F.conv2d(h, w[:, :, None, None], b))
    dm = torch.randn(s.shape, generator=g).double()
    (s * dm).sum().backward()
    maps = torch.empty(B, 3, 16, 16, device=DEV)
    hd = _bf(_nhwc(h.detach()))
    wd, bdv = w.detach().float().to(DEV).contiguous(), b.detach().float().to(DEV)
    _lib.check(L.msam_op_ais_head(_lib.ptr(hd), B, 256, C, _lib.ptr(wd), _lib.ptr(bdv), _lib.ptr(maps), _lib.cur_stream()))
    ws = torch.empty(int(L.msam_ais_head_backward_workspace(B, 256, C)), device=DEV, dtype=torch.uint8)
    dh, dw, db = torch.empty_like(hd), torch.empty(3, C, device=DEV), torch.empty(3, device=DEV)
    _lib.check(L.msam_op_ais_head_backward(_lib.ptr(hd), B, 256, C, _lib.ptr(wd), _lib.ptr(maps), _lib.ptr(dm.float().to(DEV)),
                                           _lib.ptr(ws), ws.numel(), _lib.ptr(dh), _lib.ptr(dw), _lib.ptr(db), _lib.cur_stream()))
    assert ref.rel_l2(dw, w.grad) < 1e-4 and ref.rel_l2(db, b.grad) < 1e-4
    assert ref.rel_l2(dh.permute(0, 3, 1, 2).float(), h.grad * (h.detach() > 0)) < 5e-3
    # crop + resize
    for (ih, iw), (oh, ow) in [((64, 48), (100, 75)), ((64, 64), (20, 20)), ((40, 64), (40, 64))]:
        m = torch.zeros(2, 3, 64, 64, dtype=torch.float64, requires_grad=True)
        do = torch.randn(2, 3, oh, ow, generator=g).double()
        (ref.crop_resize(m, (ih, iw), (oh, ow)) * do).sum().backward()
        tmp = torch.empty(6 * oh * iw, device=DEV)
        dm2 = torch.empty(2, 3, 64, 64, device=DEV)
        _lib.check(L.msam_op_ais_resize_backward(_lib.ptr(do.float().to(DEV)), 6, 64, 64, ih, iw, oh, ow, _lib.ptr(tmp), _lib.ptr(dm2),
                                                 _lib.cur_stream()))
        assert ref.rel_l2(dm2, m.grad) < 1e-5, (ih, iw, oh, ow)
    # loss
    for mask in (True, False):
        xl = torch.rand(2, 3, 70, 90, generator=g).double().requires_grad_(True)
        yl = torch.rand(2, 3, 70, 90, generator=g).double()
        yl[:, 0] = (yl[:, 0] > 0.4).double()
        want = ref.dice_based_distance_loss(xl, yl, mask)
        want.backward()
        xg = xl.detach().float().to(DEV).requires_grad_(True)
        got = training.DiceBasedDistanceLoss(mask)(xg, yl.float().to(DEV))
        got.backward()
        assert abs(float(got) - float(want)) < 1e-5
        assert ref.rel_l2(xg.grad, xl.grad) < 1e-4


def test_head_resize_and_loss_backward_at_1024():
    """out_conv + sigmoid backward, the crop + resize backward and the distance loss at the decoder's output size, B = 2: 2048
    chunks of NT_CHUNK pixels in the head's weight gradient, 256 chunks of DL_CHUNK per image in the loss statistics"""
    g = torch.Generator(device=DEV).manual_seed(6)
    L = _lib.lib()
    B, C, HW = 2, 64, 1024 * 1024
    h = torch.relu(torch.randn(B, C, 1024, 1024, generator=g, device=DEV)).to(torch.bfloat16).double().requires_grad_(True)
    w = (torch.randn(3, C, generator=g, device=DEV) * 0.1).double().requires_grad_(True)
    b = torch.randn(3, generator=g, device=DEV).double().requires_grad_(True)
    s = torch.sigmoid(F.conv2d(h, w[:, :, None, None], b))
    dm = torch.randn(s.shape, generator=g, device=DEV).double()
    (s * dm).sum().backward()
    hd = _bf(_nhwc(h.detach()))
    wd, bdv = w.detach().float().contiguous(), b.detach().float()
    maps = torch.empty(B, 3, 1024, 1024, device=DEV)
    _lib.check(L.msam_op_ais_head(_lib.ptr(hd), B, HW, C, _lib.ptr(wd), _lib.ptr(bdv), _lib.ptr(maps), _lib.cur_stream()))
    assert ref.rel_l2(maps, s.detach()) < 1e-5
    ws = torch.empty(int(L.msam_ais_head_backward_workspace(B, HW, C)), device=DEV, dtype=torch.uint8)
    dh, dw, db = torch.empty_like(hd), torch.empty(3, C, device=DEV), torch.empty(3, device=DEV)
    _lib.check(L.msam_op_ais_head_backward(_lib.ptr(hd), B, HW, C, _lib.ptr(wd), _lib.ptr(maps), _lib.ptr(dm.float()), _lib.ptr(ws),
                                           ws.numel(), _lib.ptr(dh), _lib.ptr(dw), _lib.ptr(db), _lib.cur_stream()))
    assert ref.rel_l2(dw, w.grad) < 1e-4 and ref.rel_l2(db, b.grad) < 1e-4
    assert ref.rel_l2(dh.permute(0, 3, 1, 2), h.grad * (h.detach() > 0)) < 5e-3
    del h, s, hd, dh, ws
    # crop + resize to a few original sizes, as postprocess_masks after the decoder
    for (ih, iw), (oh, ow) in [((1024, 768), (1536, 1152)), ((768, 1024), (600, 800)), ((1024, 1024), (1024, 1024))]:
        m = torch.zeros(B, 3, 1024, 1024, dtype=torch.float64, device=DEV, requires_grad=True)
        do = torch.randn(B, 3, oh, ow, generator=g, device=DEV).double()
        (ref.crop_resize(m, (ih, iw), (oh, ow)) * do).sum().backward()
        tmp = torch.empty(B * 3 * oh * iw, device=DEV)
        dm2 = torch.empty(B, 3, 1024, 1024, device=DEV)
        _lib.check(L.msam_op_ais_resize_backward(_lib.ptr(do.float()), B * 3, 1024, 1024, ih, iw, oh, ow, _lib.ptr(tmp), _lib.ptr(dm2),
                                                 _lib.cur_stream()))
        assert ref.rel_l2(dm2, m.grad) < 1e-4, (ih, iw, oh, ow)   # fp32 interpolation weights: 4.6e-5 at 1024 -> 1536
    # distance-based Dice loss: statistics and backward
    for mask in (True, False):
        xl = torch.rand(B, 3, 1024, 1024, generator=g, device=DEV).double().requires_grad_(True)
        yl = torch.rand(B, 3, 1024, 1024, generator=g, device=DEV).double()
        yl[:, 0] = (yl[:, 0] > 0.4).double()
        want = ref.dice_based_distance_loss(xl, yl, mask)
        want.backward()
        xg = xl.detach().float().requires_grad_(True)
        got = training.DiceBasedDistanceLoss(mask)(xg, yl.float())
        got.backward()
        assert abs(float(got) - float(want)) < 1e-5
        assert ref.rel_l2(xg.grad, xl.grad) < 1e-4


@pytest.mark.parametrize("plan", sorted(nf.CASES))
def test_decoder_backward_against_float64(plan):
    """every parameter gradient and d embedding within twice the bf16 noise floor of tests/unetr_train_noise_floor.py, on its
    case: the float64 reference is fed the same bf16-rounded weights and embedding as the device"""
    sd, z, dm = nf.case_inputs(plan)
    want, maps = nf.grads(sd, z, dm, torch.float64, False)
    floor = nf.floors(plan)
    d = _dec(sd)
    got_maps = d.forward(z.to(DEV))
    assert ref.rel_l2(got_maps, maps) < 2e-2
    dz = d.backward(dm.to(DEV))
    got = dict(d.grads, d_embedding=dz)
    # a bias in front of a training-mode BatchNorm or an InstanceNorm has gradient 0 (the norm removes a per-channel constant):
    # its value on the device is rounding noise, bounded against the gradient of the norm's own beta / the weight beside it
    # (bound: twice the float32 emulation's own value of that noise)
    emu, _ = nf.grads(sd, z, dm, torch.float32, True)
    for k in nf.zero_grad_keys(got):
        if k.endswith(".block.1.block.bias"):   # the upsamplers' biases are not bounded: see zero_grad_keys
            beta = float(want[k.replace(".1.block.bias", ".2.bias")].norm())
            assert float(got[k].norm()) < 2 * float(emu[k].norm()) + 1e-3 * beta, k
    ratio = {k: ref.rel_l2(got[k], want[k]) / floor[k] for k in floor}
    print(plan, "worst error / floor", sorted(ratio.items(), key=lambda kv: -kv[1])[:4])
    bad = {k: v for k, v in ratio.items() if not v < 2.0}
    assert not bad, bad
    st = d.state_dict()
    lv = ref.leaves(sd)
    ref.forward_maps(lv, z.double(), train=True)
    for k in lv:
        if k.endswith(("running_mean", "running_var")):
            assert ref.rel_l2(st[k], lv[k]) < 1e-3, k
        if k.endswith("num_batches_tracked"):
            assert int(st[k]) == 1


def test_determinism_and_adamw():
    sd = unetr_ref.seeded_state(seed=11, **REDUCED)
    z = torch.randn(2, 64, 4, 4, generator=torch.Generator().manual_seed(12)).to(DEV)
    dm = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(13)).to(DEV)
    runs = []
    for _ in range(2):
        d = _dec(sd)
        d.forward(z)
        dz = d.backward(dm)
        g0 = {k: v.clone() for k, v in d.grads.items()}
        d.optimizer_step(lr=1e-3, weight_decay=0.01)
        runs.append((dz, g0, {k: v.clone() for k, v in d.masters.items()}, d))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(runs[0][1][k], runs[1][1][k]) for k in runs[0][1])
    assert all(torch.equal(runs[0][2][k], runs[1][2][k]) for k in runs[0][2])
    # one AdamW step against torch.optim.AdamW in float64 from the same gradients
    params = {k: torch.nn.Parameter(v.detach().double().cpu().clone()) for k, v in d.masters.items()}
    d0 = _dec(sd)
    for k, p in params.items():
        p.data.copy_(d0.masters[k].double().cpu())
        p.grad = runs[0][1][k].double().cpu()
    opt = torch.optim.AdamW(list(params.values()), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    opt.step()
    for k, p in params.items():
        assert ref.rel_l2(runs[0][2][k] - d0.masters[k], p.data - d0.masters[k].double().cpu()) < 1e-4, k
    assert all(s == 1 for s in runs[0][3].steps.values())


def _disks(B, H, W, seed):
    """touching disks: images (B, 3, H, W) in [0, 255] and targets (foreground, center distances, boundary distances)"""
    rng = np.random.default_rng(seed)
    imgs, tgts = [], []
    yy, xx = np.mgrid[:H, :W]
    for _ in range(B):
        fg = np.zeros((H, W), np.float32)
        cd = np.ones((H, W), np.float32)
        bd = np.ones((H, W), np.float32)
        for _ in range(6):
            cy, cx, r = rng.uniform(20, H - 20), rng.uniform(20, W - 20), rng.uniform(12, 24)
            dist = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
            inside = dist < r
            fg[inside] = 1
            cd[inside] = np.minimum(cd[inside], (dist / r)[inside])
            bd[inside] = np.minimum(bd[inside], (1 - dist / r)[inside])
        img = np.stack([fg * 180 + rng.normal(30, 10, (H, W))] * 3).clip(0, 255).astype(np.float32)
        imgs.append(img)
        tgts.append(np.stack([fg, cd * fg, bd * fg]))
    return torch.from_numpy(np.stack(imgs)), torch.from_numpy(np.stack(tgts).astype(np.float32))


def test_train_export_and_reload(tmp_path):
    sam_sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    pred = util.get_sam_model("vit_test", device=DEV, state_dict=sam_sd, max_batch=2, max_prompts=16)
    net = training.get_unetr(pred.model, unetr_ref.seeded_state(seed=21, **WIDE_EMB))
    with pytest.raises(NotImplementedError):
        training.get_unetr(pred.model, out_channels=2)
    enc = {k: v.clone() for k, v in pred.model.state_dict().items()}
    x, y = _disks(2, 256, 256, 1)
    emb, _ = net.embed(x)
    losses = [float(training.instance_train_iteration(net, x, y, lr=1e-3)) for _ in range(20)]
    print("losses", losses[0], losses[-1])
    assert losses[-1] < losses[0]
    assert all(torch.equal(enc[k], v) for k, v in pred.model.state_dict().items())
    assert set(net.decoder.steps.values()) == {20}
    path = tmp_path / "trained.pt"
    training.export_instance_segmentation_model(net, path)
    p2, dec = iseg.get_predictor_and_decoder("vit_test", str(path), device=DEV)
    # the reloaded inference decoder (BatchNorm folded) against the float64 eval-mode decoder of the exported state
    want = ref.forward_maps(ref.leaves(net.decoder_state_dict()), emb.cpu(), train=False)
    got = dec.forward_maps(emb)
    assert ref.rel_l2(got, want.detach()) < 2e-2
    seg = iseg.InstanceSegmentationWithDecoder(p2, dec)
    seg.initialize(x[0, 0].numpy().astype(np.uint8))
    labels = seg.generate()
    assert labels.shape == (256, 256)


def _labelled_disks(B, H, W, seed):
    """label images (B, 1, H, W) of separate disks and their UNETR targets (foreground, center and boundary distances)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W]
    labs, tgts = np.zeros((B, 1, H, W), np.float32), np.zeros((B, 3, H, W), np.float32)
    for b in range(B):
        for k in range(16):
            cy, cx, r = 16 + 32 * (k // 4) + rng.integers(-3, 4), 16 + 32 * (k % 4) + rng.integers(-3, 4), 8 + k % 5
            dist = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
            inside = dist < r
            labs[b, 0][inside] = k + 1
            tgts[b, 0][inside], tgts[b, 1][inside], tgts[b, 2][inside] = 1, (dist / r)[inside], (1 - dist / r)[inside]
    img = np.repeat((labs > 0) * 170.0 + rng.normal(40, 8, labs.shape), 3, 1).clip(0, 255).astype(np.float32)
    return torch.from_numpy(img), torch.from_numpy(labs), torch.from_numpy(tgts)


def test_joint_iteration_steps_the_right_tensors():
    """interactive step, then the instance step through the trained encoder: the instance step updates the encoder and the UNETR
    decoder (one step each) and leaves the prompt encoder and mask decoder bit for bit as the interactive step left them"""
    sam = util.get_sam_model("vit_test", device=DEV, state_dict=sam_ref.seeded_state_dict("vit_test", seed=1), max_batch=2,
                             max_prompts=64).model
    model = training.TrainableSAM(sam)
    net = training.get_unetr(sam, unetr_ref.seeded_state(seed=22, **WIDE_EMB))
    x, labs, tgts = _labelled_disks(2, 128, 128, 3)
    np.random.seed(0)
    enc = lambda: sam._upstream(lambda k: k.startswith("image_encoder."), master=True)   # noqa: E731
    dec = lambda: sam._upstream(lambda k: k.startswith(("mask_decoder.", "prompt_encoder.")), master=True)   # noqa: E731
    sam.train()
    sam.zero_decoder_grads()
    loss = training.interactive_train_iteration(model, x, labs, 0, n_objects_per_batch=4, n_sub_iteration=2)[0]
    loss.backward()
    sam.optimizer_step(lr=1e-4)
    e1, d1 = enc(), dec()
    assert e1 and d1
    sam.zero_decoder_grads()
    u0 = {k: v.clone() for k, v in net.decoder.masters.items()}
    lu = training.instance_train_iteration(net, x, tgts, freeze_encoder=False, lr=1e-4)
    assert torch.isfinite(lu)
    e2, d2 = enc(), dec()
    assert all(torch.equal(d1[k], d2[k]) for k in d1), "the instance step touched the mask decoder or prompt encoder"
    assert sum(not torch.equal(e1[k], e2[k]) for k in e1) > len(e1) // 2, "the instance step did not train the encoder"
    assert any(not torch.equal(u0[k], v) for k, v in net.decoder.masters.items())
    assert set(net.decoder.steps.values()) == {1}
    # one joint iteration end to end
    li, lu = training.joint_train_iteration(model, net, x, labs, tgts, iteration=1, n_objects_per_batch=4, n_sub_iteration=2, lr=1e-4)
    assert torch.isfinite(li) and torch.isfinite(lu) and set(net.decoder.steps.values()) == {2}


def test_training_ops_reject_bad_arguments():
    L = _lib.lib()
    t = torch.zeros(4096, device=DEV, dtype=torch.bfloat16)
    f = torch.zeros(4096, device=DEV)
    st = _lib.cur_stream()
    assert L.msam_ais_wgrad_workspace(63, 64, 0, 1, 8, 8, 3) < 0
    assert L.msam_op_ais_wgrad(_lib.ptr(t), 64, _lib.ptr(t), 64, None, 0, 1, 8, 8, 2, _lib.ptr(f), 1 << 30, _lib.ptr(f), st) != 0
    assert L.msam_op_ais_wgrad(_lib.ptr(t), 64, _lib.ptr(t), 64, None, 0, 1, 8, 8, 3, _lib.ptr(f), 16, _lib.ptr(f), st) != 0
    assert L.msam_op_ais_wgrad(None, 64, _lib.ptr(t), 64, None, 0, 1, 8, 8, 3, _lib.ptr(f), 1 << 30, _lib.ptr(f), st) != 0
    assert L.msam_op_ais_norm_forward(_lib.ptr(t), 1, 64, 12, 1, None, 0, None, None, 1e-5, 0, 0.1, None, None, _lib.ptr(f), 1 << 20,
                                      _lib.ptr(f), _lib.ptr(f), _lib.ptr(t), st) != 0
    assert L.msam_op_ais_norm_forward(_lib.ptr(t), 1, 64, 64, 1, None, 0, None, None, 1e-5, 0, 0.1, _lib.ptr(f), _lib.ptr(f),
                                      _lib.ptr(f), 1 << 20, _lib.ptr(f), _lib.ptr(f), _lib.ptr(t), st) != 0   # running statistics on an InstanceNorm
    assert L.msam_op_ais_norm_forward(_lib.ptr(t), 1, 64, 64, 1, None, 0, None, None, 1e-5, 0, 0.1, None, None, _lib.ptr(f), 1 << 20,
                                      _lib.ptr(f), None, _lib.ptr(t), st) != 0   # mean without rstd
    assert L.msam_op_ais_norm_forward(_lib.ptr(t), 1, 64, 64, 1, ctypes.c_void_p(f.data_ptr() + 4), 1, None, None, 1e-5, 0, 0.1,
                                      None, None, _lib.ptr(f), 1 << 20, None, None, _lib.ptr(t), st) != 0   # misaligned statistics
    assert L.msam_op_ais_norm_backward(_lib.ptr(t), 64, _lib.ptr(t), 0, 32, None, 1, 64, 64, 1, None, _lib.ptr(f), _lib.ptr(f), 0,
                                       _lib.ptr(f), 1 << 20, _lib.ptr(t), 0, 64, None, None, st) != 0   # ldd < C
    assert L.msam_op_ais_upsample2_backward(_lib.ptr(t), 1, 4, 4, 12, _lib.ptr(t), st) != 0
    assert L.msam_op_ais_head_backward(_lib.ptr(t), 1, 16, 1024, _lib.ptr(f), _lib.ptr(f), _lib.ptr(f), _lib.ptr(f), 1 << 20,
                                       _lib.ptr(t), _lib.ptr(f), _lib.ptr(f), st) != 0
    assert L.msam_op_ais_resize_backward(_lib.ptr(f), 1, 8, 8, 9, 8, 4, 4, _lib.ptr(f), _lib.ptr(f), st) != 0
    assert L.msam_op_ais_dist_loss_stats(_lib.ptr(f), _lib.ptr(f), 1, 64, 1, _lib.ptr(f), 8, _lib.ptr(f), st) != 0
    assert L.msam_op_adamw(_lib.ptr(f), _lib.ptr(f), _lib.ptr(f), _lib.ptr(f), 16, 1e-3, 0.9, 0.999, 1e-8, 0.0, 0, st) != 0
    assert b"step" in L.msam_last_error()
    assert L.msam_optimizer_step_prefix(None, b"image_encoder.", 1e-3, 0.9, 0.999, 1e-8, 0.0, st) != 0
