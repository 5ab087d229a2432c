"""Decoder-based automatic instance segmentation (AIS) on the GPU: each csrc/ais.cu op against float64, the UNETR decoder
against oracle/unetr_ref.py, the post-processing bit for bit against oracle/ais_ref.py, and the public surface
(get_predictor_and_decoder, InstanceSegmentationWithDecoder, get_instance_segmentation_generator, automatic_3d_segmentation)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from micro_sam_b200 import _lib, automatic_segmentation, instance_segmentation as iseg, unetr, util
from micro_sam_b200 import multi_dimensional_segmentation as mds
from oracle import ais_ref, merge3d_ref, sam_ref, unetr_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# decoder maps (sigmoid outputs) against the float64 oracle: (rel-L2, worst pixel) bounds per plan, twice the bf16 noise floor
# that tests/ais_noise_floor.py measures on the CPU (7.25e-3 / 2.68e-2, 3.05e-3 / 8.48e-3, 8.04e-3 / 2.80e-2); DESIGN.md section 2
MAP_BOUNDS = {"production-interp": (1.45e-2, 5.4e-2), "production-transposed": (6.1e-3, 1.7e-2), "reduced-affine": (1.6e-2, 5.6e-2)}


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _bf(t):
    return t.to(DEV, torch.bfloat16).contiguous()


def _conv(x0, x1, w, b, ks, relu, transposed=False, stats=False):
    B, H, W, C0 = x0.shape
    C1 = 0 if x1 is None else x1.shape[3]
    cout = b.numel()
    out = torch.empty((B, 2 * H, 2 * W, cout) if transposed else (B, H, W, cout), device=DEV, dtype=torch.bfloat16)
    st = torch.empty(int(_lib.lib().msam_ais_conv_stats_size(B, H, W, cout, int(transposed))) // 8, device=DEV,
                     dtype=torch.float64) if stats else None
    _lib.check(_lib.lib().msam_op_ais_conv(_lib.ptr(x0), C0, _lib.ptr(x1), C1, B, H, W, ks, _lib.ptr(w), _lib.ptr(b), cout,
                                           relu, int(transposed), _lib.ptr(out), _lib.ptr(st), _lib.cur_stream()))
    return (out, st) if stats else out


def _check_stats(out, st):
    """The epilogue's partial sums, reduced per (image, channel), equal the sums of the stored bf16 outputs."""
    B, C = out.shape[0], out.shape[3]
    part = st.view(B, -1, C, 2).sum(1)
    ref = out.double().reshape(B, -1, C)
    for k, r in ((0, ref.sum(1)), (1, (ref * ref).sum(1))):
        assert float((part[..., k] - r).abs().max() / r.abs().max().clamp_min(1e-30)) < 1e-5


@pytest.mark.parametrize("C0,C1,cout,H,W,B", [(64, 0, 64, 64, 64, 2), (256, 256, 512, 64, 64, 1), (128, 128, 128, 128, 96, 1),
                                              (64, 64, 64, 512, 512, 1), (64, 64, 64, 1024, 1024, 1), (64, 64, 192, 33, 47, 2)])
def test_conv3x3_against_float64(C0, C1, cout, H, W, B):
    g = torch.Generator().manual_seed(C0 + H)
    x0 = torch.randn(B, H, W, C0, generator=g)
    x1 = torch.randn(B, H, W, C1, generator=g) if C1 else None
    w = (torch.rand(cout, C0 + C1, 3, 3, generator=g) * 2 - 1) / (9 * (C0 + C1)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    wk = w.permute(0, 2, 3, 1).reshape(cout, 9 * (C0 + C1))
    out, st = _conv(_bf(x0), None if x1 is None else _bf(x1), _bf(wk), b.to(DEV), 3, 1, stats=True)
    _check_stats(out, st)
    out = out.float()
    xin = x0 if x1 is None else torch.cat([x0, x1], 3)
    xin = xin.to(DEV, torch.bfloat16).double().permute(0, 3, 1, 2)
    ref = F.relu(F.conv2d(xin, w.to(DEV, torch.bfloat16).double(), b.to(DEV).double(), padding=1)).permute(0, 2, 3, 1)
    err = (out.double() - ref).abs()
    scale = ref.abs().max()
    assert float(err.max() / scale) < 1e-2, float(err.max() / scale)
    for edge in (err[:, 0], err[:, -1], err[:, :, 0], err[:, :, -1]):   # rows / columns where the zero padding matters
        assert float(edge.max() / scale) < 1e-2
    if B == 2:   # a batch of 2 is bit-identical per image
        one = _conv(_bf(x0[1:]).contiguous(), None if x1 is None else _bf(x1[1:]).contiguous(), _bf(wk), b.to(DEV), 3, 1)
        assert torch.equal(one[0], out[1].to(torch.bfloat16))


@pytest.mark.parametrize("transposed", [False, True])
def test_conv1x1_and_transposed(transposed):
    g = torch.Generator().manual_seed(3)
    B, H, W, cin, cout = 2, 40, 24, 128, 64
    x = torch.randn(B, H, W, cin, generator=g)
    b = torch.randn(cout, generator=g) * 0.1
    xd = x.to(DEV, torch.bfloat16).double().permute(0, 3, 1, 2)
    if transposed:
        w = torch.randn(cin, cout, 2, 2, generator=g) / cin ** 0.5
        out, st = _conv(_bf(x), None, _bf(w.permute(2, 3, 1, 0).reshape(4 * cout, cin)), b.to(DEV), 1, 0, True, stats=True)
        _check_stats(out, st)
        ref = F.conv_transpose2d(xd, w.to(DEV, torch.bfloat16).double(), b.to(DEV).double(), stride=2)
    else:
        w = torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5
        out = _conv(_bf(x), None, _bf(w[:, :, 0, 0]), b.to(DEV), 1, 0)
        ref = F.conv2d(xd, w.to(DEV, torch.bfloat16).double(), b.to(DEV).double())
    ref = ref.permute(0, 2, 3, 1)
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 1e-2


@pytest.mark.parametrize("affine", [False, True])
def test_norm_forward_instance_norm_against_float64(affine):
    g = torch.Generator().manual_seed(4)
    B, H, W, C = 2, 96, 80, 128
    x = (torch.randn(B, H, W, C, generator=g) * 3 + torch.randn(1, 1, 1, C, generator=g)).to(DEV, torch.bfloat16)
    gam, bet = (torch.rand(C, generator=g) + 0.5).to(DEV), torch.randn(C, generator=g).to(DEV)
    L = _lib.lib()
    ws = torch.empty(int(L.msam_ais_norm_workspace(B, H * W, C)), device=DEV, dtype=torch.uint8)
    out = torch.empty_like(x)
    gp, bp = (_lib.ptr(gam), _lib.ptr(bet)) if affine else (None, None)
    _lib.check(L.msam_op_ais_norm_forward(_lib.ptr(x), B, H * W, C, 1, None, 0, gp, bp, 1e-5, 0, 0.1, None, None, _lib.ptr(ws),
                                          ws.numel(), None, None, _lib.ptr(out), _lib.cur_stream()))
    ref = F.instance_norm(x.double().permute(0, 3, 1, 2), weight=gam.double() if affine else None,
                          bias=bet.double() if affine else None, eps=1e-5).permute(0, 2, 3, 1)
    assert float((out.double() - ref).abs().max()) < 3e-2
    out2 = torch.empty_like(x)
    _lib.check(L.msam_op_ais_norm_forward(_lib.ptr(x), B, H * W, C, 1, None, 0, gp, bp, 1e-5, 0, 0.1, None, None, _lib.ptr(ws),
                                          ws.numel(), None, None, _lib.ptr(out2), _lib.cur_stream()))
    assert torch.equal(out, out2)
    # with partial sums from a convolution epilogue (the decoder's path): the same normalisation
    wk = torch.eye(C).to(DEV, torch.bfloat16).contiguous()
    y, st = _conv(x, None, wk, torch.zeros(C, device=DEV), 1, 0, stats=True)
    assert torch.equal(y, x)
    out3 = torch.empty_like(x)
    _lib.check(L.msam_op_ais_norm_forward(_lib.ptr(x), B, H * W, C, 1, _lib.ptr(st), st.numel() // (2 * B * C), gp, bp, 1e-5, 0,
                                          0.1, None, None, _lib.ptr(ws), ws.numel(), None, None, _lib.ptr(out3), _lib.cur_stream()))
    assert float((out3.double() - ref).abs().max()) < 3e-2


def test_upsample_x2_against_float64():
    x = torch.randn(2, 37, 50, 64, generator=torch.Generator().manual_seed(5)).to(DEV, torch.bfloat16)
    out = torch.empty(2, 74, 100, 64, device=DEV, dtype=torch.bfloat16)
    _lib.check(_lib.lib().msam_op_ais_upsample2(_lib.ptr(x), 2, 37, 50, 64, _lib.ptr(out), _lib.cur_stream()))
    ref = F.interpolate(x.double().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 1e-2


@pytest.mark.parametrize("input_size,original_size", [((700, 1024), (700, 1024)), ((1024, 512), (1024, 512)),
                                                      ((683, 1024), (1366, 2048)), ((1024, 768), (300, 225))])
def test_crop_and_resize_against_float64(input_size, original_size):
    maps = torch.rand(1, 3, 1024, 1024, generator=torch.Generator().manual_seed(6)).to(DEV)
    out = unetr.resize_maps(maps, input_size, original_size)
    ref = unetr_ref.postprocess_masks(maps.double(), input_size, original_size)
    assert out.shape == ref.shape
    assert float((out.double() - ref).abs().max()) < 2e-4   # fp32 source coordinates, as in PyTorch's float kernel


# ------------------------------------------------------------------------------------------------ decoder end to end
@pytest.mark.parametrize("plan,kw", [("production-interp", dict()), ("production-transposed", dict(transposed=True)),
                                     ("reduced-affine", dict(emb=256, feats=(128, 64, 64, 64), deconv=(128, 64, 64, 64),
                                                             affine=True))])
def test_decoder_against_oracle(plan, kw):
    sd = unetr_ref.seeded_state(seed=7, **kw)
    dec = unetr.UNETRDecoder(sd, device=DEV)
    z = torch.randn(1, 256, 64, 64, generator=torch.Generator().manual_seed(8)) * 0.5
    maps = dec.forward_maps(z.to(DEV))
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    ref = unetr_ref.forward_maps(sdd, z.to(DEV).to(torch.bfloat16))
    rel, worst = _rel(maps, ref), float((maps.double() - ref).abs().max())
    print(f"{kw}: rel-L2 {rel:.2e}, worst pixel {worst:.2e}")
    assert rel < MAP_BOUNDS[plan][0] and worst < MAP_BOUNDS[plan][1]
    out = dec(z.to(DEV), (683, 1024), (683, 1024))
    assert out.shape == (1, 3, 683, 1024) and torch.equal(out, maps[:, :, :683])
    assert torch.equal(dec.forward_maps(z.to(DEV)), maps)   # repeats are bit-identical


# ------------------------------------------------------------------------------------------------ post-processing
def _post(fg, cd, bd, **kw):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(DEV)
    lab, n, sweeps = unetr.postprocess(t(fg), t(cd), t(bd), **kw)
    return lab.cpu().numpy().astype(np.int64), n, sweeps


POST_CASES = {
    "touching": dict(maps=dict(H=256, W=320, n=120, seed=0), kw={}),
    "many-touching-large": dict(maps=dict(H=1024, W=1024, n=1500, seed=1), kw={}),
    "sigma0": dict(maps=dict(H=200, W=150, n=40, seed=2), kw=dict(foreground_smoothing=0.0, distance_smoothing=0.0)),
    "sigma3.3": dict(maps=dict(H=200, W=260, n=40, seed=3), kw=dict(foreground_smoothing=3.3, distance_smoothing=3.3)),
    "min-size": dict(maps=dict(H=256, W=256, n=80, seed=4), kw=dict(min_size=150)),
    "unreached": dict(maps=dict(H=256, W=256, n=60, seed=5), kw=dict(center_distance_threshold=0.12,
                                                                      boundary_distance_threshold=0.2)),
}


@pytest.mark.parametrize("case", list(POST_CASES))
def test_postprocess_bit_exact(case):
    c = POST_CASES[case]
    fg, cd, bd = ais_ref.touching_disks(c["maps"]["H"], c["maps"]["W"], c["maps"]["n"], seed=c["maps"]["seed"])
    lab, n, sweeps = _post(fg, cd, bd, **c["kw"])
    ref = ais_ref.generate(fg, cd, bd, **c["kw"])
    print(f"{case}: {n} ids, {sweeps} sweeps, {int(((lab == 0) & (ref == 0)).sum())} background")
    assert n == ref.max() and n > 0
    np.testing.assert_array_equal(lab, ref)
    if case == "unreached":
        seeds, _, fmask, _ = ais_ref.markers_and_mask(fg, cd, bd, 0.5, 0.12, 0.2, 1.0, 1.6)
        assert ((ref == 0) & fmask).any()   # foreground pixels no seed reaches stay 0
    lab2, _, _ = _post(fg, cd, bd, **c["kw"])
    assert np.array_equal(lab, lab2)


def test_postprocess_empty_foreground():
    z = np.zeros((64, 80), np.float32)
    lab, n, _ = _post(z, z, z)
    assert n == 0 and not lab.any()


# ------------------------------------------------------------------------------------------------ public surface
_CACHE = {}


def _sam_sd():
    if "sd" not in _CACHE:
        _CACHE["sd"] = sam_ref.seeded_state_dict("vit_test", seed=1)
    return _CACHE["sd"]


def _checkpoint(tmp_path, **kw):
    path = tmp_path / "ais.pt"
    torch.save({"model_state": _sam_sd(), "decoder_state": unetr_ref.seeded_state(seed=9, **kw)}, path)
    return str(path)


def test_end_to_end_from_checkpoint(tmp_path):
    from micro_sam_b200.sample_data import lm_tile
    pred, dec = iseg.get_predictor_and_decoder("vit_test", _checkpoint(tmp_path), device=DEV)
    seg = iseg.get_instance_segmentation_generator(pred, is_tiled=False, decoder=dec)
    assert isinstance(seg, iseg.InstanceSegmentationWithDecoder)
    img = lm_tile((300, 400), 12, seed=2)
    seg.initialize(img)
    kw = dict(foreground_threshold=0.45, min_size=5)
    labels = seg.generate(**kw)
    st = seg.get_state()
    assert labels.dtype == np.uint32 and labels.shape == (300, 400)
    assert st["foreground"].shape == (300, 400) and st["foreground"].dtype == np.float32
    ref = ais_ref.generate(st["foreground"], st["center_distances"], st["boundary_distances"], **kw)
    np.testing.assert_array_equal(labels.astype(np.int64), ref)
    assert np.array_equal(seg.generate(**kw), labels)
    masks = seg.generate(output_mode="binary_mask", **kw)
    assert len(masks) == labels.max()
    for m in masks:
        ys, xs = np.nonzero(labels == m["seg_id"])
        assert np.array_equal(m["segmentation"], labels == m["seg_id"]) and m["area"] == len(ys)
        assert m["bbox"] == [xs.min(), xs.max() - xs.min() + 1, ys.min(), ys.max() - ys.min() + 1]
        assert m["crop_box"] == [0, 400, 0, 300]
    seg2 = iseg.InstanceSegmentationWithDecoder(pred, dec)
    seg2.set_state(st)
    assert np.array_equal(seg2.generate(**kw), labels)
    seg2.clear_state()
    assert not seg2.is_initialized
    p2, s2 = automatic_segmentation.get_predictor_and_segmenter("vit_test", checkpoint=_checkpoint(tmp_path), device=DEV)
    assert isinstance(s2, iseg.InstanceSegmentationWithDecoder)


def test_refusals(tmp_path):
    pred, dec = iseg.get_predictor_and_decoder("vit_test", _checkpoint(tmp_path), device=DEV)
    with pytest.raises(NotImplementedError):
        iseg.get_instance_segmentation_generator(pred, is_tiled=True, decoder=dec)
    with pytest.raises(NotImplementedError):
        iseg.get_instance_segmentation_generator(pred, is_tiled=False, decoder=dec, segmentation_mode="apg")
    with pytest.raises(NotImplementedError):
        iseg.AutomaticPromptGenerator(pred, dec)
    seg = iseg.InstanceSegmentationWithDecoder(pred, dec)
    z = np.zeros((32, 32), np.float32)
    seg.set_state({"foreground": z, "center_distances": z, "boundary_distances": z})
    with pytest.raises(NotImplementedError):
        seg.generate(tile_shape=(16, 16), halo=(4, 4))
    with pytest.raises(NotImplementedError):
        seg.generate(optimize_memory=True)
    from micro_sam_b200 import precompute_state as ps
    with pytest.raises(NotImplementedError):
        ps.cache_is_state()
    with pytest.raises(NotImplementedError):
        ps.precompute_state(str(tmp_path), str(tmp_path / "out"), model_type="vit_test", checkpoint_path=_checkpoint(tmp_path))


def test_ais_ops_reject_bad_arguments():
    L = _lib.lib()
    x = torch.zeros(1, 8, 8, 64, device=DEV, dtype=torch.bfloat16)
    w = torch.zeros(64, 9 * 64, device=DEV, dtype=torch.bfloat16)
    b = torch.zeros(64, device=DEV)
    o = torch.zeros_like(x)
    p, s = _lib.ptr, _lib.cur_stream()
    assert L.msam_op_ais_conv(None, 64, None, 0, 1, 8, 8, 3, p(w), p(b), 64, 1, 0, p(o), None, s) != 0
    assert L.msam_op_ais_conv(p(x), 32, None, 0, 1, 8, 8, 3, p(w), p(b), 64, 1, 0, p(o), None, s) != 0
    assert L.msam_op_ais_conv(p(x), 64, None, 0, 1, 8, 8, 3, p(w), p(b), 48, 1, 0, p(o), None, s) != 0
    assert L.msam_op_ais_conv(p(x), 64, None, 0, 1, 8, 8, 5, p(w), p(b), 64, 1, 0, p(o), None, s) != 0
    assert L.msam_op_ais_conv(p(x), 64, None, 0, 1, 8, 8, 3, p(w), p(b), 64, 1, 1, p(o), None, s) != 0
    assert L.msam_op_ais_conv(p(x), 64, None, 32, 1, 8, 8, 3, p(w), p(b), 64, 1, 0, p(o), None, s) != 0
    assert L.msam_op_ais_conv(ctypes.c_void_p(x.data_ptr() + 2), 64, None, 0, 1, 8, 8, 3, p(w), p(b), 64, 1, 0, p(o), None, s) != 0
    ws = torch.zeros(16, device=DEV, dtype=torch.uint8)
    def norm(C, stats, nchunk, gamma, ws_bytes):
        return L.msam_op_ais_norm_forward(p(x), 1, 64, C, 1, stats, nchunk, gamma, None, 1e-5, 0, 0.1, None, None, p(ws), ws_bytes,
                                          None, None, p(o), s)
    assert norm(64, None, 0, None, ws.numel()) != 0   # workspace too small
    assert norm(60, None, 0, None, 1 << 20) != 0
    assert norm(64, None, 0, p(b), 1 << 20) != 0
    assert norm(64, p(ws), 0, None, 1 << 20) != 0   # stats, 0 chunks
    assert L.msam_op_ais_upsample2(p(x), 1, 8, 8, 12, p(o), s) != 0
    assert L.msam_op_ais_upsample2(None, 1, 8, 8, 64, p(o), s) != 0
    assert L.msam_op_ais_head(p(x), 1, 64, 1024, p(b), p(b), p(b), s) != 0
    assert L.msam_op_ais_resize(p(b), 1, 8, 8, 9, 8, 4, 4, p(b), s) != 0
    n, sw = ctypes.c_int(0), ctypes.c_int(0)
    assert L.msam_ais_postprocess(p(b), p(b), p(b), 8, 8, None, 0, None, 0, 0.5, 0.5, 0.5, 0, p(ws), 16, p(o), ctypes.byref(n),
                                  ctypes.byref(sw), s) != 0
    assert L.msam_ais_postprocess_workspace(0, 8) < 0
    assert L.msam_ais_props(None, 8, 8, 1, p(b), s) != 0


def test_automatic_3d_segmentation_with_ais(tmp_path):
    from micro_sam_b200.sample_data import em_volume
    pred, dec = iseg.get_predictor_and_decoder("vit_test", _checkpoint(tmp_path), device=DEV)
    seg = iseg.InstanceSegmentationWithDecoder(pred, dec)
    vol = em_volume((3, 160, 192), seed=3)
    kw = dict(foreground_threshold=0.45)
    out, emb = mds.automatic_3d_segmentation(vol, pred, seg, verbose=False, return_embeddings=True, **kw)
    slices = []
    for i in range(vol.shape[0]):
        seg.initialize(vol[i], image_embeddings=emb, i=i)
        slices.append(seg.generate(**kw))
    assert out.dtype == np.uint32
    np.testing.assert_array_equal(out, merge3d_ref.merge(merge3d_ref.stack_slices(slices)))
