"""Pins the float64 references of tests/tinyvit_ops_ref.py against the modules of oracle/tinyvit_ref.py (Conv2d_BN after BN
folding, Attention, TinyViTBlock's pad / partition / crop, PatchEmbed.seq[0] after Sam.preprocess), so that they cannot drift
together with the kernels, and shows without a GPU that the metrics and tolerances of tests/test_gpu_tinyvit_ops.py flag the
faults they are there for: pad rows that are 0 instead of beta, pad keys masked out of the softmax, a transposed bias index, a
clamped depth-wise border, stride-2 taps one pixel off, uint8 pad pixels normalised to -mean / std, and a last window row
left unwritten."""
import pytest
import torch
import torch.nn as nn

from oracle import sam_ref, tinyvit_ref
from tests import tinyvit_ops_ref as T

OLD_BOUND = 2e-2      # the whole-stream rel-L2 bound of the encoder-level check


def _rand(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale


def _bf16(x):
    return x.to(torch.bfloat16).double()


def _randomise(m, seed):
    """Random weights and eval-mode BatchNorm statistics for every parameter / buffer of m (float64)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in list(m.named_parameters()) + list(m.named_buffers()):
            if not p.dtype.is_floating_point:
                continue
            if name.endswith("running_var"):
                p.copy_(0.5 + torch.rand(p.shape, generator=g, dtype=torch.float64))
            elif name.endswith("bn.weight") or name.endswith("norm.weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g, dtype=torch.float64))
            else:
                p.copy_(0.3 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    return m.eval()


# ------------------------------------------------------------------------------------------------ pins
def test_stem_ref_equals_preprocess_and_patch_embed_conv():
    """PatchEmbed.seq[0..1] (Conv2d_BN 3 -> 32 /2, GELU) after Sam.preprocess of a 614 x 1024 uint8 image: the pad region
    is 0 after the normalisation."""
    osam = sam_ref.build_sam("vit_t").double()
    seq = osam.image_encoder.patch_embed.seq
    _randomise(seq[0], 1)
    u8 = T.make_u8(1, 614, 1024, seed=2)
    with torch.no_grad():
        x = osam.preprocess(u8[0].permute(2, 0, 1)[None].double())
        want = seq[1](seq[0](x)).permute(0, 2, 3, 1)
        w, b = T.fold_conv_bn(seq[0])
    xp = T.preprocess_u8(u8, 1024)
    assert float((xp - x).abs().max()) == 0.0
    got, mag = T.stem_ref(xp, T.stem_weight(w), b)
    assert float((got - want).abs().max()) < 1e-12
    dead = T.stem_pad_outputs(1, 614, 1024, 1024, "cpu")
    assert int(dead.sum()) == (512 - 308) * 512 and torch.equal(got[dead], T.gelu(b)[None].expand(int(dead.sum()), -1))


def test_im2col_and_gemm_operand_equal_patch_embed_conv2():
    """im2col (stride 2) times the stem's GEMM operand [64, 288] is PatchEmbed.seq[2] (Conv2d_BN 32 -> 64 /2)."""
    m = _randomise(tinyvit_ref.Conv2d_BN(32, 64, 3, 2, 1).double(), 3)
    x = _rand((2, 32, 18, 18), 4)
    with torch.no_grad():
        want = T.rows(m(x))
        w, b = T.fold_conv_bn(m)
    col = T.im2col_ref(T.rows(x), 2, 18, 32, 2)
    assert col.shape == (2 * 81, 288)
    assert float((col @ T.gemm_conv_weight(w).t() + b - want).abs().max()) < 1e-11


@pytest.mark.parametrize("C,H,stride,act", [(16, 12, 1, 1), (24, 10, 2, 1), (8, 7, 1, 0), (32, 9, 1, 0)])
def test_dwconv_ref_equals_depthwise_conv2d_bn(C, H, stride, act):
    """MBConv.conv2 / PatchMerging.conv2 (+ GELU) and TinyViTBlock.local_conv (no activation) after BN folding."""
    m = _randomise(tinyvit_ref.Conv2d_BN(C, C, 3, stride, 1, groups=C).double(), C + H)
    x = _rand((2, C, H, H), 5)
    with torch.no_grad():
        want = m(x)
        want = T.rows(nn.GELU()(want) if act else want)
        w, b = T.fold_conv_bn(m)
    got, _ = T.dwconv_ref(T.rows(x), 2, H, C, stride, T.dw_weight(w), b, act)
    assert float((got - want).abs().max()) < 1e-12


class _Zero(nn.Module):
    def forward(self, x):
        return torch.zeros_like(x)


@pytest.mark.parametrize("H,ws,heads", [(9, 7, 2), (7, 7, 3), (15, 14, 2), (16, 7, 4)])
def test_ln_window_and_attention_refs_equal_tinyvit_block(H, ws, heads):
    """TinyViTBlock with proj, local_conv and the MLP taken out: block(x) - x is the window attention of the block's own pad /
    partition / crop (H == ws takes its no-pad branch), and equals attn.qkv applied to ln_window_ref, through attention_ref."""
    D = heads * T.HEAD_DIM
    blk = _randomise(tinyvit_ref.TinyViTBlock(D, (H, H), heads, ws, 4.0, 3).double(), H + ws)
    blk.attn.proj, blk.local_conv, blk.mlp = nn.Identity(), nn.Identity(), _Zero()
    x = _rand((1, H * H, D), 6)
    a = blk.attn
    with torch.no_grad():
        want = (blk(x) - x)[0]
        xw = T.ln_window_ref(x[0], 1, H, D, ws, a.norm.weight, a.norm.bias)
        qkv = xw @ a.qkv.weight.t() + a.qkv.bias
        got = T.attention_ref(qkv, a.attention_biases, 1, H, ws, heads)
    assert float((got - want).abs().max()) < 1e-10
    assert torch.equal(xw[T.pad_rows(1, H, ws, "cpu")], a.norm.bias.expand(int(T.pad_rows(1, H, ws, "cpu").sum()), -1))


def test_attention_ref_equals_attention_module():
    """One window through tinyvit_ref.Attention (norm and proj taken out): the [q | k | v] split per head, the scale and
    attention_biases[:, attention_bias_idxs]."""
    for ws, heads in ((7, 4), (14, 5)):
        att = _randomise(tinyvit_ref.Attention(heads * 32, 32, heads, 1, (ws, ws)).double(), ws)
        att.norm, att.proj = nn.Identity(), nn.Identity()
        x = _rand((3, ws * ws, heads * 32), 7)
        with torch.no_grad():
            want = att(x).reshape(-1, heads * 32)
            qkv = att.qkv(x).reshape(-1, heads * 96)
            got = T.attention_ref(qkv, att.attention_biases, 3, ws, ws, heads)     # H == ws: one window per "image"
        assert float((got - want).abs().max()) < 1e-12


# ------------------------------------------------------------------------------------------------ sensitivity
def _attn_flagged(got, ref, heads, tol):
    return not T.within(T.head_rows(got, heads), T.head_rows(ref, heads), ref.shape[0] * heads, tol)[0]


@pytest.fixture(scope="module")
def stage3():
    """Stage 3's attention geometry (64 x 64 tokens, 7 x 7 windows, 10 heads: the last window row holds 1 real row of 7)."""
    B, H, ws, heads = 1, 64, 7, 10
    qkv = T.make_qkv(B, H, ws, heads, seed=11)
    tab = T.make_bias_tab(heads, ws, seed=12)
    ref = T.attention_ref(qkv, tab, B, H, ws, heads)
    return dict(B=B, H=H, ws=ws, heads=heads, qkv=qkv, tab=tab, ref=ref)


def test_attention_faults_are_flagged(stage3):
    c = stage3
    B, H, ws, heads, ref = c["B"], c["H"], c["ws"], c["heads"], c["ref"]
    good = _bf16(ref)
    edge = T.edge_tokens(B, H, ws, "cpu")
    assert not _attn_flagged(good, ref, heads, T.TOL_ATTN) and not _attn_flagged(good[edge], ref[edge], heads, T.TOL_ATTN)
    bias = c["tab"].double()[:, T.bias_index(ws, "cpu")]
    # pad keys masked out of the softmax: only the edge windows change
    kb = torch.where(T.pad_rows(B, H, ws, "cpu"), float("-inf"), 0.0).view(-1, ws * ws)
    bad = _bf16(T.unpartition(T.attention_windows(c["qkv"], bias, heads, key_bias=kb), B, H, ws))
    assert _attn_flagged(bad, ref, heads, T.TOL_ATTN) and _attn_flagged(bad[edge], ref[edge], heads, T.TOL_ATTN)
    assert torch.equal(bad[~edge], good[~edge])
    # bias index transposed: |dx| * ws + |dy|
    badt = c["tab"].double()[:, T.bias_index(ws, "cpu", transposed=True)]
    bad = _bf16(T.unpartition(T.attention_windows(c["qkv"], badt, heads), B, H, ws))
    assert _attn_flagged(bad, ref, heads, T.TOL_ATTN)
    # the last window row of queries left unwritten (zeros)
    bad = good.clone().view(B, H, H, -1)
    bad[:, (H // ws) * ws:] = 0
    assert _attn_flagged(bad.view_as(ref), ref, heads, T.TOL_ATTN)


def test_transposed_bias_in_one_head_is_flagged_per_row():
    """A bias-only case (q = 0, the bias table at twice the scale) with the bias index transposed in one head of five."""
    B, H, ws, heads = 1, 64, 14, 5
    qkv = T.make_qkv(B, H, ws, heads, seed=13)
    qkv.view(-1, heads, 3, 32)[:, :, 0] = 0
    tab = T.make_bias_tab(heads, ws, seed=14, scale=2.0)
    ref = T.attention_ref(qkv, tab, B, H, ws, heads)
    assert not _attn_flagged(_bf16(ref), ref, heads, T.TOL_ATTN_PLANTED)
    bias = tab.double()[:, T.bias_index(ws, "cpu")]
    bias[2] = tab.double()[2, T.bias_index(ws, "cpu", transposed=True)]
    bad = _bf16(T.unpartition(T.attention_windows(qkv, bias, heads), B, H, ws))
    assert _attn_flagged(bad, ref, heads, T.TOL_ATTN_PLANTED)


@pytest.mark.parametrize("H,D,ws", [(64, 320, 7), (15, 160, 14)])
def test_ln_window_faults_are_flagged(H, D, ws):
    B = 1
    x = T.rand((B * H * H, D), 21, 1.0, torch.float32).double() + T.rand((B * H * H, 1), 22, 3.0, torch.float32).double()
    gamma, beta = T.make_ln(D, 23)
    ref = T.ln_window_ref(x, B, H, D, ws, gamma, beta)
    mag = (ref - beta.double()).abs() + beta.double().abs()
    n = ref.shape[0]
    good = _bf16(ref)
    pad = T.pad_rows(B, H, ws, "cpu")
    assert T.within(good, ref, n, T.TOL_LN)[0] and T.elementwise(good, ref, mag, T.LN_C, True)[0]
    assert torch.equal(good[pad], _bf16(beta.double()).expand(int(pad.sum()), -1))
    # pad rows 0 instead of LN(0) = beta
    bad = good.clone()
    bad[pad] = 0
    assert not T.within(bad, ref, n, T.TOL_LN)[0] and not T.elementwise(bad, ref, mag, T.LN_C, True)[0]
    # the last window row left unwritten
    nw = T.n_windows(H, ws)
    bad = good.clone().view(B, nw, nw, ws * ws, D)
    bad[:, nw - 1] = 0
    assert not T.within(bad.view_as(ref), ref, n, T.TOL_LN)[0]


def _dw_case(Hin, C, stride, act, seed):
    x = T.rand((2 * Hin * Hin, C), seed, 1.0)
    w, b = T.make_dw(C, seed + 1)
    ref, mag = T.dwconv_ref(x, 2, Hin, C, stride, w, b, act)
    return x, w, b, ref, mag


@pytest.mark.parametrize("Hin,C,stride", [(32, 16, 1), (32, 16, 2)])
def test_dwconv_border_and_stride_faults_are_flagged(Hin, C, stride):
    x, w, b, ref, mag = _dw_case(Hin, C, stride, 1, 31)
    Ho = Hin // stride
    border = T.border_pixels(2, Ho, "cpu")
    good = _bf16(ref)
    assert T.elementwise(good, ref, mag, T.DW_BF16_C, True)[0]
    X, W = T.nchw(x.double(), 2, Hin, C), w.double().t().reshape(C, 1, 3, 3)
    # the border clamped (replicate pad) instead of zero-padded: only border outputs change
    clamped = torch.nn.functional.conv2d(torch.nn.functional.pad(X, (1, 1, 1, 1), mode="replicate"), W, b.double(), stride,
                                         groups=C)
    bad = _bf16(T.rows(T.gelu(clamped)))
    assert torch.equal(bad[~border], good[~border])
    assert not T.elementwise(bad[border], ref[border], mag[border], T.DW_BF16_C, True)[0]
    if stride == 2:   # taps at 2 o + k instead of 2 o + k - 1
        shifted = torch.nn.functional.conv2d(torch.nn.functional.pad(X, (0, 1, 0, 1)), W, b.double(), 2, groups=C)
        bad = _bf16(T.rows(T.gelu(shifted)))
        assert bad.shape == ref.shape and not T.elementwise(bad, ref, mag, T.DW_BF16_C, True)[0]


def test_dwconv_f32_border_fault_is_flagged():
    x = T.rand((64 * 64, 32), 41, 1.0, torch.float32)
    w, b = T.make_dw(32, 42)
    ref, mag = T.dwconv_ref(x, 1, 64, 32, 1, w, b)
    good = ref.float().double()
    assert T.elementwise(good, ref, mag, T.DW_F32_C, False)[0]
    X, W = T.nchw(x.double(), 1, 64, 32), w.double().t().reshape(32, 1, 3, 3)
    clamped = torch.nn.functional.conv2d(torch.nn.functional.pad(X, (1, 1, 1, 1), mode="replicate"), W, b.double(), groups=32)
    assert not T.elementwise(T.rows(clamped).float().double(), ref, mag, T.DW_F32_C, False)[0]


def test_stem_pad_pixels_normalised_is_flagged():
    """uint8 pad pixels given the value -mean / std (normalising after the zero pad) instead of 0."""
    img, hh, ww = 64, 40, 51
    u8 = T.make_u8(2, hh, ww, seed=51)
    w, b = T.make_stem(52)
    ref, mag = T.stem_ref(T.preprocess_u8(u8, img), w, b)
    good = _bf16(ref)
    assert T.elementwise(good, ref, mag, T.STEM_C, True)[0]
    dead = T.stem_pad_outputs(2, hh, ww, img, "cpu")
    assert torch.equal(good[dead], _bf16(T.gelu(b.double())).expand(int(dead.sum()), -1))
    xp = torch.nn.functional.pad(u8.double().permute(0, 3, 1, 2), (0, img - ww, 0, img - hh))
    xp = (xp - T.MEAN.view(1, 3, 1, 1)) / T.STD.view(1, 3, 1, 1)
    bad = _bf16(T.stem_ref(xp, w, b)[0])
    assert not T.elementwise(bad, ref, mag, T.STEM_C, True)[0]
    assert not torch.equal(bad[dead], good[dead])


def test_stage3_pad_rows_zero_exceed_the_worst_token_bound():
    """The encoder-level fault the whole-stream check missed: stage 3's pad rows 0 instead of LN beta (the seeded vit_t
    weights of tests/test_gpu_real_arch.py, its 1024^2 tile).  Against the clean oracle the stage-3 token stream stays
    inside the 2e-2 rel-L2 bound while its worst token exceeds TOL_STAGE_TOKEN."""
    import numpy as np
    from micro_sam_b200 import util
    from micro_sam_b200.sample_data import lm_tile
    sd = sam_ref.seeded_state_dict("vit_t", seed=0)
    osam = sam_ref.build_sam("vit_t")
    osam.load_state_dict(sd)
    img = util._to_image(lm_tile((1024, 1024), 150, seed=0))
    enc = osam.image_encoder
    with torch.no_grad():
        x = enc.patch_embed(osam.preprocess(torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1)[None].float()))
        for layer in enc.layers[:3]:
            x = layer(x)
        clean = enc.layers[3](x)[0]
        for blk in enc.layers[3].blocks:
            norm = blk.attn.norm
            blk.attn.norm = _PadRowsZero(norm)
        bad = enc.layers[3](x)[0]
    rel, row, _ = T.errors(bad, clean, clean.shape[0])
    print(f"stage-3 pad rows 0: rel-L2 {rel:.3e}, worst token {row:.3e}")
    assert rel < OLD_BOUND and row > T.TOL_STAGE_TOKEN, (rel, row)


class _PadRowsZero(nn.Module):
    """LayerNorm that leaves all-zero input rows (the pad tokens) at 0 instead of beta."""

    def __init__(self, norm):
        super().__init__()
        self.norm = norm

    def forward(self, x):
        return torch.where((x == 0).all(-1, keepdim=True), torch.zeros_like(x), self.norm(x))
