"""Pins the float64 references of tests/encoder_ops_ref.py against the oracle's modules and against autograd, so that they
cannot drift together with the kernels, and shows without a GPU that the metrics and tolerances of
tests/test_gpu_encoder_ops.py flag faults confined to one head, one window, four keys, the low half of the bias, one
table row or the GELU derivative's approximation -- several of which (asserted where it holds) stay inside the whole-tensor rel-L2 bounds (1.5e-2 at
op level, 2e-2 end to end) that were the only check of these kernels before."""
import pytest
import torch
import torch.nn.functional as F

from oracle import sam_ref
from tests import encoder_ops_ref as R

OLD_OP_BOUND = 1.5e-2


def _rand(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale


# ------------------------------------------------------------------------------------------------ pins
@pytest.mark.parametrize("window", [True, False], ids=["window", "global"])
@pytest.mark.parametrize("hd", [64, 80])
def test_attention_ref_equals_oracle_module(hd, window):
    heads, batch = 2, 1
    dim, side = heads * hd, (14 if window else 64)
    att = sam_ref.Attention(dim, heads, (side, side)).double()
    att.proj = torch.nn.Identity()
    with torch.no_grad():
        att.rel_pos_h.copy_(_rand(att.rel_pos_h.shape, 1, 0.3))
        att.rel_pos_w.copy_(_rand(att.rel_pos_w.shape, 2, 0.3))
        x = _rand((batch, 64, 64, dim), 3)
        if window:
            xw, pad_hw = sam_ref.window_partition(x, 14)
            want = sam_ref.window_unpartition(att(xw), 14, pad_hw, (64, 64)).reshape(-1, dim)
            qkv = att.qkv(xw).reshape(-1, 3 * dim)
        else:
            want = att(x).reshape(-1, dim)
            qkv = att.qkv(x).reshape(-1, 3 * dim)
        got = R.attention_ref(qkv, att.rel_pos_h, att.rel_pos_w, batch, heads, hd, 14 if window else 0)
    assert float((got - want).abs().max()) < 1e-10


def test_gemm_ref_equals_torch_modules():
    A, W, b, r = _rand((37, 24), 1), _rand((32, 24), 2), _rand((32,), 3), _rand((5, 32), 4)
    idx = torch.arange(37) % 5
    lin = F.linear(A, W, b)
    assert torch.allclose(R.gemm_ref(A, W, b, r, 5, act=1)[0], F.gelu(lin) + r[idx], atol=1e-12)
    assert torch.allclose(R.gemm_ref(A, W, b, r, 5, act=2, act_after_res=1)[0], torch.relu(lin + r[idx]), atol=1e-12)
    g, be = _rand((32,), 5), _rand((32,), 6)
    assert torch.allclose(R.gemm_ref(A, W, None, r, 5, ln=(g, be, 1e-5))[0], F.layer_norm(F.linear(A, W) + r[idx], (32,), g, be, 1e-5),
                          atol=1e-12)


@pytest.mark.parametrize("glob", [False, True], ids=["window", "global"])
def test_attn_ds_ref_equals_autograd_through_attn_probs_ref(glob):
    geom, n, scale = R.Geom(glob), (3 if not glob else 1), 0.125
    if glob:                      # a 64 x 64 geometry is too large for a quick CPU test of the identity; shrink the side only
        geom.side, geom.n_tok, geom.nt, geom.woff = 6, 36, 32, 16
    S = _rand((n, geom.n_tok, geom.n_tok), 1).requires_grad_(True)
    T = _rand((n, geom.n_tok, geom.nt), 2).requires_grad_(True)
    dP = _rand((n, geom.n_tok, geom.n_tok), 3)
    P = R.attn_probs_ref(S, T, geom, scale)
    (P * dP).sum().backward()
    dS, dT = R.attn_ds_ref(P.detach(), dP, geom)
    assert float((S.grad - scale * dS).abs().max()) < 1e-10 and float((T.grad - dT).abs().max()) < 1e-10
    valid = torch.zeros(geom.nt, dtype=torch.bool)
    valid[:2 * geom.side - 1] = True
    valid[geom.woff:geom.woff + 2 * geom.side - 1] = True
    assert bool((dT[..., ~valid] == 0).all())


def test_elementwise_refs():
    x = _rand((1000,), 1, 3.0).requires_grad_(True)
    F.gelu(x).sum().backward()
    assert float((R.gelu_grad_ref(x.detach()) - x.grad).abs().max()) < 1e-12
    B, g, C = 2, 6, 8
    xi, y = _rand((B * g * g, C), 2), _rand((B * g * g, 9 * C), 3)
    assert abs(float((R.im2col3x3_ref(xi, B, g, C) * y).sum() - (xi * R.col2im3x3_ref(y, B, g, C)).sum())) < 1e-9
    conv = F.conv2d(xi.view(B, g, g, C).permute(0, 3, 1, 2), torch.ones(1, C, 3, 3, dtype=torch.float64), padding=1)
    assert torch.allclose(R.im2col3x3_ref(xi, B, g, C).sum(1), conv.reshape(-1), atol=1e-12)
    xt = _rand((4096, 4), 4)
    win, _ = sam_ref.window_partition(xt.view(1, 64, 64, 4), 14)
    assert torch.equal(R.window_gather_ref(xt, 1), win.reshape(-1, 4)) and torch.equal(R.unpartition(R.window_gather_ref(xt, 1), 1), xt)
    assert int(R.pad_rows_mask(1, "cpu").sum()) == 4900 - 4096


# ------------------------------------------------------------------------------------------------ sensitivity
def _bf16(x):
    return x.to(torch.bfloat16).double()


@pytest.fixture(scope="module")
def window_case():
    """3 heads, 2 images of window attention in float64, with the probabilities."""
    heads, hd, batch = 3, 64, 2
    qkv = _bf16(_rand((batch * R.WIN_ROWS, 3 * heads * hd), 1))
    rel_h, rel_w = _bf16(_rand((27, hd), 2, 0.3)), _bf16(_rand((27, hd), 3, 0.3))
    ref, P = R.attention_ref(qkv, rel_h, rel_w, batch, heads, hd, 14, return_probs=True)
    return dict(heads=heads, hd=hd, batch=batch, qkv=qkv, rel=(rel_h, rel_w), ref=ref, P=P)


def _flag(got, ref, heads, tol):
    rows = ref.shape[0] * heads
    return R.within(R.head_rows(got, heads), R.head_rows(ref, heads), rows, tol)


def test_window_faults_are_flagged(window_case):
    c = window_case
    heads, hd, ref, tol = c["heads"], c["hd"], c["ref"], R.TOL_ATTN_WINDOW
    good = _bf16(ref)
    assert _flag(good, ref, heads, tol)[0]
    # two heads swapped in image 1 (the op-level check had 2 heads and one image: blockIdx.y >= 2, blockIdx.z >= 25 never ran)
    bad = good.clone().view(2, 4096, heads, hd)
    bad[1, :, [0, 2]] = bad[1, :, [2, 0]]
    assert not _flag(bad.view_as(ref), ref, heads, tol)[0]
    # one window's output written to the neighbouring window
    img = good.clone().view(2, 64, 64, heads * hd)
    img[0, 14:28, 28:42] = img[0, 14:28, 14:28]
    assert not _flag(img.view_as(ref), ref, heads, tol)[0]
    # keys 192..195 dropped from the softmax of one head of one window: inside the old bound, flagged per row
    v = c["qkv"].view(-1, 196, 3, heads, hd)[:, :, 2]
    P = c["P"][7, 1].clone()
    P[:, 192:] = 0
    P = P / P.sum(-1, keepdim=True)
    out = torch.zeros(2 * 25, 196, heads, hd, dtype=torch.float64)
    out[7, :, 1] = P @ v[7, :, 1] - c["P"][7, 1] @ v[7, :, 1]
    bad = _bf16(ref + R.unpartition(out.reshape(-1, heads * hd), 2))
    ok, (rel, row, _) = _flag(bad, ref, heads, tol)
    assert not ok and rel < OLD_OP_BOUND, (rel, row)


@pytest.mark.parametrize("tscale", [4, 8])
def test_bias_truncated_to_bf16_is_flagged(tscale):
    """k = 0, table x tscale: a bias that keeps only the hi bf16 part of T / scale moves single rows by more than the
    bias-only bound while the whole tensor stays inside the old one."""
    heads, hd, geom = 2, 64, R.Geom(False)
    qkv = _bf16(_rand((R.WIN_ROWS, 3 * heads * hd), 5))
    qkv.view(-1, 3, heads, hd)[:, 1] = 0
    rel_h, rel_w = _bf16(_rand((27, hd), 6, 0.1 * tscale)), _bf16(_rand((27, hd), 7, 0.1 * tscale))
    ref = R.attention_ref(qkv, rel_h, rel_w, 1, heads, hd, 14)
    assert _flag(_bf16(ref), ref, heads, R.TOL_ATTN_BIAS_ONLY)[0]
    x = qkv.view(25, 196, 3, heads, hd)
    tab = R.rel_table(rel_h, rel_w, geom).double()[:, :hd]
    scale = hd ** -0.5
    out = torch.empty(25, 196, heads, hd, dtype=torch.float64)
    for h in range(heads):
        T = x[:, :, 0, h] @ tab.t()
        T = _bf16(T / scale) * scale                      # the lo part dropped
        out[:, :, h] = R.gather_bias(T, geom).softmax(-1) @ x[:, :, 2, h]
    bad = _bf16(R.unpartition(out.reshape(-1, heads * hd), 1))
    ok, (rel, row, _) = _flag(bad, ref, heads, R.TOL_ATTN_BIAS_ONLY)
    assert not ok and rel < OLD_OP_BOUND, (rel, row)


def test_global_rel_h_slice_shift_is_flagged():
    """The rel_h bias of one 128-query tile read one table row off (the 80-row slice loaded from qh0 + 1)."""
    heads, hd, geom = 1, 64, R.Geom(True)
    qkv = _bf16(_rand((4096, 3 * hd), 8))
    rel_h, rel_w = _bf16(_rand((127, hd), 9, 0.05)), _bf16(_rand((127, hd), 10, 0.05))
    ref = R.attention_ref(qkv, rel_h, rel_w, 1, heads, hd, 0)
    good = _bf16(ref)
    assert _flag(good, ref, heads, R.TOL_ATTN_GLOBAL)[0]
    q, k, v = qkv[:, :hd], qkv[:, hd:2 * hd], qkv[:, 2 * hd:]
    rows = slice(17 * 128, 18 * 128)
    ih, iw = R.bias_index(geom, "cpu")
    T = q[rows] @ R.rel_table(rel_h, rel_w, geom).double()[:, :hd].t()
    logits = hd ** -0.5 * q[rows] @ k.t() + torch.gather(T, 1, (ih[rows] + 1).clamp_max(126)) + torch.gather(T, 1, iw[rows])
    bad = good.clone()
    bad[rows] = _bf16(logits.softmax(-1) @ v)
    assert not _flag(bad, ref, heads, R.TOL_ATTN_GLOBAL)[0]


def test_dT_one_table_row_off_is_flagged():
    geom, n = R.Geom(False), 24
    P = _bf16(_rand((n, 196, 196), 11, 2.0).softmax(-1))
    dS, dT = R.attn_ds_ref(P, _rand((n, 196, 196), 12), geom)
    good = _bf16(dT)
    assert R.within(good, dT, n * 196, R.TOL_DT)[0]
    bad = good.clone()
    edge = torch.arange(196) // 14 == 13                     # queries of the last window row: rel_h entries one row off
    bad[:, edge, 1:27] = good[:, edge, 0:26]
    bad[:, edge, 0] = 0
    assert not R.within(bad, dT, n * 196, R.TOL_DT)[0]


def test_tanh_gelu_derivative_is_flagged():
    n = 1 << 17
    pre = torch.cat([torch.linspace(-10, 10, n - 8), torch.tensor([0.0, -0.0, 1.0, -1.0, 3.0, -3.0, 10.0, -10.0])])
    pre = pre.to(torch.bfloat16).float().sort()[0].double()
    dh = _bf16(_rand((n,), 101))
    ref = dh * R.gelu_grad_ref(pre)
    good, bad = _bf16(ref), _bf16(dh * R.gelu_grad_tanh(pre))
    assert R.within(good, ref, n // 64, R.TOL_GELU_BWD)[0] and R.gelu_mismatch(good, ref, pre) <= R.TOL_GELU_MISMATCH
    assert float((bad - ref).norm() / ref.norm()) < OLD_OP_BOUND          # far inside any whole-tensor bound
    assert R.gelu_mismatch(bad, ref, pre) > 5 * R.TOL_GELU_MISMATCH
