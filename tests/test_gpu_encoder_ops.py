"""The ViT encoder's kernels op by op against the float64 references of tests/encoder_ops_ref.py: window and global
attention at production head counts and batch > 1, the persistent GEMM with its tails, pitches and epilogues
(msam_op_gemm_ex), and the row-wise stages of the attention / MLP / neck backward pass.

Metrics as in test_gpu_decoder_blocks.py: rel-L2 over the whole output, the worst per-row relative error (a row = one
token of one head for attention, one output row for the fused-LayerNorm GEMM, one query row for the backward stages),
finiteness, and sentinel margins around every output buffer.  Plain GEMM outputs are bounded per element: fp32 by
C * (sum |a||w| + |bias| + |residual|), bf16 by one bf16 ulp of the reference on top of that.  Each case prints what it
measured.  The planted attention cases name the mechanism of attention_win2.cu / attention_global.cu they exercise.

Measured on one H100 80GB HBM3 at a 700 W power limit, worst case over each family as (rel-L2, worst row):
  attention, random qkv     window 1.8e-3, 3.6e-3   global 1.8e-3, 3.5e-3   (12 / 16 heads, head_dim 64 / 80, 2 .. 3 images)
  attention, bias only      2.3e-3, 3.4e-3          (k = 0, table x1 / x4 / x8, window and global)
  attention, planted        1.9e-3, 4.3e-3          (keys 192..195 dominant, uniform, monotone logits, +-60 offsets, table ends);
                            a key that leads by 40 in the exponent gives its V row bit for bit
  GEMM, plain epilogue      fp32 out: |err| <= 2.3e-7 x magnitude; bf16 out: within one bf16 ulp of the reference plus 1.2e-7 x
                            magnitude (plus gelu_fast's 3e-5 with a GELU before a bf16 store)
  GEMM, fused LayerNorm     1.7e-3, 2.0e-3
  attn_probs                1.7e-3, 3.6e-3          row sums within 2.1e-3 of 1
  attn_ds                   dS 1.7e-3, 3.7e-3       dT 1.7e-3, 3.6e-3
  gelu_bwd                  1.1e-3, 2.7e-3          no output differs from the rounded reference for |pre| <= 3
  colsum / col2im / sum_batch   |err| <= 1.8e-7 x sum |terms|
Every figure is the bf16 rounding of the output (2^-9 relative per element); the tolerances in encoder_ops_ref.py are about
twice the measured worst value.  pack_dqkv, transpose_bf16 and window_gather are bit-exact.
"""
import pytest
import torch

from tests import encoder_ops_ref as R
from tests.encoder_ops_ref import SENT_BF16, SENT_F32, guarded, margins_intact

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(scope="module")
def L():
    from micro_sam_b200 import _lib
    _lib.lib()
    return _lib


def check(name, got, ref, rows, tol):
    ok, (rel, row, finite) = R.within(got, ref, rows, tol)
    print(f"  {name}: rel-L2 {rel:.3e}  worst row {row:.3e}  finite {finite}", flush=True)
    assert ok, f"{name}: rel-L2 {rel:.3e} (<= {tol[0]:.1e}), worst row {row:.3e} (<= {tol[1]:.1e}), finite {finite}"


def rand(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV, dtype)


# ------------------------------------------------------------------------------------------------ forward attention
def run_attention(L, qkv, tab, batch, heads, hd, window):
    n = batch * 4096 * heads * hd
    buf, out = guarded(n, torch.bfloat16)
    L.check(L.lib().msam_op_attention(L.ptr(qkv), L.ptr(tab), L.ptr(out), batch, heads, hd, R.WINDOW if window else 0,
                                      hd ** -0.5, L.cur_stream()))
    torch.cuda.synchronize()
    assert margins_intact(buf, n), "attention wrote outside its output"
    return out.view(batch * 4096, heads * hd).clone()


def make_qkv(batch, heads, hd, window, seed, scale=1.0):
    """Random qkv in the kernel's row order; the pad-token rows of the windows are one constant row, as in the model
    (q = k = v = qkv.bias there)."""
    rows = batch * (R.WIN_ROWS if window else 4096)
    qkv = rand((rows, 3 * heads * hd), seed, scale)
    if window:
        qkv[R.pad_rows_mask(batch, DEV)] = rand((3 * heads * hd,), seed + 1, 0.5)
    return qkv


def make_table(hd, window, seed, scale=0.3):
    geom = R.Geom(not window)
    rel_h = rand((2 * geom.side - 1, hd), seed, scale)
    rel_w = rand((2 * geom.side - 1, hd), seed + 1, scale)
    return rel_h, rel_w, R.rel_table(rel_h, rel_w, geom)


def attention_case(L, name, qkv, rel, batch, heads, hd, window, tol):
    rel_h, rel_w, tab = rel
    got = run_attention(L, qkv, tab, batch, heads, hd, window)
    ref = R.attention_ref(qkv, rel_h, rel_w, batch, heads, hd, R.WINDOW if window else 0)
    check(name, R.head_rows(got, heads), R.head_rows(ref, heads), batch * 4096 * heads, tol)
    return got, ref


PRODUCTION = [(12, 64, 2), (16, 64, 2), (16, 80, 2), (3, 64, 3)]


@pytest.mark.parametrize("window", [True, False], ids=["window", "global"])
@pytest.mark.parametrize("heads,hd,batch", PRODUCTION)
def test_attention_production_geometry(L, heads, hd, batch, window):
    """blockIdx.y up to 12 / 16 heads and blockIdx.z beyond one image; window queries of the last window row / column (most
    of their keys are pad tokens) are bounded on their own as well."""
    qkv = make_qkv(batch, heads, hd, window, seed=heads + hd + batch)
    rel = make_table(hd, window, seed=7)
    tol = R.TOL_ATTN_WINDOW if window else R.TOL_ATTN_GLOBAL
    got, ref = attention_case(L, f"{'window' if window else 'global'} heads={heads} hd={hd} B={batch}", qkv, rel, batch, heads, hd,
                              window, tol)
    if window:
        t = torch.arange(4096, device=DEV)
        edge = ((t // 64 >= 56) | (t % 64 >= 56)).repeat(batch)
        check("  last window row / column", R.head_rows(got[edge], heads), R.head_rows(ref[edge], heads), int(edge.sum()) * heads, tol)


@pytest.mark.parametrize("window", [True, False], ids=["window", "global"])
@pytest.mark.parametrize("heads,hd,batch", [(3, 64, 3), (2, 80, 2)])
def test_attention_per_image_invariance(L, heads, hd, batch, window):
    """Image b of a batch is bit-identical to the same image run alone, and a repeat is bit-identical."""
    qkv = make_qkv(batch, heads, hd, window, seed=3 * heads + hd)
    _, _, tab = make_table(hd, window, seed=9)
    got = run_attention(L, qkv, tab, batch, heads, hd, window)
    assert torch.equal(got, run_attention(L, qkv, tab, batch, heads, hd, window)), "repeat differs"
    per = qkv.shape[0] // batch
    for b in range(batch):
        alone = run_attention(L, qkv[b * per:(b + 1) * per].contiguous(), tab, 1, heads, hd, window)
        assert torch.equal(got[b * 4096:(b + 1) * 4096], alone), f"image {b} differs from the same image run alone"


def split(qkv, heads, hd):
    return qkv.view(qkv.shape[0], 3, heads, hd)


@pytest.mark.parametrize("window", [True, False], ids=["window", "global"])
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("tscale", [1, 4, 8])
def test_attention_bias_only(L, hd, tscale, window):
    """k = 0: the logits are the rel-pos bias alone.  Window: the bias enters the S MMA as hi + lo bf16 columns (a bias
    truncated to its hi part is off by up to 2^-9 of logits that reach +-50 at tscale 8); global: the T_h / T_w gathers."""
    heads, batch = 2, 1
    qkv = make_qkv(batch, heads, hd, window, seed=hd + tscale)
    split(qkv, heads, hd)[:, 1] = 0
    rel = make_table(hd, window, seed=11, scale=0.1 * tscale)
    attention_case(L, f"bias only x{tscale} {'window' if window else 'global'} hd={hd}", qkv, rel, batch, heads, hd, window,
                   R.TOL_ATTN_BIAS_ONLY)


def planted_qkv(batch, heads, hd, window, seed, key_gain):
    """q = u + noise (u = all ones), k = key_gain[key] * u, v random and large: logit[q, key] = scale * key_gain[key] *
    (hd + noise_q), a per-query multiple of key_gain.  key_gain: [G] over the keys of a window / an image."""
    G = R.WINDOW ** 2 if window else 4096
    rows = batch * (R.WIN_ROWS if window else 4096)
    qkv = torch.empty(rows, 3 * heads * hd, device=DEV, dtype=torch.bfloat16)
    s = split(qkv, heads, hd)
    s[:, 0] = 1.0 + rand((rows, heads, hd), seed, 0.25)
    s[:, 1] = key_gain.to(DEV).repeat(rows // G)[:, None, None].to(torch.bfloat16)
    s[:, 2] = rand((rows, heads, hd), seed + 1, 4.0)
    return qkv


@pytest.mark.parametrize("hd", [64, 80])
def test_window_keys_192_to_195_dominate(L, hd):
    """Keys 192..195 are the 13th k-step of P V, whose A tile lives in spare V columns: here they carry the largest logits
    of every query (about 8 above the rest) and distinctive V rows, so the output is almost entirely theirs."""
    heads, batch = 2, 1
    gain = torch.zeros(196)
    gain[192:] = hd ** -0.5 * 8.0
    qkv = planted_qkv(batch, heads, hd, True, seed=21 + hd, key_gain=gain)
    attention_case(L, f"window keys 192..195 dominant hd={hd}", qkv, make_table(hd, True, seed=13), batch, heads, hd, True,
                   R.TOL_ATTN_PLANTED)


@pytest.mark.parametrize("window", [True, False], ids=["window", "global"])
@pytest.mark.parametrize("hd", [64, 80])
def test_attention_uniform(L, hd, window):
    """q = 0 and a zero table: every probability is 1 / 196 (1 / 4096) and the output is the mean of V -- the window kernel's
    row sum comes from a ones column in V, the global kernel's from 32 rescaled partial sums."""
    heads, batch = 2, 1
    qkv = make_qkv(batch, heads, hd, window, seed=31 + hd)
    split(qkv, heads, hd)[:, 0] = 0
    geom = R.Geom(not window)
    zero = torch.zeros(2 * geom.side - 1, hd, device=DEV, dtype=torch.bfloat16)
    got, ref = attention_case(L, f"uniform {'window' if window else 'global'} hd={hd}", qkv, (zero, zero, R.rel_table(zero, zero, geom)),
                              batch, heads, hd, window, R.TOL_ATTN_PLANTED)
    if not window:
        mean_v = split(qkv, heads, hd)[:, 2].double().mean(0).reshape(1, -1)
        assert float((ref - mean_v).abs().max()) < 1e-12
        assert float((got.double() - mean_v).abs().max()) <= float(R.bf16_ulp(mean_v).max()), "uniform attention is not the mean of V"


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("window,key", [(True, 100), (True, 195), (False, 5), (False, 2048 + 77), (False, 4095)])
def test_attention_one_key_dominates(L, hd, window, key):
    """One key leads by more than 30 in the exponent: the output is that key's V row to bf16, wherever the key sits (first,
    a middle and the last key tile of the global kernel's online softmax)."""
    heads, batch = 2, 1
    G = 196 if window else 4096
    gain = torch.zeros(G)
    gain[key] = hd ** -0.5 * 40.0
    qkv = planted_qkv(batch, heads, hd, window, seed=41 + key, key_gain=gain)
    zero = torch.zeros(2 * R.Geom(not window).side - 1, hd, device=DEV, dtype=torch.bfloat16)
    got, _ = attention_case(L, f"dominant key {key} {'window' if window else 'global'} hd={hd}", qkv,
                            (zero, zero, R.rel_table(zero, zero, R.Geom(not window))), batch, heads, hd, window, R.TOL_ATTN_PLANTED)
    per = qkv.shape[0] // batch
    if window:
        v = split(qkv, heads, hd)[:, 2].reshape(per // 196, 196, heads * hd)[:, key]       # one V row per window
        want = R.unpartition(v[:, None].expand(-1, 196, -1).reshape(per, heads * hd), batch)
    else:
        want = split(qkv, heads, hd)[key, 2].reshape(1, heads * hd).expand(4096, -1)
    assert torch.equal(got, want), "the output is not the dominant key's V row"


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("kind", ["increasing", "decreasing", "offset+60", "offset-60"])
def test_global_online_softmax(L, hd, kind):
    """Logits that increase with the key index make the online softmax rescale in every one of the 32 key tiles, decreasing
    ones never; a common offset of +-60 on every logit of a row must cancel in the max subtraction (ex2.approx.ftz would
    flush or overflow otherwise)."""
    heads, batch = 2, 1
    ramp = torch.arange(4096) / 4096.0
    if kind == "increasing":
        gain = ramp * 4.0
    elif kind == "decreasing":
        gain = (1.0 - ramp) * 4.0
    else:
        gain = torch.full((4096,), 7.5 if kind == "offset+60" else -7.5)
    qkv = planted_qkv(batch, heads, hd, False, seed=51 + hd, key_gain=gain * (hd ** -0.5 * 8.0))
    if kind.startswith("offset"):
        split(qkv, heads, hd)[:, 1] += rand((4096, heads, hd), 52, 1.0)
    attention_case(L, f"global {kind} hd={hd}", qkv, make_table(hd, False, seed=15), batch, heads, hd, False, R.TOL_ATTN_PLANTED)


@pytest.mark.parametrize("hd", [64, 80])
def test_global_rel_table_slice_ends(L, hd):
    """rel_pos_h / rel_pos_w with magnitude only at relative index 0, 63 and 126: the ends and the centre of the table, which
    sit at different rows of the 80-row slice each query tile loads from its qh0 (tiles at the top, middle and bottom of the
    image are all bounded per row)."""
    heads, batch = 2, 1
    qkv = make_qkv(batch, heads, hd, False, seed=61 + hd)
    split(qkv, heads, hd)[:, 1] = 0
    rel_h = torch.zeros(127, hd, device=DEV, dtype=torch.bfloat16)
    rel_w = torch.zeros(127, hd, device=DEV, dtype=torch.bfloat16)
    rel_h[[0, 63, 126]] = rand((3, hd), 62, 0.5)
    rel_w[[0, 63, 126]] = rand((3, hd), 63, 0.5)
    got, ref = attention_case(L, f"global table ends hd={hd}", qkv, (rel_h, rel_w, R.rel_table(rel_h, rel_w, R.Geom(True))), batch,
                              heads, hd, False, R.TOL_ATTN_PLANTED)
    for qt in (0, 15, 31):
        rows = slice(qt * 128, qt * 128 + 128)
        check(f"  query tile {qt}", R.head_rows(got[rows], heads), R.head_rows(ref[rows], heads), 128 * heads, R.TOL_ATTN_PLANTED)


# ------------------------------------------------------------------------------------------------ GEMM
def run_gemm(L, M, N, K, seed, pads=(0, 0, 0, 0), bias=True, res=None, res_rows=0, act=0, after=0, f32=True, ln=False,
             num_sms=0, offset=0.0):
    """pads = extra elements of (lda, ldw, ldc, ldr) over their minimum.  Returns got [M, N] and the call's operands."""
    pa, pw, pc, pr = pads
    A = rand((M, K + pa), seed, 0.5)[:, :K]
    W = rand((N, K + pw), seed + 1, K ** -0.5)[:, :K]
    b = rand((N,), seed + 2, 1.0, torch.float32) + offset if bias else None
    rr = res_rows if res_rows else M
    r = None
    if res:
        r = rand((rr, N + pr), seed + 3, 1.0, torch.float32 if res == "f32" else torch.bfloat16)[:, :N]
    gamma = beta = None
    if ln:
        gamma, beta = 1.0 + rand((N,), seed + 4, 0.2, torch.float32), rand((N,), seed + 5, 0.2, torch.float32)
    ldc = N + pc
    dt = torch.float32 if f32 else torch.bfloat16
    buf, out = guarded(M * ldc, dt)

    import ctypes
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())   # noqa: E731  (strided views: pass the base pointer)
    rc = L.lib().msam_op_gemm_ex(vp(A), vp(W), M, N, K, K + pa, K + pw, vp(b), vp(r), res_rows, (N + pr) if res else 0,
                                 int(res == "bf16"), vp(out), ldc, int(f32), act, after, int(ln), vp(gamma), vp(beta), 1e-5,
                                 num_sms, L.cur_stream())
    torch.cuda.synchronize()
    sent = SENT_F32 if f32 else SENT_BF16
    o2 = out.view(M, ldc)
    assert margins_intact(buf, M * ldc), "gemm wrote outside its output"
    if rc == 0:
        assert bool((o2[:, N:] == sent).all()), "gemm wrote into columns [N, ldc)"
    return rc, o2[:, :N].clone(), dict(A=A, W=W, bias=b, residual=r, res_rows=res_rows, act=act, act_after_res=after,
                                       ln=(gamma, beta, 1e-5) if ln else None), buf


def gemm_case(L, name, M, N, K, seed, **kw):
    rc, got, ops, _ = run_gemm(L, M, N, K, seed, **kw)
    assert rc == 0, L.lib().msam_last_error().decode()
    ref, _ = R.gemm_ref(**ops)
    if ops["ln"] is not None:
        check(name, got, ref, M, R.TOL_GEMM_LN)
        return got
    mag = R.gemm_magnitude(ops["A"], ops["W"], ops["bias"], ops["residual"], ops["res_rows"])
    err = (got.double() - ref).abs()
    bound = R.GEMM_F32_C * mag
    if got.dtype == torch.bfloat16:
        bound = bound + R.bf16_ulp(ref) + (R.GEMM_GELU_FAST if ops["act"] == 1 and not ops["act_after_res"] else 0.0)
        excess = float(((err - R.bf16_ulp(ref)).clamp_min(0) / mag).max())
        print(f"  {name}: bf16 out, max (err - ulp) / magnitude {excess:.3e}", flush=True)
    else:
        print(f"  {name}: fp32 out, max err / magnitude {float((err / mag).max()):.3e}", flush=True)
    assert bool(torch.isfinite(got).all())
    bad = (err > bound).nonzero()
    assert len(bad) == 0, f"{name}: {len(bad)} elements beyond their bound, first (row, col) {bad[:8].tolist()}"
    return got


_MS = [1, 63, 64, 65, 127, 129, 9800]
_NS = [32, 96, 160, 128, 384, 256, 768]
_KS = [8, 24, 72, 200, 768]
GEMM_TAILS = sorted({(M, _NS[i % 7], _KS[i % 5]) for i, M in enumerate(_MS)} | {(129, N, _KS[(i + 2) % 5]) for i, N in enumerate(_NS)} |
                    {(65, _NS[(i + 3) % 7], K) for i, K in enumerate(_KS)} | {(9800, 160, 200), (9800, 768, 72), (1, 256, 8)} |
                    {(65536, 64, 288), (65537, 64, 256)})     # TinyViT: stem conv 2 (im2col, K = 288); MBConv conv3 (below)


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "bf16"])
@pytest.mark.parametrize("M,N,K", GEMM_TAILS)
def test_gemm_tails(L, M, N, K, f32):
    """Partial last row tile, all three BN instantiations incl. a partial last column tile, K down to 8 and not a multiple
    of 32 or 64 (the TMA box zero-fills the K tail).  N = 64, K = 256 runs TinyViT's MBConv conv3 epilogue, GELU(conv3(x) +
    shortcut) with the shortcut a bf16 residual."""
    kw = dict(res="bf16", act=1, after=1) if (N, K) == (64, 256) else {}
    gemm_case(L, f"gemm M={M} N={N} K={K}{' bf16 res, GELU after' if kw else ''}", M, N, K, seed=M + N + K, f32=f32, **kw)


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "bf16"])
@pytest.mark.parametrize("pads", [(8, 0, 0, 0), (0, 24, 0, 0), (0, 0, 2, 0), (0, 0, 34, 0), (16, 8, 6, 4)])
def test_gemm_pitches(L, pads, f32):
    gemm_case(L, f"gemm pitches +{pads}", 300, 160, 72, seed=sum(pads), pads=pads, res="f32" if f32 else "bf16", f32=f32)


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "bf16"])
@pytest.mark.parametrize("res,res_rows", [("f32", 0), ("bf16", 0), ("f32", 100), ("bf16", 64)])
@pytest.mark.parametrize("act,after", [(0, 0), (1, 0), (2, 0), (1, 1), (2, 1)])
def test_gemm_epilogues(L, res, res_rows, act, after, f32):
    """fp32 and bf16 residual, the row-modulus broadcast (pos-embed), GELU / ReLU before the residual and after it."""
    gemm_case(L, f"gemm res={res} res_rows={res_rows} act={act} after={after}", 257, 384, 200, seed=5 + act + after, res=res,
              res_rows=res_rows, act=act, after=after, f32=f32)


@pytest.mark.parametrize("M", [1, 127, 129, 4096])
@pytest.mark.parametrize("res", [None, "bf16"])
@pytest.mark.parametrize("offset", [0.0, 30.0])
def test_gemm_fused_layernorm(L, M, res, offset):
    """LayerNorm(256) epilogue; rows with a common offset of 30 need the two-pass statistics."""
    gemm_case(L, f"gemm LN256 M={M} res={res} offset={offset}", M, 256, 200, seed=M, res=res, f32=False, ln=True, offset=offset)


@pytest.mark.parametrize("N,ln", [(768, False), (160, False), (256, True)])
def test_gemm_independent_of_grid_size(L, N, ln):
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    outs = [run_gemm(L, 1000, N, 200, seed=3, f32=False, ln=ln, res="bf16", num_sms=s)[1] for s in (1, 7, n_sm, 0)]
    assert all(torch.equal(outs[0], o) for o in outs[1:]), "the output depends on the number of CTAs"


@pytest.mark.parametrize("what,kw", [
    ("N % 32", dict(N=48)), ("K % 8", dict(K=36)), ("odd ldc", dict(pads=(0, 0, 1, 0))), ("LN with N != 256", dict(N=128, ln=True, f32=False)),
    ("LN with fp32 out", dict(ln=True, f32=True)), ("LN with fp32 residual", dict(ln=True, f32=False, res="f32")),
    ("LN with act", dict(ln=True, f32=False, act=1))])
def test_gemm_rejects_bad_arguments(L, what, kw):
    """Host-side rejections: -1 with a message, nothing launched, the output untouched."""
    kw = dict(dict(N=256, K=64), **kw)
    N, K = kw.pop("N"), kw.pop("K")
    n0 = L.launch_count()
    rc, _, _, buf = run_gemm(L, 64, N, K, seed=1, **kw)
    assert rc == -1 and L.lib().msam_last_error(), what
    assert L.launch_count() == n0, f"{what}: a kernel was launched"
    assert bool((buf == (SENT_F32 if buf.dtype == torch.float32 else SENT_BF16)).all()), f"{what}: the output was written"


# ------------------------------------------------------------------------------------------------ attention backward stages
def pitched(x, pitch, fill):
    """[n, q, k] -> contiguous [n, q, pitch] with `fill` in the pad columns."""
    out = torch.full(x.shape[:2] + (pitch,), fill, device=x.device, dtype=x.dtype)
    out[..., :x.shape[2]] = x
    return out


BWD_GEOMS = [(False, 300), (False, 7), (True, 3)]     # (global, n_batch): 58800 rows, 1372 rows (not a multiple of 8), 12288 rows


@pytest.mark.parametrize("offset", [0.0, 60.0, -60.0])
@pytest.mark.parametrize("glob,n", BWD_GEOMS)
def test_attn_probs(L, glob, n, offset):
    geom = R.Geom(glob)
    scale = 0.125
    S = rand((n, geom.n_tok, geom.n_tok), 71 + n, 8.0, torch.float32) + offset / scale
    T = rand((n, geom.n_tok, geom.nt), 72 + n, 1.0, torch.float32)
    Sp = pitched(S, geom.pitch, 1e30)
    buf, P = guarded(n * geom.n_tok * geom.pitch, torch.bfloat16)
    L.check(L.lib().msam_op_attn_probs(L.ptr(Sp), L.ptr(T), n, int(glob), geom.pitch, geom.pitch, scale, L.ptr(P), L.cur_stream()))
    torch.cuda.synchronize()
    assert margins_intact(buf, P.numel())
    P = P.view(n, geom.n_tok, geom.pitch)
    assert bool((P[..., geom.n_tok:] == 0).all()), "pad columns of P are not zero"
    got = P[..., :geom.n_tok]
    check(f"attn_probs global={glob} n={n} offset={offset}", got, R.attn_probs_ref(S, T, geom, scale), n * geom.n_tok, R.TOL_PROBS)
    dev = float((got.double().sum(-1) - 1).abs().max())
    print(f"    max |row sum - 1| {dev:.3e}", flush=True)
    assert dev <= 4e-3


@pytest.mark.parametrize("glob,n", BWD_GEOMS)
def test_attn_ds(L, glob, n):
    geom = R.Geom(glob)
    P = (rand((n, geom.n_tok, geom.n_tok), 81 + n, 2.0, torch.float32)).softmax(-1).to(torch.bfloat16)
    dP = rand((n, geom.n_tok, geom.n_tok), 82 + n, 1.0, torch.float32)
    Pp, dPp = pitched(P, geom.pitch, 0.0), pitched(dP, geom.pitch, 1e30)
    bs, dS = guarded(n * geom.n_tok * geom.pitch, torch.bfloat16)
    bt, dT = guarded(n * geom.n_tok * geom.nt, torch.bfloat16)
    dS.fill_(float("nan"))      # the kernel owns every element of both outputs, whatever they held before
    dT.fill_(float("nan"))
    L.check(L.lib().msam_op_attn_ds(L.ptr(Pp), L.ptr(dPp), n, int(glob), geom.pitch, geom.pitch, L.ptr(dS), L.ptr(dT), L.cur_stream()))
    torch.cuda.synchronize()
    assert margins_intact(bs, dS.numel()) and margins_intact(bt, dT.numel())
    dS, dT = dS.view(n, geom.n_tok, geom.pitch), dT.view(n, geom.n_tok, geom.nt)
    assert bool((dS[..., geom.n_tok:] == 0).all()), "pad columns of dS are not zero"
    valid = torch.zeros(geom.nt, dtype=torch.bool, device=DEV)
    valid[:2 * geom.side - 1] = True
    valid[geom.woff:geom.woff + 2 * geom.side - 1] = True
    assert bool((dT[..., ~valid] == 0).all()), "dT entries outside the two table ranges are not zero"
    rS, rT = R.attn_ds_ref(P, dP, geom)
    check(f"attn_ds dS global={glob} n={n}", dS[..., :geom.n_tok], rS, n * geom.n_tok, R.TOL_DS)
    check(f"attn_ds dT global={glob} n={n}", dT, rT, n * geom.n_tok, R.TOL_DT)
    t = torch.arange(geom.n_tok, device=DEV)
    h, w = t // geom.side, t % geom.side
    edge = (h == 0) | (h == geom.side - 1) | (w == 0) | (w == geom.side - 1)
    check("  dT, queries on the border", dT[:, edge], rT[:, edge], n * int(edge.sum()), R.TOL_DT)


@pytest.mark.parametrize("hd,heads,outer,T", [(64, 12, 50, 196), (80, 16, 3, 196), (64, 3, 2, 4096), (80, 2, 1, 4096)])
def test_pack_dqkv(L, hd, heads, outer, T):
    dq, dk, dv = (rand((outer, heads, T, hd), 90 + i, 1.0, torch.float32) for i in range(3))
    n = outer * T * 3 * heads * hd
    buf, out = guarded(n, torch.bfloat16)
    L.check(L.lib().msam_op_pack_dqkv(L.ptr(dq), L.ptr(dk), L.ptr(dv), outer, heads, T, hd, L.ptr(out), L.cur_stream()))
    torch.cuda.synchronize()
    want = torch.stack([dq, dk, dv]).permute(1, 3, 0, 2, 4).reshape(outer * T, 3 * heads * hd).to(torch.bfloat16)
    assert margins_intact(buf, n) and torch.equal(out.view_as(want), want)


@pytest.mark.parametrize("rows,cols", [(768, 2304), (1280, 5120), (33, 95), (1, 64), (256, 31)])
def test_transpose_bf16(L, rows, cols):
    x = rand((rows, cols), rows + cols)
    buf, out = guarded(rows * cols, torch.bfloat16)
    L.check(L.lib().msam_op_transpose_bf16(L.ptr(x), rows, cols, L.ptr(out), L.cur_stream()))
    torch.cuda.synchronize()
    assert margins_intact(buf, rows * cols) and torch.equal(out.view(cols, rows), x.t().contiguous())


@pytest.mark.parametrize("B,D", [(2, 768), (1, 1280), (3, 64), (1, 8)])
def test_window_gather(L, B, D):
    x = rand((B * 4096, D), B + D)
    n = B * R.WIN_ROWS * D
    buf, out = guarded(n, torch.bfloat16)
    L.check(L.lib().msam_op_window_gather(L.ptr(x), B, D, L.ptr(out), L.cur_stream()))
    torch.cuda.synchronize()
    out = out.view(B * R.WIN_ROWS, D)
    assert margins_intact(buf, n) and torch.equal(out, R.window_gather_ref(x, B))
    assert bool((out[R.pad_rows_mask(B, DEV)] == 0).all())
    assert torch.equal(R.unpartition(out, B), x)


def gelu_bwd_inputs(device):
    """pre = 2^17 sorted points over [-10, 10] incl. +-0 (bf16), dh random."""
    n = 1 << 17
    pre = torch.cat([torch.linspace(-10, 10, n - 8), torch.tensor([0.0, -0.0, 1.0, -1.0, 3.0, -3.0, 10.0, -10.0])])
    pre = pre.to(torch.bfloat16).float().sort()[0].to(device, torch.bfloat16)
    g = torch.Generator().manual_seed(101)
    return pre, torch.randn(n, generator=g).to(device, torch.bfloat16)


def test_gelu_bwd(L):
    """In place, as encode_backward calls it.  Next to the per-row and per-element bounds, nearly every output has to be the
    bf16 rounding of the reference: single roundings hide a derivative that is 1e-3 off (the tanh approximation), the share of
    flipped roundings among 256 neighbouring points does not."""
    pre, dh = gelu_bwd_inputs(DEV)
    n = pre.numel()
    ref = dh.double() * R.gelu_grad_ref(pre)
    buf, io = guarded(n, torch.bfloat16)
    io.copy_(dh)
    L.check(L.lib().msam_op_gelu_bwd(L.ptr(io), L.ptr(pre), n, L.ptr(io), L.cur_stream()))
    torch.cuda.synchronize()
    assert margins_intact(buf, n)
    check("gelu_bwd", io, ref, n // 64, R.TOL_GELU_BWD)
    assert bool(((io.double() - ref).abs() <= R.bf16_ulp(ref) + 1e-6).all()), "an element is more than one bf16 ulp off"
    mism = R.gelu_mismatch(io, ref, pre)
    print(f"    largest share of 256 neighbours that differ from the rounded reference {mism:.3e}", flush=True)
    assert mism <= R.TOL_GELU_MISMATCH


@pytest.mark.parametrize("rows", [1, 255, 256, 257, 8192])
@pytest.mark.parametrize("N", [32, 96, 768])
def test_colsum(L, rows, N):
    x = rand((rows, N), rows + N)
    start = rand((N,), 5, 1.0, torch.float32)
    buf, out = guarded(N, torch.float32)
    out.copy_(start)
    L.check(L.lib().msam_op_colsum(L.ptr(x), rows, N, L.ptr(out), L.cur_stream()))
    torch.cuda.synchronize()
    ref = start.double() + x.double().sum(0)
    mag = start.double().abs() + x.double().abs().sum(0)
    r = float(((out.double() - ref).abs() / mag).max())
    print(f"  colsum rows={rows} N={N}: max err / magnitude {r:.3e}", flush=True)
    assert margins_intact(buf, N) and r <= R.F32_SUM_C


@pytest.mark.parametrize("B,g,C", [(2, 64, 256), (1, 5, 8), (3, 7, 64)])
def test_col2im3x3(L, B, g, C):
    dcol = rand((B * g * g, 9 * C), B + g + C)
    n = B * g * g * C
    buf, out = guarded(n, torch.float32)
    L.check(L.lib().msam_op_col2im3x3(L.ptr(dcol), B, g, C, L.ptr(out), L.cur_stream()))
    torch.cuda.synchronize()
    ref = R.col2im3x3_ref(dcol, B, g, C)
    r = float(((out.view_as(ref).double() - ref).abs() / R.col2im3x3_ref(dcol.abs(), B, g, C).clamp_min(1e-30)).max())
    print(f"  col2im B={B} g={g} C={C}: max err / magnitude {r:.3e}", flush=True)
    assert margins_intact(buf, n) and r <= R.F32_SUM_C


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("nb,n", [(300, 64 * 80), (2, 4096 * 768), (1, 1000), (7, 257)])
def test_sum_batch(L, nb, n, accumulate):
    x = rand((nb, n), nb + n, 1.0, torch.float32)
    start = rand((n,), 6, 1.0, torch.float32)
    buf, out = guarded(n, torch.float32)
    out.copy_(start)
    L.check(L.lib().msam_op_sum_batch(L.ptr(x), nb, n, L.ptr(out), accumulate, L.cur_stream()))
    torch.cuda.synchronize()
    ref = x.double().sum(0) + (start.double() if accumulate else 0)
    mag = x.double().abs().sum(0) + start.double().abs()
    r = float(((out.double() - ref).abs() / mag).max())
    print(f"  sum_batch nb={nb} n={n} accumulate={accumulate}: max err / magnitude {r:.3e}", flush=True)
    assert margins_intact(buf, n) and r <= R.F32_SUM_C


@pytest.mark.parametrize("call", ["window_gather D % 8", "pack_dqkv d % 4", "gelu_bwd n % 8", "attn_probs pitch", "null pointer"])
def test_backward_stage_rejections(L, call):
    """Size preconditions and null pointers are rejected on the host: -1 with a message, nothing launched."""
    lib, st = L.lib(), L.cur_stream()
    x = torch.zeros(1 << 16, device=DEV)
    p = L.ptr(x)
    n0 = L.launch_count()
    rc = {"window_gather D % 8": lambda: lib.msam_op_window_gather(p, 1, 12, p, st),
          "pack_dqkv d % 4": lambda: lib.msam_op_pack_dqkv(p, p, p, 1, 1, 4, 6, p, st),
          "gelu_bwd n % 8": lambda: lib.msam_op_gelu_bwd(p, p, 12, p, st),
          "attn_probs pitch": lambda: lib.msam_op_attn_probs(p, p, 1, 0, 192, 200, 0.125, p, st),
          "null pointer": lambda: lib.msam_op_attn_ds(p, None, 1, 0, 200, 200, p, p, st)}[call]()
    torch.cuda.synchronize()
    assert rc == -1 and lib.msam_last_error() and L.launch_count() == n0
    assert bool((x == 0).all())
