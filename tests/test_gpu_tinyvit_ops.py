"""The TinyViT (vit_t) encoder's CUDA-core kernels op by op (msam_op_tv_*, the launches msam_encode makes) against the float64
references of tests/tinyvit_ops_ref.py: the fused-preprocess stem on square, non-square and one-pixel-thin uint8 images and
on the fp32 path, im2col, the bf16 depth-wise convolutions (stride 1 / 2, GELU) and the fp32 local conv at the production
shapes, the window LayerNorm with TinyViT's pad rule and the window attention at the production (grid, window, heads),
plus grids with no pad and with a single real row in the last window.  Sentinels surround every output.

Metrics: the convolutions are bounded per element (C * (sum |x||w| + |b|), plus one bf16 ulp of the reference for a bf16
output), border pixels on their own as well; the LayerNorm per element and as (rel-L2, worst row); attention as (rel-L2,
worst row), a row being one token of one head, with the queries of the edge windows (last window row / column) bounded on
their own.  Each case prints what it measured.

Measured on one H100 80GB HBM3 at a 700 W power limit (test_device prints the card and limit of the run), worst case over
each family:
  stem, uint8 and fp32      (err - ulp) / magnitude 4.0e-8
  dwconv bf16               (err - ulp) / magnitude 5.4e-8       (border pixels 8.2e-9)
  dwconv fp32               err / magnitude 2.5e-7               (border pixels 1.9e-7)
  ln_window                 rel-L2 1.7e-3, worst row 2.4e-3;  per element (err - ulp) / (|gamma xhat| + |beta|) 4.6e-6
  attention, random qkv     rel-L2 1.7e-3, worst row 2.9e-3      (edge-window queries 1.7e-3, 2.7e-3)
  attention, planted        rel-L2 1.7e-3, worst row 3.1e-3      (bias only, uniform); a key that leads by about 40 in the
                            exponent gives its V row bit for bit
Every figure is the bf16 rounding of the output (2^-9 relative per element), or fp32 accumulation for the fp32 local conv.
The tolerances in tinyvit_ops_ref.py are about twice these.  im2col is bit-exact; pad rows of the LayerNorm equal bf16(beta)
and stem outputs whose 3 x 3 field lies in the zero pad equal bf16(GELU(bias)) bit for bit.
"""
import pytest
import torch

from tests import tinyvit_ops_ref as T
from tests.encoder_ops_ref import guarded, margins_intact

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def L():
    from micro_sam_b200 import _lib
    _lib.lib()
    return _lib


def power_note():
    """The card and its power limit, read in the same run as the numbers they qualify."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return f"{torch.cuda.get_device_name()} at {pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000:.0f} W"
    except Exception:
        import subprocess
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", f"-i={torch.cuda.current_device()}"],
                           capture_output=True, text=True)
        return r.stdout.strip() or torch.cuda.get_device_name()


def test_device(L):
    print(f"  device: {power_note()}", flush=True)


def check_rows(name, got, ref, rows, tol):
    ok, (rel, row, finite) = T.within(got, ref, rows, tol)
    print(f"  {name}: rel-L2 {rel:.3e}  worst row {row:.3e}  finite {finite}", flush=True)
    assert ok, f"{name}: rel-L2 {rel:.3e} (<= {tol[0]:.1e}), worst row {row:.3e} (<= {tol[1]:.1e}), finite {finite}"


def check_elems(name, got, ref, mag, c, bf16_out):
    ok, excess = T.elementwise(got, ref, mag, c, bf16_out)
    print(f"  {name}: max {'(err - ulp)' if bf16_out else 'err'} / magnitude {excess:.3e}", flush=True)
    assert ok, f"{name}: {excess:.3e} beyond C = {c:.1e}"


def run(L, fn, n, dtype, *args):
    """Calls msam_op_tv_<fn>(*args with OUT replaced by a guarded output of n elements) and returns the output."""
    buf, out = guarded(n, dtype)
    a = [L.ptr(out) if x is OUT else (L.ptr(x) if isinstance(x, torch.Tensor) else x) for x in args]
    L.check(getattr(L.lib(), f"msam_op_tv_{fn}")(*a, L.cur_stream()))
    torch.cuda.synchronize()
    assert margins_intact(buf, n), f"{fn} wrote outside its output"
    return out.clone()


OUT = object()


# ------------------------------------------------------------------------------------------------ stem
@pytest.mark.parametrize("hh,ww", [(1024, 1024), (614, 1024), (1024, 683), (1, 1024), (1024, 1)])
def test_stem_u8(L, hh, ww):
    """Sam.preprocess fused into conv3x3/2 + GELU on B = 3 images: the zero pad of a resized non-square image (and of a
    one-pixel-thin one) is 0 after the normalisation."""
    B, img = 3, 1024
    u8 = T.make_u8(B, hh, ww, seed=hh + ww, device=DEV)
    w, b = T.make_stem(7, DEV)
    got = run(L, "stem", B * 512 * 512 * 32, torch.bfloat16, u8, None, B, hh, ww, img, w, b, OUT).view(B, 512, 512, 32)
    ref, mag = T.stem_ref(T.preprocess_u8(u8, img), w, b)
    check_elems(f"stem u8 {hh}x{ww}", got, ref, mag, T.STEM_C, True)
    dead = T.stem_pad_outputs(B, hh, ww, img, DEV)
    if hh < img or ww < img:
        assert torch.equal(got[dead], T.gelu(b.double()).to(torch.bfloat16).expand(int(dead.sum()), -1)), \
            "an output whose field lies in the pad is not bf16(GELU(bias))"


def test_stem_f32(L):
    B, img = 3, 1024
    x = T.rand((B, 3, img, img), 17, 1.5, torch.float32, DEV)
    w, b = T.make_stem(18, DEV)
    got = run(L, "stem", B * 512 * 512 * 32, torch.bfloat16, None, x, B, img, img, img, w, b, OUT).view(B, 512, 512, 32)
    ref, mag = T.stem_ref(x, w, b)
    check_elems("stem f32", got, ref, mag, T.STEM_C, True)
    border = T.border_pixels(B, 512, DEV).view(B, 512, 512)
    check_elems("  border outputs", got[border], ref[border], mag[border], T.STEM_C, True)


# ------------------------------------------------------------------------------------------------ im2col / depth-wise convolutions
@pytest.mark.parametrize("B,Hin,C,stride", [(2, 512, 32, 2), (3, 7, 8, 1), (2, 10, 24, 2), (1, 1, 8, 1), (2, 2, 16, 2)])
def test_im2col(L, B, Hin, C, stride):
    x = T.rand((B * Hin * Hin, C), Hin + C, 1.0, device=DEV)
    Ho = Hin // stride
    got = run(L, "im2col", B * Ho * Ho * 9 * C, torch.bfloat16, x, B, Hin, C, stride, OUT)
    assert torch.equal(got.view(B * Ho * Ho, 9 * C), T.im2col_ref(x, B, Hin, C, stride))


DW_BF16 = [(256, 256, 1), (256, 128, 2), (128, 160, 2), (64, 320, 1), (7, 8, 1), (6, 24, 2)]


@pytest.mark.parametrize("Hin,C,stride", DW_BF16)
@pytest.mark.parametrize("act", [1, 0])
def test_dwconv_bf16(L, Hin, C, stride, act):
    B, Ho = 2, Hin // stride
    x = T.rand((B * Hin * Hin, C), Hin + C + stride, 1.0, device=DEV)
    w, b = T.make_dw(C, C + stride, DEV)
    got = run(L, "dwconv_bf16", B * Ho * Ho * C, torch.bfloat16, x, B, Hin, C, stride, w, b, act, OUT).view(B * Ho * Ho, C)
    ref, mag = T.dwconv_ref(x, B, Hin, C, stride, w, b, act)
    check_elems(f"dwconv bf16 {Hin}/{C}/s{stride} act={act}", got, ref, mag, T.DW_BF16_C, True)
    e = T.border_pixels(B, Ho, DEV)
    check_elems("  border rows / columns", got[e], ref[e], mag[e], T.DW_BF16_C, True)


@pytest.mark.parametrize("Hin,C", [(128, 128), (64, 160), (64, 320), (7, 4), (15, 12)])
def test_dwconv_f32(L, Hin, C):
    B = 2
    x = T.rand((B * Hin * Hin, C), Hin + C, 1.0, torch.float32, DEV)
    w, b = T.make_dw(C, C, DEV)
    got = run(L, "dwconv_f32", B * Hin * Hin * C, torch.float32, x, B, Hin, C, w, b, OUT).view(B * Hin * Hin, C)
    ref, mag = T.dwconv_ref(x, B, Hin, C, 1, w, b)
    check_elems(f"dwconv f32 {Hin}/{C}", got, ref, mag, T.DW_F32_C, False)
    e = T.border_pixels(B, Hin, DEV)
    check_elems("  border rows / columns", got[e], ref[e], mag[e], T.DW_F32_C, False)


# ------------------------------------------------------------------------------------------------ window LayerNorm
@pytest.mark.parametrize("H,D,ws", [(128, 128, 7), (64, 160, 14), (64, 320, 7), (14, 160, 14), (7, 64, 7), (15, 160, 14), (8, 384, 7)])
def test_ln_window(L, H, D, ws):
    B = 2
    x = T.rand((B * H * H, D), H + D, 1.0, torch.float32, DEV) + T.rand((B * H * H, 1), H + D + 1, 3.0, torch.float32, DEV)
    gamma, beta = T.make_ln(D, D + ws, DEV)
    nrows = B * T.n_windows(H, ws) ** 2 * ws * ws
    got = run(L, "ln_window", nrows * D, torch.bfloat16, x, B, H, D, ws, gamma, beta, 1e-5, OUT).view(nrows, D)
    ref = T.ln_window_ref(x, B, H, D, ws, gamma, beta)
    pad = T.pad_rows(B, H, ws, DEV)
    assert torch.equal(got[pad], beta.to(torch.bfloat16).expand(int(pad.sum()), -1)), "a pad row is not bf16(beta)"
    check_rows(f"ln_window H={H} D={D} ws={ws}", got, ref, nrows, T.TOL_LN)
    check_elems("  per element", got, ref, (ref - beta.double()).abs() + beta.double().abs(), T.LN_C, True)
    nw = T.n_windows(H, ws)
    last = torch.zeros(B, nw, nw, ws * ws, dtype=torch.bool, device=DEV)
    last[:, nw - 1] = True
    last[:, :, nw - 1] = True
    last = last.view(-1) & ~pad
    check_rows("  real rows of the edge windows", got[last], ref[last], int(last.sum()), T.TOL_LN)


# ------------------------------------------------------------------------------------------------ window attention
def run_attention(L, qkv, tab, B, H, ws, heads):
    return run(L, "attention", B * H * H * heads * 32, torch.bfloat16, qkv, tab, B, H, ws, heads, OUT).view(B * H * H, heads * 32)


def attention_case(L, name, qkv, tab, B, H, ws, heads, tol):
    got = run_attention(L, qkv, tab, B, H, ws, heads)
    ref = T.attention_ref(qkv, tab, B, H, ws, heads)
    check_rows(name, T.head_rows(got, heads), T.head_rows(ref, heads), B * H * H * heads, tol)
    e = T.edge_tokens(B, H, ws, DEV)
    check_rows("  queries of the edge windows", T.head_rows(got[e], heads), T.head_rows(ref[e], heads), int(e.sum()) * heads, tol)
    return got, ref


ATTN = [(128, 7, 4), (64, 14, 5), (64, 7, 10), (7, 7, 4), (14, 14, 5), (8, 7, 2), (15, 14, 5)]


@pytest.mark.parametrize("H,ws,heads", ATTN)
def test_attention(L, H, ws, heads):
    """Production (grid, window, heads) with B = 2, H = ws (no pad) and H = ws + 1 (one real row and column in the last
    windows); the pad rows of each window are one constant row, as in the model."""
    B = 2
    qkv = T.make_qkv(B, H, ws, heads, seed=H + ws + heads, device=DEV)
    tab = T.make_bias_tab(heads, ws, seed=heads, device=DEV)
    attention_case(L, f"attention H={H} ws={ws} heads={heads}", qkv, tab, B, H, ws, heads, T.TOL_ATTN)


@pytest.mark.parametrize("H,ws,heads", [(64, 7, 10), (64, 14, 5)])
def test_attention_bias_only(L, H, ws, heads):
    """q = 0: the logits are the bias table alone, a different table per head (heads swapped or the index transposed would
    show)."""
    B = 1
    qkv = T.make_qkv(B, H, ws, heads, seed=5 + heads, device=DEV)
    qkv.view(-1, heads, 3, 32)[:, :, 0] = 0
    tab = T.make_bias_tab(heads, ws, seed=6, scale=2.0, device=DEV)
    attention_case(L, f"bias only H={H} ws={ws}", qkv, tab, B, H, ws, heads, T.TOL_ATTN_PLANTED)


@pytest.mark.parametrize("H,ws,heads", [(64, 7, 10), (64, 14, 5)])
def test_attention_uniform(L, H, ws, heads):
    """q = 0 and a zero table: every query's output is the mean of its window's V rows, the pad keys' V included."""
    B = 1
    qkv = T.make_qkv(B, H, ws, heads, seed=8 + ws, device=DEV)
    qkv.view(-1, heads, 3, 32)[:, :, 0] = 0
    tab = torch.zeros(heads, ws * ws, device=DEV)
    got, ref = attention_case(L, f"uniform H={H} ws={ws}", qkv, tab, B, H, ws, heads, T.TOL_ATTN_PLANTED)
    v = qkv.view(-1, ws * ws, heads, 3, 32)[:, :, :, 2].double().mean(1)                  # [windows, heads, 32]
    mean_v = T.unpartition(v.reshape(-1, 1, heads * 32).expand(-1, ws * ws, -1).reshape(-1, heads * 32), B, H, ws)
    assert float((ref - mean_v).abs().max()) < 1e-12
    # fp32 sum of ws * ws terms, then one bf16 rounding
    bound = T.bf16_ulp(mean_v) + T.F32_SUM_C * ws * ws * qkv.view(-1, ws * ws, heads, 3, 32)[:, :, :, 2].double().abs().mean()
    assert bool(((got.double() - mean_v).abs() <= bound).all()), "uniform attention is not the mean of V"


@pytest.mark.parametrize("ws,key", [(7, 0), (7, 48), (14, 100), (14, 195)])
def test_attention_one_key_dominates(L, ws, key):
    """q = u + noise, k = gain[key] u with one key leading by about 40 in the exponent: the output is that key's V row, bit for
    bit (first, middle and last key of the online softmax's 4-key chunks, incl. the partial last chunk of 49 keys)."""
    B, H, heads = 1, 2 * ws + 1, 3
    N = ws * ws
    rows = B * T.n_windows(H, ws) ** 2 * N
    qkv = torch.empty(rows, heads, 3, 32, device=DEV, dtype=torch.bfloat16)
    qkv[:, :, 0] = 1.0 + T.rand((rows, heads, 32), 61 + key, 0.25, device=DEV)
    gain = torch.zeros(N)
    gain[key] = 40.0 / (32 * T.SCALE)
    qkv[:, :, 1] = gain.to(DEV).repeat(rows // N)[:, None, None].to(torch.bfloat16)
    qkv[:, :, 2] = T.rand((rows, heads, 32), 62 + key, 4.0, device=DEV)
    qkv = qkv.view(rows, heads * 96)
    tab = torch.zeros(heads, N, device=DEV)
    got, _ = attention_case(L, f"dominant key {key} ws={ws}", qkv, tab, B, H, ws, heads, T.TOL_ATTN_PLANTED)
    v = qkv.view(-1, N, heads, 3, 32)[:, key, :, 2].reshape(-1, 1, heads * 32)           # one V row per window
    want = T.unpartition(v.expand(-1, N, -1).reshape(rows, heads * 32), B, H, ws)
    assert torch.equal(got, want), "the output is not the dominant key's V row"


@pytest.mark.parametrize("H,ws,heads", [(64, 14, 5), (15, 7, 4)])
def test_attention_per_image_invariance(L, H, ws, heads):
    """Image b of a batch is bit-identical to the same image run alone, and a repeat is bit-identical."""
    B = 3
    qkv = T.make_qkv(B, H, ws, heads, seed=71, device=DEV)
    tab = T.make_bias_tab(heads, ws, seed=72, device=DEV)
    got = run_attention(L, qkv, tab, B, H, ws, heads)
    assert torch.equal(got, run_attention(L, qkv, tab, B, H, ws, heads)), "repeat differs"
    per = qkv.shape[0] // B
    for b in range(B):
        alone = run_attention(L, qkv[b * per:(b + 1) * per].contiguous(), tab, 1, H, ws, heads)
        assert torch.equal(got[b * H * H:(b + 1) * H * H], alone), f"image {b} differs from the same image run alone"


# ------------------------------------------------------------------------------------------------ rejections
@pytest.mark.parametrize("call", ["stem odd img", "stem image > img", "stem both inputs", "im2col C % 8", "im2col odd Hin stride 2",
                                  "dwconv_bf16 stride 3", "dwconv_f32 C % 4", "ln D > 384", "ln D % 4", "ln ws 8", "attention ws 9",
                                  "null pointer"])
def test_rejects_bad_arguments(L, call):
    """Every precondition the kernels assume without checking is refused on the host: -1 with a message, nothing launched,
    nothing written."""
    lib, st = L.lib(), L.cur_stream()
    x = torch.zeros(1 << 16, device=DEV)
    p = L.ptr(x)
    n0 = L.launch_count()
    rc = {"stem odd img": lambda: lib.msam_op_tv_stem(p, None, 1, 7, 7, 7, p, p, p, st),
          "stem image > img": lambda: lib.msam_op_tv_stem(p, None, 1, 9, 8, 8, p, p, p, st),
          "stem both inputs": lambda: lib.msam_op_tv_stem(p, p, 1, 8, 8, 8, p, p, p, st),
          "im2col C % 8": lambda: lib.msam_op_tv_im2col(p, 1, 8, 12, 1, p, st),
          "im2col odd Hin stride 2": lambda: lib.msam_op_tv_im2col(p, 1, 7, 8, 2, p, st),
          "dwconv_bf16 stride 3": lambda: lib.msam_op_tv_dwconv_bf16(p, 1, 9, 8, 3, p, p, 0, p, st),
          "dwconv_f32 C % 4": lambda: lib.msam_op_tv_dwconv_f32(p, 1, 8, 6, p, p, p, st),
          "ln D > 384": lambda: lib.msam_op_tv_ln_window(p, 1, 7, 388, 7, p, p, 1e-5, p, st),
          "ln D % 4": lambda: lib.msam_op_tv_ln_window(p, 1, 7, 66, 7, p, p, 1e-5, p, st),
          "ln ws 8": lambda: lib.msam_op_tv_ln_window(p, 1, 8, 64, 8, p, p, 1e-5, p, st),
          "attention ws 9": lambda: lib.msam_op_tv_attention(p, p, 1, 9, 9, 1, p, st),
          "null pointer": lambda: lib.msam_op_tv_attention(p, None, 1, 7, 7, 1, p, st)}[call]()
    torch.cuda.synchronize()
    assert rc == -1 and lib.msam_last_error() and L.launch_count() == n0, call
    assert bool((x == 0).all())
