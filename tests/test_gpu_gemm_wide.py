"""The wide-tile GEMM (gemm.cu:gemm_wide_kernel, 128 x 256 tiles, wgmma m64n256 per 64-row half) against the float64
references of tests/encoder_ops_ref.py, with the per-element bounds of test_gpu_encoder_ops.py (run_gemm / gemm_case there,
called through msam_op_gemm_ex2 with an explicit kernel path):
  * every GEMM of the ViT encoder forward of vit_b / vit_l / vit_h at the benchmark's row counts, with its epilogue;
  * tails: rows that do not fill a tile, K down to 8 (the TMA box zero-fills the K tail), pitched lda / ldw / ldc / ldr;
  * every epilogue combination, and the residual stream updated in place (out aliasing the residual);
  * the output does not depend on the number of CTAs of the persistent grid;
  * the tiled kernel and the wide one on the same inputs: each output element sums the same k16 chunks in the same order, so
    the two are expected to agree bit for bit (the PTX ISA does not promise it across MMA shapes; each case prints what
    it found and bounds both against float64);
  * the default dispatch (wide tiles for the large products only) and the host-side rejections of a forced path.
"""
import ctypes

import pytest
import torch

from tests import encoder_ops_ref as R
from tests.encoder_ops_ref import SENT_BF16, SENT_F32
from tests.test_gpu_encoder_ops import gemm_case, rand, run_gemm

pytestmark = pytest.mark.gpu
DEV = "cuda"
AUTO, TILED, WIDE = 0, 1, 2   # msam_op_gemm_ex2 paths


class PathLib:
    """The _lib module as run_gemm / gemm_case use it, with msam_op_gemm_ex routed to msam_op_gemm_ex2 on one path."""

    def __init__(self, mod, path):
        self.mod, self.path = mod, path

    def lib(self):
        return self

    def msam_op_gemm_ex(self, *args):
        return self.mod.lib().msam_op_gemm_ex2(*args[:-1], self.path, args[-1])

    def msam_last_error(self):
        return self.mod.lib().msam_last_error()

    def cur_stream(self):
        return self.mod.cur_stream()

    def launch_count(self):
        return self.mod.launch_count()


@pytest.fixture(scope="module")
def lib_mod():
    from micro_sam_b200 import _lib
    _lib.lib()
    return _lib


@pytest.fixture(scope="module")
def wide(lib_mod):
    return PathLib(lib_mod, WIDE)


@pytest.fixture(scope="module")
def tiled(lib_mod):
    return PathLib(lib_mod, TILED)


def compare_paths(name, got_wide, got_tiled):
    """True if bit-identical; prints the largest difference relative to the largest magnitude otherwise."""
    if torch.equal(got_wide, got_tiled):
        print(f"  {name}: wide and tiled kernels bit-identical", flush=True)
        return True
    d = (got_wide.double() - got_tiled.double()).abs()
    print(f"  {name}: wide vs tiled: {int((d > 0).sum())} elements differ, max |diff| {float(d.max()):.3e} "
          f"(max |out| {float(got_tiled.double().abs().max()):.3e})", flush=True)
    return False


# ------------------------------------------------------------------------------------------------ encoder products
def encoder_products(D, M, Mw):
    """Every GEMM of Engine::vit_forward at embed dim D with M image tokens (Mw window-partitioned rows incl. padding), with the
    epilogue it runs: (name, M, N, K, run_gemm keywords)."""
    return [("patch_embed", M, D, 768, dict(res="f32", res_rows=4096)),
            ("qkv global", M, 3 * D, D, dict(f32=False)),
            ("qkv windowed", Mw, 3 * D, D, dict(f32=False)),
            ("proj", M, D, D, dict(res="f32")),
            ("fc1 + GELU", M, 4 * D, D, dict(act=1, f32=False)),
            ("fc2", M, D, 4 * D, dict(res="f32")),
            ("neck conv1", M, 256, D, dict(bias=False)),
            ("neck conv2", M, 256, 9 * 256, dict(bias=False))]


# bench.py runs vit_b at 16 tiles per step (65 536 tokens, 78 400 window rows) and the ViT-H line at batch 8
ENCODER_CASES = ([("vit_b", *c) for c in encoder_products(768, 65536, 78400)] +
                 [("vit_l", *c) for c in encoder_products(1024, 32768, 39200)] +
                 [("vit_h", *c) for c in encoder_products(1280, 32768, 39200)])


def deep_k_case(L, name, M, N, K, seed, **kw):
    """gemm_case for plain epilogues at any K: the fp32-accumulation term of the bound, C x magnitude with C set for K <= 768
    (encoder_ops_ref.GEMM_F32_C), grows in proportion to the number of accumulated products (the classical gamma_K bound),
    so it is scaled by K / 768 above that: fc2 and the 3x3 neck conv reduce over K = 2304 .. 5120."""
    rc, got, ops, _ = run_gemm(L, M, N, K, seed, **kw)
    assert rc == 0, L.lib().msam_last_error().decode()
    ref, _ = R.gemm_ref(**ops)
    mag = R.gemm_magnitude(ops["A"], ops["W"], ops["bias"], ops["residual"], ops["res_rows"])
    err = (got.double() - ref).abs()
    bound = R.GEMM_F32_C * max(1.0, K / 768) * mag
    if got.dtype == torch.bfloat16:
        bound = bound + R.bf16_ulp(ref) + (R.GEMM_GELU_FAST if ops["act"] == 1 and not ops["act_after_res"] else 0.0)
        err = (err - R.bf16_ulp(ref)).clamp_min(0)
    print(f"  {name}: {'bf16' if got.dtype == torch.bfloat16 else 'fp32'} out, max err (above one ulp) / magnitude "
          f"{float((err / mag).max()):.3e}", flush=True)
    assert bool(torch.isfinite(got).all())
    bad = ((got.double() - ref).abs() > bound).nonzero()
    assert len(bad) == 0, f"{name}: {len(bad)} elements beyond their bound, first (row, col) {bad[:8].tolist()}"
    return got


@pytest.mark.parametrize("arch,name,M,N,K,kw", ENCODER_CASES, ids=[f"{c[0]}-{c[1]}" for c in ENCODER_CASES])
def test_wide_encoder_products(wide, tiled, arch, name, M, N, K, kw):
    seed = M + N + K
    got = deep_k_case(wide, f"{arch} {name} M={M} N={N} K={K}", M, N, K, seed, **kw)
    ref_tiled = run_gemm(tiled, M, N, K, seed, **kw)[1]
    compare_paths(f"{arch} {name}", got, ref_tiled)


# ------------------------------------------------------------------------------------------------ tails and pitches
TAILS = [(M, N, K) for M in (1, 127, 129, 9800) for N in (256, 768) for K in (8, 72, 200)]


@pytest.mark.parametrize("M,N,K", TAILS)
def test_wide_tails_and_pitches(wide, tiled, M, N, K):
    """Partial row tiles, K tails inside one 64-deep block, and row pitches above the minimum on every operand."""
    f32 = (M + K) % 2 == 0
    kw = dict(pads=(16, 8, 6, 4), res="f32" if f32 else "bf16", f32=f32)
    got = gemm_case(wide, f"wide M={M} N={N} K={K} pitched", M, N, K, seed=M + N + K, **kw)
    compare_paths(f"M={M} N={N} K={K}", got, run_gemm(tiled, M, N, K, M + N + K, **kw)[1])


# ------------------------------------------------------------------------------------------------ epilogues
@pytest.mark.parametrize("f32", [True, False], ids=["f32", "bf16"])
@pytest.mark.parametrize("res,res_rows", [("f32", 0), ("bf16", 0), ("f32", 100), ("bf16", 64)])
@pytest.mark.parametrize("act,after", [(0, 0), (1, 0), (2, 0), (1, 1), (2, 1)])
def test_wide_epilogues(wide, tiled, res, res_rows, act, after, f32):
    """fp32 and bf16 residual, the row-modulus broadcast (pos-embed), GELU / ReLU before the residual and after it."""
    kw = dict(res=res, res_rows=res_rows, act=act, after=after, f32=f32)
    got = gemm_case(wide, f"wide res={res} res_rows={res_rows} act={act} after={after}", 257, 512, 200, seed=5 + act + after, **kw)
    compare_paths("epilogue", got, run_gemm(tiled, 257, 512, 200, 5 + act + after, **kw)[1])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("M,N,K", [(9800, 768, 768), (300, 256, 3072)])
def test_wide_residual_in_place(lib_mod, M, N, K, dtype):
    """out == residual (the residual stream of proj / fc2): every element is read before it is written."""
    A, W = rand((M, K), 11, 0.5), rand((N, K), 12, K ** -0.5)
    b = rand((N,), 13, 1.0, torch.float32)
    x = rand((M, N), 14, 1.0, dtype)
    x0 = x.clone()
    ref, _ = R.gemm_ref(A, W, bias=b, residual=x0)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    f32 = int(dtype == torch.float32)
    rc = lib_mod.lib().msam_op_gemm_ex2(vp(A), vp(W), M, N, K, K, K, vp(b), vp(x), 0, 0, 1 - f32, vp(x), 0, f32, 0, 0, 0,
                                        None, None, 1e-5, 0, WIDE, lib_mod.cur_stream())
    torch.cuda.synchronize()
    assert rc == 0, lib_mod.lib().msam_last_error().decode()
    bound = R.GEMM_F32_C * R.gemm_magnitude(A, W, b, x0) + (0.0 if f32 else R.bf16_ulp(ref))
    err = (x.double() - ref).abs()
    print(f"  in place {dtype}: max err / bound {float((err / bound).max()):.3f}", flush=True)
    assert bool((err <= bound).all())


# ------------------------------------------------------------------------------------------------ grid, paths, dispatch
@pytest.mark.parametrize("f32", [True, False], ids=["f32", "bf16"])
def test_wide_independent_of_grid_size(wide, f32):
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    outs = [run_gemm(wide, 1000, 768, 200, seed=3, f32=f32, res="bf16", act=1, num_sms=s)[1] for s in (1, 2, 7, n_sm, 0)]
    assert all(torch.equal(outs[0], o) for o in outs[1:]), "the output depends on the number of CTAs"


def test_default_dispatch(lib_mod):
    """Without a path, large plain products with N % 256 == 0 run the wide kernel; small ones, N % 256 != 0 and the fused
    LayerNorm stay on the tiled kernel; both give the forced paths' results."""
    L = lib_mod.lib()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    m_fill = 128 * ((n_sm + 2) // 3)   # N = 768: 3 tiles per 128-row block
    cases = [(m_fill, 768, 200, False, "gemm_wide"), (m_fill - 128, 768, 200, False, "gemm_bf16"),
             (8192, 384, 200, False, "gemm_bf16"), (8192, 256, 200, True, "gemm_bf16<256,ln256>")]
    for M, N, K, ln, want in cases:
        L.msam_profile(1)
        got = run_gemm(PathLib(lib_mod, AUTO), M, N, K, seed=7, f32=False, ln=ln)[1]
        names = [r["name"] for r in lib_mod.profile_report()]
        L.msam_profile(0)
        assert len(names) == 1 and names[0].startswith(want), f"M={M} N={N}: ran {names}, expected {want}"
        forced = run_gemm(PathLib(lib_mod, WIDE if want == "gemm_wide" else TILED), M, N, K, seed=7, f32=False, ln=ln)[1]
        assert torch.equal(got, forced)


@pytest.mark.parametrize("what,path,kw", [("wide with N % 256", WIDE, dict(N=384)),
                                          ("wide with the LayerNorm epilogue", WIDE, dict(N=256, ln=True, f32=False)),
                                          ("unknown path", 3, dict(N=256))])
def test_forced_path_rejections(lib_mod, what, path, kw):
    """Host-side rejections: -1 with a message, nothing launched, the output untouched."""
    N = kw.pop("N")
    n0 = lib_mod.launch_count()
    rc, _, _, buf = run_gemm(PathLib(lib_mod, path), 64, N, 64, seed=1, **kw)
    assert rc == -1 and lib_mod.lib().msam_last_error(), what
    assert lib_mod.launch_count() == n0, f"{what}: a kernel was launched"
    assert bool((buf == (SENT_F32 if buf.dtype == torch.float32 else SENT_BF16)).all()), f"{what}: the output was written"
