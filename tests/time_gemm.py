"""Time the encoder GEMMs on both kernels of gemm.cu: the tiled kernel (gemm_bf16_kernel, msam_op_gemm_ex2 path 1) and the
wide-tile kernel (gemm_wide_kernel, path 2), for every linear layer of the vit_b and vit_h encoder forward at the
benchmark's row counts (vit_b: 16 images = 65 536 tokens, 78 400 window rows; vit_h: 8 images), each with the epilogue it
runs in Engine::vit_forward.

    python tests/time_gemm.py [--lib PATH] [--iters 50] [--warmup 5] [--rounds 3] [--arch vit_b vit_h]

Per shape and path: CUDA events around `iters` back-to-back launches, `rounds` rounds with the two paths alternating; the
median round gives ms per launch, algorithmic TFLOP/s (2 M N K) and its fraction of the H100 SXM data-sheet dense bf16 peak.
Per architecture also the GEMM time of one encoder forward (each product times the number of times a forward runs it).
Prints one JSON line with the GPU name, power limit and max SM clock read in the same run.  Inputs are seeded; nothing is
written to the tree.  Not a test (no test_ prefix): it needs a GPU and only measures.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_TFLOPS = 989.0   # H100 SXM data sheet: dense bf16
PATHS = {"tiled": 1, "wide": 2}
# embed dim, depth, images, window rows per image (25 windows of 14 x 14)
ARCHS = {"vit_b": (768, 12, 16, 4900), "vit_h": (1280, 32, 8, 4900)}
N_GLOBAL = 4   # global-attention blocks of every ViT-SAM encoder


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        return dict(zip(("gpu", "power_limit", "sm_clock_max"), vals)) if len(vals) == 3 else {"nvidia_smi": r.stdout.strip()}
    except (OSError, subprocess.SubprocessError) as e:
        return {"nvidia_smi": str(e)}


def products(D, depth, nb, tw):
    """(name, M, N, K, epilogue, launches per encoder forward); epilogue = (bias, residual, res_rows, act, out_fp32)."""
    M, Mw = nb * 4096, nb * tw
    return [("patch_embed", M, D, 768, (True, True, 4096, 0, True), 1),
            ("qkv global", M, 3 * D, D, (True, False, 0, 0, False), N_GLOBAL),
            ("qkv windowed", Mw, 3 * D, D, (True, False, 0, 0, False), depth - N_GLOBAL),
            ("proj", M, D, D, (True, True, 0, 0, True), depth),
            ("fc1 + GELU", M, 4 * D, D, (True, False, 0, 1, False), depth),
            ("fc2", M, D, 4 * D, (True, True, 0, 0, True), depth),
            ("neck conv1", M, 256, D, (False, False, 0, 0, True), 1),
            ("neck conv2", M, 256, 2304, (False, False, 0, 0, True), 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libmsam_b200.so to load instead of the in-tree build")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--arch", nargs="+", default=list(ARCHS), choices=list(ARCHS))
    args = ap.parse_args()
    if args.iters < 20:
        ap.error("--iters must be at least 20")

    sys.path.insert(0, ROOT)
    import torch
    from micro_sam_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        raise SystemExit("time_gemm.py needs a CUDA device")
    torch.cuda.set_device(0)
    L = _lib.lib()
    vp = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())   # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(5)
    res = {"lib": _lib.LIB_PATH, "iters": args.iters, "rounds": args.rounds, **gpu_info()}

    for arch in args.arch:
        D, depth, nb, tw = ARCHS[arch]
        out_arch = {}
        forward_ms = {p: 0.0 for p in PATHS}
        for name, M, N, K, (has_bias, has_res, res_rows, act, f32), count in products(D, depth, nb, tw):
            A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
            W = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
            bias = torch.randn(N, device="cuda", generator=g) if has_bias else None
            out = torch.randn(M, N, device="cuda", generator=g).to(torch.float32 if f32 else torch.bfloat16)
            resid = out[:res_rows] if (has_res and res_rows) else (out if has_res else None)   # in place, as the encoder runs it

            def launch(path):
                _lib.check(L.msam_op_gemm_ex2(vp(A), vp(W), M, N, K, K, K, vp(bias), vp(resid), res_rows, 0, 0, vp(out), 0,
                                              int(f32), act, 0, 0, None, None, 1e-5, 0, path, _lib.cur_stream()))

            times = {p: [] for p in PATHS}
            for p in PATHS.values():
                for _ in range(args.warmup):
                    launch(p)
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for pname, p in PATHS.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        launch(p)
                    e1.record()
                    e1.synchronize()
                    times[pname].append(e0.elapsed_time(e1) / args.iters)
            flop = 2.0 * M * N * K
            row = {"M": M, "N": N, "K": K, "per_forward": count}
            for pname in PATHS:
                ms = statistics.median(times[pname])
                tf = flop / ms * 1e-9
                row[pname] = {"ms": round(ms, 4), "tflop_s": round(tf, 1), "frac_peak": round(tf / PEAK_TFLOPS, 3),
                              "spread_ms": round(max(times[pname]) - min(times[pname]), 4)}
                forward_ms[pname] += count * ms
            row["speedup"] = round(row["tiled"]["ms"] / row["wide"]["ms"], 3)
            out_arch[name] = row
            del A, W, bias, out, resid
        out_arch["forward_gemm_ms"] = {p: round(v, 3) for p, v in forward_ms.items()}
        out_arch["forward_gemm_ms"]["speedup"] = round(forward_ms["tiled"] / forward_ms["wide"], 3)
        res[arch] = out_arch
    print(json.dumps(res))


if __name__ == "__main__":
    main()
