"""Time the fused token -> image attention block (msam_op_dec_t2i, kernel t2i_fused) at the production AMG chunk of
P = 1024 prompts, for the three instances a decode runs: layer 0 on the shared image (l0_shared), layer 1 on each prompt's
own keys (l1_own) and the final attention on own keys (final_own).

    python tests/time_t2i.py [--lib PATH] [--tokens 7] [--iters 100] [--warmup 10]

Prints one JSON line: per instance the mean ms per launch of the t2i_fused kernel alone (the library's CUDA-event profile,
msam_profile / profile_report; the entry point also runs the q projection, the Q' prep / GEMM and the per-head value
projection, which are left out), and the TFLOP/s and GB/s of the kernel's algorithmic counts (those of prof_begin in
t2i_fused.cu) with their fractions of the H100 SXM data-sheet peaks, plus the GPU name, power limit and max SM clock.
Profile entries are matched by the prefix "t2i_fused", so a build with other t2i_fused launch names can be timed with
`--lib` as well.  --tokens 9..16 times the one-prompt-per-item path.  Inputs are seeded; nothing is written to the tree.
Not a test (no test_ prefix): it needs a GPU and only measures.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_GBS = 3350.0     # H100 SXM data sheet: HBM3
PEAK_TFLOPS = 989.0   # H100 SXM data sheet: dense bf16
INSTANCES = {"l0_shared": (0, False), "l1_own": (1, True), "final_own": (2, True)}   # which, own keys


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        vals = [v.strip() for v in r.stdout.strip().split(",")]
        return dict(zip(("gpu", "power_limit", "sm_clock_max"), vals)) if len(vals) == 3 else {"nvidia_smi": r.stdout.strip()}
    except (OSError, subprocess.SubprocessError) as e:
        return {"nvidia_smi": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libmsam_b200.so to load instead of the in-tree build")
    ap.add_argument("--prompts", type=int, default=1024)
    ap.add_argument("--tokens", type=int, default=7)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters must be at least 50")
    if not 5 <= args.tokens <= 16:
        ap.error("--tokens must be in [5, 16] (the decoder's range)")

    sys.path.insert(0, ROOT)
    import torch
    from micro_sam_b200 import _lib, util
    from oracle import sam_ref
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        raise SystemExit("time_t2i.py needs a CUDA device")
    torch.cuda.set_device(0)

    P, T = args.prompts, args.tokens
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    sam = util.get_sam_model("vit_test", device="cuda:0", state_dict=sd, max_batch=1, max_prompts=P).model
    g = torch.Generator(device="cuda").manual_seed(7)
    sam.bind_embedding(torch.randn(1, 256, 64, 64, device="cuda", generator=g))
    qpe = torch.randn(P * T, 256, device="cuda", generator=g).to(torch.bfloat16)
    keys = torch.randn(P * 4096, 256, device="cuda", generator=g).to(torch.bfloat16)
    out = torch.empty(P * T, 128, device="cuda", dtype=torch.bfloat16)
    L = _lib.lib()
    res = {"lib": _lib.LIB_PATH, "prompts": P, "tokens": T, "iters": args.iters, **gpu_info()}
    for inst, (which, own) in INSTANCES.items():
        def launch():
            _lib.check(L.msam_op_dec_t2i(sam._h, which, _lib.ptr(qpe), _lib.ptr(keys) if own else None, P, T,
                                         _lib.ptr(out), 0, _lib.cur_stream()))

        for _ in range(args.warmup):
            launch()
        torch.cuda.synchronize()
        L.msam_profile(1)
        for _ in range(args.iters):
            launch()
        rep = [r for r in _lib.profile_report() if r["name"].startswith("t2i_fused")]
        L.msam_profile(0)
        if len(rep) != 1 or rep[0]["n"] != args.iters:
            raise SystemExit(f"expected {args.iters} launches of one t2i_fused kernel in the profile, got {rep}")
        r = rep[0]
        ms = r["ms"] / args.iters
        tflops = r["flops"] / args.iters / ms * 1e-9
        gbs = r["bytes"] / args.iters / ms * 1e-6
        res[inst] = {"kernel": r["name"], "kernel_ms": round(ms, 4), "tflop_s": round(tflops, 1),
                     "frac_peak_tflop_s": round(tflops / PEAK_TFLOPS, 3), "gb_s": round(gbs, 1),
                     "frac_peak_gb_s": round(gbs / PEAK_GBS, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
