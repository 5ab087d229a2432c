"""Time the fused up-scaling + hyper-product block (msam_op_dec_upscale, kernel upscale_fused) at the production AMG chunk
of P = 1024 prompts, with multimask (nm = 3) and without (nm = 1).

    python tests/time_upscale.py [--lib PATH] [--iters 100] [--warmup 10]

Prints one JSON line: per nm the mean ms per launch over CUDA events around `--iters` back-to-back launches (after
`--warmup` launches), the algorithmic TFLOP/s and GB/s (the operation and byte counts of prof_begin in upscale_fused.cu)
and their fractions of the H100 SXM data-sheet peaks, plus the GPU name, power limit and max SM clock.  `--lib` loads
another build of libmsam_b200.so, so that two builds can be timed alternately in one session.  Inputs are seeded;
nothing is written to the tree.  Not a test (no test_ prefix): it needs a GPU and only measures.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0   # H100 SXM data sheet: dense bf16 / fp16, HBM3


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
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters must be at least 50")

    sys.path.insert(0, ROOT)
    import torch
    from micro_sam_b200 import _lib, util
    from oracle import sam_ref
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        raise SystemExit("time_upscale.py needs a CUDA device")
    torch.cuda.set_device(0)

    P = args.prompts
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    sam = util.get_sam_model("vit_test", device="cuda:0", state_dict=sd, max_batch=1, max_prompts=P).model
    g = torch.Generator(device="cuda").manual_seed(7)
    keys = torch.randn(P * 4096, 256, device="cuda", generator=g).to(torch.bfloat16)
    hyper = torch.randn(P, 4, 32, device="cuda", generator=g) * 0.5
    L = _lib.lib()
    res = {"lib": _lib.LIB_PATH, "prompts": P, "iters": args.iters, **gpu_info()}
    for multimask, nm in ((True, 3), (False, 1)):
        out = torch.empty(P, nm, 256, 256, device="cuda")

        def launch():
            _lib.check(L.msam_op_dec_upscale(sam._h, _lib.ptr(keys), _lib.ptr(hyper), P, int(multimask), _lib.ptr(out), 0,
                                             _lib.cur_stream()))

        for _ in range(args.warmup):
            launch()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.iters):
            launch()
        t1.record()
        t1.synchronize()
        ms = t0.elapsed_time(t1) / args.iters
        flops = P * 4096 * (2.0 * 256 * 256 + 4 * 2.0 * 128 * 64 + 2.0 * 512 * nm)
        nbytes = P * (4096.0 * 256 * 2 + 65536.0 * 4 * nm)
        tflops, gbs = flops / ms * 1e-9, nbytes / ms * 1e-6
        res[f"nm{nm}"] = {"ms": round(ms, 4), "tflops": round(tflops, 1), "gb_s": round(gbs, 1),
                          "frac_peak_tflops": round(tflops / PEAK_TFLOPS, 3), "frac_peak_gb_s": round(gbs / PEAK_GBS, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
