"""Time the fused image -> token block (msam_op_dec_i2t, kernel i2t_fused) at the production AMG chunk of P = 1024
prompts with T = 7 tokens each, in both modes the AMG step runs: layer 0 on the shared image (l0_shared) and layer 1 on
each prompt's own keys, updated in place (l1_inplace).

    python tests/time_i2t.py [--lib PATH] [--iters 100] [--warmup 10]

Prints one JSON line: per mode the mean ms per launch of the i2t_fused kernel alone (the library's CUDA-event profile,
msam_profile / profile_report: the entry point also runs the small Mq / V' GEMMs, which are left out), the GB/s of the
kernel's algorithmic bytes (those of prof_begin in i2t_fused.cu) and their fraction of the H100 SXM data-sheet HBM3
bandwidth, plus the GPU name, power limit and max SM clock.  `--lib` loads another build of libmsam_b200.so, so that two
builds can be timed alternately in one session.  Inputs are seeded; nothing is written to the tree.  Not a test (no test_
prefix): it needs a GPU and only measures.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_GBS = 3350.0   # H100 SXM data sheet: HBM3
MODES = {"l0_shared": (0, 1, "i2t_fused (shared image)"), "l1_inplace": (1, 0, "i2t_fused (own keys)")}   # layer, shared


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
    if not 5 <= args.tokens <= 8:
        ap.error("--tokens must be in [5, 8] (the fused kernel's range)")

    sys.path.insert(0, ROOT)
    import torch
    from micro_sam_b200 import _lib, util
    from oracle import sam_ref
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    if not torch.cuda.is_available():
        raise SystemExit("time_i2t.py needs a CUDA device")
    torch.cuda.set_device(0)

    P, T = args.prompts, args.tokens
    sd = sam_ref.seeded_state_dict("vit_test", seed=1)
    sam = util.get_sam_model("vit_test", device="cuda:0", state_dict=sd, max_batch=1, max_prompts=P).model
    g = torch.Generator(device="cuda").manual_seed(7)
    sam.bind_embedding(torch.randn(1, 256, 64, 64, device="cuda", generator=g))
    q = torch.randn(P * T, 256, device="cuda", generator=g).to(torch.bfloat16)
    qpe = (q.float() + 0.5 * torch.randn(P * T, 256, device="cuda", generator=g)).to(torch.bfloat16)
    keys = torch.randn(P * 4096, 256, device="cuda", generator=g).to(torch.bfloat16)
    L = _lib.lib()
    res = {"lib": _lib.LIB_PATH, "prompts": P, "tokens": T, "iters": args.iters, **gpu_info()}
    for mode, (layer, shared, kname) in MODES.items():
        def launch():
            _lib.check(L.msam_op_dec_i2t(sam._h, layer, _lib.ptr(q), _lib.ptr(qpe), shared, _lib.ptr(keys), P, T, 0,
                                         _lib.cur_stream()))

        for _ in range(args.warmup):
            launch()
        torch.cuda.synchronize()
        L.msam_profile(1)
        for _ in range(args.iters):
            launch()
        rep = [r for r in _lib.profile_report() if r["name"] == kname]
        L.msam_profile(0)
        if len(rep) != 1 or rep[0]["n"] != args.iters:
            raise SystemExit(f"expected {args.iters} launches of '{kname}' in the profile, got {rep}")
        ms = rep[0]["ms"] / args.iters
        gbs = rep[0]["bytes"] / args.iters / ms * 1e-6
        res[mode] = {"kernel_ms": round(ms, 4), "gb_s": round(gbs, 1), "frac_peak_gb_s": round(gbs / PEAK_GBS, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
