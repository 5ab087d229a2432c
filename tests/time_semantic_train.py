"""Times the semantic fine-tuning loss on the device (csrc/semantic_loss.cu): msam_semantic_loss_stats and
msam_semantic_loss_backward on their own (CUDA events over many launches) and compute_semantic_loss + loss.backward() end to end,
at B = 2, C = 3, originals 512^2 and 1024^2.  Rates are the algorithmic bytes (low-res logits and labels read, d low_res written)
over kernel time, against the H100 SXM data sheet's 3.35 TB/s; `moved` adds the backward pass's full-resolution intermediates.
Prints one JSON line per case, with the card's name and power limit read in the same run (and appends them to --out when given).
Usage:  python tests/time_semantic_train.py [--reps 50] [--out path.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import _lib, training  # noqa: E402
from micro_sam_b200.sam import get_preprocess_shape  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def cuda_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def case(B, C, H, W, reps, card):
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(0)
    low = torch.randn(B, C, 256, 256, device="cuda", generator=g) * 4
    lab = torch.randint(0, C, (B, H, W), device="cuda", generator=g)
    in_h, in_w = get_preprocess_shape(H, W, 1024)
    n = int(L.msam_semantic_loss_workspace(B, C, in_h, in_w, H, W, 1))
    ws = torch.empty(n, device="cuda", dtype=torch.uint8)
    st = torch.empty(3 * C + 3, device="cuda", dtype=torch.float64)
    ds = torch.randn(3 * C + 3, device="cuda", dtype=torch.float64, generator=g)
    d_lr = torch.empty_like(low)
    p, s = _lib.ptr, _lib.cur_stream()

    def stats():
        _lib.check(L.msam_semantic_loss_stats(p(low), p(lab), 1, B, C, in_h, in_w, H, W, p(ws), n, p(st), s))

    def backward():
        _lib.check(L.msam_semantic_loss_backward(p(low), p(lab), 1, p(ds), B, C, in_h, in_w, H, W, p(ws), n, p(d_lr), s))

    def step():
        x = low.clone().requires_grad_(True)
        training.compute_semantic_loss(x, lab, C).backward()

    t_stats, t_bwd, t_step = cuda_ms(stats, reps), cuda_ms(backward, reps), cuda_ms(step, max(1, reps // 5))
    lr_bytes, lab_bytes = B * C * 65536 * 4, B * H * W * 8
    stats_bytes = lr_bytes + lab_bytes
    bwd_bytes = 2 * lr_bytes + lab_bytes
    bc4 = B * C * 4   # each intermediate is written once and read once
    bwd_moved = bwd_bytes + 2 * bc4 * (H * W + in_h * 256 + (0 if (in_h, in_w) == (H, W) else H * in_w + in_h * in_w))
    return {"case": f"B{B}_C{C}_{H}x{W}", **card, "input_size": [in_h, in_w],
            "stats_ms": round(t_stats, 4), "backward_ms": round(t_bwd, 4), "loss_and_backward_end_to_end_ms": round(t_step, 4),
            "stats_GBps": round(stats_bytes / t_stats / 1e6, 1), "stats_share_of_hbm": round(stats_bytes / t_stats / 1e-3 / HBM_BYTES_PER_S, 4),
            "backward_GBps": round(bwd_bytes / t_bwd / 1e6, 1), "backward_share_of_hbm": round(bwd_bytes / t_bwd / 1e-3 / HBM_BYTES_PER_S, 4),
            "backward_moved_GBps": round(bwd_moved / t_bwd / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_semantic_train.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    card = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}
    lines = [json.dumps(case(2, 3, H, H, args.reps, card)) for H in (512, 1024)]
    for line in lines:
        print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
