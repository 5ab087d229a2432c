"""Times PerObjectDistanceTransform (the UNETR decoder's targets, csrc/distance_targets.cu) on the device: device labels to
device targets (CUDA events, warmed, windows of at least a second), the numpy -> numpy path, each kernel stage (msam_profile),
the writer's and the EDT's share of the HBM bound, and the numpy / scipy oracle's host time on the same inputs.  One JSON line
per case (Voronoi cells at 512^2 and 1024^2, B = 1 and 4), with the card's name and power limit read in the same run.
Usage:  python tests/time_distance_targets.py [--out measurements/distance_targets_h100.jsonl]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import _lib, training  # noqa: E402
from oracle import distance_targets_ref as ref  # noqa: E402
from tests.test_gpu_centers import voronoi_labels  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def cuda_ms(fn, min_s=1.0):
    """mean ms per call over a window of at least min_s seconds, after a warm-up"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps, ms = 4, 0.0
    while True:
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= 1e3 * min_s:
            return ms / reps
        reps = max(reps * 2, int(reps * 1.2e3 * min_s / max(ms, 1e-3)))


def host_s(fn, min_s=1.0):
    fn()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        if time.perf_counter() - t0 >= min_s:
            return (time.perf_counter() - t0) / n


def stages(fn, reps=20):
    _lib.lib().msam_profile(1)
    for _ in range(reps):
        fn()
    rep = _lib.profile_report()
    _lib.lib().msam_profile(0)
    return {r["name"]: {"ms": round(r["ms"] / r["n"], 4), "bytes": r["bytes"] / r["n"]} for r in rep if r["name"].startswith("dt_")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    trafo = training.PerObjectDistanceTransform()   # torch_em's defaults as micro-sam's train_sam uses them, with instances
    trafo4 = training.PerObjectDistanceTransform(instances=True)
    lines = []
    for side, seeds in ((512, 1200), (1024, 1500)):
        for B in (1, 4):
            labs = np.stack([voronoi_labels((side, side), seeds, seed=10 * B + b) for b in range(B)])
            dev = torch.from_numpy(labs).cuda()
            n = labs.size
            rec = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q, "H": side, "W": side, "B": B,
                   "objects": int(sum(len(np.unique(lab)) - 1 for lab in labs)), "channels": 4}
            rec["device_ms"] = round(cuda_ms(lambda: trafo4(dev)), 4)
            rec["device_ms_3ch"] = round(cuda_ms(lambda: trafo(dev)), 4)
            rec["numpy_to_numpy_ms"] = round(1e3 * host_s(lambda: [trafo4(lab) for lab in labs]), 3)
            st = stages(lambda: trafo4(dev))
            rec["stages"] = st
            for name in ("dt_write", "dt_edt"):
                if name in st:
                    bound = st[name]["bytes"] / HBM_BYTES_PER_S * 1e3
                    rec[f"{name}_share_of_hbm_bound"] = round(bound / st[name]["ms"], 3)
            rec["oracle_host_s"] = round(host_s(lambda: [ref.per_object_distance_transform(lab, instances=True) for lab in labs],
                                                min_s=0.1), 3)
            assert n == B * side * side
            line = json.dumps(rec)
            print(line, flush=True)
            lines.append(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
