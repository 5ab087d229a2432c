"""Times get_centers_and_bounding_boxes and segmentation_to_one_hot on the device (CUDA events, end to end from a host numpy
label image to the reference's dicts / a device one-hot tensor), the squared EDT and one-hot passes against the HBM bound, and
the numpy / scipy oracle's host time on the same inputs.  Prints one JSON line (and writes it to --out when given).
Usage:  python tests/time_centers.py [--reps 10] [--out path.json]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import _lib, util  # noqa: E402
from oracle import centers_ref  # noqa: E402
from tests.test_gpu_centers import voronoi_labels  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def cuda_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def host_s(fn):
    t = time.perf_counter()
    fn()
    return time.perf_counter() - t


def edt_pass(shape, reps):
    """the squared EDT over the padded grid of `shape` alone: ms and share of the HBM bound (first pass reads 1 byte and writes
    4 per pixel, each further pass reads and writes 4)"""
    padded = tuple(s + 2 for s in shape)
    n = int(np.prod(padded))
    rng = np.random.default_rng(0)
    m = torch.from_numpy((rng.random(padded) > 0.05).astype(np.uint8)).cuda()
    out = torch.empty(padded, dtype=torch.int32, device="cuda")
    ws = torch.empty(3 * ((4 * n + 255) // 256 * 256), dtype=torch.uint8, device="cuda")
    dims = (ctypes.c_int * len(padded))(*padded)
    L = _lib.lib()
    ms = cuda_ms(lambda: _lib.check(L.msam_op_edt_squared(_lib.ptr(m), len(padded), dims, _lib.ptr(ws), ws.numel(), _lib.ptr(out),
                                                          _lib.cur_stream())), reps)
    bound = n * (5 + 8 * (len(padded) - 1)) / HBM_BYTES_PER_S * 1e3
    return {"ms": round(ms, 4), "hbm_bound_ms": round(bound, 4), "share_of_hbm_bound": round(bound / ms, 3)}


def one_hot_pass(seg, reps):
    t = torch.from_numpy(seg).cuda()
    n_planes = int(seg.max())
    ms = cuda_ms(lambda: util.segmentation_to_one_hot(t), reps)
    bound = (n_planes + 1) * seg.size * 4 / HBM_BYTES_PER_S * 1e3   # the planes written, the int32 labels read
    return {"planes": n_planes, "ms": round(ms, 4), "hbm_bound_ms": round(bound, 4), "share_of_hbm_bound": round(bound / ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    res = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q, "cases": {}}
    for name, shape, n_seeds in (("2d_2048", (2048, 2048), 6000), ("3d_32x512x512", (32, 512, 512), 2500)):
        seg = voronoi_labels(shape, n_seeds, seed=1).astype(np.uint32)
        case = {"objects": int(len(np.unique(seg)) - 1)}
        for mode in ("v", "p"):
            case[f"device_dicts_ms_{mode}"] = round(cuda_ms(lambda: util.get_centers_and_bounding_boxes(seg, mode), args.reps), 3)
            dseg = torch.from_numpy(seg.view(np.int32)).cuda()
            case[f"device_tensors_ms_{mode}"] = round(cuda_ms(lambda: util.get_centers_and_bounding_boxes(dseg, mode, device_result=True),
                                                              args.reps), 3)
            case[f"oracle_host_s_{mode}"] = round(host_s(lambda: centers_ref.get_centers_and_bounding_boxes(seg, mode)), 3)
        case["edt"] = edt_pass(shape, args.reps)
        res["cases"][name] = case
    res["one_hot_1024_64"] = one_hot_pass(voronoi_labels((1024, 1024), 64, 2, background=0.0, sparse=False).astype(np.int32), args.reps)
    res["one_hot_2048_100"] = one_hot_pass(voronoi_labels((2048, 2048), 100, 3, background=0.0, sparse=False).astype(np.int32), args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
