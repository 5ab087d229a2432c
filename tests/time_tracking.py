"""Timing (not a test): track_from_prompts on vit_b (seeded weights), a 64 x 1024 x 1024 timeseries with its embeddings held on
the device.  A disk of radius 120 translating by (2.6, -1.9) pixels per frame is drawn in the prompt frames 0 and 1, so the
motion model shifts by non-integer steps from frame 2 on; threshold None, so every frame up to the last is tracked.  Frames per
second of the device step (csrc/volume.cu) and of the same schedule through scipy.ndimage.shift and segment_from_mask's host
glue, for each projection mode; then msam_shift_mask alone on a 1024 x 1024 plane, timed with CUDA events.  Prints the card and
its power limit.  Run from the repository root on the GPU: `python tests/time_tracking.py`."""
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import _lib, multi_dimensional_segmentation as mds, util  # noqa: E402
from micro_sam_b200.sample_data import em_volume  # noqa: E402
from oracle import sam_ref  # noqa: E402

T, S = 64, 1024
STEP = (2.6, -1.9)


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    pred = util.get_sam_model("vit_b", state_dict=sam_ref.seeded_state_dict("vit_b", seed=0), max_batch=4, max_prompts=64)
    series = em_volume((T, S, S), seed=0)
    emb = util.precompute_image_embeddings(pred, series, ndim=3, batch_size=4, to_numpy=False)
    yy, xx = np.mgrid[:S, :S]
    seg0 = np.zeros((T, S, S), np.uint32)
    slices = np.array([0, 1])
    for k in slices:
        seg0[k][(yy - 400 - STEP[0] * k) ** 2 + (xx - 600 - STEP[1] * k) ** 2 < 120 ** 2] = 1
    layer = SimpleNamespace(data=np.array([[0, 400, 600], [1, 403, 598]], float), properties={"state": np.array(["track", "track"])})
    n = T - 2
    for proj in mds.PROJECTION_MODES:
        res = {}
        for name, fn in (("device", mds.track_from_prompts), ("host glue", mds._track_from_prompts_host)):
            seg = seg0.copy()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                fn(layer, None, seg, pred, slices, emb, False, None, proj, 0.5, 0.05)
            except RuntimeError as e:   # more than 16 tokens per prompt
                res[name] = f"refused ({str(e)[:70]})"
                continue
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            res[name] = f"{n / dt:.1f} frames/s ({dt * 1e3 / n:.2f} ms/frame)"
            res[name + " seg"] = seg
        if "device seg" not in res or "host glue seg" not in res:
            same = "no series to compare"
        else:
            same = "device and host series identical" if np.array_equal(res["device seg"], res["host glue seg"]) else "series differ"
        print(f"{proj:16s} device {res['device']}; host glue {res['host glue']}; {same}", flush=True)

    L = _lib.lib()
    src = torch.from_numpy(((yy - 512) ** 2 + (xx - 512) ** 2 < 480 ** 2).astype(np.uint8)).cuda()
    dst = torch.empty_like(src)

    def run():
        _lib.check(L.msam_shift_mask(_lib.ptr(src), S, _lib.ptr(dst), S, S, S, 13.37, -7.5, _lib.cur_stream()))
    for _ in range(10):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        run()
    e1.record()
    torch.cuda.synchronize()
    print(f"msam_shift_mask, 1024 x 1024 uint8: {e0.elapsed_time(e1) / 200 * 1e3:.1f} us per call back to back from Python", flush=True)
    # the kernel alone: far shorter than a call from Python, so the events above measure the launch rate
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            run()
        torch.cuda.synchronize()
    k = [e for e in prof.key_averages() if "shift_kernel" in e.key][0]
    us = k.device_time_total / k.count
    print(f"shift_kernel (torch.profiler, {k.count} launches): {us:.2f} us, {2 * S * S / (us * 1e-6) / 1e9:.0f} GB/s "
          f"(1 byte read + 1 byte written per pixel)", flush=True)


if __name__ == "__main__":
    main()
