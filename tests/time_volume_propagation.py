"""Timing (not a test): segment_mask_in_volume on vit_b (seeded weights), a 64 x 1024 x 1024 volume with its embeddings held on
the device, one seed slice in the middle, iou_threshold = 0 (every slice is segmented).  Slices per second of the device slice
step (csrc/volume.cu) and of the same schedule through segment_from_mask's host glue, for each projection mode; then the
device prompt derivation alone (msam_mask_prompts) on a large object, a disk of radius 480 filling most of its 961 x 961 crop
of a 1024 x 1024 mask, per point mode.  Prints the
card and its power limit.  Run from the repository root on the GPU: `python tests/time_volume_propagation.py`."""
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import _lib, multi_dimensional_segmentation as mds, util  # noqa: E402
from micro_sam_b200.sample_data import em_volume  # noqa: E402
from oracle import sam_ref  # noqa: E402

Z, S = 64, 1024


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    pred = util.get_sam_model("vit_b", state_dict=sam_ref.seeded_state_dict("vit_b", seed=0), max_batch=4, max_prompts=64)
    vol = em_volume((Z, S, S), seed=0)
    emb = util.precompute_image_embeddings(pred, vol, ndim=3, batch_size=4, to_numpy=False)
    yy, xx = np.mgrid[:S, :S]
    seg0 = np.zeros((Z, S, S), np.uint32)
    seg0[Z // 2][(yy - 500) ** 2 + (xx - 480) ** 2 < 120 ** 2] = 1
    slices = np.array([Z // 2])
    for proj in mds.PROJECTION_MODES:
        res = {}
        for name, fn in (("device", mds.segment_mask_in_volume), ("host glue", mds._segment_mask_in_volume_host)):
            seg = seg0.copy()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                _, (z0, z1) = fn(seg, pred, emb, slices, False, False, 0.0, proj)
            except RuntimeError as e:   # more than 16 tokens per prompt
                res[name] = f"refused ({str(e)[:60]})"
                continue
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            n = Z - 1
            res[name] = f"{n / dt:.1f} slices/s ({dt * 1e3 / n:.2f} ms/slice, z {z0}..{z1})"
            res[name + " seg"] = seg
        same = "device and host volumes identical" if ("device seg" in res and "host glue seg" in res and
                                                       np.array_equal(res["device seg"], res["host glue seg"])) else "volumes differ"
        print(f"{proj:16s} device {res['device']}; host glue {res['host glue']}; {same}", flush=True)

    L = _lib.lib()
    m = torch.from_numpy(((yy - 512) ** 2 + (xx - 512) ** 2 < 480 ** 2).astype(np.uint8)).cuda()
    ws = torch.empty(int(L.msam_mask_prompts_workspace(S, S)), dtype=torch.uint8, device="cuda")
    st = torch.zeros(12, dtype=torch.int64, device="cuda")
    box, lg = torch.zeros(4, device="cuda"), torch.zeros(256, 256, device="cuda")
    pts, lbl = torch.zeros(64, 2, device="cuda"), torch.zeros(64, device="cuda")
    for mode, name in ((0, "box + logits"), (1, "box + logits + single point"), (2, "box + logits + points")):
        def run():
            _lib.check(L.msam_mask_prompts(_lib.ptr(m), S, S, S, 0.0, 1, mode, 64, _lib.ptr(ws), ws.numel(), _lib.ptr(st), _lib.ptr(box),
                                           _lib.ptr(lg), _lib.ptr(pts), _lib.ptr(lbl), None, _lib.cur_stream()))
        for _ in range(3):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            run()
        e1.record()
        torch.cuda.synchronize()
        print(f"msam_mask_prompts, disk r=480 in 1024 x 1024, {name}: {e0.elapsed_time(e1) / 20:.3f} ms", flush=True)


if __name__ == "__main__":
    main()
