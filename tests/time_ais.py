"""Timing of AIS per 1024x1024 image on one GPU (run: PYTHONPATH=. python tests/time_ais.py).  Every figure is the median of
REPEATS windows of at least WINDOW_S seconds each, with the spread (min .. max) beside it:
  - the UNETR decoder (UNETRDecoder.__call__), and per kernel from msam_profile's CUDA events over a window of its own, with
    TFLOP/s against the H100 SXM's dense bf16 data-sheet peak (989 TFLOP/s);
  - the post-processing with its watershed sweeps, on the decoder's maps and on synthetic touching disks;
  - InstanceSegmentationWithDecoder.initialize (from precomputed embeddings) + generate (label image on the host).
Seeded production-plan decoder weights; a seeded vit_test predictor only provides the embedding."""
import statistics
import subprocess
import time

import numpy as np
import torch

from micro_sam_b200 import _lib, instance_segmentation as iseg, unetr, util
from micro_sam_b200.sample_data import lm_tile
from oracle import ais_ref, sam_ref, unetr_ref

PEAK = 989e12
WINDOW_S, REPEATS = 1.0, 5
DEV = "cuda:0"


def timed(fn):
    """median and (min, max) ms per call over REPEATS windows of >= WINDOW_S seconds"""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    n = max(3, int(WINDOW_S / max(time.perf_counter() - t0, 1e-4)))
    ms = []
    for _ in range(REPEATS):
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) / n * 1e3)
    return statistics.median(ms), min(ms), max(ms), n


def fmt(t):
    return f"{t[0]:.3f} ms (min {t[1]:.3f} .. max {t[2]:.3f}, {REPEATS} windows of {t[3]} calls)"


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    dec = unetr.UNETRDecoder(unetr_ref.seeded_state(seed=0), device=DEV)
    z = torch.randn(1, 256, 64, 64, device=DEV) * 0.5
    t_dec = timed(lambda: dec(z, (1024, 1024), (1024, 1024)))
    L = _lib.lib()
    dec(z, (1024, 1024), (1024, 1024))
    torch.cuda.synchronize()
    L.msam_profile(1)
    n_prof = max(3, t_dec[3])
    for _ in range(n_prof):
        dec(z, (1024, 1024), (1024, 1024))
    torch.cuda.synchronize()
    rows = _lib.profile_report()
    L.msam_profile(0)
    flops = sum(r["flops"] for r in rows) / n_prof
    print(f"decoder: {fmt(t_dec)}; {flops / 1e12:.3f} TFLOP per image, {flops / t_dec[0] / 1e9:.1f} TFLOP/s "
          f"({flops / (t_dec[0] * 1e-3) / PEAK:.2f} of the bf16 peak)")
    for r in sorted(rows, key=lambda r: -r["ms"]):
        ms = r["ms"] / n_prof
        tf = r["flops"] / (r["ms"] * 1e-3) / 1e12 if r["flops"] else 0.0
        print(f"  {r['name']:<32s} {r['n'] / n_prof:5.1f} launches {ms:8.3f} ms per image"
              + (f"  {tf:6.1f} TFLOP/s ({tf * 1e12 / PEAK:.2f} of peak)" if tf else ""))
    maps = dec(z, (1024, 1024), (1024, 1024))[0]
    fg, cd, bd = ais_ref.touching_disks(1024, 1024, 1500, seed=1)
    syn = [torch.from_numpy(a).to(DEV) for a in (fg, cd, bd)]
    for src, m in (("decoder maps (seeded weights)", [maps[0], maps[1], maps[2]]), ("synthetic touching disks", syn)):
        _, ids, sweeps = unetr.postprocess(*m)
        print(f"post-processing on {src}: {fmt(timed(lambda: unetr.postprocess(*m)))}, {ids} ids, {sweeps} watershed sweeps")
    pred = util.get_sam_model("vit_test", device=DEV, state_dict=sam_ref.seeded_state_dict("vit_test", seed=1), max_batch=1,
                              max_prompts=64)
    img = lm_tile((1024, 1024), 150, seed=2)
    emb = util.precompute_image_embeddings(pred, img, verbose=False)
    seg = iseg.InstanceSegmentationWithDecoder(pred, dec)
    print(f"initialize (precomputed embeddings): {fmt(timed(lambda: seg.initialize(img, image_embeddings=emb)))}")
    print(f"generate (label image on the host): {fmt(timed(lambda: seg.generate()))}")
    print(f"initialize + generate: {fmt(timed(lambda: (seg.initialize(img, image_embeddings=emb), seg.generate())))}")


if __name__ == "__main__":
    main()
