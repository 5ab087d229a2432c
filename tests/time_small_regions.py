"""Timing of msam_remove_small_regions on one GPU (run: PYTHONPATH=. python tests/time_small_regions.py): 128 masks of
1024^2 and of 2048^2, holes then islands with min_mask_region_area = 100, as AMG's generate(min_mask_region_area > 0)
calls it per chunk of 128 masks.  Every call starts from the same seeded masks (blobs with specks and pin holes), restored
by a device copy that is timed on its own and subtracted.  Every figure is the median of REPEATS windows of at least WINDOW_S
seconds, with the spread (min .. max) beside it; the card's name and power limit are read in the same run."""
import json
import statistics
import subprocess
import time

import torch

from micro_sam_b200 import _lib

WINDOW_S, REPEATS = 1.0, 5
DEV = "cuda:0"
N, AREA = 128, 100


def timed(fn):
    """median, min, max ms per call over REPEATS windows of >= WINDOW_S seconds"""
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
    return statistics.median(ms), min(ms), max(ms)


def seeded_masks(n, side, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    low = torch.randn(n, 1, side // 64, side // 64, generator=g, device=DEV)
    m = torch.nn.functional.interpolate(low, (side, side), mode="bicubic")[:, 0] > 0.3
    m |= torch.rand(n, side, side, generator=g, device=DEV) > 0.9995      # specks (islands)
    m &= ~(torch.rand(n, side, side, generator=g, device=DEV) > 0.999)    # pin holes
    return m.to(torch.uint8).contiguous()


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    L = _lib.lib()
    for side in (1024, 2048):
        src = seeded_masks(N, side, seed=side)
        masks = torch.empty_like(src)
        ws = torch.empty(N * (2 * side * side + 4), dtype=torch.int32, device=DEV)
        ch = torch.zeros(2, N, dtype=torch.int32, device=DEV)

        def run():
            masks.copy_(src)
            for q, holes in enumerate((1, 0)):
                _lib.check(L.msam_remove_small_regions(_lib.ptr(masks), N, side, side, AREA, holes, _lib.ptr(ch[q]), _lib.ptr(ws),
                                                       _lib.cur_stream()))

        t_all = timed(run)
        t_copy = timed(lambda: masks.copy_(src))
        run()
        torch.cuda.synchronize()
        print(json.dumps({"gpu": gpu, "n": N, "side": side, "area": AREA, "holes_then_islands_ms": round(t_all[0] - t_copy[0], 3),
                          "with_copy_ms": [round(x, 3) for x in t_all], "copy_ms": [round(x, 3) for x in t_copy],
                          "changed": [int(ch[0].sum()), int(ch[1].sum())],
                          "checksum": int(masks.view(N, -1).sum(1, dtype=torch.int64).mul(torch.arange(1, N + 1, device=DEV)).sum())}),
              flush=True)


if __name__ == "__main__":
    main()
