"""Timing (not a test): object features (micro_sam_b200.object_classification.compute_object_features, csrc/objfeat.cu).

1. One 1024 x 1024 tile with about 400 objects and random embeddings on the device: msam_object_features alone (CUDA events
   over 50 calls) and compute_object_features end to end (relabel, pooling, copy of the result to the host); then the kernels
   alone on objects whose boxes are much larger than their area (100 thin diagonal strokes), on one large disk, and on that
   disk with a 1024 x 1024 resize grid.
2. A 64 x 2048 x 2048 volume with tiled embeddings on the device (tile 1024, halo 64: 4 tiles per slice, 256 units) and about
   180 objects per slice, each through four slices: compute_object_features end to end, then the same inputs through the fp64
   oracle (oracle/objfeat_ref.py) on every host core, and the largest difference between the two.
Prints the card and its power limit.  Run from the repository root on the GPU: `python tests/time_object_features.py`.
"""
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import util  # noqa: E402
from micro_sam_b200 import object_classification as oc  # noqa: E402
from oracle import objfeat_ref as ref  # noqa: E402

Z, S, TILE, HALO = 64, 2048, 1024, 64


def blocky_labels(z, n_side, side, gen):
    """labels constant on n_side x n_side blocks of a side x side plane, ids shared by runs of four slices, 30 % background"""
    cell = side // n_side
    ids = torch.arange(1, n_side * n_side + 1, device="cuda").view(n_side, n_side) + (z // 4) * 100000
    ids = torch.where(torch.rand(n_side, n_side, generator=gen, device="cuda") < 0.3, 0, ids)
    return ids.repeat_interleave(cell, 0).repeat_interleave(cell, 1).to(torch.int32)


def _oracle_unit(args):
    seg, emb = args
    return ref.compute_unit(emb, seg)


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)

    # ---- 1. one 1024 x 1024 tile
    seg = blocky_labels(0, 24, 1024 - 1024 % 24, gen)
    seg = torch.nn.functional.pad(seg, (0, 1024 - seg.shape[1], 0, 1024 - seg.shape[0]))
    emb = torch.randn(1, 256, 64, 64, generator=gen, device="cuda")
    dense, ids = oc._relabel(seg, seg.device)
    pool = oc._Pool(int(ids.numel()), seg.device)
    e = emb[0].contiguous()
    for _ in range(5):
        pool.add(e, dense, (256, 256))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        pool.add(e, dense, (256, 256))
    e1.record()
    torch.cuda.synchronize()
    print(f"1024 x 1024 tile, {int(ids.numel())} objects: msam_object_features {e0.elapsed_time(e1) / 50:.3f} ms per tile", flush=True)
    d = {"features": emb, "input_size": (1024, 1024), "original_size": (1024, 1024)}
    for _ in range(3):
        oc.compute_object_features(d, seg, verbose=False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(20):
        oc.compute_object_features(d, seg, verbose=False)
    torch.cuda.synchronize()
    print(f"1024 x 1024 tile: compute_object_features end to end {(time.perf_counter() - t0) / 20 * 1e3:.3f} ms", flush=True)

    # objects whose r-grid box is much larger than their area, and a fine resize grid: the label kernel's gather visits every
    # cell of an object's box, so its cost follows the box, not the pixel count
    yy, xx = torch.meshgrid(torch.arange(1024, device="cuda"), torch.arange(1024, device="cuda"), indexing="ij")
    diag = torch.zeros(1024, 1024, dtype=torch.int32, device="cuda")
    for k in range(100):   # 100 diagonal strokes 3 pixels wide across the whole tile
        diag[((xx - yy - (k - 50) * 20).abs() <= 1)] = k + 1
    disk = (((yy - 512) ** 2 + (xx - 512) ** 2) < 500 ** 2).to(torch.int32)
    for name, lab, shape in (("100 diagonal strokes", diag, (256, 256)), ("one disk of radius 500", disk, (256, 256)),
                             ("one disk of radius 500, resize_embedding_shape (1024, 1024)", disk, (1024, 1024))):
        dense, ids = oc._relabel(lab, lab.device)
        pool = oc._Pool(int(ids.numel()), lab.device)
        for _ in range(3):
            pool.add(e, dense, shape)
        e0.record()
        for _ in range(20):
            pool.add(e, dense, shape)
        e1.record()
        torch.cuda.synchronize()
        print(f"1024 x 1024 tile, {name}: msam_object_features {e0.elapsed_time(e1) / 20:.3f} ms per tile", flush=True)

    # ---- 2. 64 x 2048 x 2048 tiled volume
    vol = torch.stack([blocky_labels(z, 16, S, gen) for z in range(Z)])
    feats = util._MemGroup()
    feats.attrs.update({"shape": (S, S), "tile_shape": (TILE, TILE), "halo": (HALO, HALO)})
    n_tiles = (S // TILE) ** 2
    for t in range(n_tiles):
        feats[str(t)] = util._MemDataset(torch.randn(Z, 1, 256, 64, 64, generator=gen, device="cuda"), {})
    emb = {"features": feats, "input_size": None, "original_size": None}
    oc.compute_object_features(emb, vol[:2], verbose=False)   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids, got = oc.compute_object_features(emb, vol, verbose=False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"{Z} x {S} x {S} tiled volume ({Z * n_tiles} units, {len(ids)} objects): compute_object_features {dt * 1e3:.1f} ms "
          f"({dt * 1e3 / (Z * n_tiles):.3f} ms per unit)", flush=True)

    host = util._MemGroup()
    host.attrs.update(feats.attrs)
    for k, ds in feats.items():
        host[k] = util._MemDataset(ds.data.cpu().numpy(), {})
    vol_h = vol.cpu().numpy()
    del feats, emb
    torch.cuda.empty_cache()
    n_proc = os.cpu_count()
    with mp.get_context("spawn").Pool(n_proc) as pool_h:
        t0 = time.perf_counter()
        want_ids, want = ref.merge(ref.units({"features": host, "input_size": None}, vol_h), vol_h,
                                   unit_fn=lambda it: pool_h.imap(_oracle_unit, it, chunksize=1))
        dt_o = time.perf_counter() - t0
    assert np.array_equal(ids, want_ids) and np.array_equal(got[:, 0], want[:, 0])
    err = np.abs(got[:, 1:].astype(np.float64) - want[:, 1:]).max()
    print(f"oracle (fp64 restatement, {n_proc} host processes): {dt_o:.1f} s; {dt_o / dt:.0f}x the device; ids and areas equal, "
          f"max mean difference {err:.2e} (max|E| {max(float(np.abs(d.data).max()) for d in host.values()):.2f})", flush=True)


if __name__ == "__main__":
    main()
