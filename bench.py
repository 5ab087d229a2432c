#!/usr/bin/env python
"""bench.py -- BASELINE.json metric: 1024x1024 tiles/s for embedding precompute + AMG (vit_b, 32x32 point grid, batch of 16
synthetic LM tiles = BASELINE.json configs[1]) on N H100s, plus the ViT-H encoder forward as a fraction of the bf16
tensor-core roofline.

  python bench.py --gpus N --steps K --warmup W            # ours (torchrun for N > 1, one rank per GPU, weak scaling)
  python bench.py --impl reference --gpus N --steps K ...  # the reference algorithm's CPU path (oracle port) on host cores
  python bench.py --config cfg1|cfg3|cfg4|cfg5 ...                   # the other BASELINE.json GPU configurations (extra JSON lines)
  python bench.py ... --dump-outputs DIR                   # also write what the last timed step computed, as DIR/<name>.npy

One "step" = one pass of the hot path over one batch of 16 tiles per GPU.  BOTH arms run the same workload
(`workload_config`): same tiles, same seeded weights, same point grid and the same generate() thresholds, chosen so that
the filters keep a realistic number of masks with the random-init weights (the reference defaults 0.88 / 0.95 keep none);
the thresholds-0.0 worst case (every mask reaches the NMS) is timed as an extra line (`worst_case`).
  value : tiles/s, inputs resident in HBM (uint8 tiles on the device), device-side AMG result (painted label image)
  e2e   : tiles/s through the reference-facing API (precompute_image_embeddings + AutomaticMaskGenerator.initialize /
          generate) from HOST uint16 tiles to HOST uint32 label images; H2D / D2H inside the timed region.
Timing: CUDA events on the launching stream, barrier + synchronize on both sides, max over ranks.  Every step streams
multi-GB decoder activations (>> 50 MB L2), so no extra L2 flush is needed ("l2": "working_set_exceeds_l2").
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_TILES = 16
TILE = 1024
GRID = 32
# algorithmic FLOPs (SURVEY.md 8d)
ENC_FLOPS = {"vit_b": 0.9376e12, "vit_l": 2.8370e12, "vit_h": 5.6418e12}
DEC_FLOPS_PER_PROMPT = 2.817e9      # hoisted decoder (SURVEY.md 8d); + 0.805e9 once per tile
# generate() thresholds of the benchmark (both arms).  With the seeded random-init weights the predicted IoUs have median
# 0.23 / 90 % quantile 0.51 and the stability scores median 0.125 (noise masks), so the reference defaults (0.88 / 0.95)
# filter everything; and because every noise mask has a near-full-tile box (pairwise box IoU ~ 0.99) the default box-NMS
# threshold 0.7 keeps exactly one mask per tile.  The benchmark therefore uses ~ the 90 % / 50 % quantiles of the seeded
# vit_b model's predictions (`threshold_calibration` in the JSON line) and box_nms_thresh 1.0 (NMS runs but suppresses
# nothing): O(100-200) survivors per tile reach the NMS, the painter and the connected-component pass, which is the order
# of a real LM tile.  The thresholds-0.0 worst case (all 3072 masks into the NMS) is reported as `worst_case`.
BENCH_THRESH = {"pred_iou_thresh": 0.5, "stability_score_thresh": 0.125, "box_nms_thresh": 1.0}


def workload_config(args):
    """Identical in both arms (the driver compares the two `config` objects)."""
    return {"workload": f"{args.model} AutomaticMaskGenerator, 32x32 point grid, batch of 16 synthetic 1024x1024 LM tiles per "
                        "GPU (BASELINE.json configs[1]); seeded random-init weights; embed + AMG initialize + generate",
            "tiles_per_step_per_gpu": N_TILES, "points_per_side": GRID,
            "pred_iou_thresh": args.pred_iou_thresh, "stability_score_thresh": args.stability_score_thresh,
            "box_nms_thresh": args.box_nms_thresh,
            "l2": "gpu arm: working_set_exceeds_l2 (multi-GB decoder activations per step)",
            "parallelism": "tile shards, one process per GPU, no collective (reference arm: host threads of rank 0)"}


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d, "measured"
    # NVIDIA H100 SXM data sheet (700 W card): 3.35 TB/s HBM3, 989 TFLOP/s dense BF16; no sustained rate has been measured
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0}, "datasheet"


class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, dev):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", str(dev), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                       "-lms", "100"], stdout=self.f, stderr=subprocess.DEVNULL)
        except Exception:  # noqa: BLE001
            self.p = None

    def stop(self):
        if self.p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:  # noqa: BLE001
            self.p.kill()
        self.f.flush()
        rows = [l.strip().split(", ") for l in open(self.f.name) if l.strip()]
        os.unlink(self.f.name)
        sm = [float(r[1]) for r in rows if len(r) >= 9]
        mx = [float(r[2]) for r in rows if len(r) >= 9]
        reasons = set()
        for r in rows:
            if len(r) < 9:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                if v.strip().lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def make_tiles(seed0=0, n=N_TILES):
    from micro_sam_b200.sample_data import lm_tile
    return np.stack([lm_tile((TILE, TILE), 150, seed=seed0 + i) for i in range(n)])


def best_cpu_threads():
    """All host threads are allowed, but PyTorch's CPU GEMMs peak below the logical-core count on SMT hosts: pick the
    thread count that runs an encoder-sized matmul fastest (candidates: all, 1/2, 1/4 of the logical cores)."""
    n = os.cpu_count() or 1
    a, b = torch.randn(4096, 768), torch.randn(768, 3072)
    best, best_t = n, None
    for c in sorted({n, max(1, n // 2), max(1, n // 4)}, reverse=True):
        torch.set_num_threads(c)
        a @ b
        t0 = time.perf_counter()
        for _ in range(3):
            a @ b
        t = time.perf_counter() - t0
        if best_t is None or t < best_t:
            best, best_t = c, t
    return best


# ---------------------------------------------------------------------------------------------------- reference arm
def cpu_baseline(args, n_point_batches=1, threads=None):
    """The reference algorithm's CPU path (oracle port of segment_anything + micro-sam's AMG) on the host cores, on a
    BOUNDED sample of the same workload with the SAME generate() thresholds as the GPU arm: 1 tile embedding +
    `n_point_batches` x 64 grid points (every 16/n-th batch of the 16) through predict_torch / _to_mask_data, + generate;
    the AMG part is scaled to the 16-batch (1024 point) grid."""
    from oracle import amg_ref, sam_ref
    threads = threads or best_cpu_threads()
    torch.set_num_threads(threads)
    sam = sam_ref.build_seeded_sam(args.model, seed=0)
    pred = sam_ref.SamPredictor(sam)
    img = make_tiles(0, 1)[0]
    t0 = time.perf_counter()
    emb = amg_ref.precompute_image_embeddings_2d(pred, img)
    t_embed = time.perf_counter() - t0
    amg = amg_ref.AutomaticMaskGenerator(pred, points_per_side=GRID, points_per_batch=64)
    stride = 16 // n_point_batches
    rows = np.concatenate([np.arange(64 * b, 64 * b + 64) for b in range(0, 16, stride)][:n_point_batches])
    amg.point_grids = [amg.point_grids[0][rows]]
    t0 = time.perf_counter()
    amg.initialize(img, image_embeddings=emb)
    t_init = time.perf_counter() - t0
    t0 = time.perf_counter()
    seg = amg.generate(pred_iou_thresh=args.pred_iou_thresh, stability_score_thresh=args.stability_score_thresh,
                       box_nms_thresh=args.box_nms_thresh)
    t_gen = time.perf_counter() - t0
    scale = (GRID * GRID) / (64 * n_point_batches)
    per_tile = t_embed + t_init * scale + t_gen * scale
    return {
        "value": 1.0 / per_tile, "unit": "tiles/s", "cores": threads, "kind": "port",
        "sample": f"1 tile: embed {t_embed:.2f}s + {n_point_batches}x64 of 1024 grid points {t_init:.2f}s + generate "
                  f"{t_gen:.2f}s ({int(seg.max())} instances in the sample), AMG part scaled x{scale:.0f}",
        "seconds_per_tile": per_tile,
    }


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    vals = []
    for _ in range(max(1, args.warmup > 0)):
        cpu_baseline(args, 1)
    t_all = time.perf_counter()
    for _ in range(args.steps):
        cb = cpu_baseline(args, 1)
        vals.append(cb)
    v = float(np.mean([c["value"] for c in vals]))
    cb = vals[-1]
    cb["value"] = v
    out = {
        "impl": "reference", "metric": "1024x1024 tiles/s, embed + AMG", "value": v, "unit": "tiles/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * (time.perf_counter() - t_all) / args.steps,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(args),
        "cpu_baseline": cb, "e2e": {"value": v, "unit": "tiles/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(out))


# ---------------------------------------------------------------------------------------------------- our arm
def vit_h_roofline(device, steps=3):
    """ViT-H encoder forward: ms/tile and fraction of the bf16 tensor roofline.  Measured at batch 4 and 8 tiles (distinct
    uint8 tiles each step, so nothing is cached); the better of the two is reported together with its batch."""
    from oracle import sam_ref  # weights only (seeded generator); nothing of the oracle is timed here
    from micro_sam_b200 import _lib
    from micro_sam_b200.sam import B200Sam
    sd = {k: v for k, v in sam_ref.seeded_state_dict("vit_h", seed=0).items() if k.startswith("image_encoder.")}
    sam = B200Sam("vit_h", sd, device=device, max_batch=8, max_prompts=1)
    best = None
    for batch in (8, 4):
        xs = [torch.randint(0, 255, (batch, TILE, TILE, 3), dtype=torch.uint8, device=device) for _ in range(steps)]
        for _ in range(2):
            sam.encode_u8(xs[0])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(steps):
            sam.encode_u8(xs[k])
        e1.record()
        torch.cuda.synchronize()
        ms_tile = e0.elapsed_time(e1) / steps / batch
        if best is None or ms_tile < best[0]:
            best = (ms_tile, batch)
    # per-kernel table at the better batch
    L = _lib.lib()
    x = torch.randint(0, 255, (best[1], TILE, TILE, 3), dtype=torch.uint8, device=device)
    L.msam_profile(1)
    sam.encode_u8(x)
    rep = _lib.profile_report()
    L.msam_profile(0)
    del sam
    torch.cuda.empty_cache()
    return best, [dict(r, ms_per_tile=r["ms"] / best[1]) for r in rep]


def kernel_table(rep, steps, pk, dev_ms_per_step):
    """Per-kernel rows from the library's CUDA-event records: time share, achieved algorithmic TFLOP/s and GB/s against the
    two rooflines; `bound` = the roofline that gives the larger lower bound on the kernel's time."""
    rows = []
    for r in sorted(rep, key=lambda r: -r["ms"]):
        ms = r["ms"] / steps
        n = r["n"] / steps
        tf = r["flops"] / (r["ms"] * 1e-3) / 1e12 if r["ms"] > 0 else 0.0
        gbs = r["bytes"] / (r["ms"] * 1e-3) / 1e9 if r["ms"] > 0 else 0.0
        f_t, f_h = tf / pk["bf16_tflops_sustained"], gbs / pk["hbm_gbs"]
        row = {"kernel": r["name"], "ms_per_step": ms, "launches_per_step": n, "share_of_step": ms / dev_ms_per_step,
               "tflops": tf, "gbs": gbs, "frac_tensor": f_t, "frac_hbm": f_h, "bound": "tensor" if f_t >= f_h else "hbm"}
        rows.append(row)
    return rows


def dump_outputs(path, last):
    """Writes what the last timed step returned to its caller, as float32 .npy files (~25 MB in all): `iou_preds` [16, 3072]
    (every tile), and fixed seeded samples of the larger outputs -- `labels` [16, 262144] (the same pixels of every tile's
    label image) and `features` [2097152] (elements of the [16, 256, 64, 64] image embeddings)."""
    os.makedirs(path, exist_ok=True)
    rng = np.random.default_rng(1234)
    pix = torch.from_numpy(np.sort(rng.choice(TILE * TILE, 262144, replace=False)))
    feat = last["features"].reshape(-1)
    idx = torch.from_numpy(np.sort(rng.choice(feat.numel(), 2097152, replace=False)))
    arrays = {
        "labels": torch.stack([l.reshape(-1)[pix.to(l.device)] for l in last["labels"]]).float(),
        "iou_preds": torch.stack([v.reshape(-1) for v in last["iou_preds"]]).float(),
        "features": feat[idx.to(feat.device)].float(),
    }
    for name, a in arrays.items():
        np.save(os.path.join(path, f"{name}.npy"), a.cpu().numpy().astype(np.float32))


def run_ours(args):
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    from oracle import sam_ref  # seeded weight generator only
    from micro_sam_b200 import _lib, instance_segmentation as iseg, sam as sam_mod, util
    pk, pk_src = peaks()

    sd = sam_ref.seeded_state_dict(args.model, seed=0)
    pred = util.get_sam_model(args.model, device=device, state_dict=sd, max_batch=args.enc_batch, max_prompts=args.max_prompts)
    sam = pred.model
    amg = iseg.AutomaticMaskGenerator(pred, points_per_side=GRID)
    tiles = make_tiles(seed0=rank * N_TILES)                                   # host uint16 (16,1024,1024)
    tiles_u8 = torch.from_numpy(np.stack([util._to_image(t) for t in tiles])).to(device)   # device-resident inputs
    gen_kw = dict(pred_iou_thresh=args.pred_iou_thresh, stability_score_thresh=args.stability_score_thresh,
                  box_nms_thresh=args.box_nms_thresh)
    worst_kw = dict(pred_iou_thresh=0.0, stability_score_thresh=0.0, box_nms_thresh=args.box_nms_thresh)
    survivors = []
    last = {}   # what the last timed step computed (--dump-outputs; the label buffer is reused per tile, so it is copied)

    def step_device(kw=gen_kw, count=False, capture=False):
        feats = sam.encode_u8(tiles_u8)
        out = None
        labels, ious = [], []
        for t in range(N_TILES):
            emb = {"features": feats[t:t + 1], "input_size": (TILE, TILE), "original_size": (TILE, TILE)}
            amg.initialize(tiles[t], image_embeddings=emb)
            out = amg.generate_device(**kw)
            if capture:   # `_crop_list`, not `crop_list`: the property would materialise the lazily skipped statistics
                labels.append(out.clone())
                ious.append(amg._crop_list[0]["iou_preds"].clone())
            if count:
                survivors.append(amg._n_keep_dev.clone())
        if capture:
            last.update(features=feats, labels=labels, iou_preds=ious)
        return out

    def step_e2e():
        emb = util.precompute_image_embeddings(pred, tiles, ndim=3, batch_size=N_TILES, to_numpy=False)
        segs = []
        for z in range(N_TILES):
            amg.initialize(tiles[z], image_embeddings=emb, i=z)
            segs.append(amg.generate(**gen_kw))
        return segs

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        ms = max(e0.elapsed_time(e1), 0.0)
        t = torch.tensor([ms, wall * 1e3], device=device, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        barrier()
        return float(t[0]), float(t[1])

    L = _lib.lib()
    # ---- device-resident throughput (value): the timed region itself is NOT instrumented
    sampler = ClockSampler(local) if rank == 0 else None
    for _ in range(args.warmup):
        step_device()
    l0 = _lib.launch_count()
    n_timed = [0]

    def timed_step():
        n_timed[0] += 1
        return step_device(capture=bool(args.dump_outputs) and n_timed[0] == args.steps)

    dev_ms, _ = timed(timed_step, args.steps, 0)
    launches = (_lib.launch_count() - l0) / args.steps
    clocks = sampler.stop() if sampler else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last)
    value = world * N_TILES * args.steps / (dev_ms / 1e3)
    # ---- end to end through the reference-facing API (host in, host out)
    e2e_ms, e2e_wall = timed(step_e2e, args.steps, max(1, args.warmup // 2))
    e2e_time = max(e2e_ms, e2e_wall)  # host work after the last kernel is part of the step
    e2e_val = world * N_TILES * args.steps / (e2e_time / 1e3)
    # ---- worst case: thresholds 0.0, every mask reaches the NMS (SURVEY.md 8d)
    worst_ms, _ = timed(lambda: step_device(worst_kw), max(1, args.steps // 2), 1)
    worst_val = world * N_TILES * max(1, args.steps // 2) / (worst_ms / 1e3)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    # ---- instrumented passes (outside the timed regions): per-kernel CUDA events inside the library, stage events here
    L.msam_profile(1)
    step_device()
    rep = _lib.profile_report()
    L.msam_profile(0)
    prof_ms = sum(r["ms"] for r in rep)
    table = kernel_table(rep, 1, pk, dev_ms / args.steps)

    stage = {}

    def wrap(name, fn):
        def inner(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **k)
            e1.record()
            stage.setdefault(name, []).append((e0, e1))
            return r
        return inner

    orig = (sam.encode_u8, pred.decode_low_res)
    sam.encode_u8 = wrap("encode", sam.encode_u8)
    pred.decode_low_res = wrap("decode", pred.decode_low_res)

    class _LWrap:  # the two generate() tail calls go through the ctypes handle
        def __init__(self, lib):
            self._lib = lib
            self.msam_mask_stats_lazy = wrap("mask_stats (lazy: masks passing the IoU filter)", lib.msam_mask_stats_lazy)
            self.msam_amg_filter_nms = wrap("filter_nms", lib.msam_amg_filter_nms)
            self.msam_paint_min_area = wrap("paint", lib.msam_paint_min_area)
            self.msam_finish_segmentation = wrap("finish_segmentation", lib.msam_finish_segmentation)

        def __getattr__(self, k):
            return getattr(self._lib, k)

    _lib._lib = _LWrap(L)
    survivors.clear()
    step_device(count=True)
    torch.cuda.synchronize()
    _lib._lib = L
    sam.encode_u8, pred.decode_low_res = orig
    stages = {k: sum(a.elapsed_time(b) for a, b in v) / N_TILES for k, v in stage.items()}
    surv = [int(s.item()) for s in survivors]
    # per-stage survivor counts of the last tile (filters evaluated with torch on the device's own statistics)
    d = amg.crop_list[0]
    n_iou = int((d["iou_preds"] > args.pred_iou_thresh).sum())
    n_stab = int(((d["iou_preds"] > args.pred_iou_thresh) & (d["stability_score"] >= args.stability_score_thresh)).sum())
    qs = torch.tensor([0.5, 0.8, 0.9, 0.95], device=device)
    stab_valid = d["stability_score"][~torch.isnan(d["stability_score"])]
    calib = {"iou_pred_quantiles_50_80_90_95": [round(float(v), 4) for v in torch.quantile(d["iou_preds"], qs)],
             "stability_quantiles_50_80_90_95": [round(float(v), 4) for v in torch.quantile(stab_valid, qs)]}

    dom = table[0]
    bound = dom["bound"]
    roof = {"bound": bound, "kernel": dom["kernel"],
            "achieved": dom["tflops"] if bound == "tensor" else dom["gbs"],
            "peak": pk["bf16_tflops_sustained"] if bound == "tensor" else pk["hbm_gbs"],
            "unit": "TFLOP/s" if bound == "tensor" else "GB/s",
            "frac": dom["frac_tensor"] if bound == "tensor" else dom["frac_hbm"],
            "peak_source": f"{pk_src} " + ("bf16_tflops_sustained" if bound == "tensor" else "hbm_gbs"),
            "launches_per_step": dom["launches_per_step"], "share_of_step": dom["share_of_step"],
            "avg_launch_ms": dom["ms_per_step"] / max(dom["launches_per_step"], 1),
            "note": "dominant kernel of the step by summed CUDA-event time (library-side events on the launching stream, "
                    "separate instrumented pass); achieved = ALGORITHMIC flops or bytes / that time",
            "whole_step": {"algorithmic_tflop_per_tile": (ENC_FLOPS[args.model] + 0.805e9 + GRID * GRID * DEC_FLOPS_PER_PROMPT) / 1e12,
                           "tflops": (ENC_FLOPS[args.model] + 0.805e9 + GRID * GRID * DEC_FLOPS_PER_PROMPT) * N_TILES
                                     / (dev_ms / args.steps * 1e-3) / 1e12,
                           "peak": pk["bf16_tflops_sustained"]},
            "kernels": table, "instrumented_kernel_ms_per_step": prof_ms}
    roof["whole_step"]["frac"] = roof["whole_step"]["tflops"] / pk["bf16_tflops_sustained"]
    out = {
        "metric": "1024x1024 tiles/s, embed + AMG", "value": value, "unit": "tiles/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": dev_ms / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": workload_config(args),
        "e2e": {"value": e2e_val, "unit": "tiles/s", "ms_per_step": e2e_time / args.steps,
                "h2d_bytes_per_step": int(N_TILES * TILE * TILE * 2 + N_TILES * GRID * GRID * 12),
                "d2h_bytes_per_step": int(N_TILES * TILE * TILE * 4)},
        "gpu_launches": launches, "clocks": clocks, "roofline": roof,
        "stages_ms_per_tile": stages,
        "survivors": {"per_tile_after_nms": surv, "last_tile": {"masks": int(d["iou_preds"].shape[0]), "after_iou_filter": n_iou,
                                                                 "after_stability_filter": n_stab, "after_box_nms": surv[-1]}},
        "survivors_last_tile": surv[-1],
        "threshold_calibration": calib,
        "worst_case": {"value": worst_val, "unit": "tiles/s", "ms_per_step": worst_ms / max(1, args.steps // 2),
                       "config": dict(workload_config(args), pred_iou_thresh=0.0, stability_score_thresh=0.0)},
    }
    if world == 1 and not args.no_cpu_baseline:
        out["cpu_baseline"] = cpu_baseline(args, 1)
    if world == 1 and not args.no_vith:
        del pred, sam, amg
        torch.cuda.empty_cache()
        (ms_tile, vith_batch), vith_rep = vit_h_roofline(device)
        tf = ENC_FLOPS["vit_h"] / (ms_tile * 1e-3) / 1e12
        out["vit_h_encoder"] = {"ms_per_tile": ms_tile, "tflops": tf, "frac_of_peak": tf / pk["bf16_tflops_sustained"],
                                "frac_of_burst_peak": tf / pk["bf16_tflops"],
                                "peak": pk["bf16_tflops_sustained"], "batch": vith_batch, "algorithmic_tflop_per_tile": 5.6418,
                                "kernels_ms_per_tile": {r["name"]: round(r["ms_per_tile"], 4) for r in vith_rep}}
    print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="cfg2", choices=["cfg1", "cfg2", "cfg3", "cfg4", "cfg5"])
    ap.add_argument("--model", default=None)
    ap.add_argument("--max-prompts", type=int, default=1024)
    ap.add_argument("--enc-batch", type=int, default=16, help="tiles per encoder pass (the engine chunks the 16-tile batch)")
    ap.add_argument("--pred-iou-thresh", type=float, default=BENCH_THRESH["pred_iou_thresh"])
    ap.add_argument("--stability-score-thresh", type=float, default=BENCH_THRESH["stability_score_thresh"])
    ap.add_argument("--box-nms-thresh", type=float, default=BENCH_THRESH["box_nms_thresh"])
    ap.add_argument("--no-vith", action="store_true")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write what the last timed step computed to DIR/<name>.npy (float32, fixed seeded samples)")
    args = ap.parse_args()
    if args.model is None:
        args.model = {"cfg1": "vit_t", "cfg2": "vit_b", "cfg3": "vit_l", "cfg4": "vit_h", "cfg5": "vit_b"}[args.config]
    if args.config != "cfg2":
        import bench_configs
        return bench_configs.main(args)
    if args.impl == "reference":
        run_reference(args)
    else:
        if not torch.cuda.is_available():
            raise SystemExit("bench.py: no CUDA device (the GPU path has no CPU fallback; use --impl reference)")
        run_ours(args)


if __name__ == "__main__":
    main()
