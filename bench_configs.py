"""bench.py --config cfg1 | cfg3 | cfg4: the other configurations of BASELINE.json, as extra JSON lines with bench.py's contract
(one rank per GPU under torchrun, barrier + CUDA events + max over ranks, `--impl reference` = the oracle port on host cores).

cfg1  vit_t (MobileSAM / TinyViT) precompute_image_embeddings on 512 x 512 float32 LM tiles (the reference's CPU-runnable
      case): a step = 16 tiles, one call per tile as the reference does it (util.py:902 _compute_2d).  `value` = device-resident
      (resized uint8 tiles in HBM, batch of 16 through the encoder), `e2e` = host float32 tile -> host embedding through
      precompute_image_embeddings (normalise + PIL resize 512 -> 1024 + H2D + encoder + D2H per tile).

cfg5  vit_b fine-tuning step on LIVECell-shaped batches (2 images of 512 x 512 per GPU, 25 box-prompted objects each): preprocess
      (torch resize) + encoder forward keeping activations + prompt encoder / mask decoder forward (training mode) + loss (dice +
      IoU MSE) + loss.backward() through the decoder and the encoder + gradient all-reduce over the ranks (NCCL, one flat fp32
      buffer, averaged) + AdamW update on the device.  One prompting iteration per step (the reference's further sub-iterations
      feed mask prompts, which have no backward pass here).  metric: images/s.
cfg3  vit_l tiled 3-D embedding precompute: uint8 EM volume 64 x 2048 x 2048, tile_shape (1024, 1024), halo (128, 128)
      -> 4 outer tiles of 1152^2 per plane, 256 encoder tiles, written to a zarr container (1 GiB of embeddings).
      The volume is FIXED (strong scaling): ranks take contiguous shards of the (z, tile) list, each writes its own chunks,
      rank 0 writes the signature; no collective.  metric: tiles/s, host volume -> container on disk (always end to end:
      the host crop / normalise / resize / D2H / chunk writes are the workload).
cfg4  vit_h batched_inference with 256 box prompts per tile over 128 synthetic 1024^2 tiles (box recipe of
      development/benchmark.py:108-116): tiles are sharded over the ranks (strong scaling), every rank embeds its tiles and
      decodes the boxes.  metric: tiles/s; `value` = device-resident (uint8 tiles + boxes in HBM, label images stay on the
      device), `e2e` = host uint16 tiles -> host uint32 label images through precompute_image_embeddings + batched_inference.
"""
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CFG3 = dict(shape=(64, 2048, 2048), tile_shape=(1024, 1024), halo=(128, 128), batch=16)
CFG4 = dict(n_tiles=128, n_boxes=256, tile=1024, enc_batch=8)


CFG1 = dict(n_tiles=16, tile=512)
CFG5 = dict(batch=2, tile=512, n_obj=25)


def _config(args):
    if args.config == "cfg1":
        return {"workload": f"{args.model} (MobileSAM TinyViT) precompute_image_embeddings, 16 synthetic 512x512 float32 LM tiles, one call "
                            "per tile (BASELINE.json configs[0]); seeded random-init weights",
                "tiles_per_step_per_gpu": CFG1["n_tiles"], "l2": "flushed between steps (256 MB buffer write)",
                "parallelism": "tile shards, one process per GPU, no collective (reference arm: host threads of rank 0)"}
    if args.config == "cfg5":
        return {"workload": f"{args.model} fine-tuning step, batch of 2 synthetic 512x512 images per GPU with 25 box-prompted objects each "
                            "(BASELINE.json configs[4]); seeded random-init weights; encoder + decoder forward, dice + IoU loss, backward through "
                            "decoder and encoder, gradient all-reduce, AdamW update; one prompting iteration",
                "images_per_step_per_gpu": CFG5["batch"], "objects_per_image": CFG5["n_obj"], "sub_iterations": 1,
                "l2": "working_set_exceeds_l2 (GBs of saved activations per step)",
                "parallelism": "data parallel replicas, one process per GPU, one NCCL all-reduce of the flat gradient buffer per step"}
    if args.config == "cfg3":
        return {"workload": f"{args.model} tiled 3d embedding precompute, 64x2048x2048 uint8 EM-like volume, tile_shape=(1024,1024) "
                            "halo=(128,128) -> 256 tiles of 1152^2, zarr container (BASELINE.json configs[2]); seeded random-init weights",
                "tiles_total": 256, "batch_size": CFG3["batch"], "l2": "gpu arm: working_set_exceeds_l2 (distinct tiles every batch)",
                "parallelism": "(z, tile) shards, one process per GPU, no collective (reference arm: host threads of rank 0)"}
    return {"workload": f"{args.model} batched_inference, 256 box prompts per tile, 128 synthetic 1024x1024 LM tiles "
                        "(BASELINE.json configs[3]); seeded random-init weights; embed + decode + paint",
            "tiles_total": CFG4["n_tiles"], "boxes_per_tile": CFG4["n_boxes"], "multimasking": False,
            "l2": "gpu arm: working_set_exceeds_l2 (distinct tiles every batch)",
            "parallelism": "tile shards, one process per GPU, no collective (reference arm: host threads of rank 0)"}


def _volume():
    """Band-limited uint8 noise (Gaussian-filtered white noise, sigma 3) -- generated plane by plane (seed = z)."""
    from scipy import ndimage
    z, h, w = CFG3["shape"]
    vol = np.empty((z, h, w), np.uint8)
    for k in range(z):
        v = ndimage.gaussian_filter(np.random.default_rng(k).standard_normal((h, w)).astype(np.float32), 3)
        vol[k] = ((v - v.min()) / (v.max() - v.min() + 1e-7) * 255).astype(np.uint8)
    return vol


def _dist():
    import torch.distributed as dist
    world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    return dist, world, rank, local, device


def _timed(dist, world, device, fn, steps, warmup):
    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
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
    t = torch.tensor([e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    barrier()
    return max(float(t[0]), float(t[1]))   # host work after the last kernel is part of the step


def run_cfg3(args):
    from bench import ClockSampler, peaks, ENC_FLOPS
    from oracle import sam_ref
    from micro_sam_b200 import _lib, util
    dist, world, rank, local, device = _dist()
    pk, _ = peaks()
    sd = {k: v for k, v in sam_ref.seeded_state_dict(args.model, seed=0).items() if k.startswith("image_encoder.")}
    pred = util.get_sam_model(args.model, device=device, state_dict=sd, max_batch=CFG3["batch"], max_prompts=1)
    vol = _volume()
    base = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    path = os.path.join(base, "msam_cfg3_bench.zarr")

    def step():
        if rank == 0 and os.path.exists(path):
            shutil.rmtree(path)
        if world > 1:
            dist.barrier()
        util.precompute_image_embeddings(pred, vol, save_path=path, tile_shape=CFG3["tile_shape"], halo=CFG3["halo"],
                                         batch_size=CFG3["batch"], rank=rank, world_size=world)

    sampler = ClockSampler(local) if rank == 0 else None
    l0 = _lib.launch_count()
    ms = _timed(dist, world, device, step, args.steps, min(args.warmup, 1))
    launches = (_lib.launch_count() - l0) / (args.steps + min(args.warmup, 1))
    clocks = sampler.stop() if sampler else None
    if rank == 0:
        from micro_sam_b200 import zarr_store
        f = zarr_store.open_group(path)
        ok = "input_size" in f.attrs and sorted(f["features"].keys()) == ["0", "1", "2", "3"] and \
            f["features"]["3"].shape == (64, 1, 256, 64, 64) and np.count_nonzero(f["features"]["2"][63]) > 0
        value = 256 * args.steps / (ms / 1e3)
        # encoder-only device rate for the roofline of the dominant kernels
        L = _lib.lib()
        x = torch.randint(0, 255, (CFG3["batch"], 1024, 1024, 3), dtype=torch.uint8, device=device)
        pred.model.encode_u8(x)
        L.msam_profile(1)
        pred.model.encode_u8(x)
        rep = sorted(_lib.profile_report(), key=lambda r: -r["ms"])
        L.msam_profile(0)
        enc_ms = sum(r["ms"] for r in rep) / CFG3["batch"]
        dom = rep[0]
        tf = dom["flops"] / (dom["ms"] * 1e-3) / 1e12
        out = {"metric": "1024x1024 tiles/s, tiled 3d embedding precompute to a zarr container", "value": value, "unit": "tiles/s",
               "n_gpus": world, "steps": args.steps, "warmup": min(args.warmup, 1), "ms_per_step": ms / args.steps,
               "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
               "config": _config(args),
               "e2e": {"value": value, "unit": "tiles/s", "h2d_bytes_per_step": 256 * 1024 * 1024 * 3,
                       "d2h_bytes_per_step": 256 * 256 * 64 * 64 * 4, "note": "this configuration is end to end by definition"},
               "gpu_launches": launches, "clocks": clocks, "container_ok": bool(ok),
               "roofline": {"bound": "tensor", "kernel": dom["name"], "achieved": tf, "peak": pk["bf16_tflops_sustained"],
                            "unit": "TFLOP/s", "frac": tf / pk["bf16_tflops_sustained"], "traffic": None,
                            "encoder_kernel_ms_per_tile": enc_ms,
                            "encoder_only_tiles_per_s": 1e3 / enc_ms,
                            "encoder_tflops": ENC_FLOPS[args.model] / (enc_ms * 1e-3) / 1e12,
                            "kernels_ms_per_tile": {r["name"]: round(r["ms"] / CFG3["batch"], 4) for r in rep}}}
        print(json.dumps(out))
        shutil.rmtree(path, ignore_errors=True)
    if world > 1:
        dist.destroy_process_group()


def run_cfg1(args):
    from bench import ClockSampler, peaks
    from oracle import sam_ref
    from micro_sam_b200 import _lib, util
    from micro_sam_b200.sam import ResizeLongestSide
    from micro_sam_b200.sample_data import lm_tile
    dist, world, rank, local, device = _dist()
    pk, _ = peaks()
    sd = {k: v for k, v in sam_ref.seeded_state_dict(args.model, seed=0).items() if k.startswith("image_encoder.")}
    pred = util.get_sam_model(args.model, device=device, state_dict=sd, max_batch=CFG1["n_tiles"], max_prompts=1)
    n = CFG1["n_tiles"]
    tiles = [lm_tile((CFG1["tile"],) * 2, 40, seed=rank * n + t).astype(np.float32) for t in range(n)]
    rs = ResizeLongestSide(1024)
    tiles_u8 = torch.from_numpy(np.stack([rs.apply_image(util._to_image(t)) for t in tiles])).to(device)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)

    def step_device():
        flush.fill_(1)
        return pred.model.encode_u8(tiles_u8)

    def step_e2e():
        flush.fill_(1)
        return [util.precompute_image_embeddings(pred, t, ndim=2)["features"] for t in tiles]

    sampler = ClockSampler(local) if rank == 0 else None
    l0 = _lib.launch_count()
    ms = _timed(dist, world, device, step_device, args.steps, args.warmup)
    launches = (_lib.launch_count() - l0) / (args.steps + args.warmup)
    ms_e2e = _timed(dist, world, device, step_e2e, args.steps, 1)
    clocks = sampler.stop() if sampler else None
    if rank == 0:
        L = _lib.lib()
        L.msam_profile(1)
        pred.model.encode_u8(tiles_u8)
        rep = sorted(_lib.profile_report(), key=lambda r: -r["ms"])
        L.msam_profile(0)
        dom = rep[0]
        tf, gbs = dom["flops"] / (dom["ms"] * 1e-3) / 1e12, dom["bytes"] / (dom["ms"] * 1e-3) / 1e9
        bound = "tensor" if tf / pk["bf16_tflops_sustained"] >= gbs / pk["hbm_gbs"] else "hbm"
        feats = step_e2e()
        out = {"metric": "512x512 tiles/s, vit_t precompute_image_embeddings", "value": n * world * args.steps / (ms / 1e3), "unit": "tiles/s",
               "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
               "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic", "config": _config(args),
               "e2e": {"value": n * world * args.steps / (ms_e2e / 1e3), "unit": "tiles/s", "ms_per_step": ms_e2e / args.steps,
                       "h2d_bytes_per_step": n * 1024 * 1024 * 3, "d2h_bytes_per_step": n * 256 * 64 * 64 * 4},
               "gpu_launches": launches, "clocks": clocks, "embedding_shape": list(np.asarray(feats[-1]).shape),
               "roofline": {"bound": bound, "kernel": dom["name"], "achieved": tf if bound == "tensor" else gbs,
                            "peak": pk["bf16_tflops_sustained"] if bound == "tensor" else pk["hbm_gbs"],
                            "unit": "TFLOP/s" if bound == "tensor" else "GB/s",
                            "frac": tf / pk["bf16_tflops_sustained"] if bound == "tensor" else gbs / pk["hbm_gbs"], "traffic": None,
                            "share_of_step": dom["ms"] / (ms / args.steps),
                            "kernels_ms_per_tile": {r["name"]: round(r["ms"] / n, 4) for r in rep}}}
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def _cfg5_batch(seed0):
    """LIVECell-like: 512 x 512 uint8 images with non-overlapping disks; the first n_obj disks become box prompts + targets."""
    rng = np.random.default_rng(seed0)
    S, n = CFG5["tile"], CFG5["n_obj"]
    recs, targets = [], []
    yy, xx = np.mgrid[:S, :S]
    for b in range(CFG5["batch"]):
        img = rng.normal(60, 8, (S, S)).astype(np.float32)
        boxes, masks, tries = [], [], 0
        while len(boxes) < n and tries < 5000:
            tries += 1
            r = rng.integers(8, 22)
            cy, cx = rng.integers(r + 1, S - r - 1, 2)
            if any((cy - py) ** 2 + (cx - px) ** 2 < (r + pr + 2) ** 2 for py, px, pr in masks):
                continue
            masks.append((cy, cx, r))
            boxes.append([cx - r, cy - r, cx + r, cy + r])
            img[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] += 90
        img = np.clip(img, 0, 255)
        tg = np.stack([((yy - cy) ** 2 + (xx - cx) ** 2 < r * r)[None] for cy, cx, r in masks]).astype(np.float32)
        recs.append({"image": torch.from_numpy(np.repeat(img[None], 3, 0)), "original_size": (S, S),
                     "boxes": torch.tensor(boxes, dtype=torch.float32) * (1024.0 / S)})
        targets.append(torch.from_numpy(tg))
    return recs, targets


def run_cfg5(args):
    from bench import ClockSampler, peaks, ENC_FLOPS
    from oracle import sam_ref
    from micro_sam_b200 import _lib, training, util
    dist, world, rank, local, device = _dist()
    pk, _ = peaks()
    pred = util.get_sam_model(args.model, device=device, state_dict=sam_ref.seeded_state_dict(args.model, seed=0),
                              max_batch=CFG5["batch"], max_prompts=64)
    sam = pred.model.train()
    m = training.TrainableSAM(sam)
    recs, targets = _cfg5_batch(100 + rank)
    state = {}

    def step():
        rr = [dict(r) for r in recs]
        sam.zero_decoder_grads()
        emb, rr = m.image_embeddings_oft(rr)                      # encoder forward, activations kept
        out = m(rr, emb, multimask_output=True, return_masks=False)   # prompt encoder + mask decoder, training mode
        loss = training.compute_loss(out, targets)
        loss[0].backward()                                        # loss -> decoder -> encoder
        n = sam.allreduce_grads(world)                            # one NCCL all-reduce of the flat gradient buffer, averaged
        sam.optimizer_step(lr=1e-5)                               # AdamW on the device + operand refresh
        state["loss"], state["n"] = float(loss[0]), n
        return n

    sampler = ClockSampler(local) if rank == 0 else None
    l0 = _lib.launch_count()
    ms = _timed(dist, world, device, step, args.steps, args.warmup)
    launches = (_lib.launch_count() - l0) / (args.steps + args.warmup)
    clocks = sampler.stop() if sampler else None
    # the instrumented step contains the gradient all-reduce: EVERY rank runs it (a rank-0-only step would wait for its peers until
    # the NCCL timeout), only rank 0 records the kernel events
    L = _lib.lib()
    if rank == 0:
        L.msam_profile(1)
    step()
    if rank == 0:
        rep = sorted(_lib.profile_report(), key=lambda r: -r["ms"])
        L.msam_profile(0)
        dom = rep[0]
        tf = dom["flops"] / (dom["ms"] * 1e-3) / 1e12
        n_img = CFG5["batch"] * world
        enc_flops = 3 * ENC_FLOPS[args.model] * CFG5["batch"]     # forward + ~2x backward, algorithmic
        out = {"metric": "images/s, fine-tuning step (forward + loss + backward + gradient all-reduce)", "value": n_img * args.steps / (ms / 1e3), "unit": "images/s",
               "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
               "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic", "config": _config(args),
               "e2e": {"value": n_img * args.steps / (ms / 1e3), "unit": "images/s", "h2d_bytes_per_step": CFG5["batch"] * 3 * 512 * 512 * 4,
                       "d2h_bytes_per_step": 4, "note": "host float images -> device every step; the loss value is read back"},
               "gpu_launches": launches, "clocks": clocks, "loss": state.get("loss"), "gradient_elements": state.get("n"),
               "roofline": {"bound": "tensor", "kernel": dom["name"], "achieved": tf, "peak": pk["bf16_tflops_sustained"], "unit": "TFLOP/s",
                            "frac": tf / pk["bf16_tflops_sustained"], "traffic": None, "share_of_step": dom["ms"] / (ms / args.steps),
                            "encoder_fwd_bwd_tflops": enc_flops / (ms / args.steps * 1e-3) / 1e12,
                            "kernels_ms_per_step": {r["name"]: round(r["ms"], 3) for r in rep}}}
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def _cfg4_inputs(rank, world):
    from micro_sam_b200.sample_data import lm_tile, random_boxes
    lo, hi = (CFG4["n_tiles"] * rank) // world, (CFG4["n_tiles"] * (rank + 1)) // world
    tiles = np.stack([lm_tile((CFG4["tile"],) * 2, 150, seed=t) for t in range(lo, hi)])
    boxes = [random_boxes(CFG4["n_boxes"], (CFG4["tile"],) * 2, seed=t) for t in range(lo, hi)]
    return tiles, boxes


def run_cfg4(args):
    from bench import ClockSampler, peaks
    from oracle import sam_ref
    from micro_sam_b200 import _lib, inference, util
    dist, world, rank, local, device = _dist()
    pk, _ = peaks()
    pred = util.get_sam_model(args.model, device=device, state_dict=sam_ref.seeded_state_dict(args.model, seed=0),
                              max_batch=CFG4["enc_batch"], max_prompts=CFG4["n_boxes"])
    tiles, boxes = _cfg4_inputs(rank, world)
    n_local = len(tiles)
    tiles_u8 = torch.from_numpy(np.stack([util._to_image(t) for t in tiles])).to(device)
    T = CFG4["tile"]

    def step_e2e():
        segs = []
        for b0 in range(0, n_local, CFG4["enc_batch"]):
            emb = util.precompute_image_embeddings(pred, tiles[b0:b0 + CFG4["enc_batch"]], ndim=3, batch_size=CFG4["enc_batch"],
                                                   to_numpy=False)
            for k in range(emb["features"].shape[0]):
                util.set_precomputed(pred, emb, i=k)
                segs.append(inference.batched_inference(pred, None, batch_size=CFG4["n_boxes"], boxes=boxes[b0 + k]))
        return segs

    def step_device():
        out = None
        for b0 in range(0, n_local, CFG4["enc_batch"]):
            feats = pred.model.encode_u8(tiles_u8[b0:b0 + CFG4["enc_batch"]])
            for k in range(feats.shape[0]):
                util.set_precomputed(pred, {"features": feats[k:k + 1], "input_size": (T, T), "original_size": (T, T)})
                out = inference.batched_inference(pred, None, batch_size=CFG4["n_boxes"], boxes=boxes[b0 + k], device_result=True)
        return out

    sampler = ClockSampler(local) if rank == 0 else None
    l0 = _lib.launch_count()
    ms = _timed(dist, world, device, step_device, args.steps, min(args.warmup, 1))
    launches = (_lib.launch_count() - l0) / (args.steps + min(args.warmup, 1))
    clocks = sampler.stop() if sampler else None
    ms_e2e = _timed(dist, world, device, step_e2e, args.steps, 1)
    if rank == 0:
        L = _lib.lib()
        L.msam_profile(1)
        step_device()
        rep = sorted(_lib.profile_report(), key=lambda r: -r["ms"])
        L.msam_profile(0)
        dom = rep[0]
        tf, gbs = dom["flops"] / (dom["ms"] * 1e-3) / 1e12, dom["bytes"] / (dom["ms"] * 1e-3) / 1e9
        bound = "tensor" if tf / pk["bf16_tflops_sustained"] >= gbs / pk["hbm_gbs"] else "hbm"
        seg = step_e2e()[-1]
        out = {"metric": "1024x1024 tiles/s, embed + batched_inference (256 boxes/tile)", "value": CFG4["n_tiles"] * args.steps / (ms / 1e3),
               "unit": "tiles/s", "n_gpus": world, "steps": args.steps, "warmup": min(args.warmup, 1), "ms_per_step": ms / args.steps,
               "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
               "config": _config(args),
               "e2e": {"value": CFG4["n_tiles"] * args.steps / (ms_e2e / 1e3), "unit": "tiles/s", "ms_per_step": ms_e2e / args.steps,
                       "h2d_bytes_per_step": n_local * (T * T * 2 + CFG4["n_boxes"] * 16), "d2h_bytes_per_step": n_local * T * T * 4},
               "gpu_launches": launches, "clocks": clocks, "instances_last_tile": int(seg.max()),
               "roofline": {"bound": bound, "kernel": dom["name"], "achieved": tf if bound == "tensor" else gbs,
                            "peak": pk["bf16_tflops_sustained"] if bound == "tensor" else pk["hbm_gbs"],
                            "unit": "TFLOP/s" if bound == "tensor" else "GB/s",
                            "frac": tf / pk["bf16_tflops_sustained"] if bound == "tensor" else gbs / pk["hbm_gbs"], "traffic": None,
                            "share_of_step": dom["ms"] / (ms / args.steps),
                            "kernels_ms_per_tile": {r["name"]: round(r["ms"] / n_local, 4) for r in rep}}}
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def run_reference(args):
    """The oracle port on the host cores, bounded sample: cfg1 = 4 of the 16 tiles (normalise + resize + TinyViT encoder each);
    cfg3 = one 1152^2 tile (normalise + resize + vit_l encoder); cfg4 = one tile (vit_h encoder) + 32 of its 256 boxes through
    batched_inference (decoder part scaled x8)."""
    if int(os.environ.get("RANK", "0")) != 0:
        return
    from bench import best_cpu_threads
    from oracle import amg_ref, sam_ref
    threads = best_cpu_threads()
    torch.set_num_threads(threads)
    sam = sam_ref.build_seeded_sam(args.model, seed=0)
    pred = sam_ref.SamPredictor(sam)
    vals, t_all = [], time.perf_counter()
    for it in range(args.steps + (1 if args.warmup > 0 else 0)):
        if args.config == "cfg5":
            from oracle import train_ref
            recs, targets = _cfg5_batch(100)
            recs, targets = recs[:1], targets[:1]
            om = train_ref.TrainableSAM(sam)
            for p in sam.parameters():
                p.requires_grad_(True)
            t0 = time.perf_counter()
            emb, rr = om.image_embeddings_oft([dict(r) for r in recs])
            loss = train_ref.compute_loss(om(rr, emb, multimask_output=True), targets)
            loss[0].backward()
            per_tile = time.perf_counter() - t0
            sam.zero_grad(set_to_none=True)
            sample = f"1 of 2 images: forward + loss ({float(loss[0]):.3f}) + backward (torch autograd, fp32) {per_tile:.1f}s"
        elif args.config == "cfg1":
            from micro_sam_b200.sample_data import lm_tile
            tiles = [lm_tile((CFG1["tile"],) * 2, 40, seed=t).astype(np.float32) for t in range(4)]
            t0 = time.perf_counter()
            for t in tiles:
                amg_ref.precompute_image_embeddings_2d(pred, t)
            per_tile = (time.perf_counter() - t0) / len(tiles)
            sample = f"4 of 16 tiles (512^2 -> 1024^2, {args.model} encoder) {per_tile:.2f}s each"
        elif args.config == "cfg3":
            from scipy import ndimage
            v = ndimage.gaussian_filter(np.random.default_rng(0).standard_normal((1152, 1152)).astype(np.float32), 3)
            tile = ((v - v.min()) / (v.max() - v.min() + 1e-7) * 255).astype(np.uint8)
            t0 = time.perf_counter()
            amg_ref.precompute_image_embeddings_2d(pred, tile)
            per_tile = time.perf_counter() - t0
            sample = f"1 of 256 tiles (1152^2 -> 1024^2, {args.model} encoder) {per_tile:.2f}s"
        else:
            from micro_sam_b200.sample_data import lm_tile, random_boxes
            img, bx = lm_tile((1024, 1024), 150, seed=0), random_boxes(CFG4["n_boxes"], (1024, 1024), seed=0)
            t0 = time.perf_counter()
            emb = amg_ref.precompute_image_embeddings_2d(pred, img)
            t_emb = time.perf_counter() - t0
            t0 = time.perf_counter()
            amg_ref.batched_inference(pred, img, batch_size=32, boxes=bx[:32], image_embeddings=emb)
            t_dec = time.perf_counter() - t0
            per_tile = t_emb + 8 * t_dec
            sample = f"1 of 128 tiles: embed {t_emb:.2f}s + 32 of 256 boxes {t_dec:.2f}s (scaled x8)"
        if it > 0 or args.warmup == 0:
            vals.append(1.0 / per_tile)
    v = float(np.mean(vals))
    cb = {"value": v, "unit": "tiles/s", "cores": threads, "kind": "port", "sample": sample}
    unit = "images/s" if args.config == "cfg5" else "tiles/s"
    cb["unit"] = unit
    print(json.dumps({"impl": "reference", "metric": {"cfg1": "512x512 tiles/s", "cfg5": "images/s, fine-tuning step (forward + loss + backward + gradient all-reduce)"}.get(args.config, "1024x1024 tiles/s"), "value": v, "unit": unit, "n_gpus": args.gpus,
                      "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * (time.perf_counter() - t_all) / max(args.steps, 1),
                      "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                      "config": _config(args), "cpu_baseline": cb,
                      "e2e": {"value": v, "unit": unit, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))


def main(args):
    if args.impl == "reference":
        return run_reference(args)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the GPU path has no CPU fallback; use --impl reference)")
    return {"cfg1": run_cfg1, "cfg3": run_cfg3, "cfg4": run_cfg4, "cfg5": run_cfg5}[args.config](args)
