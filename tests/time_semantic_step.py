"""Times one semantic fine-tuning step at vit_b widths (seeded weights), C = 3, 1024^2 inputs, B = 2 and 8: the encoder's training
forward, the prompt-free decode of the whole batch in one slot, the loss (compute_semantic_loss), loss.backward() (loss adjoint,
decoder backward, encoder backward) and the AdamW step.  Each stage is bracketed by CUDA events; the table is the mean over the
timed steps after warm-up.  At B = 8 it also times the decoder alone, forward + backward on fixed embeddings, for the prompt-free
batch in one slot and for B per-image decodes with one box each (the prompted path, one slot per image).  Then it tries a vit_b
training forward (encoder + decode) at B = 16 and reports the device memory in use after it, or the error if it did not run.
Prints one JSON line per case, with the card's name and power limit read in the same run (and appends them to --out when given).
Usage:  python tests/time_semantic_step.py [--steps 5] [--warmup 2] [--out path.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import training  # noqa: E402
from oracle import sam_ref  # noqa: E402

STAGES = ("encoder_forward", "decode", "loss", "backward", "optimizer_step")


def labels(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(0, 3, (B, 1, H // 32, W // 32), generator=g)
    return y.repeat_interleave(32, 2).repeat_interleave(32, 3).contiguous()


def step_case(sd, B, steps, warmup, card):
    model = training.get_trainable_sam_model("vit_b", state_dict=sd, max_batch=B)
    sam = model.sam
    g = torch.Generator().manual_seed(B)
    x = (torch.rand(B, 3, 1024, 1024, generator=g) * 255).cuda()
    y = labels(B, 1024, 1024, B).cuda()
    times = {s: 0.0 for s in STAGES}
    for it in range(warmup + steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
        sam.zero_decoder_grads()
        batched = training.ConvertToSemanticSamInputs()(x, y)
        ev[0].record()
        emb, batched = model.image_embeddings_oft(batched)
        ev[1].record()
        outs = model(batched, emb, multimask_output=True, return_masks=False)
        ev[2].record()
        loss = training.compute_semantic_loss(outs, y, 3)
        ev[3].record()
        loss.backward()
        ev[4].record()
        sam.optimizer_step(lr=1e-5)
        ev[5].record()
        ev[5].synchronize()
        if it >= warmup:
            for i, s in enumerate(STAGES):
                times[s] += ev[i].elapsed_time(ev[i + 1]) / steps
    out = {"case": f"vit_b_semantic_step_B{B}_1024", **card, "steps": steps, "warmup": warmup,
           **{f"{s}_ms": round(t, 3) for s, t in times.items()}, "step_ms": round(sum(times.values()), 3),
           "images_per_s": round(B / sum(times.values()) * 1e3, 2)}
    return model, out


def decoder_case(model, B, steps, warmup, card):
    """decoder forward + backward on fixed embeddings: one prompt-free batch in one slot against B one-box decodes in B slots"""
    sam = model.sam
    g = torch.Generator().manual_seed(7)
    emb = torch.randn(B, 256, 64, 64, generator=g).cuda()
    d_low = (torch.randn(B, 3, 256, 256, generator=g) / 256).cuda()
    box = torch.tensor([[100.0, 120.0, 600.0, 700.0]], device="cuda")

    def free():
        e = emb.clone().requires_grad_(True)
        low, _ = sam.decoder_train_images(e, True, slot=0)
        low.backward(d_low)

    def per_image():
        for b in range(B):
            e = emb[b].clone().requires_grad_(True)
            low, _ = sam.decoder_train(e, None, box, True, slot=b)
            low.backward(d_low[b:b + 1])

    res = {}
    for name, fn in (("prompt_free_one_slot", free), ("one_box_per_image_slots", per_image)):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        b.synchronize()
        res[f"{name}_ms"] = round(a.elapsed_time(b) / steps, 3)
    return {"case": f"vit_b_decoder_forward_backward_B{B}", **card, **res}


def memory_case(sd, card):
    """a vit_b training forward (encoder + prompt-free decode) at B = 16, with the device memory in use after it"""
    B = 16
    out = {"case": "vit_b_training_forward_B16_1024", **card}
    try:
        model = training.get_trainable_sam_model("vit_b", state_dict=sd, max_batch=B)
        x = torch.rand(B, 3, 1024, 1024, device="cuda") * 255
        y = labels(B, 1024, 1024, 3).cuda()
        emb, batched = model.image_embeddings_oft(training.ConvertToSemanticSamInputs()(x, y))
        model(batched, emb, multimask_output=True, return_masks=False)
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        out.update(ran=True, device_memory_in_use_GiB=round((total - free) / 2**30, 2), device_memory_GiB=round(total / 2**30, 2))
        del model, emb
    except Exception as exc:   # reported, not hidden: the record says it did not run and why
        out.update(ran=False, error=f"{type(exc).__name__}: {exc}"[:300])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_semantic_step.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    card = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}
    sd = sam_ref.seeded_state_dict("vit_b", seed=0)
    lines = []
    for B in (2, 8):
        model, rec = step_case(sd, B, args.steps, args.warmup, card)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
        if B == 8:
            lines.append(json.dumps(decoder_case(model, B, args.steps, args.warmup, card)))
            print(lines[-1], flush=True)
        del model
        torch.cuda.empty_cache()
    lines.append(json.dumps(memory_case(sd, card)))
    print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
