"""Timing (not a test) at the cfg 5 training shape -- vit_b, B = 2 images of 512 x 512, 25 objects, 8 sub-iterations:
  1. one iterative prompt update (`training.IterativePromptUpdate`, csrc/prompts.cu) on the best low-res logits;
  2. the same update the reference's way on the same GPU: per object torch.where on the full-size masks and targets, then
     np.random.choice on the host (IterativePromptGenerator + SamTrainer._update_prompts, oracle/prompt_ref.py);
  3. one whole `training.interactive_train_iteration` against `compute_iterative_loss` driven by the reference-style update
     (which needs the full-size masks of every pass), same prompts of pass 0.
Seeded vit_b weights.  Prints the card and its power limit.  Run from the repository root on the GPU:
`python tests/time_prompt_update.py`."""
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import training, util  # noqa: E402
from micro_sam_b200.sample_data import lm_tile  # noqa: E402
from oracle import sam_ref  # noqa: E402
from oracle.prompt_ref import ReferenceStyleUpdate  # noqa: E402

B, S, N_OBJ, N_SUB = 2, 512, 25, 8


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    sd = sam_ref.seeded_state_dict("vit_b", seed=0)
    sam = util.get_sam_model("vit_b", state_dict=sd, max_batch=B, max_prompts=64).model
    sam.train()
    m = training.TrainableSAM(sam)
    x = torch.stack([torch.from_numpy(np.repeat(lm_tile((S, S), 40, seed=b, dtype="uint8")[None], 3, 0).astype("float32")) for b in range(B)])
    yy, xx = np.mgrid[:S, :S]
    y = np.zeros((B, 1, S, S), np.float32)
    rng = np.random.default_rng(0)
    for b in range(B):
        for k in range(40):
            cy, cx, r = rng.integers(20, S - 20, 2).tolist() + [int(rng.integers(6, 20))]
            y[b, 0][(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = k + 1
    y = torch.from_numpy(y)

    # 1 / 2: one prompt update on the outputs of one decoder pass
    np.random.seed(0)
    conv = training.ConvertToSamInputs(m.transform)
    recs, ids = conv(x, y, 1, 0, False, N_OBJ)
    recs, y1h = training.preprocess_batch(recs, y, ids)
    with torch.no_grad():
        emb, recs = m.image_embeddings_oft(recs)
        outs = m(recs, emb.detach(), multimask_output=True, return_masks=True)
        masks, logits = training.get_best_masks(outs)

    def fresh():
        return [{k: v for k, v in r.items()} for r in recs]

    def time_update(upd, full, n):
        for _ in range(2):
            upd(fresh(), masks if full else None, logits)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        s.record()
        for _ in range(n):
            upd(fresh(), masks if full else None, logits)
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / n, (time.perf_counter() - t0) * 1e3 / n

    lib_upd = training.IterativePromptUpdate(y1h, m.transform, 0.5)
    ref_upd = ReferenceStyleUpdate(y1h, m.transform, 0.5)
    for rep in range(3):
        a = time_update(lib_upd, False, 50)
        b = time_update(ref_upd, True, 3)
        print(f"rep {rep}: prompt update, library {a[0]:.3f} ms (events) / {a[1]:.3f} ms (host, synchronised); "
              f"reference-style {b[0]:.1f} ms / {b[1]:.1f} ms", flush=True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        lib_upd(fresh(), None, logits)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "iterative_kernel" in ev.key:
            print(f"iterative_kernel (B * n_obj = {B * N_OBJ} CTAs): {ev.device_time_total / 1000:.3f} ms device time", flush=True)

    # 3: whole step
    def step_library(seed):
        np.random.seed(seed); random.seed(seed)
        sam.zero_decoder_grads()
        loss = training.interactive_train_iteration(m, x, y, 0, n_objects_per_batch=N_OBJ, n_sub_iteration=N_SUB, mask_prob=0.5)[0]
        loss.backward()

    def step_reference_style(seed):
        np.random.seed(seed); random.seed(seed)
        sam.zero_decoder_grads()
        n_pos, n_neg, get_boxes, mm = training.get_prompt_and_multimasking_choices(0)
        r, i = training.ConvertToSamInputs(m.transform)(x, y, n_pos, n_neg, get_boxes, N_OBJ)
        r, yo = training.preprocess_batch(r, y, i)
        loss = training.compute_iterative_loss(m, r, yo, N_SUB, mm, ReferenceStyleUpdate(yo, m.transform, 0.5), full_masks=True)[0]
        loss.backward()

    for f in (step_library, step_reference_style):
        f(0)
    torch.cuda.synchronize()
    for rep in range(3):
        res = []
        for f in (step_library, step_reference_style):
            t0 = time.perf_counter()
            for k in range(3):
                f(k + 1)
            torch.cuda.synchronize()
            res.append((time.perf_counter() - t0) * 1e3 / 3)
        print(f"rep {rep}: training step ({N_SUB} passes, forward + backward), interactive_train_iteration {res[0]:.1f} ms; "
              f"compute_iterative_loss with the reference-style update {res[1]:.1f} ms", flush=True)


if __name__ == "__main__":
    main()
