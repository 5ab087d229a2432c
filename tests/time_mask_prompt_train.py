"""Timing (not a test): the training-mode mask decoder, forward + backward of one image's P = 25 box prompts (the cfg 5 shape), with
and without mask prompts, alternating; then the mask-downscaling block alone and its kernels under torch.profiler.  The decoder
of every SAM size is the same, so the seeded vit_test model stands for vit_b here.  Run from the repository root on the GPU:
`python tests/time_mask_prompt_train.py`."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from micro_sam_b200 import util
from oracle import sam_ref
sd = sam_ref.seeded_state_dict("vit_test", seed=1)
sam = util.get_sam_model("vit_test", state_dict=sd, max_batch=2, max_prompts=64).model
sam.train()
P = 25
g = torch.Generator().manual_seed(0)
emb = torch.randn(256, 64, 64, generator=g).cuda()
xy = torch.rand(P, 2, generator=g) * 600 + 50
boxes = torch.cat([xy, xy + 200], 1).cuda()
masks = (torch.randn(P, 1, 256, 256, generator=g) * 4).cuda()
d_low = (torch.randn(P, 1, 256, 256, generator=g) / 256).cuda()
d_iou = torch.randn(P, 1, generator=g).cuda()
def run(mk):
    e = emb.clone().requires_grad_(True)
    low, iou = sam.decoder_train(e, None, boxes, False, slot=0, masks=mk)
    torch.autograd.backward([low, iou], [d_low, d_iou])
def timeit(mk, n=20):
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); s.record()
    for _ in range(n): run(mk)
    t.record(); torch.cuda.synchronize()
    return s.elapsed_time(t) / n
import subprocess
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
for mk in (None, masks):
    run(mk)
    run(mk)
res = {"unmasked": [], "masked": []}
for r in range(5):
    res["unmasked"].append(timeit(None)); res["masked"].append(timeit(masks))
med = {k: sorted(v)[2] for k, v in res.items()}
print("decoder_train fwd+bwd P=25 ms per pass (5 alternating reps of 20):", {k: [round(x, 3) for x in v] for k, v in res.items()}, "median", med,
      f"overhead {100 * (med['masked'] / med['unmasked'] - 1):.1f}%")
# the mask kernels alone, through the op entry point
from micro_sam_b200 import _lib
dd = torch.randn(P, 4096, 256, device="cuda"); dense = torch.empty_like(dd); gr = torch.empty(4684, device="cuda")
def op():
    _lib.check(_lib.lib().msam_op_mask_downscaling_train(sam._h, _lib.ptr(masks), P, _lib.ptr(dd), _lib.ptr(dense), _lib.ptr(gr), _lib.cur_stream()))
op(); torch.cuda.synchronize()
s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s.record()
for _ in range(50): op()
t.record(); torch.cuda.synchronize()
print(f"msam_op_mask_downscaling_train P=25 (forward + backward of the block alone): {s.elapsed_time(t) / 50:.3f} ms")
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    run(masks); torch.cuda.synchronize()
for ev in prof.key_averages():
    if "md_" in ev.key or "src_" in ev.key:
        print("kernel", ev.key[:60], f"{ev.device_time_total / 1000:.3f} ms")
