"""bf16 noise floor of the UNETR decoder's training step (forward + backward), measured on the CPU.  The float64 training-mode
restatement (tests/unetr_train_ref.py) is compared with the device mirror of tests/unetr_train_mirror.py run in float32, which
rounds to bf16 where the kernels of csrc/ais.cu / csrc/ais_train.cu do (that module lists the rounding points).  Both are fed
the same bf16-rounded weights and embedding, so the floor is what the device's own rounding adds.  Prints the floor per
parameter tensor and for d embedding, per plan, as JSON; the GPU bounds of tests/test_gpu_unetr_train.py are twice these."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import unetr_ref  # noqa: E402
from tests import unetr_train_mirror as mirror  # noqa: E402
from tests import unetr_train_ref as ref  # noqa: E402

REDUCED = dict(emb=64, feats=(128, 64, 64, 64), deconv=(64, 64, 64, 64), head_in=64)
# (state dict kwargs, embedding shape): the whole-decoder cases of the GPU test
CASES = {"interp": (dict(transposed=False, affine=False, **REDUCED), (2, 64, 16, 16)),
         "transposed": (dict(transposed=True, affine=False, **REDUCED), (2, 64, 16, 16)),
         "affine": (dict(transposed=False, affine=True, **REDUCED), (2, 64, 16, 16))}
STATE_SEED, DATA_SEED = 7, 8


def case_inputs(name):
    """(state dict with bf16-rounded weights, bf16-rounded embedding, upstream gradient of the maps)"""
    kw, shape = CASES[name]
    sd = unetr_ref.seeded_state(seed=STATE_SEED, **kw)
    sd = mirror.device_weights(sd)
    g = torch.Generator().manual_seed(DATA_SEED)
    z = mirror.bf(torch.randn(shape, generator=g))
    dm = torch.randn(shape[0], 3, 16 * shape[2], 16 * shape[3], generator=g)
    return sd, z, dm


def grads(sd, z, dm, dtype, emulate):
    """(gradients with "d_embedding", maps): the device mirror of tests/unetr_train_mirror.py (emulate) or the float64
    restatement"""
    if emulate:
        g, maps, _ = mirror.run(sd, z, dm, dtype)
        return g, maps
    lv = ref.leaves(sd)
    zz = z.to(dtype).requires_grad_(True)
    maps = ref.forward_maps(lv, zz, train=True)
    (maps * dm.to(dtype)).sum().backward()
    out = {k: v.grad for k, v in lv.items() if isinstance(v, torch.Tensor) and v.grad is not None}
    out["d_embedding"] = zz.grad
    return out, maps.detach()


zero_grad_keys = mirror.zero_grad_keys


def floors(name):
    sd, z, dm = case_inputs(name)
    g64, _ = grads(sd, z, dm, torch.float64, False)
    g32, _ = grads(sd, z, dm, torch.float32, True)
    skip = zero_grad_keys(g64)
    return {k: ref.rel_l2(g32[k], g64[k]) for k in g64 if k not in skip}


def main():
    for name in CASES:
        f = floors(name)
        print(json.dumps({"plan": name, "max": max(f.values()), "d_embedding": f["d_embedding"], "per_tensor": f}))


if __name__ == "__main__":
    main()
