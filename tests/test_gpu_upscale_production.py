"""The fused up-scaling block (msam_op_dec_upscale) at the production AMG chunk of P = 1024 prompts, with multimask on and
off, against the float64 reference of test_gpu_decoder_blocks.

At this size every CTA of the persistent kernel runs hundreds of (prompt, token row) items, its two consumer warpgroups
alternate over them and each reloads its hyper-network tile at every prompt change; CTA ranges start in the middle of
prompts.  The block tests stop at P = 64, so this covers what only the benchmark's chunk size reaches.  A seeded sample of
32 prompts -- 16 of the prompts in which a CTA range starts, the first and last prompt and random others --
is compared under TOL_UP; the whole output must be finite, fully written (no sentinel left inside) and the margins
around it untouched.

Measured on one H100 80GB HBM3 at a 700 W power limit: rel-L2 8.5e-4, worst row 1.33e-3 (multimask) and 8.2e-4, 1.26e-3
(single mask), inside the same bounds as the block tests.
"""
import random

import pytest
import torch

from tests.test_gpu_decoder_blocks import DC, DEV, NI, SENT_F32, TOL_UP, check, env, ref_up, run_up  # noqa: F401

P = 1024
ITEMS_PER_PROMPT = 64   # the kernel's work item is one row of 64 image tokens


@pytest.fixture(scope="module")
def prod(env):  # noqa: F811
    from micro_sam_b200 import util
    pred = util.get_sam_model("vit_test", state_dict=env["sd"], max_batch=1, max_prompts=P)
    g = torch.Generator(device=DEV).manual_seed(1234)
    keys = torch.randn(P * NI, DC, device=DEV, generator=g).to(torch.bfloat16)
    hyper = torch.randn(P, 4, 32, device=DEV, generator=g) * 0.5
    return pred.model, keys, hyper


def sample_prompts(n_sm, n=32):
    """Prompts whose items are split between two CTAs at a grid of n_sm CTAs, then the ends and seeded random others."""
    total = P * ITEMS_PER_PROMPT
    split = sorted({(total * b // n_sm) // ITEMS_PER_PROMPT for b in range(1, n_sm) if (total * b // n_sm) % ITEMS_PER_PROMPT})
    rng = random.Random(5)
    pick = set(rng.sample(split, min(16, len(split)))) | {0, P - 1}
    rest = [p for p in range(P) if p not in pick]
    pick |= set(rng.sample(rest, n - len(pick)))
    return sorted(pick), split


@pytest.mark.gpu
@pytest.mark.parametrize("multimask", [True, False])
def test_upscale_production_chunk(env, prod, multimask):  # noqa: F811
    sam, keys, hyper = prod
    got = run_up(env, keys, hyper, P, multimask, sam=sam)
    nm = got.shape[1]
    assert bool(torch.isfinite(got).all()), "non-finite logits"
    assert int((got == SENT_F32).sum()) == 0, "some logits were never written"
    idx, split = sample_prompts(env["n_sm"])
    assert len(split) > 0 and any(p in split for p in idx)
    sel = torch.tensor(idx, device=DEV)
    ref = ref_up(env["md"], keys.view(P, NI, DC)[sel].reshape(-1, DC), hyper[sel], len(idx), multimask)
    check(f"upscale P={P} mm={multimask} ({len(idx)} prompts)", got[sel], ref, len(idx) * nm * 256, TOL_UP)
