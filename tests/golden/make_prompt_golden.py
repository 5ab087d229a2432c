"""Generates tests/golden/prompt_regions.npz by EXECUTING THE REFERENCE's own micro_sam/prompt_generators.py in this container (run
once here; the GPU box has no /root/reference).  It records the sets the reference samples prompt points from: every
single-argument `torch.where` call the generator makes.  Each object is passed alone, so the last such call of a method is the set
its point is drawn from (after the reference's own fallbacks):
  * PointAndBoxPromptGenerator: `_sample_positive_points` (the object), `_sample_negative_points` (the ring
    |box widened by ds - dilated object|), `_ensure_num_points` (the fill-up background);
  * IterativePromptGenerator: `_get_positive_points` (false negatives, else the overlap) and `_get_negative_points` (false
    positives, else the box ring, else the background).
kornia is not installed: `kornia.morphology.dilation(x, ones(3, 3), engine="convolution")` is stood in for by a 3 x 3 max-pool
that pads with -inf (kornia's geodesic border).  That stand-in is UNPINNED: the dilation itself is not the reference's code.
Usage:  python tests/golden/make_prompt_golden.py
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

REF = "/root/reference/micro_sam"
OUT = os.path.dirname(os.path.abspath(__file__))


def load_prompt_generators():
    kornia = types.ModuleType("kornia")
    morphology = types.ModuleType("kornia.morphology")

    def dilation(x, kernel, engine="convolution"):
        assert tuple(kernel.shape) == (3, 3) and bool((kernel == 1).all())
        return torch.nn.functional.max_pool2d(torch.nn.functional.pad(x, (1, 1, 1, 1), value=-float("inf")), 3, stride=1)

    morphology.dilation = dilation
    kornia.morphology = morphology
    sys.modules["kornia"], sys.modules["kornia.morphology"] = kornia, morphology
    spec = importlib.util.spec_from_file_location("ref_prompt_generators", os.path.join(REF, "prompt_generators.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class WhereRecorder:
    """records the results of single-argument torch.where calls as boolean planes"""

    def __init__(self, shape):
        self.shape, self.calls, self._orig = shape, [], torch.where

    def __enter__(self):
        def where(*args, **kw):
            out = self._orig(*args, **kw)
            if len(args) == 1 and not kw:
                plane = np.zeros(self.shape, bool)
                plane[out[-2].numpy(), out[-1].numpy()] = True
                self.calls.append(plane)
            return out
        torch.where = where
        return self

    def __exit__(self, *exc):
        torch.where = self._orig


def label_images():
    rng = np.random.default_rng(0)
    H, W = 48, 40
    yy, xx = np.mgrid[:H, :W]
    lab = np.zeros((H, W), np.int64)
    for k in range(5):
        cy, cx, r = rng.integers(6, H - 6), rng.integers(6, W - 6), rng.integers(2, 6)
        lab[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = k + 1
    lab[20:26, 0:5] = 6; lab[20:26, 5:9] = 7          # touching, on the border
    lab[0:3, W - 4:W] = 8                               # corner
    lab[H - 1, 10] = 9                                  # 1 pixel
    lab[30:46, 15:38] = 10
    lab[35:40, 20:25] = 11                              # hole in object 10
    return lab


def main():
    pg = load_prompt_generators()
    lab = label_images()
    ids = np.unique(lab)[1:]
    objs = np.stack([lab == i for i in ids])
    boxes = []
    for o in objs:
        ys, xs = np.nonzero(o)
        boxes.append([ys.min(), xs.min(), ys.max() + 1, xs.max() + 1])
    boxes = np.array(boxes, np.int64)
    boxes_big = boxes.copy()                            # distorted-style boxes: larger than the object
    boxes_big[:, :2] = np.maximum(boxes[:, :2] - 2, 0)
    boxes_big[:, 2] = np.minimum(boxes[:, 2] + 3, lab.shape[0]); boxes_big[:, 3] = np.minimum(boxes[:, 3] + 3, lab.shape[1])
    out = {"label": lab, "ids": ids, "boxes": boxes, "boxes_big": boxes_big}
    np.random.seed(0)
    for ds in (0, 1, 3, 10):
        for name, bx in (("box", boxes), ("bigbox", boxes_big)):
            gen = pg.PointAndBoxPromptGenerator(1, 1, ds)
            pos, ring, fill = [], [], []
            for o, b in zip(objs, bx):
                m = torch.from_numpy(o.astype(np.float32))
                with WhereRecorder(o.shape) as r:
                    gen._sample_positive_points(m, None, [], [])
                pos.append(r.calls[-1])
                with WhereRecorder(o.shape) as r:
                    gen._sample_negative_points(m, tuple(int(v) for v in b), [], [])
                ring.append(r.calls[-1])
                with WhereRecorder(o.shape) as r:
                    gen._ensure_num_points(m, [], [])
                fill.append(r.calls[-1])
            out[f"pb_{name}_ds{ds}_positive"] = np.stack(pos)
            out[f"pb_{name}_ds{ds}_ring"] = np.stack(ring)
            out[f"pb_{name}_ds{ds}_fill"] = np.stack(fill)
    # iterative: targets = the objects, predictions = planted variants covering every fallback
    H, W = lab.shape
    preds = []
    rng = np.random.default_rng(1)
    for k, o in enumerate(objs):
        v = k % 5
        if v == 0:
            p = o.copy()                                  # perfect: overlap / box ring (or background)
        elif v == 1:
            p = np.zeros_like(o)                          # empty: FN / box ring
        elif v == 2:
            p = np.roll(o, 2, axis=1)                     # shifted: FN / FP
        elif v == 3:
            p = o.copy(); p[rng.integers(0, H), rng.integers(0, W)] = True    # FP only (or nothing)
        else:
            p = np.ones_like(o)                           # everything: overlap / FP
        preds.append(p)
    full_t = np.ones((H, W), bool); full_t[0, 0] = False  # the box ring is the one pixel left
    targets = np.concatenate([objs, full_t[None]])
    preds = np.concatenate([np.stack(preds), full_t[None]])
    gen = pg.IterativePromptGenerator()
    ipos, ineg = [], []
    for t, p in zip(targets, preds):
        tt = torch.from_numpy(t.astype(np.float32))[None, None]
        pp = torch.from_numpy(p.astype(np.float32))[None, None]
        diff = pp - tt
        with WhereRecorder(t.shape) as r:
            gen._get_positive_points(diff == -1, torch.logical_and(pp == 1, tt == 1).float(), False)
        ipos.append(r.calls[-1])
        with WhereRecorder(t.shape) as r:
            gen._get_negative_points((diff == 1).float(), tt, False)
        ineg.append(r.calls[-1])
    out.update(it_targets=targets, it_preds=preds, it_positive=np.stack(ipos), it_negative=np.stack(ineg))
    np.savez_compressed(os.path.join(OUT, "prompt_regions.npz"), **out)
    print("wrote", os.path.join(OUT, "prompt_regions.npz"), {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
