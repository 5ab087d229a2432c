"""Generates tests/golden/centers.npz by EXECUTING THE REFERENCE's own code (run once where micro_sam's source is at hand; the
GPU machines do not need it).  `get_centers_and_bounding_boxes` and `segmentation_to_one_hot` are extracted from
micro_sam/util.py with `ast` and exec'ed unchanged.  Their absent dependencies are stubbed:
  * skimage's `regionprops`: label, bbox, image and centroid (the mean of the pixel coordinates as float64, as skimage computes
    it), ascending labels;
  * skimage's `find_boundaries(mode="inner")`: oracle/centers_ref.inner_boundaries (DESIGN.md section 2);
  * bioimage_cpp's `distance_transform`: scipy.ndimage.distance_transform_edt;
  * skimage's `relabel_sequential`: oracle/centers_ref.relabel_sequential.
Usage:  python tests/golden/make_centers_golden.py [path to micro_sam]
"""
import ast
import os
import sys
from typing import Dict, Optional, Tuple

import numpy as np
import torch
from scipy import ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import centers_ref  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/micro_sam"
NAMES = ("get_centers_and_bounding_boxes", "segmentation_to_one_hot")


class _Region:
    def __init__(self, label, idx):
        self.label = int(label)
        lo = [int(i.min()) for i in idx]
        hi = [int(i.max()) + 1 for i in idx]
        self.bbox = tuple(lo + hi)
        self.image = np.zeros([h - l for l, h in zip(lo, hi)], bool)
        self.image[tuple(i - l for i, l in zip(idx, lo))] = True
        self.centroid = tuple(np.stack(idx, 1).astype(np.float64).mean(axis=0))


def regionprops(seg):
    return [_Region(lab, np.nonzero(seg == lab)) for lab in np.unique(seg) if lab != 0]


def find_boundaries(label_img, mode="thick"):
    assert mode == "inner"
    return centers_ref.inner_boundaries(label_img)


def relabel_sequential(seg):
    return centers_ref.relabel_sequential(seg), None, None


def load():
    src = open(os.path.join(REF, "util.py")).read()
    ns = {"np": np, "torch": torch, "regionprops": regionprops, "find_boundaries": find_boundaries,
          "distance_transform": ndimage.distance_transform_edt, "relabel_sequential": relabel_sequential,
          "Dict": Dict, "Tuple": Tuple, "Optional": Optional}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in NAMES:
            node.returns = None
            for a in node.args.args:
                a.annotation = None
            exec(compile(ast.Module(body=[node], type_ignores=[]), "util.py", "exec"), ns)
    missing = [n for n in NAMES if n not in ns]
    assert not missing, missing
    return ns


def disk(shape, c, r):
    g = np.indices(shape)
    return sum((gi - ci) ** 2 for gi, ci in zip(g, c)) < r * r


def cases(rng):
    c = {}
    s = np.zeros((24, 31), np.int64)          # touching and diagonally touching objects
    s[2:9, 3:12] = 1
    s[2:9, 12:20] = 2                          # shares an edge with 1
    s[9:15, 20:27] = 3                         # touches 2 only at a corner
    s[15:22, 4:10] = 4
    s[15:22, 10:14] = 5
    c["touching"] = s
    s = np.zeros((29, 33), np.int64)          # concave: a C and a ring, centroids outside the object
    s[3:20, 3:15] = 1
    s[7:16, 8:15] = 0
    ring = disk((29, 33), (14, 24), 7) & ~disk((29, 33), (14, 24), 4)
    s[ring] = 2
    s[22:27, 3:30] = 3
    c["concave"] = s
    s = np.zeros((17, 23), np.int64)          # every border and corner
    s[0:3, 0:4], s[0:3, 19:23], s[14:17, 0:5], s[13:17, 20:23] = 1, 2, 3, 4
    s[0:2, 8:15], s[15:17, 8:15], s[6:11, 0:2], s[6:11, 21:23] = 5, 6, 7, 8
    s[6:11, 8:15] = 9
    c["borders"] = s
    s = np.zeros((15, 19), np.int64)          # 1-pixel and 1-wide objects
    s[2, 3] = 1
    s[5, 2:15] = 2
    s[7:14, 9] = 3
    s[0, 18] = 4
    s[10:13, 2:5] = 5
    s[11, 3] = 6                               # a pixel inside another object
    c["thin"] = s
    s = np.zeros((20, 26), np.int64)          # sparse ids
    s[2:10, 2:12] = 3
    s[11:18, 4:20] = 1000
    s[1:9, 14:24] = 2 ** 31 - 1
    c["sparse_ids"] = s
    s = np.zeros((21, 23), np.int64)          # no background
    s[:, :11], s[:, 11:] = 1, 2
    c["no_background"] = s
    r = np.zeros((40, 48), np.int64)          # random disks, overlapping: later ones paint over earlier ones
    for k in range(1, 26):
        r[disk(r.shape, rng.uniform(0, [40, 48]), rng.uniform(2, 9))] = k
    c["random_disks"] = r
    v = np.zeros((9, 22, 25), np.int64)       # 3-D stack: balls, a slab on the z borders and a 1-voxel object
    for k in range(1, 8):
        v[disk(v.shape, rng.uniform(0, [9, 22, 25]), rng.uniform(2, 6))] = k
    v[0, 2:6, 2:9] = 8
    v[8, 15:20, 3:12] = 9
    v[4, 20, 23] = 10
    v[:, 0:2, 20:25] = 11
    c["stack3d"] = v
    return c


def main():
    ns = load()
    rng = np.random.default_rng(0)
    res = {}
    for name, seg in cases(rng).items():
        res[f"{name}__seg"] = seg
        for mode in ("v", "p"):
            centers, boxes = ns["get_centers_and_bounding_boxes"](seg.copy(), mode=mode)
            ids = np.array(sorted(centers), np.int64)
            assert list(centers) == list(ids) and list(boxes) == list(ids)
            res[f"{name}__ids"] = ids
            res[f"{name}__centers_{mode}"] = np.array([centers[i] for i in ids], np.int64 if mode == "v" else np.float64)
            res[f"{name}__boxes"] = np.array([boxes[i] for i in ids], np.int64)
    one_hot = {
        "touching": None, "stack3d": None, "thin": [2, 5, 6],
        "random_disks": [7, 3, 25, 11],               # unsorted subset
        "borders": [2, 40, 5, 9],                     # 40 is absent: later objects move forward, the last plane is empty
        "concave": [17, 99],                          # nothing selected is present
    }
    for name, ids in one_hot.items():
        seg = res[f"{name}__seg"]
        out = ns["segmentation_to_one_hot"](seg.copy(), None if ids is None else np.array(ids))
        res[f"onehot_{name}__ids"] = np.array([] if ids is None else ids, np.int64)
        res[f"onehot_{name}__out"] = out.numpy().astype(np.uint8)
    np.savez_compressed(os.path.join(HERE, "centers.npz"), **res)
    print(f"wrote {len(res)} arrays")


if __name__ == "__main__":
    main()
