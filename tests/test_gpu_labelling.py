"""msam_remove_small_regions (segment_anything's remove_small_regions over a batch of masks, on the shared connected-component
labeller of csrc/postprocess.cu) against oracle/amg_ref.remove_small_regions, mask for mask and flag for flag."""
import numpy as np
import pytest
import torch

from micro_sam_b200 import _lib
from oracle import amg_ref

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _remove(masks, area_thresh, holes):
    """masks: uint8 [n, h, w] device tensor, edited in place; returns the changed flags"""
    n, h, w = masks.shape
    ws = torch.empty(n * (2 * h * w + 4), dtype=torch.int32, device=DEV)
    ch = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    _lib.check(_lib.lib().msam_remove_small_regions(_lib.ptr(masks), n, h, w, int(area_thresh), holes, _lib.ptr(ch), _lib.ptr(ws),
                                                     _lib.cur_stream()))
    return ch


def _planted(h, w):
    """masks that each pin one rule down"""
    ms = []
    m = np.zeros((h, w), bool); m[10:12, 20:22] = True; m[40:42, 5:7] = True; m[30, 60] = True
    ms.append(m)                                    # every island small, two tie for largest: the first in raster order stays
    m = np.zeros((h, w), bool); m[40:42, 5:7] = True; m[10:12, 20:22] = True
    ms.append(m)                                    # the same tie, written in the other order
    m = np.zeros((h, w), bool)
    for k in range(8): m[20 + k, 30 + k] = True     # a diagonal line: one 8-connected island of 8 pixels
    m[5, 5] = m[6, 6] = m[5, 7] = True              # three pixels joined only through corners
    m[60:64, 100:104] = True
    ms.append(m)
    m = np.ones((h, w), bool)
    for k in range(6): m[30 + k, 40 + k] = False    # a diagonal hole of 6 pixels: one component under 8-connectivity
    m[0:3, 0:3] = False; m[h - 1, w - 1] = False    # holes touching the border and the corner
    m[50, 0:w] = False                              # a background band across the whole width
    ms.append(m)
    m = np.zeros((h, w), bool); m[0:h, 0:4] = True; m[0:4, 0:w] = True; m[h - 20:h, w - 20:w] = True
    ms.append(m)                                    # islands touching every border, none small: unchanged
    ms.append(np.zeros((h, w), bool))               # empty mask
    ms.append(np.ones((h, w), bool))                # full mask
    return np.stack(ms)


def _random(n, h, w, seed):
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    mk = (torch.nn.functional.interpolate(torch.randn(n, 1, h // 9 + 2, w // 9 + 2, generator=g), (h, w), mode="bicubic")[:, 0]
          > 0.3).numpy()
    mk |= rng.random(mk.shape) > 0.995              # specks (islands)
    mk &= ~(rng.random(mk.shape) > 0.99)            # pin holes
    return mk


@pytest.mark.parametrize("n,h,w,area", [(7, 96, 130, 12), (200, 96, 130, 12), (130, 128, 128, 30), (3, 257, 300, 40)])
def test_remove_small_regions_against_oracle(n, h, w, area):
    """holes then islands, as AMG's generate(min_mask_region_area > 0) applies them; n = 200 and 130 are not multiples of 128"""
    mk = _random(n, h, w, seed=n + h)
    pl = _planted(h, w)
    mk[: min(n, len(pl))] = pl[: min(n, len(pl))]
    dm = torch.from_numpy(mk).to(DEV).to(torch.uint8).contiguous()
    ref = mk.copy()
    for holes, mode in ((1, "holes"), (0, "islands")):
        ch = _remove(dm, area, holes).cpu().numpy()
        ref_ch = np.zeros(n, bool)
        for k in range(n):
            ref[k], ref_ch[k] = amg_ref.remove_small_regions(ref[k], area, mode)
        np.testing.assert_array_equal(dm.cpu().numpy().astype(bool), ref, err_msg=mode)
        np.testing.assert_array_equal(ch != 0, ref_ch, err_msg=mode)
        assert set(np.unique(ch)) <= {0, 1}
        if n >= len(pl):
            assert ref_ch.any() and not ref_ch.all()    # both outcomes occur


def test_remove_small_regions_in_passes():
    """3 masks of 27000 x 27000: n * h * w >= 2^31, so the masks are labelled in more than one pass.  Every mask has a large
    square with one-pixel holes and a small island; small squares at the bottom of one mask and the top of the next would be
    one large island if the masks were linked."""
    N, A = 27000, 100
    if torch.cuda.get_device_properties(DEV).total_memory < 40 << 30:
        pytest.skip("needs about 22 GB of device memory")
    masks = torch.zeros(3, N, N, dtype=torch.uint8, device=DEV)
    want = torch.zeros_like(masks)
    for m in range(3):
        y, x = 1000 + 9000 * m, 26000 - 12000 * m
        masks[m, y:y + 500, x:x + 700] = 1          # the large square: stays
        want[m, y:y + 500, x:x + 700] = 1
        masks[m, y + 10, x + 10] = 0                # holes: filled
        masks[m, y + 490 - m, x + 300] = 0
        masks[m, N // 2: N // 2 + 5, 7 * m: 7 * m + 5] = 1   # a small island: removed
    masks[0, N - 8:, 100:107] = 1                   # 56 + 56 pixels across the seams between masks 0 / 1 and 1 / 2
    masks[1, :8, 100:107] = 1
    masks[1, N - 8:, 200:207] = 1
    masks[2, :8, 200:207] = 1
    torch.cuda.synchronize()
    ch = _remove(masks, A, 1)
    assert ch.tolist() == [1, 1, 1]
    ch = _remove(masks, A, 0)
    assert ch.tolist() == [1, 1, 1]
    assert torch.equal(masks, want)
    del masks, want
    torch.cuda.empty_cache()
