"""numpy / scipy restatement of InstanceSegmentationWithDecoder.generate's post-processing with the rules DESIGN.md section 2
fixes (unpinned: the reference calls vigra, elf and skimage):
  smoothing    separable, taps exp(-k^2 / 2 s^2) normalised, radius floor(3 s + 0.5), scipy 'mirror' border, fp64 with the taps
               summed from -r to r, rounded to fp32 once; s = 0 leaves the map as it is
  markers      (cd_s < t_cd) & (bd_s < t_bd) & (fg_s > t_fg), 8-connected components numbered 1.. in raster order
  watershed    on h = bd_s inside fg, 4-neighbourhoods: B(p) = max(h(p), min over in-mask neighbours B(q)), B(seed) = h(seed);
               label(p) = the smallest seed id reachable by stepping to neighbours of minimal B; unreached pixels stay 0
  size filter  ids with fewer than min_size pixels -> 0, the rest renumbered in id order
The rule is computed twice (watershed_relax and watershed_dijkstra); heap_flood restates skimage's priority flood only to
measure how far the rule is from it."""
import heapq

import numpy as np
from scipy import ndimage

NB4 = ((-1, 0), (1, 0), (0, -1), (0, 1))   # N, S, W, E


def gaussian_taps(sigma):
    if sigma == 0:
        return np.zeros(0, np.float64)
    r = int(3.0 * sigma + 0.5)
    k = np.arange(-r, r + 1, dtype=np.float64)
    w = np.exp(-(k * k) / (2.0 * sigma * sigma))
    return w / w.sum()


def mirror_index(i, n):
    if n == 1:
        return np.zeros_like(i)
    p = 2 * n - 2
    i = np.mod(i, p)
    return np.where(i < n, i, p - i)


def _smooth_axis(x, taps, axis):
    r = len(taps) // 2
    n = x.shape[axis]
    idx = np.arange(n)
    acc = np.zeros(x.shape, np.float64)
    for k in range(-r, r + 1):
        acc = acc + taps[k + r] * np.take(x, mirror_index(idx + k, n), axis=axis)
    return acc


def smooth(x, sigma):
    x = np.asarray(x, np.float32)
    if sigma == 0:
        return x.copy()
    t = gaussian_taps(sigma)
    return _smooth_axis(_smooth_axis(x.astype(np.float64), t, 0), t, 1).astype(np.float32)


def markers_and_mask(fg, cd, bd, t_cd, t_bd, t_fg, s_fg, s_d):
    fg_s, cd_s, bd_s = smooth(fg, s_fg), smooth(cd, s_d), smooth(bd, s_d)
    fmask = fg_s > np.float32(t_fg)
    markers = (cd_s < np.float32(t_cd)) & (bd_s < np.float32(t_bd)) & fmask
    lab, n = ndimage.label(markers, structure=np.ones((3, 3), int))   # numbered in raster order of first pixel
    return lab.astype(np.int64), n, fmask, bd_s


def _neighbours(H, W, y, x):
    for dy, dx in NB4:
        v, u = y + dy, x + dx
        if 0 <= v < H and 0 <= u < W:
            yield v, u


def _shifted(a, fill):
    """a's N, S, W, E neighbour values per pixel (fill outside the image)."""
    H, W = a.shape
    out = np.full((4, H, W), fill, dtype=a.dtype)
    out[0, 1:] = a[:-1]
    out[1, :-1] = a[1:]
    out[2, :, 1:] = a[:, :-1]
    out[3, :, :-1] = a[:, 1:]
    return out


def watershed_relax(h, fmask, seeds):
    """The rule by plain Jacobi relaxation of both fixpoints."""
    h = np.asarray(h, np.float32)
    seed = seeds > 0
    free = fmask & ~seed
    B = np.where(seed, h, np.float32(np.inf)).astype(np.float32)
    while True:
        m = _shifted(B, np.float32(np.inf)).min(0)
        nb = np.where(free, np.maximum(h, m), B)
        if np.array_equal(nb, B):
            break
        B = nb
    BIG = np.iinfo(np.int64).max
    L = np.where(seed, seeds, np.where(fmask, BIG, 0)).astype(np.int64)
    nbB = _shifted(B, np.float32(np.inf))
    m = nbB.min(0)
    act = free & np.isfinite(B)
    is_min = nbB == m[None]
    while True:
        nl = _shifted(L, BIG)
        cand = np.where(is_min, nl, BIG).min(0)
        nL = np.where(act, np.minimum(L, cand), L)
        if np.array_equal(nL, L):
            break
        L = nL
    return np.where(L == BIG, 0, L), B


def watershed_dijkstra(h, fmask, seeds):
    """The rule by a Dijkstra flood on the barrier and a breadth-first search, in seed id order, over the reversed
    steepest-step edges."""
    h = np.asarray(h, np.float32)
    H, W = h.shape
    seed = seeds > 0
    B = np.full((H, W), np.float32(np.inf), np.float32)
    heap = []
    for y, x in zip(*np.nonzero(seed)):
        B[y, x] = h[y, x]
        heap.append((float(h[y, x]), y * W + x))
    heapq.heapify(heap)
    done = np.zeros((H, W), bool)
    while heap:
        b, i = heapq.heappop(heap)
        y, x = divmod(i, W)
        if done[y, x]:
            continue
        done[y, x] = True
        for v, u in _neighbours(H, W, y, x):
            if fmask[v, u] and not seed[v, u] and not done[v, u]:
                nb = max(h[v, u], np.float32(b))
                if nb < B[v, u]:
                    B[v, u] = nb
                    heapq.heappush(heap, (float(nb), v * W + u))
    rev = [[] for _ in range(H * W)]   # q -> p when q is a minimal-B neighbour of p
    for y in range(H):
        for x in range(W):
            if not fmask[y, x] or seed[y, x] or not np.isfinite(B[y, x]):
                continue
            nbs = [(B[v, u], v * W + u) for v, u in _neighbours(H, W, y, x)]
            m = min(b for b, _ in nbs)
            for b, j in nbs:
                if b == m:
                    rev[j].append(y * W + x)
    L = np.zeros(H * W, np.int64)
    order = sorted(zip(seeds[seed].tolist(), np.flatnonzero(seed).tolist()))
    by_id = {}
    for sid, i in order:
        by_id.setdefault(sid, []).append(i)
    for sid in sorted(by_id):
        stack = list(by_id[sid])
        for i in stack:
            L[i] = sid
        while stack:
            j = stack.pop()
            for p in rev[j]:
                if L[p] == 0:
                    L[p] = sid
                    stack.append(p)
    return L.reshape(H, W), B


def heap_flood(h, fmask, seeds):
    """skimage.segmentation.watershed's priority flood restated: (value, age) ordered heap, 4-neighbourhoods, each pixel takes
    the label of the neighbour that pushed it first."""
    h = np.asarray(h, np.float32)
    H, W = h.shape
    L = np.where(fmask, seeds, 0).astype(np.int64)
    heap, age = [], 0
    for y, x in zip(*np.nonzero(L)):
        heap.append((float(h[y, x]), age, y * W + x))
        age += 1
    heapq.heapify(heap)
    while heap:
        _, _, i = heapq.heappop(heap)
        y, x = divmod(i, W)
        for v, u in _neighbours(H, W, y, x):
            if fmask[v, u] and L[v, u] == 0:
                L[v, u] = L[y, x]
                heapq.heappush(heap, (float(h[v, u]), age, v * W + u))
                age += 1
    return L


def size_filter(labels, min_size):
    if min_size <= 0 or labels.max() == 0:
        return labels
    cnt = np.bincount(labels.ravel())
    keep = cnt >= min_size
    keep[0] = False
    new = np.zeros(len(cnt), np.int64)
    new[keep] = np.arange(1, keep.sum() + 1)
    return new[labels]


def generate(fg, cd, bd, center_distance_threshold=0.5, boundary_distance_threshold=0.5, foreground_threshold=0.5,
             foreground_smoothing=1.0, distance_smoothing=1.6, min_size=0, watershed=watershed_relax):
    seeds, _, fmask, bd_s = markers_and_mask(fg, cd, bd, center_distance_threshold, boundary_distance_threshold,
                                             foreground_threshold, foreground_smoothing, distance_smoothing)
    labels, _ = watershed(bd_s, fmask, seeds)
    return size_filter(labels, min_size)


def touching_disks(H, W, n, seed=0, noise=0.05):
    """Synthetic decoder maps: n random disks (touching and overlapping), foreground probability, center distance (0 at the
    center, 1 at the rim) and boundary distance (0 deep inside, 1 at the boundary), from distance_transform_edt, plus noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W]
    lab = np.zeros((H, W), np.int64)
    cdist = np.ones((H, W))
    for k in range(1, n + 1):
        cy, cx, r = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(6, 18)
        d = np.hypot(yy - cy, xx - cx) / r
        inside = (d < 1) & (d < cdist)
        lab[inside] = k
        cdist = np.where(inside, d, cdist)
    fg = (lab > 0).astype(np.float64)
    bd = np.ones((H, W))
    for k in np.unique(lab)[1:]:
        m = lab == k
        e = ndimage.distance_transform_edt(m)
        bd[m] = 1 - e[m] / max(e.max(), 1)
    f = lambda a: np.clip(a + noise * rng.standard_normal((H, W)), 0, 1).astype(np.float32)
    return f(fg), f(cdist), f(bd)
