"""Exact integer statement of word instances (``GlobalHeatMap.word_instances``): the 8-connected components of a mask
and each component's area, box, index sums and peak, ranked and cut to K as the kernels rank them. Pure numpy, so the
GPU tests need no scipy; ``tests/test_word_instances_host.py`` pins :func:`label8` and :func:`components64` to
``scipy.ndimage.label`` / ``find_objects``."""
import numpy as np

# the neighbours before a pixel in raster order (W, NW, N, NE): every 8-adjacent pair is one of these once
_BACK = ((0, -1), (-1, -1), (-1, 0), (-1, 1))


def label8(mask) -> np.ndarray:
    """int64 ``[H, W]``: each foreground pixel's component root, the smallest raster index in its 8-connected
    component; -1 on the background. Union-find over the pairs of 8-adjacent foreground pixels: each round hooks every
    root under the smallest root it shares a pair with, then flattens the forest by pointer jumping."""
    mask = np.asarray(mask, dtype=bool)
    h, w = mask.shape
    idx = np.arange(h * w, dtype=np.int64).reshape(h, w)
    a_parts, b_parts = [], []
    for dy, dx in _BACK:
        y0, x0, x1 = -dy, max(0, -dx), min(w, w - dx)
        if y0 >= h or x0 >= x1:
            continue
        both = mask[y0:, x0:x1] & mask[y0 + dy:h + dy, x0 + dx:x1 + dx]
        a_parts.append(idx[y0:, x0:x1][both])
        b_parts.append(idx[y0 + dy:h + dy, x0 + dx:x1 + dx][both])
    a, b = np.concatenate(a_parts or [idx[:0, 0]]), np.concatenate(b_parts or [idx[:0, 0]])
    parent = np.arange(h * w, dtype=np.int64)
    while True:
        ra, rb = parent[a], parent[b]
        apart = ra != rb
        if not apart.any():
            break
        a, b, ra, rb = a[apart], b[apart], ra[apart], rb[apart]
        np.minimum.at(parent, np.maximum(ra, rb), np.minimum(ra, rb))
        while True:                                             # pointer jumping until every node points at a root
            jumped = parent[parent]
            if np.array_equal(jumped, parent):
                break
            parent = jumped
    return np.where(mask.ravel(), parent, -1).reshape(h, w)


def components64(mask, pre=None):
    """Every component of ``mask`` in raster order of its first pixel (scipy.ndimage.label's order): a dict of
    ``root`` (the first pixel), ``area``, ``box`` ``[n, 4]`` (half-open ``(y0, x0, y1, x1)``), ``sum_yx`` ``[n, 2]``
    (int64), and with ``pre`` (fp32 ``[H, W]``) ``peak`` (max of ``pre``) and ``peak_yx`` (its first pixel)."""
    mask = np.asarray(mask, dtype=bool)
    h, w = mask.shape
    lab = label8(mask).ravel()
    p = np.flatnonzero(lab >= 0)
    roots, inv = np.unique(lab[p], return_inverse=True)
    order = np.argsort(inv, kind='stable')                     # groups of components, each in raster order
    p = p[order]
    area = np.bincount(inv, minlength=len(roots)).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(area)[:-1]]).astype(np.int64)
    y, x = p // w, p % w
    out = dict(root=roots, area=area)
    if len(roots) == 0:
        out.update(box=np.zeros((0, 4), np.int64), sum_yx=np.zeros((0, 2), np.int64))
        if pre is not None:
            out.update(peak=np.zeros(0, np.float32), peak_yx=np.zeros((0, 2), np.int64))
        return out
    ends = starts + area - 1
    out['box'] = np.stack([y[starts], np.minimum.reduceat(x, starts), y[ends] + 1, np.maximum.reduceat(x, starts) + 1], 1)
    out['sum_yx'] = np.stack([np.add.reduceat(y, starts), np.add.reduceat(x, starts)], 1).astype(np.int64)
    if pre is not None:
        v = np.asarray(pre, dtype=np.float32).ravel()[p]
        peak = np.maximum.reduceat(v, starts)
        group = np.repeat(np.arange(len(roots)), area)
        first = np.minimum.reduceat(np.where(v == peak[group], p, h * w), starts)
        out.update(peak=peak, peak_yx=np.stack([first // w, first % w], 1))
    return out


def instances64(pre, threshold, k):
    """What ``word_instances`` returns for one plane ``pre`` (fp32 ``[H, W]``, the expanded map without threshold):
    ``count`` and the ``k`` largest components of ``pre > fp32(threshold)`` by (area desc, first pixel asc), the slots
    past the count zero: ``area`` ``[k]``, ``box`` ``[k, 4]``, ``sum_yx`` ``[k, 2]``, ``peak`` ``[k]``, ``peak_yx``
    ``[k, 2]``."""
    pre = np.asarray(pre, dtype=np.float32)
    c = components64(pre > np.float32(threshold), pre)
    n = len(c['root'])
    keep = np.lexsort((c['root'], -c['area']))[:k]
    m = len(keep)
    out = dict(count=np.int64(n), area=np.zeros(k, np.int64), box=np.zeros((k, 4), np.int64),
               sum_yx=np.zeros((k, 2), np.int64), peak=np.zeros(k, np.float32), peak_yx=np.zeros((k, 2), np.int64))
    for f in ('area', 'box', 'sum_yx', 'peak', 'peak_yx'):
        out[f][:m] = c[f][keep]
    return out


def instances64_stack(pre, threshold, k):
    """:func:`instances64` of every plane of ``pre`` ``[..., H, W]``, stacked: each field gets the leading axes."""
    pre = np.asarray(pre, dtype=np.float32)
    lead = pre.shape[:-2]
    planes = [instances64(p, threshold, k) for p in pre.reshape((-1,) + pre.shape[-2:])]
    return {f: np.stack([p[f] for p in planes]).reshape(lead + np.shape(planes[0][f])) if planes else
            np.zeros(lead + np.shape(instances64(np.zeros((1, 1), np.float32), 1.0, k)[f]))
            for f in ('count', 'area', 'box', 'sum_yx', 'peak', 'peak_yx')}
