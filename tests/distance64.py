"""The exact signed squared distance transform of masks, the reference of the word-distance tests.

``signed_d2(masks)`` takes each plane's nearest pixel of the other class from ``scipy.ndimage.distance_transform_edt``
(``return_indices=True``) and recomputes the squared distance from the indices as integers, never by squaring floats:
``min d2`` to the mask at a pixel outside it, ``-min d2`` to the pixels outside it (image pixels only) at a pixel of
it, ``+NONE`` everywhere for an empty mask and ``-NONE`` for a full one. ``brute_force`` (all pairs) and ``separable``
(a column pass and a per-row minimum over every column, in int64) compute the same thing independently of scipy; the
host tests pin the reference to both.
"""
import numpy as np
from scipy import ndimage

NONE = 2 ** 31 - 1


def _nearest_d2(other: np.ndarray) -> np.ndarray:
    """int64 ``[H, W]``: the squared distance from every pixel to the nearest ``True`` pixel of ``other`` (at least
    one), from scipy's indices."""
    _, idx = ndimage.distance_transform_edt(~other, return_indices=True)
    yy, xx = np.indices(other.shape, dtype=np.int64)
    return (yy - idx[0]) ** 2 + (xx - idx[1]) ** 2


def signed_d2_plane(m: np.ndarray) -> np.ndarray:
    m = np.asarray(m, bool)
    if not m.any():
        return np.full(m.shape, NONE, np.int32)
    if m.all():
        return np.full(m.shape, -NONE, np.int32)
    out = np.where(m, -_nearest_d2(~m), _nearest_d2(m))
    return out.astype(np.int32)


def signed_d2(masks) -> np.ndarray:
    """int32, the shape of ``masks`` (``[..., H, W]``, any nonzero inside)."""
    masks = np.asarray(masks) != 0
    flat = masks.reshape((-1,) + masks.shape[-2:])
    return np.stack([signed_d2_plane(m) for m in flat]).reshape(masks.shape) if flat.shape[0] else \
        np.zeros(masks.shape, np.int32)


def brute_force(m: np.ndarray) -> np.ndarray:
    """``signed_d2_plane`` by the minimum over all pairs of pixels."""
    m = np.asarray(m, bool)
    h, w = m.shape
    yy, xx = np.indices((h, w), dtype=np.int64)
    p = np.stack([yy.ravel(), xx.ravel()], 1)
    d2 = ((p[:, None, :] - p[None, :, :]) ** 2).sum(-1)                  # [n, n]
    flat = m.ravel()
    out = np.empty(h * w, np.int64)
    for i in range(h * w):
        other = flat != flat[i]
        out[i] = (-1 if flat[i] else 1) * (d2[i, other].min() if other.any() else NONE)
    return out.reshape(h, w).astype(np.int32)


def separable(m: np.ndarray) -> np.ndarray:
    """``signed_d2_plane`` from the column distances g and ``min_x' (x - x')^2 + g(y, x')^2`` over every column."""
    m = np.asarray(m, bool)
    h, w = m.shape
    out = np.empty((h, w), np.int64)
    big = np.int64(1) << 40
    for cls in (False, True):
        other = m != cls                                                  # the pixels to measure to
        g = np.full((h, w), big, np.int64)                                # vertical distance to `other` in the column
        for x in range(w):
            yo = np.nonzero(other[:, x])[0].astype(np.int64)
            if yo.size:
                g[:, x] = np.abs(np.arange(h, dtype=np.int64)[:, None] - yo[None, :]).min(1)
        g2 = np.where(g < big, g * g, big)
        xs = np.arange(w, dtype=np.int64)
        d2 = ((xs[:, None] - xs[None, :]) ** 2)[None] + g2[:, None, :]    # [h, x, x']
        best = d2.min(-1)
        sel = m == cls
        out[sel] = np.where(best >= big, NONE, best)[sel] * (-1 if cls else 1)
    return out.astype(np.int32)


def kinds(seed, h, w):
    """Empty, full, a single pixel, a corner pixel, a checkerboard, a border-touching block, thin lines, random blobs."""
    g = np.random.default_rng(seed)
    out = [np.zeros((h, w), bool), np.ones((h, w), bool)]
    m = np.zeros((h, w), bool)
    m[g.integers(h), g.integers(w)] = True
    out.append(m)
    m = np.zeros((h, w), bool)
    m[-1, -1] = True
    out.append(m)
    out.append(np.indices((h, w)).sum(0) % 2 == 1)
    m = np.zeros((h, w), bool)
    m[:g.integers(1, h + 1), g.integers(w):] = True
    out.append(m)
    m = np.zeros((h, w), bool)
    m[g.integers(h), :] = True
    m[:, g.integers(w)] = True
    out.append(m)
    out.append(ndimage.binary_opening(g.random((h, w)) < 0.45) | (g.random((h, w)) < 0.02))
    out.append(~out[-1])
    return np.stack(out)
