"""Float64 reference of the guided filter behind GlobalHeatMap.refine_words / daam_refine_words, and the error bound
the fp32 device result must meet.

With ``m`` ``[..., H, W]`` the expanded word maps, ``I`` the image's bytes / 255 and ``mean`` the box mean over the
``(2r+1)^2`` window clipped to the image (He's ``boxfilter(f) ./ boxfilter(1)``):
``mu = mean(I)``, ``Sigma = mean(I I^T) - mu mu^T``, ``c = mean(I m) - mu mean(m)``, ``a = (Sigma + eps Id)^-1 c``,
``b = mean(m) - a . mu`` and ``q = mean(a) . I + mean(b)``. The image's window sums are int64 and exact; those of ``m``
are float64 cumulative sums, whose error (about 2^-53 times a row's or column's sum) is far below the fp32 bound."""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24               # unit roundoff of fp32


def window_bounds(n: int, r: int):
    """``(lo, hi)``: the window ``[lo, hi)`` of every index of an axis of ``n``, clipped to it."""
    i = np.arange(n)
    return np.maximum(0, i - r), np.minimum(n, i + r + 1)


def window_count(h: int, w: int, r: int) -> np.ndarray:
    """``N`` ``[h, w]``: pixels in each clipped window."""
    ylo, yhi = window_bounds(h, r)
    xlo, xhi = window_bounds(w, r)
    return (yhi - ylo)[:, None] * (xhi - xlo)[None, :]


def box_sum(f: np.ndarray, r: int) -> np.ndarray:
    """Sum of ``f`` ``[..., h, w]`` over each clipped window, by cumulative sums along the rows, then the columns
    (exact for integers)."""
    h, w = f.shape[-2:]
    c = np.concatenate([np.zeros(f.shape[:-1] + (1,), f.dtype), np.cumsum(f, -1)], -1)
    lo, hi = window_bounds(w, r)
    g = c[..., hi] - c[..., lo]
    c = np.concatenate([np.zeros(g.shape[:-2] + (1, w), g.dtype), np.cumsum(g, -2)], -2)
    lo, hi = window_bounds(h, r)
    return c[..., hi, :] - c[..., lo, :]


def guide64(image: np.ndarray, r: int, eps: float):
    """``(mu [3, h, w], inv [h, w, 3, 3], I [3, h, w])`` of a uint8 ``[h, w, 3]`` image: Sigma from exact int64 window
    sums, then ``(Sigma + eps Id)^-1`` in float64."""
    px = np.moveaxis(image.astype(np.int64), -1, 0)                  # [3, h, w]
    h, w = px.shape[1:]
    n = window_count(h, w, r).astype(np.int64)
    s = box_sum(px, r)
    scd = box_sum(px[:, None] * px[None, :], r)                      # [3, 3, h, w]
    sigma = (n * scd - s[:, None] * s[None, :]) / (65025.0 * n.astype(np.float64) ** 2)
    a = np.moveaxis(sigma, (0, 1), (-2, -1)) + eps * np.eye(3)
    return s / (255.0 * n), np.linalg.inv(a), px / 255.0


def refine64(m: np.ndarray, image: np.ndarray, r: int, eps: float, parts: bool = False):
    """The guided filter of ``m`` ``[..., h, w]`` with ``image`` uint8 ``[h, w, 3]`` as guide, in float64. ``eps`` is
    taken as given (pass the fp32 value the device sees). ``parts``: also return ``dict(a, b, c)``, ``a`` and ``c``
    ``[..., 3, h, w]``."""
    m = np.asarray(m, dtype=np.float64)
    h, w = m.shape[-2:]
    mu, inv, img = guide64(image, r, eps)
    n = window_count(h, w, r).astype(np.float64)
    p = box_sum(m, r) / n
    mi = box_sum(img * m[..., None, :, :], r) / n                    # [..., 3, h, w]
    c = mi - mu * p[..., None, :, :]
    a = np.einsum('hwcd,...dhw->...chw', inv, c)
    b = p - (a * mu).sum(-3)
    q = (box_sum(a, r) / n * img).sum(-3) + box_sum(b, r) / n
    return (q, dict(a=a, b=b, c=c)) if parts else q


def refine_brute(m: np.ndarray, image: np.ndarray, r: int, eps: float) -> np.ndarray:
    """The definition pixel by pixel, windows walked explicitly: for pinning :func:`refine64` at small sizes."""
    m = np.asarray(m, dtype=np.float64)
    img = image.astype(np.float64) / 255.0                           # [h, w, 3]
    h, w = m.shape

    def win(y, x):
        return slice(max(0, y - r), min(h, y + r + 1)), slice(max(0, x - r), min(w, x + r + 1))

    a = np.zeros((h, w, 3))
    b = np.zeros((h, w))
    for y in range(h):
        for x in range(w):
            ys, xs = win(y, x)
            gi = img[ys, xs].reshape(-1, 3)
            pm = m[ys, xs].reshape(-1)
            mu = gi.mean(0)
            sigma = (gi[:, :, None] * gi[:, None, :]).mean(0) - np.outer(mu, mu)
            c = (gi * pm[:, None]).mean(0) - mu * pm.mean()
            a[y, x] = np.linalg.solve(sigma + eps * np.eye(3), c)
            b[y, x] = pm.mean() - a[y, x] @ mu
    q = np.zeros((h, w))
    for y in range(h):
        for x in range(w):
            ys, xs = win(y, x)
            q[y, x] = a[ys, xs].reshape(-1, 3).mean(0) @ img[y, x] + b[ys, xs].mean()
    return q


def refine_bound(m: np.ndarray, parts: dict, r: int, eps: float) -> np.ndarray:
    """An upper bound on ``|q_fp32 - q|`` per ``[..., h, w]`` plane (one number per plane, broadcast ``[..., 1, 1]``),
    from the fp32 operations of refine.cu over exact guide statistics. With L_x = min(2r + 1, w), L_y = min(2r + 1, h)
    and delta = (L_x + L_y + 1) u, a window mean of fp32 values x (a row sum of at most L_x terms, a column sum of at
    most L_y row sums, one division) is within delta max|x| of the exact mean of those values. M, A, B, C are the
    plane's max |m|, |a|, |b|, |c| (float64), and K = sqrt(3) / eps bounds ||(Sigma + eps Id)^-1||_inf
    (||.||_2 <= 1 / eps, Sigma being positive semi-definite):
      mean(m): delta M;  mean(I m): (delta + 2u) M (I = byte / 255 and the product rounded once each)
      c:       dc = (2 delta + 7u) M (mu rounded once, mu p and the difference rounded)
      a:       da = K (dc + 4u (C + dc)) (the stored inverse within u of each entry; the 3-term product)
      b:       db = delta M + 3 (da + u A') + 4u (M + 3 A'), A' = A + da
      q:       3 (da + delta A' + u A') + db + delta B' + 5u (3 A' + B'), B' = B + db
    The sum, times 1.25 for the second-order terms the list leaves out."""
    h, w = m.shape[-2:]
    lead = m.shape[:-2]
    delta = (min(2 * r + 1, w) + min(2 * r + 1, h) + 1) * U
    def peak(x):                                                     # max |x| per plane
        return np.abs(x).reshape(lead + (-1,)).max(-1)

    big_m, big_a, big_b, big_c = peak(m), peak(parts['a']), peak(parts['b']), peak(parts['c'])
    k = math.sqrt(3.0) / eps
    dc = (2 * delta + 7 * U) * big_m
    da = k * (dc + 4 * U * (big_c + dc))
    a1 = big_a + da
    db = delta * big_m + 3 * (da + U * a1) + 4 * U * (big_m + 3 * a1)
    b1 = big_b + db
    dq = 3 * (da + delta * a1 + U * a1) + db + delta * b1 + 5 * U * (3 * a1 + b1)
    return (1.25 * dq)[..., None, None]
