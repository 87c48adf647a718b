"""Float64 reference of the CRF mean field behind GlobalHeatMap.segment_crf / daam_segment_crf, and the error bound one
fp32 update must meet.

With ``z`` ``[L, H, W]`` the unary logits (``scale`` times the scores: the threshold plane, if any, then the word maps),
``Q`` ``[L, H, W]`` the current marginals, ``I`` the image's RGB bytes and ``W(x)`` the ``(2r+1)^2`` window around
``x`` clipped to the image, one update is
``msg_l(x) = sum_{y in W(x), y != x} (A[y - x] exp(-|I_x - I_y|^2 coef) + S[y - x]) Q_l(y)`` and
``Q' = softmax_l(z + msg)``. A mean-field error bound compounded over iterations says nothing useful, so the device is
checked one update at a time: its own ``Q_k`` goes in, and its ``Q_{k+1}`` must lie within :func:`crf_bound` of
:func:`crf_step64`'s."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24               # unit roundoff of fp32


def f32(v) -> float:
    """``v`` rounded to fp32, as the C entry receives it."""
    return float(np.float32(v))


def crf_tables(r: int, appearance: float, sigma_xy: float, smoothness: float, sigma_smooth: float,
               sigma_rgb: float) -> dict:
    """``A``, ``S`` ``[2r+1, 2r+1]`` (row-major over ``(o_y, o_x)``, centre 0) and ``coef = 1 / (2 sigma_rgb^2)``, in
    float64 from the fp32 arguments. Each table is normalised over the window's offsets ``o != 0``."""
    o = np.arange(-r, r + 1, dtype=np.float64)
    d2 = o[:, None] ** 2 + o[None, :] ** 2

    def table(weight, sigma):
        g = np.exp(-d2 / (2.0 * f32(sigma) ** 2))
        g[r, r] = 0.0
        return f32(weight) * g / g.sum()

    return dict(A=table(appearance, sigma_xy), S=table(smoothness, sigma_smooth),
                coef=1.0 / (2.0 * f32(sigma_rgb) ** 2))


def logits64(m: np.ndarray, threshold=None, scale: float = 16.0) -> np.ndarray:
    """``z`` ``[L, H, W]`` from the expanded word maps ``m`` ``[n_words, H, W]`` (fp32 values): the threshold plane
    first when ``threshold`` is in effect (Python truthiness), every plane times ``scale``."""
    s = np.asarray(m, dtype=np.float64)
    if threshold:
        s = np.concatenate([np.full((1,) + s.shape[1:], f32(threshold)), s])
    return f32(scale) * s


def softmax64(t: np.ndarray) -> np.ndarray:
    e = np.exp(t - t.max(0))
    return e / e.sum(0)


def crf_step64(z: np.ndarray, q: np.ndarray, image: np.ndarray, tables: dict, r: int, rows=None, parts: bool = False):
    """One mean-field update from ``q`` ``[L, H, W]``: ``Q'`` ``[L, y1 - y0, W]`` over output rows ``rows = (y0, y1)``
    (all by default). ``parts``: also return ``dict(t=z + msg, mass=sum_y (A + S) Q)``, what :func:`crf_bound` takes."""
    L, h, w = q.shape
    y0, y1 = rows or (0, h)
    img = np.asarray(image, dtype=np.int64)
    q = np.asarray(q, dtype=np.float64)
    msg = np.zeros((L, y1 - y0, w))
    mass = np.zeros((L, y1 - y0, w))
    for dy in range(-r, r + 1):
        ya, yb = max(y0, -dy), min(y1, h - dy)            # output rows whose row y + dy is in the image
        if ya >= yb:
            continue
        for dx in range(-r, r + 1):
            if dy == 0 and dx == 0:
                continue
            xa, xb = max(0, -dx), min(w, w - dx)
            if xa >= xb:
                continue
            d2 = ((img[ya:yb, xa:xb] - img[ya + dy:yb + dy, xa + dx:xb + dx]) ** 2).sum(-1)
            a, s = tables['A'][dy + r, dx + r], tables['S'][dy + r, dx + r]
            src = q[:, ya + dy:yb + dy, xa + dx:xb + dx]
            msg[:, ya - y0:yb - y0, xa:xb] += (a * np.exp(-d2 * tables['coef']) + s) * src
            mass[:, ya - y0:yb - y0, xa:xb] += (a + s) * src
    t = z[:, y0:y1] + msg
    out = softmax64(t)
    return (out, dict(t=t, mass=mass)) if parts else out


def crf_brute(z: np.ndarray, q: np.ndarray, image: np.ndarray, tables: dict, r: int) -> np.ndarray:
    """The definition pixel by pixel, windows walked explicitly: for pinning :func:`crf_step64` at small sizes."""
    L, h, w = q.shape
    img = np.asarray(image, dtype=np.float64)
    out = np.zeros((L, h, w))
    for y in range(h):
        for x in range(w):
            t = np.array(z[:, y, x], dtype=np.float64)
            for yy in range(max(0, y - r), min(h, y + r + 1)):
                for xx in range(max(0, x - r), min(w, x + r + 1)):
                    if (yy, xx) == (y, x):
                        continue
                    k = tables['A'][yy - y + r, xx - x + r] * np.exp(-((img[y, x] - img[yy, xx]) ** 2).sum() *
                                                                      tables['coef'])
                    t += (k + tables['S'][yy - y + r, xx - x + r]) * q[:, yy, xx]
            e = np.exp(t - t.max())
            out[:, y, x] = e / e.sum()
    return out


def crf_bound(parts: dict, r: int):
    """``(bound, dt)``: an upper bound on ``|Q'_fp32 - Q'|`` per element ``[L, rows, W]`` for one update of crf.cu from
    the same ``Q`` and exact ``z`` (``scale`` a power of two), and a bound ``dt`` ``[rows, W]`` on every label's fp32
    logit error at a pixel. From the fp32 operations, with ``N = (2r+1)^2`` and ``gamma_n = n u / (1 - n u)``:
      weight:  ``k = fma(A, expf(-d2 * coef), S)`` with ``A``, ``S``, ``coef`` each rounded once. ``d2`` is exact; the
               argument ``t = d2 coef`` carries a relative error of 2u, which moves ``exp(-t)`` by at most
               ``2u t e^{-t} <= 2u / e``; CUDA's ``expf`` adds 2 ulp (4u relative); so ``|dk| <= 8u (A + S)``;
      message: a sequential sum of at most ``N - 1`` fused products, ``|dmsg| <= (8u + gamma_N) mass`` with
               ``mass = sum (A + S) Q``, plus ``N 2^-149`` for products that fall below fp32's normal range;
      logit:   ``z + msg`` rounded once: ``dt_l = |dmsg_l| + u |t_l|``; ``dt = max_l dt_l``;
      softmax: a logit error of at most ``dt`` moves ``Q'_l`` by a factor within ``e^{+-2 dt}``; the device's own
               softmax adds, relative to ``Q'_l``, ``eps_l + max_k eps_k + gamma_L + u`` with
               ``eps_l = (1 + expm1(u |t_l - max t|)) (1 + 4u) - 1`` (the rounded difference, then ``expf``), for the
               sum in label order and the division.
    The bound is ``1.25 Q'_l (expm1(2 dt) + e^{2 dt} (eps_l + max eps + gamma_L + u)) + 2^-125``: the factor 1.25 for
    the second-order terms the list leaves out, the last term for results below fp32's normal range."""
    t, mass = parts['t'], parts['mass']
    L = t.shape[0]
    n = (2 * r + 1) ** 2
    gamma = lambda k: k * U / (1 - k * U)
    dmsg = (8 * U + gamma(n)) * mass + n * 2.0 ** -149
    dt = (dmsg + U * np.abs(t)).max(0)
    q = softmax64(t)
    eps = (1 + np.expm1(U * np.abs(t - t.max(0)))) * (1 + 4 * U) - 1
    rel = eps + eps.max(0) + gamma(L) + U
    bound = 1.25 * q * (np.expm1(2 * dt) + np.exp(2 * dt) * rel) + 2.0 ** -125
    return bound, dt
