"""Float64 statement of word segmentation (``GlobalHeatMap.segment``) and the fp32 error bound its labels are compared
under. ``tests/test_segment_host.py`` pins :func:`segment64` to the oracle's ``port_word_heat_map`` + ``port_expand_as``
followed by an argmax; ``tests/test_segment_gpu.py`` compares the kernel's labels with it."""
import torch

from tests.reference64 import FP32_EPS, bicubic64


def segment64(maps, rows_per_word, hw, absolute, threshold):
    """float64 word maps (mean of ``rows_per_word[w]`` of ``maps``) -> ``B_y @ W @ B_x^T`` to ``hw`` -> float64 min-max
    normalisation unless ``absolute`` -> ``(labels, max, top-two margin, word maps, B_y, B_x)``; labels are
    ``argmax + 1``, 0 where ``threshold`` is truthy and the max is not above it."""
    words = torch.stack([maps[rows].double().mean(0) for rows in rows_per_word])
    by, bx = bicubic64(maps.shape[-2], hw[0], maps.device), bicubic64(maps.shape[-1], hw[1], maps.device)
    up = by @ words @ bx.T                                                   # [n_words, H, W]
    if not absolute:
        lo, hi = up.amin((1, 2), keepdim=True), up.amax((1, 2), keepdim=True)
        up = (up - lo) / (hi - lo + 1e-8)
    top = up.topk(min(2, up.shape[0]), dim=0).values
    margin = top[0] - top[1] if up.shape[0] > 1 else torch.full_like(top[0], float('inf'))
    labels = up.argmax(0) + 1
    if threshold:
        labels = torch.where(top[0] > threshold, labels, torch.zeros_like(labels))
    return labels, top[0], margin, words, by, bx


def label_bound(words, by, bx, rows_per_word, absolute):
    """Per-word bound on |fp32 normalised value - float64 value|, from the error analysis, not from observed errors:

    * word map: a mean of ``k`` fp32 rows, relative error below ``(k + 1) 2^-24``;
    * interpolation: a 16-tap stencil in fp32, error below ``32 2^-24 N_y N_x max|W|`` (``N`` the largest row 1-norm of
      the bicubic matrix of each axis, as in ``finalize_tolerance``), plus the word map's error times ``N_y N_x``;
    * normalisation: with ``E`` that bound for v, lo and hi (lo and hi are values of v) and ``D = hi - lo + 1e-8``,
      ``|d((v - lo) / D)| <= 2E / D + 2E / D + 3 2^-24`` (the quotient is at most 1).
    Absolute maps keep ``E``."""
    ny = float(by.abs().sum(1).max())
    nx = float(bx.abs().sum(1).max())
    out = []
    for w, rows in zip(words, rows_per_word):
        vmax = float(w.abs().max())
        e = 32 * FP32_EPS * ny * nx * vmax + (len(rows) + 1) * FP32_EPS * vmax * ny * nx
        if absolute:
            out.append(e)
        else:
            up = by @ w @ bx.T
            d = float(up.max() - up.min()) + 1e-8
            out.append(4 * e / d + 3 * FP32_EPS)
    return max(out)
