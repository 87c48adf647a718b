"""Float64 statement of word segmentation (``GlobalHeatMap.segment``) and the fp32 error bound its labels are compared
under. ``tests/test_segment_host.py`` pins :func:`segment64` to the oracle's ``port_word_heat_map`` + ``port_expand_as``
followed by an argmax; ``tests/test_segment_gpu.py`` compares the kernel's labels with it."""
import torch

from tests.reference64 import bicubic64
from tests.words64 import expand64, expand_bound


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
    """Per pixel, a bound on |fp32 value - float64 value| of every word: :func:`tests.words64.expand_bound` (the fp32
    row mean, the 16-tap stencil, the fp32 source coordinate of ``make_taps`` and, unless ``absolute``, the min-max
    normalisation) for each word at the pixel, the largest over the words. ``words``: the float64 word maps of
    non-negative global maps."""
    out_hw = (by.shape[0], bx.shape[0])
    bound = expand_bound(words, out_hw, absolute, [len(r) for r in rows_per_word], exp=expand64(words, out_hw, True))
    return bound.amax(0)
