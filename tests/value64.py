"""Float64 statements of value-weighted heat maps, in torch so that they run on the GPU next to the kernels.

* :func:`value_norms64` is ``daam_value_norms``: ``n[b, h, j] = ||W_h v_{b,h,j}||`` over the fp32 values of both
  operands, and :func:`value_norms_bound` bounds what its fixed fp32 ``fmaf`` order may make of the squares.
* :func:`weighted_map64` is ``daam_finalize_parts_weighted`` for one map: ``(1/K) sum_k w_k[t] clamp(bicubic(key_k[t]))``,
  optionally normalised; :func:`weighted_tolerance` is ``reference64.rect_tolerance`` with every key's error scaled by
  the largest weight.
* :func:`trace_weighted_map64` states a traced generation's weighted map from the recorded Q, K, V and output weights.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from tests.reference64 import FP32_EPS, _normalize, layer_maps64, rect_tolerance, up64


def value_norms64(value: torch.Tensor, weight: torch.Tensor, heads: int) -> torch.Tensor:
    """``value [S, T, heads*d]`` (the samples kept), ``weight [C_out, heads*d]`` -> ``[S, heads, T]`` float64 norms."""
    s, t, c = value.shape
    d = c // heads
    v = value.double().reshape(s, t, heads, d)
    w = weight.double().reshape(weight.shape[0], heads, d)
    y = torch.einsum('sthe,che->shtc', v, w)
    return y.square().sum(-1).sqrt()


def value_norms_bound(value: torch.Tensor, weight: torch.Tensor, heads: int) -> torch.Tensor:
    """``[S, heads, T]``: the bound on ``|n_hat^2 - n^2|`` of the kernel's fp32 arithmetic, ``(d + C_out + 2) 2^-24
    sum_c (sum_e |W_ce v_e|)^2`` -- d roundings in each fma chain over e, C_out in the chain over c, and one each for
    squaring and the square root's input."""
    s, t, c = value.shape
    d = c // heads
    v = value.double().abs().reshape(s, t, heads, d)
    w = weight.double().abs().reshape(weight.shape[0], heads, d)
    a = torch.einsum('sthe,che->shtc', v, w).square().sum(-1)
    return (d + weight.shape[0] + 2) * FP32_EPS * a


def weighted_map64(keys: Sequence[torch.Tensor], weights: Sequence[torch.Tensor], grid: Tuple[int, int], n_rows: int,
                   normalize: bool = False, head_sel: Optional[int] = None) -> torch.Tensor:
    """``keys[g]`` ``[heads, tokens, h, w]`` and ``weights[g]`` ``[heads, tokens]`` of every group of one map ->
    ``[n_rows, *grid]`` float64; ``head_sel`` keeps one head of every group."""
    total, n = None, 0
    for stack, wts in zip(keys, weights):
        sel = slice(None) if head_sel is None else slice(head_sel, head_sel + 1)
        k, w = stack[sel, :n_rows], wts[sel, :n_rows].double()
        part = (up64(k, grid).clamp_(min=0.0) * w[:, :, None, None]).sum(dim=0)
        total = part if total is None else total + part
        n += k.shape[0]
    out = total / n
    return _normalize(out) if normalize else out


def weighted_tolerance(keys: Sequence[torch.Tensor], weights: Sequence[torch.Tensor], n_keys: int,
                       grid: Tuple[int, int]) -> Tuple[float, float]:
    """``(rtol, atol)`` of a weighted fp32 map against :func:`weighted_map64`: the sum of ``n_keys`` non-negative fma
    terms errs relatively by ``(n_keys + 1) 2^-24`` at most, as in ``rect_tolerance``; each key's stencil error is
    ``rect_tolerance``'s atol, times its weight, and the mean of those is below the largest weight times it."""
    rtol, atol = rect_tolerance(keys, n_keys, grid)
    wmax = max(float(w.abs().max()) for w in weights)
    return rtol, atol * max(wmax, 1.0)


def trace_weighted_map64(calls, layers, rows: Sequence[int], grid: Tuple[int, int], sample: int, n_rows_total: int,
                         images: int = 1, image_idx: Optional[int] = None, normalize: bool = False) -> torch.Tensor:
    """A traced generation's weighted map in float64: ``calls`` are the recorded ``(layer_idx, q, k, v, W, heads,
    scale)`` of every traced layer call, ``layers`` ``{layer_idx: (h, w)}`` the layers the read keeps (in read order).
    The per-key sums are the softmax of every call of the layer; the norms those of the layer's LAST call (a valid
    weighted read has one set per generation). ``sample``: the first kept sample of the batch (the conditional half
    starts at B / 2; ``negative``: 0), then ``images`` samples per prompt of which ``image_idx`` (or all) are read.
    ``rows``: the context rows of the map (compact rows of a long context). Returns ``[len(rows), *grid]``."""
    total, n = None, 0
    for layer_idx, (h, w) in layers.items():
        own = [c for c in calls if c[0] == layer_idx]
        acc, norms = None, None
        for _, q, k, v, wt, heads, scale in own:
            b = q.shape[0]
            pair = torch.cat([torch.arange(sample, sample + images), torch.arange(sample, sample + images)])
            # layer_maps64 keeps the second half of a CFG batch: feed it (kept, kept) so the kept samples come out
            m = layer_maps64(q[pair], k[pair], heads, scale)                   # [images, heads, T, hw]
            acc = m if acc is None else acc + m
            norms = value_norms64(v[sample:sample + images], wt, heads)     # [images, heads, T]
        sel = range(images) if image_idx is None else [image_idx]
        for i in sel:
            keys = acc[i][:, rows].reshape(acc.shape[1], len(rows), h, w)
            part = (up64(keys, grid).clamp_(min=0.0) * norms[i][:, rows][:, :, None, None]).sum(dim=0)
            total = part if total is None else total + part
            n += acc.shape[1]
    out = total / n
    return _normalize(out) if normalize else out
