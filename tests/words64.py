"""Float64 statement of the word-list pipeline (``daam_b200/csrc/words.cu``) and the fp32 error bound its kernels are
compared under.

* :func:`word_maps64`: a word's map, the float64 mean of its rows of a global map (heatmap.py:121-123).
* :func:`expand64`: ``expand_as`` of each word map: ``B_y @ W @ B_x^T`` with the matrices of ``math_bicubic_matrix``,
  float64 min-max normalisation unless ``absolute``, then the threshold.
* :func:`expand_bound`: per element, a bound on ``|m_fp32 - m64|`` before the threshold, derived from the kernels'
  arithmetic (``word_mean``, ``make_taps``, ``bicubic_shared``, ``minmax_normalize``), not from observed errors.
* :func:`src_error`: the part of it that comes from the fp32 source coordinate of ``make_taps``.

The kernels themselves never see these; ``tests/test_word_geometry_host.py`` checks the bound against fp32 emulations
of ``make_taps`` and of the 16-tap stencil, ``tests/test_word_geometry_gpu.py`` checks the kernels against it."""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from tests.reference64 import FP32_EPS, bicubic64

U = FP32_EPS                                          # unit roundoff of fp32, 2^-24
DENOM_EPS = 1e-8                                      # minmax_normalize's + 1e-8 (1e-8f in the kernel)
CUBIC_CURVE = 15.0                                    # sum_j max |W_j''| of the A = -0.75 cubic: 4.5 + 4.5 + 3 + 3


def word_maps64(maps: torch.Tensor, rows_per_word: Sequence[Sequence[int]]) -> torch.Tensor:
    """``[n_words, h, w]`` float64: word ``i`` is the mean of rows ``rows_per_word[i]`` of ``maps`` ``[n_rows, h, w]``
    (negative rows count from the end, as torch indexes them)."""
    return torch.stack([maps[list(rows)].double().mean(0) for rows in rows_per_word])


def expand64(word_maps: torch.Tensor, out_hw: Tuple[int, int], absolute: bool,
             threshold: Optional[float] = None) -> SimpleNamespace:
    """``expand_as`` of each of ``word_maps`` ``[n_words, h, w]`` to ``out_hw`` in float64. Returns ``v`` (the bicubic
    up-sample), ``lo`` / ``hi`` (its per-word min / max, ``[n_words, 1, 1]``), ``pre`` (``v`` normalised unless
    ``absolute``) and ``m`` (``pre`` thresholded when ``threshold`` is truthy, as ``if threshold:`` reads it), plus the
    bicubic matrices ``by`` / ``bx``. ``threshold`` should be the fp32 value the kernel compares with."""
    w = word_maps.double()
    by = bicubic64(w.shape[-2], out_hw[0], w.device)
    bx = bicubic64(w.shape[-1], out_hw[1], w.device)
    v = by @ w @ bx.T
    lo, hi = v.amin((1, 2), keepdim=True), v.amax((1, 2), keepdim=True)
    pre = v if absolute else (v - lo) / (hi - lo + DENOM_EPS)
    m = (pre > threshold).double() if threshold else pre
    return SimpleNamespace(v=v, lo=lo, hi=hi, pre=pre, m=m, by=by, bx=bx)


def src_error(n_in: int, n_out: int) -> np.ndarray:
    """``[n_out]``: how far ``make_taps``'s fp32 coordinate (``floor(src) + t``) lies from the exact
    ``src = (dst + 0.5) n_in / n_out - 0.5``, for either arithmetic nvcc may emit. The kernel computes
    ``scale = fl(n_in / n_out)`` (a correctly rounded division) and ``src = fl(fl(scale (dst + 0.5)) - 0.5)``
    (``dst + 0.5`` is exact), or with the last two contracted into one fma, ``fl(scale (dst + 0.5) - 0.5)``; then
    ``t = fl(src - floor(src))``, exact unless ``src`` is negative (``src + 1`` rounds). Each of these roundings is
    applied exactly here: ``scale (dst + 0.5)`` and ``scale (dst + 0.5) - 0.5`` are exact in float64, so both
    candidate values are the kernel's bits, and the larger of the two distances is returned. Dyadic ratios round
    nowhere and give 0."""
    f32 = lambda x: np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)
    d = np.arange(n_out, dtype=np.float64) + 0.5
    scale = float(f32(n_in / n_out))
    exact = d * n_in / n_out - 0.5
    worst = np.zeros(n_out)
    for src in (f32(f32(scale * d) - 0.5), f32(scale * d - 0.5)):          # separate roundings; one fma
        base = np.floor(src)
        worst = np.maximum(worst, np.abs(base + f32(src - base) - exact))
    return worst


def _norm(b: torch.Tensor) -> float:
    """The largest row 1-norm of a bicubic matrix."""
    return float(b.abs().sum(1).max())


def row_motion(n_in: int, n_out: int) -> np.ndarray:
    """``[n_out]`` bound on the 1-norm by which row ``dst`` of the bicubic matrix moves when its coordinate moves by
    ``ds`` (:func:`src_error`). A row is ``W_j(t)`` on taps ``floor(src) - 1 + j``; it is continuously differentiable
    in ``src``, across a change of ``floor(src)`` too (Keys' kernel is C1). So the move is at most
    ``ds (S(t) + 15 ds)``, with ``S(t) = sum_j |W_j'(t)|`` at the exact ``t`` (1.5 at t = 0, 3 at t = 1/2) and 15 the
    sum of the weights' largest second derivatives."""
    a = -0.75
    src = (np.arange(n_out, dtype=np.float64) + 0.5) * n_in / n_out - 0.5
    t = src - np.floor(src)
    near = lambda x: 3 * (a + 2) * x * x - 2 * (a + 3) * x                  # W' of |x| <= 1
    far = lambda x: 3 * a * x * x - 10 * a * x + 8 * a                       # W' of 1 <= |x| <= 2
    slope = np.abs(far(t + 1)) + np.abs(near(t)) + np.abs(near(1 - t)) + np.abs(far(2 - t))
    ds = src_error(n_in, n_out)
    return ds * (slope + CUBIC_CURVE * ds)


def expand_bound(word_maps: torch.Tensor, out_hw: Tuple[int, int], absolute: bool, n_rows=1,
                 mean_abs: Optional[torch.Tensor] = None, exp: Optional[SimpleNamespace] = None) -> torch.Tensor:
    """Per element, ``[n_words, H, W]``: a bound on ``|m_fp32 - m64|`` before the threshold, for the fp32 value the
    word-list kernels compute from the fp32 global map (``word_maps`` the float64 :func:`word_maps64`, ``n_rows`` the
    row count ``k`` of each word, an int or one per word; ``mean_abs`` the float64 mean of the absolute rows, by
    default ``|word_maps|``, which it is for non-negative maps; ``exp``: :func:`expand64` of ``word_maps``, if at hand).
    With ``u = 2^-24``, ``N_y`` / ``N_x`` the largest row 1-norms of the bicubic matrices and ``M`` the word map's
    largest magnitude:

    1. word map (``word_mean``): ``k`` fp32 adds and one division, below ``(k + 1) u`` times the mean of ``|rows|``;
       the stencil carries it to the output with gain ``N_y N_x``;
    2. the 16-tap stencil (``bicubic_shared``): fp32 weights from an fp32 ``t``, their products and sums, below
       ``32 u N_y N_x M`` (``finalize_tolerance``'s stencil bound);
    3. the source coordinate: ``floor(src) + t`` lies within ``ds`` (:func:`src_error`) of the exact ``src``, so row
       ``dst`` of each bicubic matrix moves by at most ``g(dst)`` in 1-norm (:func:`row_motion`: ``ds`` times the
       weights' slope, at most 3), and ``v = B_y W B_x^T`` by at most ``g_y(oy) N_x M + g_x(ox) N_y M``;
    4. normalised maps: with ``E`` the bound of 1-3 at the element, ``E*`` its largest value over the word (``lo`` and
       ``hi`` are values of ``v``, so each errs by at most ``E*``), ``D = hi - lo + 1e-8``, ``r = (v - lo) / D`` in
       ``[0, 1)`` and ``rho = 2 u D + 2^-50`` (the two roundings of the denominator, and ``1e-8f`` against ``1e-8``):
       the computed numerator is ``(r D + dv - dlo)(1 + d1)`` and denominator ``D' = D + dhi - dlo + rho'``, so
       ``m' - m = (D (dv - (1 - r) dlo - r dhi) + d1 num D - r D rho') / (D D')``, and
       ``|dm| <= (E + E* + u (r D + E + E*) + r rho) / (D - 2 E* - rho)``, plus the rounding of the quotient,
       ``u (r + |dm|)``.

    Absolute maps keep 1-3; a normalised 1-pixel output is 0 exactly."""
    w = word_maps.double()
    n_words, mh, mw = w.shape
    if exp is None:
        exp = expand64(w, out_hw, absolute=True)
    ny, nx = _norm(exp.by), _norm(exp.bx)
    ks = torch.as_tensor([n_rows] * n_words if isinstance(n_rows, int) else list(n_rows), dtype=torch.float64,
                         device=w.device).view(-1, 1, 1)
    mabs = (w.abs() if mean_abs is None else mean_abs.double()).amax((1, 2), keepdim=True)
    big_m = w.abs().amax((1, 2), keepdim=True)
    gy = torch.from_numpy(row_motion(mh, out_hw[0])).to(w.device).view(1, -1, 1)
    gx = torch.from_numpy(row_motion(mw, out_hw[1])).to(w.device).view(1, 1, -1)
    e = (ks + 1) * U * mabs * ny * nx + 32 * U * ny * nx * big_m
    e = e + big_m * (gy * nx + gx * ny)                                        # [n_words, H, W]
    if absolute:
        return e
    if out_hw[0] * out_hw[1] == 1:                       # one pixel: v - lo is 0 on both sides, and so is m
        return torch.zeros_like(e)
    v, lo, hi = exp.v, exp.lo, exp.hi
    den = hi - lo + DENOM_EPS
    e_star = e.amax((1, 2), keepdim=True)
    rho = 2 * U * den + 2.0 ** -50
    low_den = den - 2 * e_star - rho
    assert bool((low_den > 0).all()), 'the bound cannot separate lo from hi: the word map is too flat'
    r = (v - lo) / den
    a = e + e_star
    dm = (a + U * (r * den + a) + r * rho) / low_den
    return dm + U * (r + dm)


def bound_for(maps: torch.Tensor, rows_per_word: Sequence[Sequence[int]], out_hw: Tuple[int, int], absolute: bool,
              threshold: Optional[float] = None) -> Tuple[SimpleNamespace, torch.Tensor]:
    """:func:`expand64` of the words of ``maps`` ``[n_rows, h, w]`` and :func:`expand_bound` for them."""
    wm = word_maps64(maps, rows_per_word)
    mean_abs = word_maps64(maps.abs(), rows_per_word)
    exp = expand64(wm, out_hw, absolute, threshold)
    exp.word_maps = wm
    return exp, expand_bound(wm, out_hw, absolute, [len(r) for r in rows_per_word], mean_abs, exp)


def threshold_unsure(pre: torch.Tensor, bound: torch.Tensor, threshold: float) -> torch.Tensor:
    """The elements whose thresholded value the bound cannot decide: ``pre`` within ``bound`` of ``threshold``."""
    return (pre - threshold).abs() <= bound


def row_mean_bound(maps: torch.Tensor, rows_per_word: Sequence[Sequence[int]]) -> torch.Tensor:
    """``[n_words, h, w]``: ``(k + 1) u`` times the mean of ``|rows|``, the bound of the fp32 ``word_mean``."""
    mean_abs = word_maps64(maps.abs(), rows_per_word)
    ks = torch.tensor([len(r) for r in rows_per_word], dtype=torch.float64, device=maps.device).view(-1, 1, 1)
    return (ks + 1) * U * mean_abs


def fp32(x: float) -> float:
    """``x`` rounded to fp32, as the kernel receives a threshold."""
    return float(np.float32(x))

