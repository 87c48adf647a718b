"""Float64 numpy reference of the region ranking scores (GlobalHeatMap.region_ranking, daam_region_ranking).

For one plane of values ``v`` (the fp32 expand_words values, compared as numbers: -0 and +0 tie) and a region ``inside``
(bool), with P the pixels inside, N the others and the distinct values in ascending order:

* ``u2 = sum_{p in P} sum_{q in N} (2 [v_p > v_q] + [v_p == v_q])``, from int64 counts per distinct value;
* ``ap = sum_k (TP_k - TP_{k-1}) / n_p * TP_k / (TP_k + FP_k)`` over the distinct values in descending order, NaN when
  n_p = 0 (sklearn's ``average_precision_score``);
* ``groups``: the number of distinct values (tie groups), which bounds the rounding of the ap sum.
"""
import numpy as np


def plane_groups(values):
    """``(inverse, n_groups)``: each pixel's tie group, numbered by ascending value."""
    uniq, inv = np.unique(np.asarray(values, dtype=np.float64).ravel(), return_inverse=True)
    return inv.ravel(), len(uniq)


def ranking64(values, inside, groups=None):
    """``(u2, ap, n_groups)`` of one plane ``values`` against one region ``inside`` (same shape). ``groups``: what
    :func:`plane_groups` returns for ``values``, to share it over several regions."""
    inv, k = plane_groups(values) if groups is None else groups
    pos = np.asarray(inside, dtype=bool).ravel()
    cnt_p = np.bincount(inv[pos], minlength=k).astype(np.int64)
    cnt_n = np.bincount(inv[~pos], minlength=k).astype(np.int64)
    n_p = int(cnt_p.sum())
    neg_below = np.cumsum(cnt_n) - cnt_n                  # negatives strictly below each value
    u2 = int((cnt_p * (2 * neg_below + cnt_n)).sum())
    if n_p == 0:
        return u2, float('nan'), k
    tp, fp = cnt_p[::-1], cnt_n[::-1]                     # descending values
    tp_le, fp_le = np.cumsum(tp), np.cumsum(fp)
    ap = float(np.sum(tp / n_p * (tp_le / (tp_le + fp_le))))
    return u2, ap, k


def ranking64_all(m, regions):
    """``(u2 int64 [R, W], ap float64 [R, W], groups [W])`` of a stack ``m`` [W, H, W'] against ``regions`` [R, H, W']
    (nonzero inside)."""
    m = np.asarray(m)
    inside = np.asarray(regions) != 0
    n_words, n_regions = m.shape[0], inside.shape[0]
    u2 = np.zeros((n_regions, n_words), dtype=np.int64)
    ap = np.zeros((n_regions, n_words), dtype=np.float64)
    groups = np.zeros(n_words, dtype=np.int64)
    for w in range(n_words):
        g = plane_groups(m[w])
        groups[w] = g[1]
        for r in range(n_regions):
            u2[r, w], ap[r, w], _ = ranking64(None, inside[r], g)
    return u2, ap, groups


def ap_bound(ap, groups):
    """The largest |ap - ap64| two float64 sums of the same ``groups`` positive terms can differ by: each side rounds
    every term at most three times and adds them in some order, so each is within (groups + 3) * 2^-53 * ap of the
    exact value."""
    return 2 * (np.asarray(groups, dtype=np.float64) + 3) * 2.0 ** -53 * np.abs(ap)
