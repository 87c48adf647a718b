"""Float64 reference of the boundary scores (daam_region_boundary / daam_mask_boundary, RegionBoundary), with numpy and
scipy, straight from the definitions:

* the boundary of a mask M is M & ~binary_erosion(M, cross, border_value=0): the pixels of M with a 4-neighbour outside
  M or outside the image;
* d2(p, S) is the squared Euclidean distance between pixel centres to the nearest pixel of S, taken from scipy's exact
  distance_transform_edt as rint(d * d);
* a boundary pixel is within tolerance theta when d2 <= theta^2, theta the fp32 tolerance widened to float64.

brute_force() computes the same outputs from every pairwise distance, for pinning the reference on small masks.
"""
import math

import numpy as np
from scipy import ndimage

CROSS = ndimage.generate_binary_structure(2, 1)


def boundary(mask: np.ndarray) -> np.ndarray:
    m = np.asarray(mask) != 0
    return m & ~ndimage.binary_erosion(m, CROSS, border_value=0)


def d2_map(s: np.ndarray) -> np.ndarray:
    """int64 squared distance from every pixel to the nearest pixel of the nonempty set ``s``."""
    d = ndimage.distance_transform_edt(~s)
    return np.rint(d * d).astype(np.int64)


def tolerances2(tolerances) -> np.ndarray:
    t = np.asarray(tolerances, dtype=np.float32).astype(np.float64)
    return t * t


def _direction(d2: np.ndarray, tol2: np.ndarray):
    """hits per tolerance, max d2 and the float64 sum of roots (math.fsum: the exactly rounded sum) of the d2 values of
    one direction's boundary pixels."""
    hits = [(d2.astype(np.float64) <= t).sum() for t in tol2]
    return hits, int(d2.max()), math.fsum(np.sqrt(d2.astype(np.float64)).tolist())


def _scores(planes, regions, tolerances, d2_between):
    planes = np.asarray(planes).reshape(-1, *np.shape(planes)[-2:])
    regions = np.asarray(regions).reshape(-1, *np.shape(regions)[-2:])
    tol2 = tolerances2(tolerances)
    P, R, T = planes.shape[0], regions.shape[0], len(tol2)
    da = [boundary(m) for m in planes]
    db = [boundary(m) for m in regions]
    out = dict(word_boundary=np.array([int(a.sum()) for a in da], dtype=np.int32),
               region_boundary=np.array([int(b.sum()) for b in db], dtype=np.int32),
               word_hits=np.zeros((P, T, R), np.int32), region_hits=np.zeros((P, T, R), np.int32),
               max_d2=np.full((P, R, 2), -1, np.int64), sum_dist=np.zeros((P, R, 2), np.float64))
    for p in range(P):
        for r in range(R):
            if not da[p].any() or not db[r].any():
                continue
            for k, (src, dst) in enumerate(((da[p], db[r]), (db[r], da[p]))):
                hits, mx, s = _direction(d2_between(src, dst), tol2)
                (out['word_hits'] if k == 0 else out['region_hits'])[p, :, r] = hits
                out['max_d2'][p, r, k] = mx
                out['sum_dist'][p, r, k] = s
    return out


def boundary64(planes, regions, tolerances):
    """The outputs of daam_mask_boundary for ``planes`` ``[P, H, W]`` (nonzero: inside) and ``regions`` ``[R, H, W]``:
    ``word_boundary`` ``[P]``, ``region_boundary`` ``[R]``, ``word_hits`` / ``region_hits`` ``[P, T, R]``, ``max_d2`` /
    ``sum_dist`` ``[P, R, 2]``."""
    cache = {}

    def d2_between(src, dst):
        if id(dst) not in cache:
            cache[id(dst)] = d2_map(dst)
        return cache[id(dst)][src]
    return _scores(planes, regions, tolerances, d2_between)


def brute_force(planes, regions, tolerances):
    """boundary64 from every pairwise distance between the two boundaries."""
    def d2_between(src, dst):
        a, b = np.argwhere(src), np.argwhere(dst)
        diff = a[:, None, :] - b[None, :, :]
        return (diff * diff).sum(-1).min(1)
    return _scores(planes, regions, tolerances, d2_between)


def as_stack(out, n_maps: int, n_words: int):
    """boundary64's plane-major outputs as RegionBoundary's ``[maps, T, R, W]`` / ``[maps, R, W, 2]`` layout."""
    T, R = out['word_hits'].shape[1:]
    return dict(word_boundary=out['word_boundary'].reshape(n_maps, n_words),
                region_boundary=out['region_boundary'],
                word_hits=out['word_hits'].reshape(n_maps, n_words, T, R).transpose(0, 2, 3, 1),
                region_hits=out['region_hits'].reshape(n_maps, n_words, T, R).transpose(0, 2, 3, 1),
                max_d2=out['max_d2'].reshape(n_maps, n_words, R, 2).transpose(0, 2, 1, 3),
                sum_dist=out['sum_dist'].reshape(n_maps, n_words, R, 2).transpose(0, 2, 1, 3))


def sum_bound(out):
    """The allowed |error| of each sum_dist entry: n 2^-52 of the exact sum for n terms (each root and each addition
    rounded once, in float64)."""
    n = np.stack([np.broadcast_to(out['word_boundary'][..., None, :], out['max_d2'].shape[:-1]),
                  np.broadcast_to(out['region_boundary'][:, None], out['max_d2'].shape[:-1])], -1)
    return n * 2.0 ** -52 * np.abs(out['sum_dist'])
