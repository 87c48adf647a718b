"""The numpy reference of the superpixel calls (daam_image_superpixels, daam_segment_superpixels): the SLIC partition in
integers and float64 exactly as include/daam_b200.h defines it, so the device must match it bit for bit, and the
pooled word means in float64."""
import math

import numpy as np

MAX_CELLS = 65536


def grid(h: int, w: int, k: int):
    """``(ny, nx)``: ``S = sqrt(H W / K)`` in float64, ``clamp(floor(H / S + 0.5), 1, H)`` rows, columns likewise."""
    s = math.sqrt(float(h * w) / k)
    return min(max(math.floor(h / s + 0.5), 1), h), min(max(math.floor(w / s + 0.5), 1), w)


def cell_begin(c, n_cells: int, n: int):
    """The first pixel row (column) of cell row (column) ``c``: ``floor(c n / n_cells)``."""
    return np.asarray(c, dtype=np.int64) * n // n_cells


def cell_of(y, n_cells: int, n: int):
    """The cell row (column) of pixel row (column) ``y``: ``floor(((y + 1) n_cells - 1) / n)``."""
    return ((np.asarray(y, dtype=np.int64) + 1) * n_cells - 1) // n


def wxy(c: float, ny: int, nx: int, h: int, w: int) -> float:
    """``c c (ny nx) / (H W)``, left to right in float64 from the fp32 ``c``."""
    c = float(np.float32(c))
    return c * c * float(ny * nx) / float(h * w)


def initial_state(img: np.ndarray, ny: int, nx: int) -> np.ndarray:
    """int64 ``[ny nx, 6]``: each cluster's ``(sum r, g, b, y, x, n)`` of the pixel at the middle of its cell."""
    h, w = img.shape[:2]
    yb, xb = cell_begin(np.arange(ny + 1), ny, h), cell_begin(np.arange(nx + 1), nx, w)
    ys = np.repeat((yb[:-1] + yb[1:] - 1) // 2, nx)
    xs = np.tile((xb[:-1] + xb[1:] - 1) // 2, ny)
    st = np.empty((ny * nx, 6), dtype=np.int64)
    st[:, :3] = img[ys, xs].astype(np.int64)
    st[:, 3], st[:, 4], st[:, 5] = ys, xs, 1
    return st


def assign(img: np.ndarray, state: np.ndarray, ny: int, nx: int, c: float) -> np.ndarray:
    """One assignment pass: int32 ``[H, W]``, each pixel's nearest of the up to 9 clusters around its cell, every
    float64 operation rounded on its own, the lowest cluster on ties."""
    h, w = img.shape[:2]
    mu = state[:, :5].astype(np.float64) / state[:, 5:6].astype(np.float64)
    cy = cell_of(np.arange(h), ny, h)[:, None]
    cx = cell_of(np.arange(w), nx, w)[None, :]
    pix = img.astype(np.float64)
    fy = np.arange(h, dtype=np.float64)[:, None]
    fx = np.arange(w, dtype=np.float64)[None, :]
    k_wxy = wxy(c, ny, nx, h, w)
    best = np.full((h, w), np.inf)
    lab = np.zeros((h, w), dtype=np.int64)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            ky, kx = cy + dy, cx + dx
            ok = (ky >= 0) & (ky < ny) & (kx >= 0) & (kx < nx)
            k = np.clip(ky, 0, ny - 1) * nx + np.clip(kx, 0, nx - 1)
            m = mu[k]                                       # [H, W, 5]
            er, eg, eb = pix[..., 0] - m[..., 0], pix[..., 1] - m[..., 1], pix[..., 2] - m[..., 2]
            ey, ex = fy - m[..., 3], fx - m[..., 4]
            d = ((er * er + eg * eg) + eb * eb) + k_wxy * ((ey * ey) + (ex * ex))
            take = ok & (d < best)                          # ascending k: strict keeps the lowest on ties
            best = np.where(take, d, best)
            lab = np.where(take, k, lab)
    return lab.astype(np.int32)


def sums(img: np.ndarray, lab: np.ndarray, cells: int) -> np.ndarray:
    """int64 ``[cells, 6]``: the exact ``(sum r, g, b, y, x, n)`` of each cluster's pixels."""
    h, w = img.shape[:2]
    out = np.zeros((cells, 6), dtype=np.int64)
    flat = lab.reshape(-1).astype(np.int64)
    yy, xx = np.meshgrid(np.arange(h, dtype=np.int64), np.arange(w, dtype=np.int64), indexing='ij')
    cols = [img[..., 0], img[..., 1], img[..., 2], yy, xx, np.ones((h, w), dtype=np.int64)]
    for i, v in enumerate(cols):
        np.add.at(out[:, i], flat, v.reshape(-1).astype(np.int64))
    return out


def slic(img: np.ndarray, n_segments: int, compactness: float, iterations: int) -> np.ndarray:
    """int32 ``[H, W]``: the partition after ``iterations`` passes; between passes a cluster with pixels takes their
    sums, one without keeps its own."""
    h, w = img.shape[:2]
    ny, nx = grid(h, w, n_segments)
    assert ny * nx <= MAX_CELLS
    state = initial_state(img, ny, nx)
    for t in range(iterations):
        lab = assign(img, state, ny, nx, compactness)
        if t + 1 < iterations:
            new = sums(img, lab, ny * nx)
            state = np.where(new[:, 5:6] > 0, new, state)
    return lab


def slic_brute(img: np.ndarray, n_segments: int, compactness: float, iterations: int) -> np.ndarray:
    """The same partition pixel by pixel in plain Python, from the definitions."""
    h, w = img.shape[:2]
    s = math.sqrt(float(h * w) / n_segments)
    ny, nx = min(max(math.floor(h / s + 0.5), 1), h), min(max(math.floor(w / s + 0.5), 1), w)
    yb = [c * h // ny for c in range(ny + 1)]
    xb = [c * w // nx for c in range(nx + 1)]
    state = []
    for cy in range(ny):
        for cx in range(nx):
            y, x = (yb[cy] + yb[cy + 1] - 1) // 2, (xb[cx] + xb[cx + 1] - 1) // 2
            state.append([int(img[y, x, 0]), int(img[y, x, 1]), int(img[y, x, 2]), y, x, 1])
    cf = float(np.float32(compactness))
    k_wxy = cf * cf * float(ny * nx) / float(h * w)
    for t in range(iterations):
        lab = [[0] * w for _ in range(h)]
        for y in range(h):
            cy = next(c for c in range(ny) if yb[c] <= y < yb[c + 1])
            for x in range(w):
                cx = next(c for c in range(nx) if xb[c] <= x < xb[c + 1])
                best, arg = math.inf, -1
                for ky in range(cy - 1, cy + 2):
                    for kx in range(cx - 1, cx + 2):
                        if not (0 <= ky < ny and 0 <= kx < nx):
                            continue
                        k = ky * nx + kx
                        n = float(state[k][5])
                        mu = [float(v) / n for v in state[k][:5]]
                        px = [float(img[y, x, 0]), float(img[y, x, 1]), float(img[y, x, 2]), float(y), float(x)]
                        e = [px[i] - mu[i] for i in range(5)]
                        d = ((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]) + k_wxy * ((e[3] * e[3]) + (e[4] * e[4]))
                        if d < best:
                            best, arg = d, k
                lab[y][x] = arg
        if t + 1 < iterations:
            new = [[0] * 6 for _ in state]
            for y in range(h):
                for x in range(w):
                    acc = new[lab[y][x]]
                    for i, v in enumerate((int(img[y, x, 0]), int(img[y, x, 1]), int(img[y, x, 2]), y, x, 1)):
                        acc[i] += v
            state = [nw if nw[5] else old for nw, old in zip(new, state)]
    return np.array(lab, dtype=np.int32)


def pooled64(m: np.ndarray, lab: np.ndarray):
    """``(mean, count)``: float64 ``[n_words, cells]`` means of ``m`` ``[n_words, H, W]`` over each cluster of ``lab``
    (NaN where empty) and int64 ``[cells]`` pixel counts, ``cells = lab.max() + 1``."""
    flat = lab.reshape(-1).astype(np.int64)
    cells = int(flat.max()) + 1
    count = np.bincount(flat, minlength=cells)
    mean = np.stack([np.bincount(flat, weights=mw.reshape(-1).astype(np.float64), minlength=cells) for mw in m])
    with np.errstate(invalid='ignore', divide='ignore'):
        return mean / count, count


def pooled_labels64(m: np.ndarray, lab: np.ndarray, threshold=None):
    """``(labels, scores, top2)``: what daam_segment_superpixels gives with float64 means rounded to fp32 -- uint8 and
    fp32 ``[H, W]`` -- and the fp32 gap between each pixel's two highest means (inf with one word)."""
    mean, _ = pooled64(m, lab)
    mean32 = mean.astype(np.float32)
    arg = np.argmax(mean32, axis=0)                      # the first word on ties
    best = mean32.max(axis=0)
    srt = np.sort(mean32, axis=0)
    gap = (srt[-1] - srt[-2]) if len(m) > 1 else np.full_like(best, np.inf)
    lab_c = (arg + 1).astype(np.uint8)
    if threshold:
        lab_c = np.where(best > np.float32(threshold), lab_c, 0).astype(np.uint8)
    return lab_c[lab], best[lab], gap[lab]
