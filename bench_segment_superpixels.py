#!/usr/bin/env python
"""Benchmark of superpixel word segmentation on one GPU: ``GlobalHeatMap.segment_superpixels`` /
``GlobalHeatMapStack.segment_superpixels`` (``daam_segment_superpixels``: the word maps, ``2 * iterations`` SLIC
launches, then the per-tile sums, the per-superpixel means and the labels) against the same algorithm written in torch
on the device:

* SLIC: per pass the 9 candidate centres' distances as separate float64 ops, stacked and ``argmin``-ed (the first
  minimum, so the lowest cluster wins a tie), then the integer sums of the next centres by ``index_add_``;
* pooling: ``expand_words(..., to_cpu=False)``, its float64 sums per superpixel by ``index_add_``, over the pixel
  counts, then the max and argmax over the words;
* for a history (one image for every step): the partition once, the pooling once per step.

    python bench_segment_superpixels.py [--steps K] [--warmup W] [--rounds R]

Workloads, all with a threshold of 0.4, compactness 20 and 10 passes: SD-2.1 at 512x512 with 8 and 24 words and 1024
segments; SDXL at 1024x1024 and 1216x832 with 8 words and 1024 segments (grids as the tracer makes them: 64x64,
128x128, 76x52); a 50-step history at 512x512 with 8 words; SD-2.1 at 512x512 with 8 words and 256 and 4096 segments.
Maps are uniform random rows; the image is flat random-coloured blocks with a little noise, so that it has edges.

Before timing, the two forms are checked against each other: the partitions equal, the scores within
``SCORE_TOLERANCE`` and the labels equal on all but ``LABEL_MISMATCH`` of the pixels (the torch form's float64 sums
run in atomic order, which can flip a superpixel whose two best means tie to within rounding). Timing: warm-up, then
blocks of K calls queued behind a spin kernel and timed with CUDA events; the fused call and the torch form alternate,
R rounds each, and the median is reported. The card name and power limit are read in the same run. One JSON line per
workload goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import math
import os
import sys

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench_aspect import card           # noqa: E402
from bench_segment_crf import _size, make_image   # noqa: E402

# name, grid, image (h, w), words, maps (0: one global map), n_segments
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 0, 1024), ('sd21', (64, 64), (512, 512), 24, 0, 1024),
             ('sdxl', (128, 128), (1024, 1024), 8, 0, 1024), ('sdxl', (76, 52), (1216, 832), 8, 0, 1024),
             ('sd21-history', (64, 64), (512, 512), 8, 50, 1024),
             ('sd21', (64, 64), (512, 512), 8, 0, 256), ('sd21', (64, 64), (512, 512), 8, 0, 4096)]
SP = dict(threshold=0.4, compactness=20.0, iterations=10)
N_PROMPT_WORDS = 30
SCORE_TOLERANCE = 1e-6   # max |score_torch - score_fused| accepted
LABEL_MISMATCH = 1e-3    # largest share of pixels whose labels may differ


def torch_slic(image, n_segments):
    """The partition of daam_image_superpixels in torch: int64 ``[h * w]`` cluster ids and ``[cells]`` pixel counts."""
    h, w = image.shape[:2]
    dev = image.device
    s = math.sqrt(float(h * w) / n_segments)
    ny, nx = min(max(math.floor(h / s + 0.5), 1), h), min(max(math.floor(w / s + 0.5), 1), w)
    cells = ny * nx
    c = float(torch.tensor(SP['compactness'], dtype=torch.float32))
    wxy = c * c * float(cells) / float(h * w)
    yb = torch.arange(ny + 1, device=dev) * h // ny
    xb = torch.arange(nx + 1, device=dev) * w // nx
    cy = ((torch.arange(h, device=dev) + 1) * ny - 1) // h
    cx = ((torch.arange(w, device=dev) + 1) * nx - 1) // w
    sy, sx = (yb[:-1] + yb[1:] - 1) // 2, (xb[:-1] + xb[1:] - 1) // 2
    ys, xs = sy.repeat_interleave(nx), sx.repeat(ny)
    yy, xx = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing='ij')
    feats = torch.cat([image.long(), yy[..., None], xx[..., None], torch.ones_like(yy)[..., None]], -1).reshape(-1, 6)
    state = feats.view(h, w, 6)[ys, xs]
    pix = torch.cat([image.double(), yy[..., None].double(), xx[..., None].double()], -1)
    for t in range(SP['iterations']):
        mu = state[:, :5].double() / state[:, 5:].double()
        ds = []
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                ky, kx = cy[:, None] + dy, cx[None, :] + dx
                ok = (ky >= 0) & (ky < ny) & (kx >= 0) & (kx < nx)
                e = pix - mu[ky.clamp(0, ny - 1) * nx + kx.clamp(0, nx - 1)]
                d = ((e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]) + \
                    wxy * ((e[..., 3] * e[..., 3]) + (e[..., 4] * e[..., 4]))
                ds.append(torch.where(ok, d, torch.inf))
        pick = torch.stack(ds).argmin(0)                # the first minimum: ascending k
        ky = cy[:, None] + pick // 3 - 1
        kx = cx[None, :] + pick % 3 - 1
        lab = (ky * nx + kx).reshape(-1)
        new = torch.zeros((cells, 6), dtype=torch.int64, device=dev).index_add_(0, lab, feats)
        if t + 1 < SP['iterations']:
            state = torch.where(new[:, 5:] > 0, new, state)
    return lab, new[:, 5]


def torch_pool(m, lab, count):
    """labels uint8 and scores fp32 ``[h, w]`` of the word values ``m`` ``[W, h, w]`` pooled over ``lab``."""
    n_words, h, w = m.shape
    sums = torch.zeros((n_words, count.numel()), dtype=torch.float64, device=m.device)
    sums.index_add_(1, lab, m.reshape(n_words, -1).double())
    mean = (sums / count.clamp(min=1).double()).float()
    best, arg = mean.max(0)
    labels = torch.where(best > SP['threshold'], arg + 1, 0).to(torch.uint8)
    return labels[lab].view(h, w), best[lab].view(h, w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.heatmap import GlobalHeatMap, TimeHeatMaps
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    torch.cuda.set_device(0)
    _native.load()
    name, power = card()
    stream = torch.cuda.current_stream()

    def block_us(fn, size, spin_ms):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(spin_ms * 1.9e6))          # the host queues the whole block while the GPU spins
        e0.record(stream)
        for _ in range(size):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / size * 1e3

    med = lambda v: sorted(v)[len(v) // 2]
    tok = WhitespaceTokenizer()
    prompt = ' '.join(f'w{i}' for i in range(N_PROMPT_WORDS))
    g = torch.Generator(device='cuda').manual_seed(0)
    for workload, grid, hw, n_words, stack, k in WORKLOADS:
        out_hw = (hw[1], hw[0]) if grid[0] == grid[1] else hw
        image = make_image(*out_hw, g)
        words = [f'w{i}' for i in range(n_words)]
        n_maps = max(1, stack)
        maps = torch.rand((n_maps, N_PROMPT_WORDS + 2) + grid, generator=g, device='cuda')
        target = TimeHeatMaps(tok, prompt, maps) if stack else GlobalHeatMap(tok, prompt, maps[0])
        singles = [target[i] for i in range(n_maps)] if stack else [target]
        fused = lambda: target.segment_superpixels(words, image, n_segments=k, to_cpu=False, **SP)

        def composition():
            lab, count = torch_slic(image, k)
            return lab, [torch_pool(ghm.expand_words(words, _size(image), to_cpu=False)[1], lab, count)
                         for ghm in singles]

        # the answers before timing: the torch form against the fused call
        _, labels, scores, sp = fused()
        labels, scores = labels.reshape(n_maps, *out_hw), scores.reshape(n_maps, *out_hw)
        lab, comp = composition()
        assert torch.equal(lab.view(out_hw).int(), sp), workload
        s_diff = max(float((cs - scores[i]).abs().max()) for i, (_, cs) in enumerate(comp))
        mismatch = max(float((cl != labels[i]).float().mean()) for i, (cl, _) in enumerate(comp))
        assert s_diff <= SCORE_TOLERANCE and mismatch <= LABEL_MISMATCH, (workload, k, s_diff, mismatch)
        del comp
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        size = max(1, args.steps // max(1, n_maps // 5))
        loop_size = max(1, size // 4)
        for _ in range(max(1, args.warmup)):
            fused(); composition()
        torch.cuda.synchronize()
        a, b = [], []
        for _ in range(args.rounds):                     # alternated rounds
            a.append(block_us(fused, size, 5.0 + 0.5 * size * n_maps))
            b.append(block_us(composition, loop_size, 5.0 + 10.0 * loop_size * n_maps))
        fused_us, torch_us = med(a), med(b)
        bench.emit({'workload': workload, 'image': f'{out_hw[0]}x{out_hw[1]}', 'grid': list(grid),
                    'words': n_words, 'maps': n_maps, 'n_segments': k, 'iterations': SP['iterations'],
                    'fused_us': round(fused_us, 1), 'torch_us': round(torch_us, 1),
                    'speedup_vs_torch': round(torch_us / fused_us, 2), 'fused_launches': launches,
                    'torch_max_score_diff': float(f'{s_diff:.3g}'), 'label_mismatch': float(f'{mismatch:.3g}'),
                    'timing': f'median of {args.rounds} alternated rounds of {size} calls ({loop_size} torch)',
                    'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
