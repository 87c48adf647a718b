#!/usr/bin/env python
"""Benchmark of boundary scores on one GPU: ``GlobalHeatMap.region_boundary`` / ``GlobalHeatMapStack.region_boundary``
(``daam_region_boundary``: the regions' boundaries and column distances, then per round of planes the values, the
planes' boundaries and column distances, one nearest-boundary query pass and a fixed-order reduction) and
``evaluate.boundary_scores`` (``daam_mask_boundary``) against what a user writes today: ``expand_words(...,
threshold)`` copied to the host, then scipy's ``binary_erosion`` and ``distance_transform_edt`` once per region and once
per (map, word) plane, and the hit counts, maximum and sum of distances per (plane, region) pair. scipy takes seconds,
so it is timed on a few regions, planes and pairs and scaled to all of them (``scipy_scaled``: true).

    python bench_region_boundary.py [--steps K] [--warmup W] [--rounds R]

Workloads: SD-2.1 at 512x512 with 8 words and 4 regions, 8 x 16 and 24 x 4; SDXL at 1024x1024 with 8 x 4 and 24 x 4;
SDXL at 1216x832 with 8 x 4 (grids as the tracer makes them: 64x64, 128x128, 76x52); a 50-step history and 15 layer
maps at 512x512 with 8 x 4; the far-apart worst case at 1024x1024 (``boundary_scores`` of 8 masks of 30 % noise in the
bottom-right quadrant, every mask pixel a likely boundary pixel, against 4 small squares in the top-left corner: every
query scans most of its row); ``boundary_scores`` of ``refine_words(..., threshold=0.4)`` at 512x512 with 8 words and
4 regions. Regions are random rectangles, maps uniform random rows, the threshold 0.5 and the tolerance DAVIS's
default.

Timing: warm-up, then blocks of K calls queued behind a spin kernel and timed with CUDA events, R rounds, median. Every
fused result is checked equal to the scipy computation (the counts and maxima exactly, the sums within 1e-9 relative)
before timing: every plane for one map, the first two maps of a stack. The card name and power limit are read in the
same run. One JSON line per workload goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import math
import os
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench_aspect import card           # noqa: E402

# name, grid, image (h, w), words, regions, maps (0: one global map), kind
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 4, 0, None), ('sd21', (64, 64), (512, 512), 8, 16, 0, None),
             ('sd21', (64, 64), (512, 512), 24, 4, 0, None),
             ('sdxl', (128, 128), (1024, 1024), 8, 4, 0, None), ('sdxl', (128, 128), (1024, 1024), 24, 4, 0, None),
             ('sdxl', (76, 52), (1216, 832), 8, 4, 0, None),
             ('sd21-history', (64, 64), (512, 512), 8, 4, 50, 'time'),
             ('sd21-layers', (64, 64), (512, 512), 8, 4, 15, 'layer'),
             ('far-apart', (128, 128), (1024, 1024), 8, 4, 0, 'far'),
             ('sd21-refined', (64, 64), (512, 512), 8, 4, 0, 'refine')]
N_PROMPT_WORDS = 30
THRESHOLD = 0.5
TIMED_REGIONS, TIMED_PLANES, TIMED_PAIRS = 2, 2, 4


def scipy_scores(planes, regions, tol2):
    """What a user writes today, on host masks ``planes`` [P, H, W] and ``regions`` [R, H, W]: per set the boundary and
    its distance transform, then per pair the hits per tolerance, the maxima and the sums of distances, both ways.
    Returns the six outputs in daam_mask_boundary's layout and the seconds spent on regions, planes and pairs."""
    from scipy import ndimage
    cross = ndimage.generate_binary_structure(2, 1)

    def prep(m):
        b = m & ~ndimage.binary_erosion(m, cross, border_value=0)
        d = ndimage.distance_transform_edt(~b) if b.any() else None
        return b, d

    t0 = time.perf_counter()
    rb = [prep(r) for r in regions]
    t1 = time.perf_counter()
    pb = [prep(p) for p in planes]
    t2 = time.perf_counter()
    P, R, T = len(planes), len(regions), len(tol2)
    out = dict(word_boundary=np.array([b.sum() for b, _ in pb]), region_boundary=np.array([b.sum() for b, _ in rb]),
               word_hits=np.zeros((P, T, R), np.int64), region_hits=np.zeros((P, T, R), np.int64),
               max_d2=np.full((P, R, 2), -1, np.int64), sum_dist=np.zeros((P, R, 2)))
    for p, (ba, da) in enumerate(pb):
        for r, (bb, db) in enumerate(rb):
            if da is None or db is None:
                continue
            for k, d in enumerate((db[ba], da[bb])):
                d2 = np.rint(d * d)
                (out['word_hits'] if k == 0 else out['region_hits'])[p, :, r] = [(d2 <= t).sum() for t in tol2]
                out['max_d2'][p, r, k] = int(d2.max())
                out['sum_dist'][p, r, k] = np.sqrt(d2).sum()
    t3 = time.perf_counter()
    return out, (t1 - t0, t2 - t1, t3 - t2)


def check(flat, ref, what):
    for f in ('word_boundary', 'region_boundary', 'word_hits', 'region_hits', 'max_d2'):
        assert np.array_equal(flat[f], ref[f]), (what, f)
    assert np.allclose(flat['sum_dist'], ref['sum_dist'], rtol=1e-9, atol=0), what


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.evaluate import boundary_scores
    from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, TimeHeatMaps
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
    gc = torch.Generator().manual_seed(0)
    for workload, grid, hw, n_words, n_regions, stack, kind in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        h, w = out_hw = (hw[1], hw[0]) if grid[0] == grid[1] else hw
        words = [f'w{i}' for i in range(n_words)]
        n_maps = max(1, stack)
        maps = torch.rand((n_maps, N_PROMPT_WORDS + 2) + grid, generator=g, device='cuda')
        regions = torch.zeros((n_regions,) + out_hw, dtype=torch.bool)
        for r in range(n_regions):
            if kind == 'far':                              # small squares in the top-left corner
                regions[r, 4 * r:4 * r + 12, 4 * r:4 * r + 12] = True
                continue
            y0, x0 = int(torch.randint(0, h - 8, (1,), generator=gc)), int(torch.randint(0, w - 8, (1,), generator=gc))
            y1 = int(torch.randint(y0 + 8, h + 1, (1,), generator=gc))
            x1 = int(torch.randint(x0 + 8, w + 1, (1,), generator=gc))
            regions[r, y0:y1, x0:x1] = True
        regions = regions.cuda()
        if kind == 'time':
            target = TimeHeatMaps(tok, prompt, maps)
        elif kind == 'layer':
            target = LayerHeatMaps(tok, prompt, maps, range(stack), [f'layer{i}' for i in range(stack)], [1] * stack)
        else:
            target = GlobalHeatMap(tok, prompt, maps[0])
        singles = [target[i] for i in range(n_maps)] if stack else [target]
        tol = [float(math.ceil(0.008 * math.hypot(h, w)))]
        tol2 = np.array(tol) ** 2

        if kind == 'far':
            masks = torch.zeros((n_words,) + out_hw, dtype=torch.bool)
            masks[:, h // 2:, w // 2:] = torch.rand((n_words, h - h // 2, w - w // 2), generator=gc) < 0.3
            masks = masks.cuda()
            fused = lambda: boundary_scores(masks, regions, to_cpu=False)
            host_masks = lambda i: masks.cpu().numpy()
        elif kind == 'refine':
            img = torch.randint(0, 256, out_hw + (3,), dtype=torch.uint8, generator=gc)
            _, refined = target.refine_words(words, img, threshold=0.4, to_cpu=False)
            fused = lambda: boundary_scores(refined > 0, regions, to_cpu=False)
            host_masks = lambda i: (refined > 0).cpu().numpy()
        else:
            fused = lambda: target.region_boundary(words, image, regions, THRESHOLD, to_cpu=False)[1]
            host_masks = lambda i: singles[i].expand_words(words, image, threshold=THRESHOLD, to_cpu=True)[1].numpy() > 0

        # same answer before timing: every plane of one map, the first two maps of a stack
        b = fused()
        reg_np = regions.cpu().numpy()
        for i in range(min(n_maps, 2)):
            bi = b.map(i) if stack else b
            got = dict(word_boundary=bi.word_boundary.cpu().numpy(), region_boundary=bi.region_boundary.cpu().numpy(),
                       word_hits=bi.word_hits.permute(2, 0, 1).cpu().numpy(),
                       region_hits=bi.region_hits.permute(2, 0, 1).cpu().numpy(),
                       max_d2=bi.max_d2.permute(1, 0, 2).cpu().numpy(), sum_dist=bi.sum_dist.permute(1, 0, 2).cpu().numpy())
            ref, _ = scipy_scores(host_masks(i), reg_np, tol2)
            check(got, ref, (workload, i))
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        # the baseline, timed on a few regions, planes and pairs and scaled to all of them
        t0 = time.perf_counter()
        m0 = host_masks(0)                                  # one map's masks and copy, for every map
        copy_s = (time.perf_counter() - t0) * n_maps
        _, (reg_s, plane_s, _) = scipy_scores(m0[:TIMED_PLANES], reg_np[:TIMED_REGIONS], tol2)
        _, (_, _, pair_s) = scipy_scores(m0[:1], reg_np[:TIMED_PAIRS], tol2)
        n_planes, n_pairs = n_maps * n_words, n_maps * n_words * n_regions
        scipy_us = (copy_s + reg_s / TIMED_REGIONS * n_regions + plane_s / TIMED_PLANES * n_planes
                    + pair_s / TIMED_PAIRS * n_pairs) * 1e6

        size = max(1, args.steps // max(1, n_maps // 5))
        for _ in range(max(1, args.warmup)):
            fused()
        torch.cuda.synchronize()
        a = [block_us(fused, size, 5.0 + 0.5 * size * n_maps * n_words) for _ in range(args.rounds)]
        fused_us = med(a)
        bench.emit({'workload': workload, 'image': f'{h}x{w}', 'grid': list(grid), 'words': n_words,
                    'regions': n_regions, 'maps': n_maps, 'tolerance_px': tol[0], 'fused_us': round(fused_us, 1),
                    'scipy_us': round(scipy_us), 'scipy_scaled': True,
                    'speedup_vs_scipy': round(scipy_us / fused_us, 1), 'fused_launches': launches,
                    'timing': f'median of {args.rounds} rounds of {size} calls', 'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
