#!/usr/bin/env python
"""Benchmark of word distance maps on one GPU: ``GlobalHeatMap.word_distance`` / ``GlobalHeatMapStack.word_distance``
(``daam_word_distance``: per round of planes the word maps, the values, the column pass and the row pass) and
``evaluate.distance_transform`` (``daam_mask_distance``: the column and row passes) against what a user writes today:
``expand_words(..., threshold, to_cpu=False)`` copied to the host, then scipy's ``distance_transform_edt`` twice per
(map, word) plane, once to the mask and once to its outside. scipy takes tens of milliseconds a plane, so it is timed
on a few planes and scaled to all of them (``scipy_scaled``: true).

    python bench_word_distance.py [--steps K] [--warmup W] [--rounds R]

Workloads: SD-2.1 at 512x512 with 8 and 24 words; SDXL at 1024x1024 with 8 and 24 words; SDXL at 1216x832 with 8
words (grids as the tracer makes them: 64x64, 128x128, 76x52); a 50-step history and 15 layer maps at 512x512 with 8
words; ``distance_transform`` of 8 random-blob masks at 1024x1024, and the far-apart case: 8 one-pixel masks in the
top-left corner at 1024x1024, whose distances reach the far corner (a search that grows with the distance would be
slowest here). Maps are uniform random rows, the threshold 0.5.

Timing: warm-up, then blocks of K calls queued behind a spin kernel and timed with CUDA events, R rounds, median. Every
fused result is checked equal to the scipy result (``rint`` of the squared float distances, signed by the class)
before timing: every plane of one map, the first two maps of a stack. The card name and power limit are read in the
same run. One JSON line per workload goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
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

# name, grid, image (h, w), words, maps (0: one global map), kind
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 0, None), ('sd21', (64, 64), (512, 512), 24, 0, None),
             ('sdxl', (128, 128), (1024, 1024), 8, 0, None), ('sdxl', (128, 128), (1024, 1024), 24, 0, None),
             ('sdxl', (76, 52), (1216, 832), 8, 0, None),
             ('sd21-history', (64, 64), (512, 512), 8, 50, 'time'),
             ('sd21-layers', (64, 64), (512, 512), 8, 15, 'layer'),
             ('masks-random', (128, 128), (1024, 1024), 8, 0, 'random'),
             ('far-apart', (128, 128), (1024, 1024), 8, 0, 'far')]
N_PROMPT_WORDS = 30
THRESHOLD = 0.5
TIMED_PLANES = 2


def scipy_signed_d2(planes):
    """What a user writes today, on host masks ``planes`` [P, H, W] (each neither empty nor full): two Euclidean
    distance transforms per plane, the squared distances rounded to integers and signed by the class. Returns the int64
    result and the seconds spent."""
    from scipy import ndimage
    t0 = time.perf_counter()
    out = []
    for m in planes:
        d_out = ndimage.distance_transform_edt(~m)          # outside: distance to the mask
        d_in = ndimage.distance_transform_edt(m)            # inside: distance to the outside
        out.append(np.where(m, -np.rint(d_in * d_in), np.rint(d_out * d_out)).astype(np.int64))
    return np.stack(out), time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.evaluate import distance_transform
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
    for workload, grid, hw, n_words, stack, kind in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        h, w = out_hw = (hw[1], hw[0]) if grid[0] == grid[1] else hw
        words = [f'w{i}' for i in range(n_words)]
        n_maps = max(1, stack)
        maps = torch.rand((n_maps, N_PROMPT_WORDS + 2) + grid, generator=g, device='cuda')
        if kind == 'time':
            target = TimeHeatMaps(tok, prompt, maps)
        elif kind == 'layer':
            target = LayerHeatMaps(tok, prompt, maps, range(stack), [f'layer{i}' for i in range(stack)], [1] * stack)
        else:
            target = GlobalHeatMap(tok, prompt, maps[0])
        singles = [target[i] for i in range(n_maps)] if stack else [target]

        if kind in ('random', 'far'):
            if kind == 'far':
                masks = torch.zeros((n_words,) + out_hw, dtype=torch.bool)
                masks[:, 0, 0] = True
            else:
                coarse = torch.rand(n_words, 1, h // 32, w // 32, generator=gc)
                masks = torch.nn.functional.interpolate(coarse, size=out_hw, mode='bilinear')[:, 0] > 0.6
            masks = masks.cuda()
            fused = lambda: distance_transform(masks, to_cpu=False)
            host_masks = lambda i: masks.cpu().numpy()
        else:
            fused = lambda: target.word_distance(words, image, THRESHOLD, to_cpu=False)[1]
            host_masks = lambda i: singles[i].expand_words(words, image, threshold=THRESHOLD,
                                                           to_cpu=False)[1].cpu().numpy() > 0

        # same answer before timing: every plane of one map, the first two maps of a stack
        wd = fused()
        for i in range(min(n_maps, 2)):
            got = (wd.map(i) if stack else wd).signed_d2.cpu().numpy()
            ref, _ = scipy_signed_d2(host_masks(i))
            assert np.array_equal(got, ref), (workload, i)
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        # the baseline, timed on a few planes and scaled to all of them
        t0 = time.perf_counter()
        m0 = host_masks(0)                                  # one map's masks and copy, for every map
        copy_s = (time.perf_counter() - t0) * n_maps
        _, plane_s = scipy_signed_d2(m0[:TIMED_PLANES])
        n_planes = n_maps * n_words
        scipy_us = (copy_s + plane_s / TIMED_PLANES * n_planes) * 1e6

        size = max(1, args.steps // max(1, n_maps // 5))
        for _ in range(max(1, args.warmup)):
            fused()
        torch.cuda.synchronize()
        a = [block_us(fused, size, 5.0 + 0.2 * size * n_planes) for _ in range(args.rounds)]
        fused_us = med(a)
        bench.emit({'workload': workload, 'image': f'{h}x{w}', 'grid': list(grid), 'words': n_words,
                    'maps': n_maps, 'fused_us': round(fused_us, 1), 'fused_us_per_plane': round(fused_us / n_planes, 2),
                    'scipy_us': round(scipy_us), 'scipy_scaled': True,
                    'speedup_vs_scipy': round(scipy_us / fused_us, 1), 'fused_launches': launches,
                    'timing': f'median of {args.rounds} rounds of {size} calls', 'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
