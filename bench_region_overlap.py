#!/usr/bin/env python
"""Benchmark of word-region overlap on one GPU: ``GlobalHeatMap.region_overlap`` / ``TimeHeatMaps.region_overlap``
(``daam_region_overlap``, three launches) against (a) ``expand_words(to_cpu=False)`` plus one ``einsum`` per map and
(b) the reference's evaluation pattern, ``expand_words`` then ``compute_iou`` for every (word, region) pair.

    python bench_region_overlap.py [--steps K] [--warmup W] [--rounds R]

Workloads: SD-2.1 at 512x512 and SDXL at 1024x1024 with 8 and 24 words and 4 and 16 regions; SDXL at 1216x832 with 8
words and 4 regions (grids as the tracer makes them: 64x64, 64x64, 76x52); and a 50-step history at 512x512 with 8 words
and 4 regions, in one call against the per-step loops. Threshold 0.4 throughout; regions are random binary masks.

Timing as in ``bench_segment.py``: warm-up, then blocks of K calls queued behind a spin kernel and timed with CUDA
events; the forms alternate, R rounds each, and the median is reported. Form (b) syncs on every pair (``.item()``), so
it is timed one call per block without the spin. The fused and einsum results are checked to be equal before timing.
The card name and power limit are read in the same run. One JSON line per workload goes to stdout; nothing is written
anywhere.
"""
from __future__ import annotations

import argparse
import os
import sys
from types import SimpleNamespace

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench_aspect import card           # noqa: E402

# name, grid, image (h, w), words, regions, steps (0: one global map)
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 4, 0), ('sd21', (64, 64), (512, 512), 8, 16, 0),
             ('sd21', (64, 64), (512, 512), 24, 4, 0), ('sd21', (64, 64), (512, 512), 24, 16, 0),
             ('sdxl', (64, 64), (1024, 1024), 8, 4, 0), ('sdxl', (64, 64), (1024, 1024), 8, 16, 0),
             ('sdxl', (64, 64), (1024, 1024), 24, 4, 0), ('sdxl', (64, 64), (1024, 1024), 24, 16, 0),
             ('sdxl', (76, 52), (1216, 832), 8, 4, 0), ('sd21-history', (64, 64), (512, 512), 8, 4, 50)]
THRESHOLD = 0.4
N_PROMPT_WORDS = 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.evaluate import compute_iou
    from daam_b200.heatmap import GlobalHeatMap, TimeHeatMaps
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    torch.cuda.set_device(0)
    _native.load()
    name, power = card()
    stream = torch.cuda.current_stream()

    def block_us(fn, size, spin_ms):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if spin_ms:
            torch.cuda._sleep(int(spin_ms * 1.9e6))      # the host queues the whole block while the GPU spins
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
    for workload, grid, hw, n_words, n_regions, steps in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        words = [f'w{i}' for i in range(n_words)]
        n_rows = N_PROMPT_WORDS + 2
        regions = torch.rand((n_regions,) + hw, generator=g, device='cuda') < 0.3
        region_f = regions.float()
        if steps:
            tm = TimeHeatMaps(tok, prompt, torch.rand((steps, n_rows) + grid, generator=g, device='cuda'))
            maps = [tm[t] for t in range(steps)]
            fused = lambda: tm.region_overlap(words, image, regions, threshold=THRESHOLD, to_cpu=False)
        else:
            maps = [GlobalHeatMap(tok, prompt, torch.rand((n_rows,) + grid, generator=g, device='cuda'))]
            fused = lambda: maps[0].region_overlap(words, image, regions, threshold=THRESHOLD, to_cpu=False)

        def einsum_form():
            out = []
            for ghm in maps:
                m = ghm.expand_words(words, image, threshold=THRESHOLD, to_cpu=False)[1]
                out.append((torch.einsum('nhw,rhw->rn', m, region_f), m.sum((-1, -2))))
            return out

        def pair_form():
            for ghm in maps:
                m = ghm.expand_words(words, image, threshold=THRESHOLD, to_cpu=False)[1]
                for w in range(n_words):
                    for r in range(n_regions):
                        compute_iou(m[w], region_f[r])

        # same answer before timing
        _, ov = fused()
        ref = einsum_form()
        inter = ov.intersection.reshape(-1, n_regions, n_words)
        area = ov.word_area.reshape(-1, n_words)
        for t, (i_ref, a_ref) in enumerate(ref):
            assert torch.equal(inter[t], i_ref) and torch.equal(area[t], a_ref), (workload, t)
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        n_maps = max(1, steps)
        size = max(1, args.steps // max(1, steps // 10)) if steps else args.steps
        spin = 5.0 + 0.4 * size * n_maps
        for _ in range(max(3, args.warmup)):
            fused(); einsum_form()
        pair_form()
        torch.cuda.synchronize()
        a, b, c = [], [], []
        for _ in range(args.rounds):                     # alternated rounds
            a.append(block_us(fused, size, spin))
            b.append(block_us(einsum_form, size, spin))
            c.append(block_us(pair_form, 1, 0))
        fused_us, einsum_us, pair_us = med(a), med(b), med(c)
        bench.emit({'workload': workload, 'image': f'{hw[0]}x{hw[1]}', 'grid': list(grid), 'words': n_words,
                    'regions': n_regions, 'maps': n_maps, 'fused_us': round(fused_us, 2),
                    'einsum_us': round(einsum_us, 2), 'pairs_us': round(pair_us, 1),
                    'speedup_vs_einsum': round(einsum_us / fused_us, 2), 'speedup_vs_pairs': round(pair_us / fused_us, 1),
                    'fused_launches': launches,
                    'timing': f'median of {args.rounds} alternated rounds of {size} calls (pairs: 1 call)',
                    'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
