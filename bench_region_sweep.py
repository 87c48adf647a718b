#!/usr/bin/env python
"""Benchmark of threshold sweeps of word-region overlap on one GPU: ``GlobalHeatMap.region_sweep`` /
``TimeHeatMaps.region_sweep`` (``daam_region_sweep``, one memset and three launches) against a loop of T
``region_overlap(threshold=t, to_cpu=False)`` calls, and one ``region_overlap`` call for scale.

    python bench_region_sweep.py [--steps K] [--warmup W] [--rounds R]

Workloads: those of ``bench_region_overlap.py`` -- SD-2.1 at 512x512 and SDXL at 1024x1024 with 8 and 24 words and 4
and 16 regions; SDXL at 1216x832 with 8 words and 4 regions (grids as the tracer makes them: 64x64, 64x64, 76x52); and
a 50-step history at 512x512 with 8 words and 4 regions -- each at T = 19 thresholds (0.05, 0.10, ..., 0.95) and at
T = 64 (0.01 ... 0.955 in equal steps). Regions are random binary masks, maps uniform random rows.

Timing as in ``bench_region_overlap.py``: warm-up, then blocks of K calls queued behind a spin kernel and timed with
CUDA events; the forms alternate, R rounds each, and the median is reported. Every slice of the sweep is checked equal
to the loop's call at its threshold before timing. The card name and power limit are read in the same run. One JSON
line per workload goes to stdout; nothing is written anywhere.
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
SWEEPS = {19: [round(0.05 * i, 2) for i in range(1, 20)], 64: [0.01 + 0.945 * i / 63 for i in range(64)]}
N_PROMPT_WORDS = 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=5)
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
    for workload, grid, hw, n_words, n_regions, steps in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        words = [f'w{i}' for i in range(n_words)]
        n_rows = N_PROMPT_WORDS + 2
        regions = torch.rand((n_regions,) + hw, generator=g, device='cuda') < 0.3
        if steps:
            target = TimeHeatMaps(tok, prompt, torch.rand((steps, n_rows) + grid, generator=g, device='cuda'))
        else:
            target = GlobalHeatMap(tok, prompt, torch.rand((n_rows,) + grid, generator=g, device='cuda'))
        n_maps = max(1, steps)
        for n_thr, taus in SWEEPS.items():
            sweep = lambda: target.region_sweep(words, image, regions, taus, to_cpu=False)
            loop = lambda: [target.region_overlap(words, image, regions, threshold=t, to_cpu=False) for t in taus]
            one = lambda: target.region_overlap(words, image, regions, threshold=taus[n_thr // 2], to_cpu=False)

            # same answer before timing
            _, ov = sweep()
            for k, (_, ref) in enumerate(loop()):
                assert torch.equal(ov.intersection[..., k, :, :], ref.intersection), (workload, n_thr, k)
                assert torch.equal(ov.word_area[..., k, :], ref.word_area), (workload, n_thr, k)
            before = _native.launch_count()
            sweep()
            launches = _native.launch_count() - before

            size = max(1, args.steps // max(1, steps // 10)) if steps else args.steps
            loop_size = max(1, size // 8)
            for _ in range(max(3, args.warmup)):
                sweep(); loop(); one()
            torch.cuda.synchronize()
            a, b, c = [], [], []
            for _ in range(args.rounds):                 # alternated rounds
                a.append(block_us(sweep, size, 5.0 + 0.4 * size * n_maps))
                b.append(block_us(loop, loop_size, 5.0 + 0.4 * loop_size * n_maps * n_thr))
                c.append(block_us(one, size, 5.0 + 0.4 * size * n_maps))
            sweep_us, loop_us, one_us = med(a), med(b), med(c)
            bench.emit({'workload': workload, 'image': f'{hw[0]}x{hw[1]}', 'grid': list(grid), 'words': n_words,
                        'regions': n_regions, 'maps': n_maps, 'thresholds': n_thr, 'sweep_us': round(sweep_us, 2),
                        'loop_us': round(loop_us, 2), 'one_call_us': round(one_us, 2),
                        'speedup_vs_loop': round(loop_us / sweep_us, 2), 'sweep_vs_one_call': round(sweep_us / one_us, 2),
                        'sweep_launches': launches,
                        'timing': f'median of {args.rounds} alternated rounds of {size} calls ({loop_size} loops)',
                        'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
