#!/usr/bin/env python
"""Benchmark of heat-map overlays on one GPU: ``GlobalHeatMap.overlay_words`` (``daam_overlay_words``, two launches)
against the torch composition it replaces, ``expand_words(to_cpu=False)`` + jet table gather + alpha blend + round +
cast to uint8.

    python bench_overlay.py [--steps K] [--warmup W] [--rounds R]

Workloads: SD-2.1 at 512x512 and 768x768 with 8 words; SDXL at 1024x1024 with 8 and 24 words; SDXL at 1216x832 with
8 words (grids as the tracer makes them: 64x64, 96x96, 64x64, 76x52); and a 50-step history at 512x512 with 8 words,
``TimeHeatMaps.overlay_words`` in one call against the per-step loop of the composition. Colour normalisation on, no
threshold; the image is a device tensor, so neither form copies it.

Timing as in ``bench_segment.py``: warm-up, then blocks of K calls queued behind a spin kernel and timed with CUDA
events; the two forms alternate, R rounds each, and the median is reported. Bytes are algorithmic: the word's rows
read, the word maps written (and, fused, read back), the image read once per map, then per word and output pixel the
fused call writes 3 bytes, while the composition writes and reads the ``[n_words, H, W]`` fp32 stack and writes the
3-byte frames. The card name and power limit are read in the same run. One JSON line per workload goes to stdout;
nothing is written anywhere.
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

# name, grid, image (h, w), words, steps (0: one global map)
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 0), ('sd21', (96, 96), (768, 768), 8, 0),
             ('sdxl', (64, 64), (1024, 1024), 8, 0), ('sdxl', (64, 64), (1024, 1024), 24, 0),
             ('sdxl', (76, 52), (1216, 832), 8, 0), ('sd21-history', (64, 64), (512, 512), 8, 50)]
N_PROMPT_WORDS = 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.heatmap import GlobalHeatMap, TimeHeatMaps, jet_colormap
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    torch.cuda.set_device(0)
    _native.load()
    name, power = card()
    stream = torch.cuda.current_stream()
    table = jet_colormap().cuda()

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

    def compare(fused, composed, size, spin_ms):
        for _ in range(max(3, args.warmup)):
            fused()
            composed()
        torch.cuda.synchronize()
        a, b = [], []
        for _ in range(args.rounds):                     # alternated rounds
            a.append(block_us(fused, size, spin_ms))
            b.append(block_us(composed, size, spin_ms))
        med = lambda v: sorted(v)[len(v) // 2]
        return med(a), med(b)

    def compose(m, image):
        """The overlay of ``m`` ``[n_words, H, W]`` over ``image`` in torch: autoscaled jet colour, alpha blend."""
        lo, hi = m.amin((-2, -1), keepdim=True), m.amax((-2, -1), keepdim=True)
        c = torch.where(hi == lo, torch.zeros_like(m), (m - lo) / (hi - lo))
        k = (c * 256.0).to(torch.int64).clamp(max=255)
        a = m.clamp(0, 1).unsqueeze(-1)
        return ((1 - a) * image.float() + a * table[k]).round().clamp(0, 255).to(torch.uint8)

    tok = WhitespaceTokenizer()
    prompt = ' '.join(f'w{i}' for i in range(N_PROMPT_WORDS))
    g = torch.Generator(device='cuda').manual_seed(0)
    for workload, grid, hw, n_words, steps in WORKLOADS:
        size_ns = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        image = torch.randint(0, 256, hw + (3,), generator=g, device='cuda', dtype=torch.uint8)
        words = [f'w{i}' for i in range(n_words)]
        n_rows = N_PROMPT_WORDS + 2
        if steps:
            tm = TimeHeatMaps(tok, prompt, torch.rand((steps, n_rows) + grid, generator=g, device='cuda'))
            maps = [tm[t] for t in range(steps)]
            fused = lambda: tm.overlay_words(words, image, to_cpu=False)
        else:
            maps = [GlobalHeatMap(tok, prompt, torch.rand((n_rows,) + grid, generator=g, device='cuda'))]
            fused = lambda: maps[0].overlay_words(words, image, to_cpu=False)

        def composed():
            for ghm in maps:
                compose(ghm.expand_words(words, size_ns, to_cpu=False)[1], image)

        # same answer before timing
        frames = fused()[1]
        want = compose(maps[-1].expand_words(words, size_ns, to_cpu=False)[1], image)
        assert torch.equal(frames.reshape((-1, n_words) + hw + (3,))[-1], want)
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        size = max(1, args.steps // max(1, steps // 10)) if steps else args.steps
        n_maps = max(1, steps)
        fused_us, composed_us = compare(fused, composed, size, 5.0 + 0.6 * size * n_maps)
        px, xx = hw[0] * hw[1], grid[0] * grid[1]
        rows_read = n_maps * n_words * xx * 4
        fused_bytes = rows_read + 2 * n_maps * n_words * xx * 4 + n_maps * px * 3 + n_maps * n_words * px * 3
        composed_bytes = rows_read + n_maps * n_words * xx * 4 + n_maps * (px * 3 + n_words * px * (2 * 4 + 3))
        bench.emit({'workload': workload, 'image': f'{hw[0]}x{hw[1]}', 'grid': list(grid), 'words': n_words,
                    'maps': n_maps, 'overlay_us': round(fused_us, 2), 'composition_us': round(composed_us, 2),
                    'speedup': round(composed_us / fused_us, 2), 'overlay_launches': launches,
                    'overlay_bytes': fused_bytes, 'composition_bytes': composed_bytes,
                    'overlay_tbps': round(fused_bytes / fused_us / 1e6, 3),
                    'timing': f'median of {args.rounds} alternated rounds of {size} calls',
                    'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
