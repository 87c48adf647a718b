#!/usr/bin/env python
"""Benchmark of word instances on one GPU: ``GlobalHeatMap.word_instances`` / ``GlobalHeatMapStack.word_instances``
(``daam_word_instances``, ``to_cpu=True``) against what a user does without it: ``expand_words(threshold=t)``, the
``[n_words, H, W]`` masks copied to the host, then per (map, word) plane ``scipy.ndimage.label`` (8-connected),
``find_objects`` and per-label area and index sums, the largest K kept. Both forms end with the results on the host,
so each is timed call to result.

    python bench_word_instances.py [--rounds R]

Workloads (threshold 0.4, K = 16, grids as the tracer makes them): SD-2.1 at 512x512 with 8 words; SDXL at 1024x1024
with 8 and 24 words; SDXL at 1216x832 with 8 words; a 50-step history at 512x512 with 8 words; a 15-map layer stack
at 512x512 with 8 words. Maps are uniform random rows, whose upsampled word maps make many blobs.

Both forms run once and are checked equal (count, area, box, index sums) before timing. Then the forms alternate, R
rounds each, each round one call timed with a host clock after a device synchronise, and the median is reported. The
card name and power limit are read in the same run. One JSON line per workload goes to stdout; nothing is written
anywhere.
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

# name, grid, image (h, w), words, maps (0: one global map)
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 0), ('sdxl', (64, 64), (1024, 1024), 8, 0),
             ('sdxl', (64, 64), (1024, 1024), 24, 0), ('sdxl', (76, 52), (1216, 832), 8, 0),
             ('sd21-history', (64, 64), (512, 512), 8, 50), ('sd21-layers', (64, 64), (512, 512), 8, 15)]
THRESHOLD = 0.4
K = 16
N_PROMPT_WORDS = 30


def host_instances(masks: np.ndarray, k: int):
    """The host form's per-plane work on ``masks`` ``[planes, H, W]``: ``(count, area, box, sum_yx)`` of the k
    largest 8-connected components (ties to the first pixel in raster order), zero-padded."""
    from scipy import ndimage
    planes, h, w = masks.shape
    count = np.zeros(planes, np.int64)
    area = np.zeros((planes, k), np.int64)
    box = np.zeros((planes, k, 4), np.int64)
    sums = np.zeros((planes, k, 2), np.int64)
    yy, xx = np.indices((h, w))
    for i, m in enumerate(masks):
        lab, n = ndimage.label(m, structure=np.ones((3, 3)))
        count[i] = n
        if n == 0:
            continue
        flat = lab.ravel()
        a = np.bincount(flat, minlength=n + 1)[1:]
        sy = np.bincount(flat, weights=yy.ravel(), minlength=n + 1)[1:]
        sx = np.bincount(flat, weights=xx.ravel(), minlength=n + 1)[1:]
        keep = np.argsort(-a, kind='stable')[:k]              # labels in raster order: ties stay in it
        objs = ndimage.find_objects(lab)
        area[i, :len(keep)] = a[keep]
        box[i, :len(keep)] = [[objs[j][0].start, objs[j][1].start, objs[j][0].stop, objs[j][1].stop] for j in keep]
        sums[i, :len(keep)] = np.stack([sy[keep], sx[keep]], 1).round().astype(np.int64)
    return count, area, box, sums


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    torch.cuda.set_device(0)
    _native.load()
    name, power = card()

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    med = lambda v: sorted(v)[len(v) // 2]
    tok = WhitespaceTokenizer()
    prompt = ' '.join(f'w{i}' for i in range(N_PROMPT_WORDS))
    g = torch.Generator(device='cuda').manual_seed(0)
    for workload, grid, hw, n_words, n_maps in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        words = [f'w{i}' for i in range(n_words)]
        n_rows = N_PROMPT_WORDS + 2
        if n_maps:
            stack = GlobalHeatMapStack(tok, prompt, torch.rand((n_maps, n_rows) + grid, generator=g, device='cuda'))
            maps = [stack[t] for t in range(n_maps)]
            fused = lambda: stack.word_instances(words, image, THRESHOLD, max_instances=K)[1]
        else:
            maps = [GlobalHeatMap(tok, prompt, torch.rand((n_rows,) + grid, generator=g, device='cuda'))]
            fused = lambda: maps[0].word_instances(words, image, THRESHOLD, max_instances=K)[1]

        def host_form():
            out = []
            for ghm in maps:
                m = ghm.expand_words(words, image, threshold=THRESHOLD)[1]       # a CPU [n_words, H, W] stack
                out.append(host_instances(m.numpy() > 0, K))
            return [np.concatenate(f) for f in zip(*out)]

        # same answer before timing
        inst = fused()
        count, area, box, sums = host_form()
        got = [inst.count.reshape(-1), inst.area.reshape(-1, K), inst.box.reshape(-1, K, 4), inst.sum_yx.reshape(-1, K, 2)]
        for a, b, f in zip(got, (count, area, box, sums), ('count', 'area', 'box', 'sum_yx')):
            assert np.array_equal(a.numpy(), b), (workload, f)
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before
        for _ in range(2):
            fused()
        a, b = [], []
        for _ in range(args.rounds):                     # alternated rounds
            a.append(timed(fused)[0])
            b.append(timed(host_form)[0])
        fused_ms, host_ms = med(a), med(b)
        planes = max(1, n_maps) * n_words
        bench.emit({'workload': workload, 'image': f'{hw[0]}x{hw[1]}', 'grid': list(grid), 'words': n_words,
                    'maps': max(1, n_maps), 'planes': planes, 'components_median': int(np.median(count)),
                    'fused_ms': round(fused_ms, 3), 'host_ms': round(host_ms, 2),
                    'speedup': round(host_ms / fused_ms, 1), 'fused_launches': launches,
                    'timing': f'median of {args.rounds} alternated rounds, one call each, host clock after a sync',
                    'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
