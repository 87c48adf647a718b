#!/usr/bin/env python
"""Benchmark of threshold-free ranking scores on one GPU: ``GlobalHeatMap.region_ranking`` /
``GlobalHeatMapStack.region_ranking`` (``daam_region_ranking``: region masks, then per round of planes the values, a
four-pass radix sort and the tie-group counts) against what a user writes today:

* torch on the device: ``expand_words(..., to_cpu=False)``, then per (map, word) plane a descending ``torch.sort``,
  the region bits gathered in that order, ``cumsum`` per region and the tie-group sums of u2 and ap;
* sklearn on the host (when importable): ``roc_auc_score`` and ``average_precision_score`` per (map, word, region)
  pair on the copied ``expand_words`` values. It takes seconds, so it is timed on a few pairs and scaled to all of them
  (``sklearn_pairs_timed``), plus one ``expand_words`` and copy per map (timed on one map).

    python bench_region_ranking.py [--steps K] [--warmup W] [--rounds R]

Workloads: SD-2.1 at 512x512 with 8 and 24 words against 4 and 16 regions; SDXL at 1024x1024 with 8 and 24 words and
4 regions; SDXL at 1216x832 with 8 words and 4 regions (grids as the tracer makes them: 64x64, 128x128, 76x52); a
50-step history and 15 layer maps at 512x512 with 8 words and 4 regions. Regions are random binary masks, maps uniform
random rows.

Timing: warm-up, then blocks of K calls queued behind a spin kernel and timed with CUDA events; the fused call and the
torch loop alternate, R rounds each, and the median is reported. The fused u2 is checked equal to the torch loop's
before timing, and its ap within 1e-12. The card name and power limit are read in the same run. One JSON line per
workload goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import os
import sys
import time
from types import SimpleNamespace

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench_aspect import card           # noqa: E402

# name, grid, image (h, w), words, regions, maps (0: one global map), stack kind
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 4, 0, None), ('sd21', (64, 64), (512, 512), 8, 16, 0, None),
             ('sd21', (64, 64), (512, 512), 24, 4, 0, None), ('sd21', (64, 64), (512, 512), 24, 16, 0, None),
             ('sdxl', (128, 128), (1024, 1024), 8, 4, 0, None), ('sdxl', (128, 128), (1024, 1024), 24, 4, 0, None),
             ('sdxl', (76, 52), (1216, 832), 8, 4, 0, None),
             ('sd21-history', (64, 64), (512, 512), 8, 4, 50, 'time'),
             ('sd21-layers', (64, 64), (512, 512), 8, 4, 15, 'layer')]
N_PROMPT_WORDS = 30
SKLEARN_PAIRS = 4


def torch_plane(v, inside):
    """u2 int64 [R] and ap float64 [R] of one plane ``v`` [n] against ``inside`` bool [R, n], in torch on the device."""
    n = v.numel()
    s, order = torch.sort(v, descending=True)
    ends = torch.ones(n, dtype=torch.bool, device=v.device)
    ends[:-1] = s[1:] != s[:-1]
    tp_le = inside[:, order].cumsum(1)[:, ends]                       # positives at or above each group's end
    pos_le = torch.arange(1, n + 1, device=v.device)[ends]
    fp_le = pos_le - tp_le
    tp = torch.diff(tp_le, dim=1, prepend=torch.zeros_like(tp_le[:, :1]))
    fp = torch.diff(fp_le, dim=1, prepend=torch.zeros_like(fp_le[:, :1]))
    n_p = tp_le[:, -1:]
    u2 = (tp * (2 * (n - n_p - fp_le) + fp)).sum(1)
    ap = (tp.double() / n_p * tp_le.double() / pos_le).sum(1)
    return u2, ap


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, TimeHeatMaps
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    try:
        from sklearn.metrics import average_precision_score, roc_auc_score
    except ImportError:
        roc_auc_score = None
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
    for workload, grid, hw, n_words, n_regions, stack, kind in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1])
        out_hw = (hw[1], hw[0]) if grid[0] == grid[1] else hw
        words = [f'w{i}' for i in range(n_words)]
        n_rows = N_PROMPT_WORDS + 2
        regions = torch.rand((n_regions,) + out_hw, generator=g, device='cuda') < 0.3
        inside = regions.flatten(1)
        n_maps = max(1, stack)
        maps = torch.rand((n_maps, n_rows) + grid, generator=g, device='cuda')
        if kind == 'time':
            target = TimeHeatMaps(tok, prompt, maps)
        elif kind == 'layer':
            target = LayerHeatMaps(tok, prompt, maps, range(stack), [f'layer{i}' for i in range(stack)], [1] * stack)
        else:
            target = GlobalHeatMap(tok, prompt, maps[0])
        singles = [target[i] for i in range(n_maps)] if stack else [target]

        fused = lambda: target.region_ranking(words, image, regions, to_cpu=False)

        def loop():
            out = []
            for ghm in singles:
                _, m = ghm.expand_words(words, image, to_cpu=False)
                out.append([torch_plane(m[w].flatten(), inside) for w in range(n_words)])
            return out

        # same answer before timing
        _, rk = fused()
        u2 = rk.u2.reshape(n_maps, n_regions, n_words)
        apf = rk.ap.reshape(n_maps, n_regions, n_words)
        for i, planes in enumerate(loop()):
            for w, (tu2, tap) in enumerate(planes):
                assert torch.equal(u2[i, :, w], tu2), (workload, i, w)
                assert torch.allclose(apf[i, :, w], tap, rtol=1e-12, atol=0), (workload, i, w)
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        size = max(1, args.steps // max(1, n_maps // 5))
        loop_size = max(1, size // 4)
        for _ in range(max(1, args.warmup)):
            fused(); loop()
        torch.cuda.synchronize()
        a, b = [], []
        for _ in range(args.rounds):                     # alternated rounds
            a.append(block_us(fused, size, 5.0 + 0.5 * size * n_maps * n_words))
            b.append(block_us(loop, loop_size, 5.0 + 1.0 * loop_size * n_maps * n_words))
        fused_us, torch_us = med(a), med(b)
        row = {'workload': workload, 'image': f'{out_hw[0]}x{out_hw[1]}', 'grid': list(grid), 'words': n_words,
               'regions': n_regions, 'maps': n_maps, 'fused_us': round(fused_us, 1), 'torch_loop_us': round(torch_us, 1),
               'speedup_vs_torch': round(torch_us / fused_us, 2), 'fused_launches': launches}
        if roc_auc_score is not None:
            t0 = time.perf_counter()                      # one map's expand_words and copy, for every map
            m0 = singles[0].expand_words(words, image, to_cpu=True)[1].flatten(1).double().numpy()
            copy_s = (time.perf_counter() - t0) * n_maps
            labels = inside.cpu().numpy()
            pairs = [(i, w, r) for i in range(n_maps) for w in range(n_words) for r in range(n_regions)]
            t0 = time.perf_counter()
            for i, w, r in pairs[:SKLEARN_PAIRS]:
                roc_auc_score(labels[r], m0[w])           # map 0's values stand in for map i's
                average_precision_score(labels[r], m0[w])
            per_pair = (time.perf_counter() - t0) / min(SKLEARN_PAIRS, len(pairs))
            row['sklearn_us'] = round((copy_s + per_pair * len(pairs)) * 1e6)
            row['speedup_vs_sklearn'] = round(row['sklearn_us'] / fused_us, 1)
            row['sklearn_pairs_timed'] = min(SKLEARN_PAIRS, len(pairs))
        row.update({'timing': f'median of {args.rounds} alternated rounds of {size} calls ({loop_size} loops)',
                    'device': name, 'power_limit': power})
        bench.emit(row)


if __name__ == '__main__':
    main()
