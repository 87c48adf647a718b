#!/usr/bin/env python
"""Benchmark of word-pair overlap on one GPU: ``GlobalHeatMap.word_overlap`` / ``relation_overlap`` and the stack forms
(``daam_word_overlap``, three launches) against the compositions a user writes without them.

    python bench_word_overlap.py [--steps K] [--warmup W] [--rounds R]

Workloads:
* ``notebook``: the DAAM paper's visuosyntactic sweep for one SD-2.1 caption (64x64 grid, 12 words, 12 dependency edges,
  ``absolute``, t = 0.15): the notebook's per-edge ``iou`` / ``ioa`` loop on the word heat maps (reproduced below)
  against one ``relation_overlap(..., to_cpu=True)``. Both end in a host sync, so each is timed one call per block.
* ``pairs``: ``word_overlap`` at 512x512, 1024x1024 and 1216x832 with 8 and 24 words, threshold 0.4 and none, against
  ``expand_words(to_cpu=False)`` then ``m.flatten(1) @ m.flatten(1).T`` in fp32 with TF32 off, plus ``m.sum``.
* ``pairs`` at the 64x64 grid (``image=None``) with 24 words, t = 0.15 and no threshold: a tile's windows of 24 words
  do not fit one staging pass, so without a threshold the kernel stages them again for each 256-pixel chunk.
* ``history`` / ``layers``: a 50-step 512x512 history with 8 words, and 60 layer maps at the 64x64 grid (``image=None``,
  12 words at the notebook's threshold, and 24 words without one), one call against the per-map composition loop.

Timing as in ``bench_region_overlap.py``: warm-up, then blocks of K calls queued behind a spin kernel and timed with
CUDA events; the forms alternate, R rounds each, and the median is reported. Results are checked equal (thresholded:
bit for bit; without: rtol 1e-4) before timing. The card name and power limit are read in the same run. One JSON line per
workload goes to stdout; nothing is written anywhere.
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

# name, grid, image (h, w) or None (the grid), words, threshold, maps (0: one global map)
WORKLOADS = [('pairs', (64, 64), (512, 512), 8, 0.4, 0), ('pairs', (64, 64), (512, 512), 8, None, 0),
             ('pairs', (64, 64), (512, 512), 24, 0.4, 0), ('pairs', (64, 64), (512, 512), 24, None, 0),
             ('pairs', (128, 128), (1024, 1024), 8, 0.4, 0), ('pairs', (128, 128), (1024, 1024), 8, None, 0),
             ('pairs', (128, 128), (1024, 1024), 24, 0.4, 0), ('pairs', (128, 128), (1024, 1024), 24, None, 0),
             ('pairs', (76, 52), (1216, 832), 8, 0.4, 0), ('pairs', (76, 52), (1216, 832), 8, None, 0),
             ('pairs', (76, 52), (1216, 832), 24, 0.4, 0), ('pairs', (76, 52), (1216, 832), 24, None, 0),
             ('pairs', (64, 64), None, 24, 0.15, 0), ('pairs', (64, 64), None, 24, None, 0),
             ('history', (64, 64), (512, 512), 8, 0.4, 50), ('layers', (64, 64), None, 12, 0.15, 60),
             ('layers', (64, 64), None, 24, None, 60)]
N_PROMPT_WORDS = 30
CAPTION = 'a large brown dog is chasing a small red ball across the green grass of a sunny park'
EDGES = [('chasing', 'dog', 'nsubj'), ('dog', 'large', 'amod'), ('dog', 'brown', 'amod'), ('chasing', 'ball', 'obj'),
         ('ball', 'small', 'amod'), ('ball', 'red', 'amod'), ('chasing', 'grass', 'obl'), ('grass', 'green', 'amod'),
         ('grass', 'park', 'nmod'), ('park', 'sunny', 'amod'), ('chasing', 'is', 'aux'), ('grass', 'across', 'case')]


def notebook_iou(a, b, t: float = 0.15) -> float:
    """notebooks/1-visuosyntactic-analyses.ipynb, cell 14."""
    i = ((a > t) & (b > t)).float().sum()
    u = ((a > t) | (b > t)).float().sum()
    if u < 1e-6:
        return 0.0
    else:
        return (i / u).item()


def notebook_ioa(a, b, t: float = 0.15) -> float:
    i = ((a > t) & (b > t)).float().sum()
    a = (a > t).float().sum()
    if a < 1e-6:
        return 0.0
    else:
        return (i / a).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, TimeHeatMaps
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    torch.cuda.set_device(0)
    torch.backends.cuda.matmul.allow_tf32 = False
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
    g = torch.Generator(device='cuda').manual_seed(0)

    # ---- the notebook's sweep for one caption ----
    n_rows = len(CAPTION.split()) + 2
    ghm = GlobalHeatMap(tok, CAPTION, torch.rand((n_rows, 64, 64), generator=g, device='cuda') * 0.4)

    def notebook_form():
        word_maps = {}
        for w in {x for h, d, _ in EDGES for x in (h, d)}:
            word_maps[w] = ghm.compute_word_heat_map(w).value
        return [(notebook_iou(word_maps[h], word_maps[d]), notebook_ioa(word_maps[d], word_maps[h]),
                 notebook_ioa(word_maps[h], word_maps[d])) for h, d, _ in EDGES]

    fused_rel = lambda: ghm.relation_overlap(EDGES, absolute=True, threshold=0.15, to_cpu=True)
    rel = fused_rel()
    got = [(float(a), float(b), float(c)) for a, b, c in zip(rel.iou, rel.iod, rel.ioh)]
    assert got == notebook_form(), 'relation_overlap differs from the notebook loop'
    for _ in range(max(3, args.warmup)):
        fused_rel(); notebook_form()
    a, b = [], []
    for _ in range(args.rounds):
        a.append(block_us(fused_rel, 1, 0))
        b.append(block_us(notebook_form, 1, 0))
    bench.emit({'workload': 'notebook', 'grid': [64, 64], 'words': len(rel.words), 'edges': len(EDGES),
                'fused_us': round(med(a), 1), 'notebook_us': round(med(b), 1),
                'speedup_vs_notebook': round(med(b) / med(a), 1),
                'timing': f'median of {args.rounds} alternated rounds of 1 call (both sync on the host)',
                'device': name, 'power_limit': power})

    # ---- word_overlap against expand_words + matmul ----
    prompt = ' '.join(f'w{i}' for i in range(N_PROMPT_WORDS))
    n_rows = N_PROMPT_WORDS + 2
    for workload, grid, hw, n_words, threshold, n_maps in WORKLOADS:
        image = SimpleNamespace(size=(hw[1], hw[0]), height=hw[0], width=hw[1]) if hw else None
        eimage = image or SimpleNamespace(size=grid[::-1], height=grid[0], width=grid[1])
        words = [f'w{i}' for i in range(n_words)]
        kw = dict(absolute=workload == 'layers', threshold=threshold)
        if n_maps:
            stack_cls = TimeHeatMaps if workload == 'history' else LayerHeatMaps
            heat = torch.rand((n_maps, n_rows) + grid, generator=g, device='cuda') * (0.4 if kw['absolute'] else 1)
            extra = {} if stack_cls is TimeHeatMaps else dict(layers=range(n_maps), names=[''] * n_maps,
                                                             factors=[1] * n_maps)
            stack = stack_cls(tok, prompt, heat, **extra)
            maps = [stack[t] for t in range(n_maps)]
            fused = lambda: stack.word_overlap(words, image, to_cpu=False, **kw)
        else:
            maps = [GlobalHeatMap(tok, prompt, torch.rand((n_rows,) + grid, generator=g, device='cuda'))]
            fused = lambda: maps[0].word_overlap(words, image, to_cpu=False, **kw)

        def matmul_form():
            out = []
            for one in maps:
                m = one.expand_words(words, eimage, to_cpu=False, **kw)[1].flatten(1)
                out.append((m @ m.T, m.sum(1)))
            return out

        _, ov = fused()
        inter = ov.intersection.reshape(-1, n_words, n_words)
        area = ov.word_area.reshape(-1, n_words)
        for t, (i_ref, a_ref) in enumerate(matmul_form()):
            if threshold:
                assert torch.equal(inter[t], i_ref) and torch.equal(area[t], a_ref), (workload, t)
            else:
                torch.testing.assert_close(inter[t], i_ref, rtol=1e-4, atol=1e-3)
                torch.testing.assert_close(area[t], a_ref, rtol=1e-4, atol=1e-3)
        before = _native.launch_count()
        fused()
        launches = _native.launch_count() - before

        n = max(1, n_maps)
        size = max(1, args.steps // max(1, n_maps // 10)) if n_maps else args.steps
        spin = 5.0 + 0.4 * size * n
        for _ in range(max(3, args.warmup)):
            fused(); matmul_form()
        torch.cuda.synchronize()
        a, b = [], []
        for _ in range(args.rounds):                     # alternated rounds
            a.append(block_us(fused, size, spin))
            b.append(block_us(matmul_form, size, spin))
        fused_us, matmul_us = med(a), med(b)
        bench.emit({'workload': workload, 'image': f'{hw[0]}x{hw[1]}' if hw else 'grid', 'grid': list(grid),
                    'words': n_words, 'threshold': threshold, 'maps': n, 'fused_us': round(fused_us, 2),
                    'composition_us': round(matmul_us, 2), 'speedup': round(matmul_us / fused_us, 2),
                    'fused_launches': launches,
                    'timing': f'median of {args.rounds} alternated rounds of {size} calls',
                    'device': name, 'power_limit': power})


if __name__ == '__main__':
    main()
