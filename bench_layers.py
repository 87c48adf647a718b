#!/usr/bin/env python
"""Benchmark of the layer- and factor-resolved heat maps: every layer's (or resolution's) map in one finalize launch.

    python bench_layers.py [--workload sd21|sdxl|both] [--iters K] [--warmup W]

The finalize reads fp32 slabs whatever the pipeline dtype, so the legs run on seeded fp32 key stacks shaped like the
workload's traced layers (``bench.traced_layers``: SD-2.1's 15 layers / 175 keys, 55 MB; SDXL's 60 layers / 1100 keys,
441 MB) through the same ``_native`` calls the tracer makes, at 12 and at 77 rows, onto the 64 x 64 grid. Per leg, the
median over 5 rounds of K timed calls (CUDA events, after W warm-up calls; the legs of a comparison alternate within
every round), in µs:

  (a) every layer's map: ``compute_layer_heat_maps`` (one ``daam_finalize_parts``, one map per layer) against the loop
      of ``compute_global_heat_map(layer_idx=l)`` (one ``daam_finalize`` per layer);
  (b) every factor's map: ``compute_factor_heat_maps`` (one ``daam_finalize_parts`` over the groups sorted by factor)
      against the loop of ``compute_global_heat_map(factors={f})``;
  (c) the IoU of 8 words against 4 regions of a 512 x 512 image in every layer: the layer stack and one
      ``daam_region_overlap`` over it against the per-layer loop of ``daam_finalize`` and ``daam_region_overlap``;
  (d) for scale, the plain ``daam_finalize`` over every key (``compute_global_heat_map()``): it reads the same bytes
      as (a) and (b).

One JSON line goes to stdout, with the card's name and power limit. Nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from daam_b200 import _native           # noqa: E402

GRID = 64                               # SD-2.1 at 512 px and SDXL at 1024 px both map to 64 x 64
ROWS = (12, 77)
WORDS, REGIONS, IMAGE = 8, 4, 512


def _slabs(workload, seed=0):
    """One fp32 slab [heads, 77, h * w] per traced layer: (tensor, heads, side)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    return [(torch.rand(h, 77, hw, generator=g, device='cuda'), h, int(round(hw ** 0.5)))
            for hw, h, _ in bench.traced_layers(workload)]


def _time(legs, iters, warmup):
    """``legs``: {name: callable}. Median over 5 rounds of ``iters`` event-timed calls; the legs alternate in a round."""
    stream = torch.cuda.current_stream()
    for fn in legs.values():
        for _ in range(warmup):
            fn()
    rounds = {name: [] for name in legs}
    for _ in range(5):
        for name, fn in legs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            for _ in range(iters):
                fn()
            b.record(stream)
            b.synchronize()
            rounds[name].append(a.elapsed_time(b) * 1000.0 / iters)
    return {name: round(statistics.median(v), 2) for name, v in rounds.items()}


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:       # nvidia-smi absent: the name alone
        return torch.cuda.get_device_name()


def _workload(workload, iters, warmup):
    lib = _native.load()
    x, stream = GRID, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    slabs = _slabs(workload)
    n = len(slabs)
    groups = [_native.DaamKeyGroup(acc=t.data_ptr(), heads=h, h=s, w=s, tokens=77, head_sel=-1, n_blocks=0)
              for t, h, s in slabs]
    factors = [x // s for _, _, s in slabs]
    order = sorted(range(n), key=lambda i: factors[i])          # the tracer's stable partition by factor
    found = sorted(set(factors))
    runs = [(min(p for p, i in enumerate(order) if factors[i] == f), factors.count(f)) for f in found]
    res = {'layers': n, 'keys': sum(h for _, h, _ in slabs), 'factors': found,
           'slab_mb': round(sum(t.numel() for t, _, _ in slabs) * 4 / 1e6, 1)}

    # every argument array is built before timing, so the legs time the launches, not Python
    def packed(gs):
        return (_native.DaamKeyGroup * len(gs))(*gs), len(gs)

    def ok(rc):
        if rc != 0:
            raise RuntimeError(lib.daam_last_error().decode())

    def finalize(arr_n, rows, out_ptr):
        ok(lib.daam_finalize(arr_n[0], arr_n[1], x, x, rows, 0, out_ptr, stream))

    def parts_call(arr_n, sel):
        ok(lib.daam_finalize_parts(arr_n[0], arr_n[1], sel, len(sel), x, x, 0, stream))

    def parts(ranges, rows, out):
        return (_native.DaamMapPart * len(ranges))(*[
            _native.DaamMapPart(group_begin=b, group_count=c, n_rows=rows, out=out[m].data_ptr())
            for m, (b, c) in enumerate(ranges)])

    g = torch.Generator(device='cuda').manual_seed(1)
    regions = (torch.rand(REGIONS, IMAGE, IMAGE, generator=g, device='cuda') < 0.3).to(torch.uint8)
    word_args = _native._word_list(x, [[1 + w] for w in range(WORDS)], IMAGE, IMAGE, False, 0.4)
    word_maps = torch.empty(n, WORDS, x, x, device='cuda')
    inter = torch.empty(n, REGIONS, WORDS, device='cuda')
    area = torch.empty(n, WORDS, device='cuda')
    scratch = torch.empty(_native.region_scratch_floats(n, WORDS, REGIONS, IMAGE, IMAGE), device='cuda')

    def ptrs(t):
        return [ctypes.c_void_p(t[i].data_ptr()) for i in range(n)]

    word_map_ptrs, inter_ptrs, area_ptrs = ptrs(word_maps), ptrs(inter), ptrs(area)
    regions_ptr, scratch_ptr = ctypes.c_void_p(regions.data_ptr()), ctypes.c_void_p(scratch.data_ptr())

    def overlap(map_ptrs, first, n_maps, rows):
        ok(lib.daam_region_overlap(map_ptrs[first], n_maps, rows, *word_args, word_map_ptrs[first], regions_ptr,
                                   REGIONS, inter_ptrs[first], area_ptrs[first], scratch_ptr, stream))

    whole = packed(groups)
    per_layer = [packed([groups[i]]) for i in range(n)]
    sorted_groups = packed([groups[i] for i in order])
    per_factor = [packed([groups[i] for i in order[b:b + c]]) for b, c in runs]
    for rows in ROWS:
        out = torch.empty(n, rows, x, x, device='cuda')
        o = ptrs(out)
        layer_parts = parts([(i, 1) for i in range(n)], rows, out)
        factor_parts = parts(runs, rows, out)
        r = {}
        r.update(_time({'a_loop_us': lambda: [finalize(per_layer[i], rows, o[i]) for i in range(n)],
                        'a_parts_us': lambda: parts_call(whole, layer_parts)}, iters, warmup))
        r.update(_time({'b_loop_us': lambda: [finalize(per_factor[j], rows, o[j]) for j in range(len(runs))],
                        'b_parts_us': lambda: parts_call(sorted_groups, factor_parts)}, iters, warmup))
        r.update(_time({'c_loop_us': lambda: [(finalize(per_layer[i], rows, o[i]), overlap(o, i, 1, rows))
                                              for i in range(n)],
                        'c_stack_us': lambda: (parts_call(whole, layer_parts), overlap(o, 0, n, rows))},
                       iters, warmup))
        r.update(_time({'d_finalize_us': lambda: finalize(whole, rows, o[0])}, iters, warmup))
        res[f'rows{rows}'] = r
    torch.cuda.synchronize()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='both', choices=['sd21', 'sdxl', 'both'])
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_layers.py needs a CUDA device')
    res = {'card': _card(), 'grid': GRID, 'words': WORDS, 'regions': REGIONS, 'image': IMAGE}
    for workload in (('sd21', 'sdxl') if args.workload == 'both' else (args.workload,)):
        res[workload] = _workload(workload, args.iters, args.warmup)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
