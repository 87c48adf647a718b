#!/usr/bin/env python
"""Benchmark of value-weighted heat maps: every key's map scaled by its value norm ``||W_h v||``.

    python bench_value_weighted.py [--iters K] [--warmup W]

The finalize reads fp32 slabs whatever the pipeline dtype, so legs (a) and (b) run on seeded fp32 key stacks shaped like
the workload's traced layers (``bench.traced_layers``: SD-2.1's 15 layers / 175 keys, SDXL's 60 layers / 1100 keys)
and seeded norms, through the same ``_native`` calls the tracer makes, at 12 and 77 rows, onto the 64 x 64 grid. Per
leg, the median over 5 rounds of K timed calls (CUDA events, after W warm-up calls; the legs of a comparison alternate
within every round), in µs:

  (a) ``compute_global_heat_map(value_weighted=True)`` (one ``daam_finalize_parts_weighted``) against the plain
      ``compute_global_heat_map()`` (``daam_finalize``), and the weighted layer stack against the plain one (one
      ``daam_finalize_parts`` / ``_weighted`` with one map per layer);
  (b) the weighted map against what a user writes without it: ``compute_per_head_heat_maps()`` (one
      ``daam_finalize_per_key``), times every key's norms, summed over the keys and divided by their count, on the device;
  (c) the one-time ``daam_value_norms`` cost of a generation: one call per traced layer of SD-2.1 (15 layers) and SDXL
      with its mid block (70 layers), fp16 values and output weights (``[channels, channels]``), one prompt's
      conditional half of a CFG batch.

One JSON line goes to stdout, with the card's name, power limit and largest SM clock. Nothing is written anywhere.
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

GRID = 64
ROWS = (12, 77)


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


def _ok(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.daam_last_error().decode())


def _maps(workload, iters, warmup):
    lib = _native.load()
    x, stream = GRID, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device='cuda').manual_seed(0)
    layers = bench.traced_layers(workload)
    slabs = [(torch.rand(h, 77, hw, generator=g, device='cuda'), h, int(round(hw ** 0.5))) for hw, h, _ in layers]
    norms = [torch.rand(h, 77, generator=g, device='cuda') * 4 for _, h, _ in layers]
    n = len(slabs)
    n_keys = sum(h for _, h, _ in slabs)
    groups = (_native.DaamKeyGroup * n)(*[_native.DaamKeyGroup(acc=t.data_ptr(), heads=h, h=s, w=s, tokens=77,
                                                               head_sel=-1, n_blocks=0) for t, h, s in slabs])
    weights = (ctypes.c_void_p * n)(*[w.data_ptr() for w in norms])
    key_norms = torch.cat(norms)                                   # [keys, 77], the per-head read's key order
    res = {'layers': n, 'keys': n_keys}
    for rows in ROWS:
        out = torch.empty(n, rows, x, x, device='cuda')
        per_key = torch.empty(n_keys, rows, x, x, device='cuda')
        one = (_native.DaamMapPart * 1)(_native.DaamMapPart(group_begin=0, group_count=n, n_rows=rows,
                                                            out=out[0].data_ptr()))
        stack = (_native.DaamMapPart * n)(*[_native.DaamMapPart(group_begin=i, group_count=1, n_rows=rows,
                                                                out=out[i].data_ptr()) for i in range(n)])
        w_rows = key_norms[:, :rows, None, None].contiguous()

        def plain():
            _ok(lib, lib.daam_finalize(groups, n, x, x, rows, 0, ctypes.c_void_p(out[0].data_ptr()), stream))

        def weighted():
            _ok(lib, lib.daam_finalize_parts_weighted(groups, n, one, 1, x, x, 0, weights, stream))

        def plain_stack():
            _ok(lib, lib.daam_finalize_parts(groups, n, stack, n, x, x, 0, stream))

        def weighted_stack():
            _ok(lib, lib.daam_finalize_parts_weighted(groups, n, stack, n, x, x, 0, weights, stream))

        def by_hand():                    # compute_per_head_heat_maps(), then weight, sum and divide on the device
            _ok(lib, lib.daam_finalize_per_key(groups, n, x, x, rows, 0, ctypes.c_void_p(per_key.data_ptr()), stream))
            torch.mul(per_key, w_rows).sum(0).div_(n_keys)

        r = {}
        r.update(_time({'a_plain_us': plain, 'a_weighted_us': weighted}, iters, warmup))
        r.update(_time({'a_plain_stack_us': plain_stack, 'a_weighted_stack_us': weighted_stack}, iters, warmup))
        r.update(_time({'b_weighted_us': weighted, 'b_by_hand_us': by_hand}, iters, warmup))
        r['a_ratio'] = round(r['a_weighted_us'] / r['a_plain_us'], 3)
        r['a_stack_ratio'] = round(r['a_weighted_stack_us'] / r['a_plain_stack_us'], 3)
        r['b_speedup'] = round(r['b_by_hand_us'] / r['b_weighted_us'], 1)
        # the two weighted maps agree (the by-hand sum runs in another order: fp32 rounding apart)
        weighted()
        ref = torch.mul(per_key, w_rows).sum(0).div_(n_keys)
        r['b_max_rel_diff'] = float(((out[0] - ref).abs().max() / ref.abs().max()).item())
        res[f'rows{rows}'] = r
    torch.cuda.synchronize()
    return res


def _norms(workload, iters, warmup):
    """One ``daam_value_norms`` per traced layer, as the tracer issues them at a generation's first step."""
    g = torch.Generator(device='cuda').manual_seed(1)
    layers = bench.traced_layers(workload)
    calls = []
    for _, heads, d in layers:
        c = heads * d
        value = torch.randn(2, 77, c, generator=g, device='cuda').half()           # to_v of a CFG batch of one prompt
        weight = (torch.randn(c, c, generator=g, device='cuda') / c ** 0.5).half()
        out = torch.empty(1, heads, 77, device='cuda')
        calls.append((value, weight, out, heads, d))
    stream = torch.cuda.current_stream().cuda_stream

    def run():
        for value, weight, out, heads, d in calls:
            _native.value_norms(value[1].data_ptr(), _native.DAAM_F16, (value.stride(0), value.stride(1), d),
                                weight.data_ptr(), _native.DAAM_F16, weight.stride(0), 1, heads, 77, d,
                                weight.shape[0], out.data_ptr(), stream)

    t = _time({'norms_us': run}, max(1, iters // 5), warmup)
    return {'layers': len(layers), 'all_layers_us': t['norms_us']}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_value_weighted.py needs a CUDA device')
    res = {'card': _card(), 'grid': GRID}
    for workload in ('sd21', 'sdxl'):
        res[workload] = _maps(workload, args.iters, args.warmup)
    res['norms'] = {w: _norms(w, args.iters, args.warmup) for w in ('sd21', 'sdxl70')}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
