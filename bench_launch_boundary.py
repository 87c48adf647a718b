#!/usr/bin/env python
"""Per-launch cost of the accumulate step on one GPU: what one more `daam_accumulate` launch costs on top of its bytes.

    python bench_launch_boundary.py [--workload sd21|sd21_768|sdxl|sdxl70|sd15] [--steps K] [--warmup W]
                                    [--dtype bf16|fp16|fp32] [--prompts 1 2 4 8]

Two measurements on the resident prompt sets, rotation and block medians of ``bench.py``'s value leg (whose workload
shapes, byte counts and set builder it imports):

  packed    two prompt sets as ONE `daam_accumulate` call (their layers packed into one launch; 2 x 15 = 30 layers for
            SD-2.1, within the 32 layers of one launch) against the same two sets as two calls. The same tiles and bytes
            run either way, so the difference is the cost of the second launch: the launch boundary, measured directly.
  prompts   the value leg (`bench.leg_value`) at each ``--prompts`` count, and the least-squares fit of
            T = F + bytes / BW over those points: F is the fixed cost per launch, BW the streaming rate.

One JSON line goes to stdout: `packed` times are µs per pair of prompt sets, `prompts` times µs per step (one prompt
set's layers). Nothing is written anywhere.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='sd21', choices=['sd21', 'sd21_768', 'sdxl', 'sdxl70', 'sd15'])
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--dtype', default=None, choices=['bf16', 'fp16', 'fp32'])
    ap.add_argument('--prompts', type=int, nargs='+', default=[1, 2, 4, 8])
    args = ap.parse_args()
    if args.steps < 2:
        ap.error('--steps must be >= 2')
    if args.dtype is None:
        args.dtype = {'sd21': 'bf16', 'sd21_768': 'bf16', 'sdxl': 'fp16', 'sdxl70': 'fp16', 'sd15': 'fp32'}[args.workload]
    args.warmup = max(3, args.warmup)
    bench.capture_stdout()

    from daam_b200 import _native, ops
    D = bench.Dist(1)
    _native.load()
    dtype = {'bf16': torch.bfloat16, 'fp16': torch.float16, 'fp32': torch.float32}[args.dtype]
    esize = 4 if dtype == torch.float32 else 2
    layers = bench.traced_layers(args.workload)
    if 2 * len(layers) > 32:
        ap.error(f'{args.workload}: two prompt sets ({2 * len(layers)} layers) do not fit one launch (32 layers)')
    stream = torch.cuda.current_stream()
    flags = _native.ACC_AUTO | _native.ACC_EARLY_LOADS       # as in bench.py's value leg: Q/K are resident inputs
    t_start = time.time()

    with torch.no_grad():
        # ---- packed: sets 2m and 2m+1 as one launch vs as two ----
        n_sets, _ = bench.value_sets(layers, 1)
        n_sets += n_sets % 2
        sets = bench.build_sets(layers, 1, dtype, n_sets, 1234)
        pairs = []
        for m in range(n_sets // 2):
            descs = [ops.make_layer_desc(q, k, acc, heads, d ** -0.5)
                     for (_, keep) in sets[2 * m:2 * m + 2] for (q, k, acc), (_, heads, d) in zip(keep, layers)]
            pairs.append(ops.pack(descs))

        def two_calls(i):
            m = i % len(pairs)
            ops.accumulate(sets[2 * m][0], 'cuda', stream, flags)
            ops.accumulate(sets[2 * m + 1][0], 'cuda', stream, flags)

        def one_call(i):
            ops.accumulate(pairs[i % len(pairs)], 'cuda', stream, flags)

        def timed(fn, steps):
            """Median over blocks of the device time per call of ``fn``; each block is queued behind a spin kernel so that
            host launch pacing is not timed."""
            for i in range(args.warmup):
                fn(i)
            torch.cuda.synchronize()
            block_us, i = [], args.warmup
            for size in bench.block_sizes(steps):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda._sleep(int(max(2.0, size * 0.08) * 1.9e6))
                e0.record(stream)
                for _k in range(size):
                    fn(i)
                    i += 1
                e1.record(stream)
                torch.cuda.synchronize()
                block_us.append(e0.elapsed_time(e1) / size * 1e3)
            return sorted(block_us)[len(block_us) // 2]

        launches0 = _native.launch_count()
        one_call(0)
        torch.cuda.synchronize()
        one_launch = _native.launch_count() - launches0 == 1
        # alternate the two forms block by block: clock drift and neighbours hit both alike
        two, one = [], []
        for _ in range(3):
            two.append(timed(two_calls, args.steps // 2))
            one.append(timed(one_call, args.steps // 2))
        two_us, one_us = sorted(two)[1], sorted(one)[1]
        del sets, pairs
        torch.cuda.empty_cache()

        # ---- prompts: the value leg at several prompt counts, and T = F + bytes / BW ----
        points = []
        for p in args.prompts:
            a = SimpleNamespace(steps=args.steps, warmup=args.warmup, prompts=p)
            ms, launches, n, _, outputs = bench.leg_value(a, layers, dtype, D, [])
            del outputs
            torch.cuda.empty_cache()
            points.append({'prompts': p, 'us_per_step': round(ms / args.steps * 1e3, 3),
                           'launches_per_step': launches / args.steps,
                           'bytes': bench.algorithmic_bytes_per_step(layers, p, esize), 'sets': n})

    fit = None
    if len(points) >= 2:
        y = torch.tensor([pt['us_per_step'] / pt['launches_per_step'] for pt in points], dtype=torch.float64)
        xs = torch.tensor([float(pt['bytes']) / pt['launches_per_step'] for pt in points], dtype=torch.float64)
        A = torch.stack([torch.ones_like(xs), xs], dim=1)
        coef = torch.linalg.lstsq(A, y.unsqueeze(1)).solution.squeeze(1)
        f_us, us_per_byte = float(coef[0]), float(coef[1])
        fit = {'fixed_us_per_launch': round(f_us, 3),
               'stream_gbs': round(1e-3 / us_per_byte, 1) if us_per_byte > 0 else None,
               'max_rel_residual': round(float(((A @ coef - y) / y).abs().max()), 5),
               'model': 'us per launch = F + bytes per launch / BW, least squares over the prompt counts'}
    bench.emit({
        'workload': bench.workload_name(SimpleNamespace(workload=args.workload, prompts=1, dtype=args.dtype)),
        'dtype': args.dtype, 'device': torch.cuda.get_device_name(0),
        'packed': {'two_calls_us': round(two_us, 3), 'one_call_us': round(one_us, 3),
                   'per_launch_us': round(two_us - one_us, 3), 'one_call_is_one_launch': one_launch,
                   'two_calls_us_runs': [round(v, 3) for v in two], 'one_call_us_runs': [round(v, 3) for v in one],
                   'bytes': 2 * bench.algorithmic_bytes_per_step(layers, 1, esize),
                   'what': 'two prompt sets per call: as one daam_accumulate launch vs as two (same tiles, same bytes); '
                           'median of 3 alternating runs, each the median block'},
        'prompts': points, 'fit': fit,
        'timing': f'blocks of K={args.steps} steps (CUDA events, launches queued behind a spin kernel), rotating over '
                  f'independent resident prompt sets, {time.time() - t_start:.1f} s',
    })


if __name__ == '__main__':
    main()
