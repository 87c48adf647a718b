#!/usr/bin/env python
"""Benchmark of the per-step device work of ``trace(pipe, time_resolved=True)`` on one GPU.

    python bench_time_resolved.py [--workload sd21|sd21_768|sdxl|sdxl70|sd15] [--steps K] [--warmup W] [--prompts P]
                                  [--dtype bf16|fp16|fp32] [--dump-outputs DIR]

Per denoising step, time-resolved tracing runs ``daam_accumulate_steps`` (the accumulate that also stores each step's
addend into a step slab per layer) and one ``daam_finalize`` per prompt over those step slabs into a history slot. This
script times both on the same resident prompt sets, rotation, blocks and medians as the value leg of ``bench.py``
(whose workload shapes and byte counts it imports): the accumulate alone, the finalize alone, and both per step, in µs
per step, with their algorithmic bytes. The finalize reduces all 77 rows (the longest prompt), so it reads every step
slab once. A last leg times ``daam_accumulate_range`` (the accumulate of ``trace(pipe, step_ranges=[...])`` while a step
lies in a declared range: it also adds each step's addend into a range slab per layer) on the same sets. One JSON line
goes to stdout.

``--dump-outputs DIR`` writes the step slabs of the last timed step (``step_layerNN.npy``, float32, sampled above 64 MB
like ``bench.py --dump-outputs``). Nothing is written anywhere else.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench import TOKENS                # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='sd21', choices=['sd21', 'sd21_768', 'sdxl', 'sdxl70', 'sd15'])
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--prompts', type=int, default=1)
    ap.add_argument('--dtype', default=None, choices=['bf16', 'fp16', 'fp32'])
    ap.add_argument('--dump-outputs', metavar='DIR', default=None)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error('--steps must be >= 1')
    if args.dtype is None:
        args.dtype = {'sd21': 'bf16', 'sd21_768': 'bf16', 'sdxl': 'fp16', 'sdxl70': 'fp16', 'sd15': 'fp32'}[args.workload]
    args.warmup = max(3, args.warmup)
    bench.capture_stdout()

    from daam_b200 import _native, ops
    torch.cuda.set_device(0)
    _native.load()
    dtype = {'bf16': torch.bfloat16, 'fp16': torch.float16, 'fp32': torch.float32}[args.dtype]
    layers = bench.traced_layers(args.workload)
    n_sets, _ = bench.value_sets(layers, args.prompts)
    x = 96 if max(hw for hw, _, _ in layers) == 9216 else 64
    n_rows = TOKENS
    stream = torch.cuda.current_stream()
    flags = _native.ACC_AUTO | _native.ACC_EARLY_LOADS      # Q/K are resident inputs, as in bench.py's value leg

    with torch.no_grad():
        sets = bench.build_sets(layers, args.prompts, dtype, n_sets, 1234)
        slabs, ptrs, groups, ranges, range_ptrs = [], [], [], [], []
        for _, keep in sets:
            step = [torch.empty_like(acc) for _, _, acc in keep]
            slabs.append(step)
            ptrs.append(_native.StepPointers([s.data_ptr() for s in step]))
            ranges.append([torch.zeros_like(acc) for _, _, acc in keep])
            range_ptrs.append(_native.StepPointers([r.data_ptr() for r in ranges[-1]]))
            groups.append([[_native.DaamKeyGroup(acc=s[p].data_ptr(), heads=s.shape[1], h=int(hw ** 0.5),
                                                 w=int(hw ** 0.5), tokens=TOKENS, head_sel=-1, reserved=0)
                            for s, (hw, _, _) in zip(step, layers)] for p in range(args.prompts)])
        history = torch.empty(args.prompts, args.warmup + args.steps, n_rows, x, x, device='cuda')

        def accumulate(i):
            ops.accumulate_steps(sets[i % n_sets][0], ptrs[i % n_sets], 'cuda', stream, flags)

        def finalize(i):
            for p in range(args.prompts):
                _native.finalize(groups[i % n_sets][p], x, n_rows, False, history[p, i % history.shape[1]].data_ptr(),
                                 stream.cuda_stream)

        def both(i):
            accumulate(i)
            finalize(i)

        def accumulate_range(i):
            ops.accumulate_range(sets[i % n_sets][0], range_ptrs[i % n_sets], 'cuda', stream, flags)

        def timed(fn):
            """Median over blocks of the per-step device time; each block is queued behind a spin kernel so that host
            launch pacing is not timed."""
            for i in range(args.warmup):
                fn(i)
            torch.cuda.synchronize()
            block_us, step = [], args.warmup
            for size in bench.block_sizes(args.steps):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda._sleep(int(max(2.0, size * 0.08) * 1.9e6))
                e0.record(stream)
                for _k in range(size):
                    fn(step)
                    step += 1
                e1.record(stream)
                torch.cuda.synchronize()
                block_us.append(e0.elapsed_time(e1) / size * 1e3)
            return sorted(block_us)[len(block_us) // 2], step

        t0 = time.time()
        acc_us, _ = timed(accumulate)
        fin_us, _ = timed(finalize)
        both_us, last = timed(both)
        range_us, _ = timed(accumulate_range)
        wall = time.time() - t0

    esize = 4 if dtype == torch.float32 else 2
    px = bench.px_per_step(layers, args.prompts)
    plain_bytes = bench.algorithmic_bytes_per_step(layers, args.prompts, esize)
    acc_bytes = plain_bytes + px * 4                                              # + the step-slab write
    fin_bytes = px * 4 + args.prompts * n_rows * x * x * 4                        # step slabs read, maps written
    range_bytes = plain_bytes + 2 * px * 4                                        # + the range-slab read and write
    peak, peak_src = bench.measured_peak()
    if args.dump_outputs:
        bench.dump_outputs(args.dump_outputs, {f'step_layer{i:02d}': s for i, s in enumerate(slabs[(last - 1) % n_sets])})
    bench.emit({
        'workload': bench.workload_name(args), 'dtype': args.dtype, 'device': torch.cuda.get_device_name(0),
        'accumulate_steps_us': round(acc_us, 3), 'finalize_us': round(fin_us, 3), 'step_us': round(both_us, 3),
        'plain_bytes': plain_bytes, 'step_slab_bytes': px * 4,
        'accumulate_steps_bytes': acc_bytes, 'finalize_bytes': fin_bytes,
        'accumulate_steps_gbs': round(acc_bytes / (acc_us * 1e-6) / 1e9, 1),
        'finalize_gbs': round(fin_bytes / (fin_us * 1e-6) / 1e9, 1),
        'accumulate_steps_frac_of_peak': round(acc_bytes / (acc_us * 1e-6) / 1e9 / peak, 4),
        'accumulate_range_us': round(range_us, 3), 'accumulate_range_bytes': range_bytes,
        'accumulate_range_gbs': round(range_bytes / (range_us * 1e-6) / 1e9, 1),
        'accumulate_range_frac_of_peak': round(range_bytes / (range_us * 1e-6) / 1e9 / peak, 4),
        'peak_gbs': peak, 'peak_source': peak_src, 'finalize_rows': n_rows, 'x': x,
        'timing': f'median of {len(bench.block_sizes(args.steps))} blocks of K={args.steps} steps (CUDA events, launches '
                  f'queued behind a spin kernel), rotating over {n_sets} prompt sets, {wall:.1f} s',
    })


if __name__ == '__main__':
    main()
