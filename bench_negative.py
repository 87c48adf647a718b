#!/usr/bin/env python
"""Step time of ``trace(pipe)`` against ``trace(pipe, negative=True)`` on one GPU.

    python bench_negative.py [--steps K] [--warmup W] [--prompts P] [--rounds R]

With ``negative=True`` each traced layer's one descriptor covers the whole CFG batch ``[uncond x P, cond x P]`` from
sample 0 into a slab twice as tall, so the step launch does twice the tiles: it reads Q of both halves and reads and
writes the accumulator of both halves (K is small). This script times both forms of the step on the same resident
Q/K, with the value leg of ``bench.py`` (whose workload shapes and byte counts it imports): the same rotation over
resident prompt sets, blocks, spin kernel and medians. The workloads are SD-2.1-base in bf16 and SDXL (60 layers) in
fp16. The two forms are alternated ``--rounds`` times in one process; the JSON gives every round and the median. One
JSON line goes to stdout, and nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402

WORKLOADS = [('sd21', torch.bfloat16, 'bf16'), ('sdxl', torch.float16, 'fp16')]


def card():
    """The GPU's name, power limit and maximum SM clock, as nvidia-smi reports them (read only)."""
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def negative_sets(layers, sets):
    """For every plain prompt set: the same Q/K, one whole-batch descriptor per layer into a [2P] slab."""
    from daam_b200 import ops
    out = []
    for _, keep in sets:
        descs, accs = [], []
        for (q, k, acc), (_, heads, d) in zip(keep, layers):
            storage = torch.zeros((2 * acc.shape[0],) + tuple(acc.shape[1:]), dtype=torch.float32, device='cuda')
            descs.append(ops.make_layer_desc(q, k, storage, heads, d ** -0.5, whole_batch=True))
            accs.append(storage)
        out.append((ops.pack(descs), accs))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--prompts', type=int, default=1)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1:
        ap.error('--steps and --rounds must be >= 1')
    args.warmup = max(3, args.warmup)
    bench.capture_stdout()

    from daam_b200 import _native, ops
    torch.cuda.set_device(0)
    _native.load()
    stream = torch.cuda.current_stream()
    flags = _native.ACC_AUTO | _native.ACC_EARLY_LOADS      # Q/K are resident inputs, as in bench.py's value leg

    def timed(sets):
        """Median over blocks of the per-step device time; each block is queued behind a spin kernel so that host
        launch pacing is not timed."""
        n = len(sets)
        for i in range(args.warmup):
            ops.accumulate(sets[i % n][0], 'cuda', stream, flags)
        torch.cuda.synchronize()
        block_us, step = [], args.warmup
        for size in bench.block_sizes(args.steps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(int(max(2.0, size * 0.08) * 1.9e6))
            e0.record(stream)
            for _k in range(size):
                ops.accumulate(sets[step % n][0], 'cuda', stream, flags)
                step += 1
            e1.record(stream)
            torch.cuda.synchronize()
            block_us.append(e0.elapsed_time(e1) / size * 1e3)
        return sorted(block_us)[len(block_us) // 2]

    t0 = time.time()
    results = []
    for workload, dtype, dname in WORKLOADS:
        layers = bench.traced_layers(workload)
        n_sets, _ = bench.value_sets(layers, args.prompts)
        with torch.no_grad():
            plain = bench.build_sets(layers, args.prompts, dtype, n_sets, 1234)
            negative = negative_sets(layers, plain)
            rounds = []
            for _ in range(args.rounds):                      # alternate the two forms: drift hits both alike
                rounds.append((timed(plain), timed(negative)))
        plain_us = sorted(p for p, _ in rounds)[len(rounds) // 2]
        neg_us = sorted(n for _, n in rounds)[len(rounds) // 2]
        plain_bytes = bench.algorithmic_bytes_per_step(layers, args.prompts, 2)
        neg_bytes = bench.algorithmic_bytes_per_step(layers, 2 * args.prompts, 2)   # both halves: Q, K, accumulator
        results.append({
            'workload': f'{workload} ({len(layers)} traced layers, {args.prompts} prompt(s)), {dname}',
            'plain_us': round(plain_us, 2), 'negative_us': round(neg_us, 2), 'ratio': round(neg_us / plain_us, 3),
            'plain_rounds_us': [round(p, 2) for p, _ in rounds], 'negative_rounds_us': [round(n, 2) for _, n in rounds],
            'plain_bytes': plain_bytes, 'negative_bytes': neg_bytes,
            'plain_gbs': round(plain_bytes / (plain_us * 1e-6) / 1e9, 1),
            'negative_gbs': round(neg_bytes / (neg_us * 1e-6) / 1e9, 1),
            'prompt_sets': n_sets,
        })
        del plain, negative
        torch.cuda.empty_cache()
    bench.emit({
        'device': torch.cuda.get_device_name(0), 'card': card(), 'results': results,
        'timing': f'per workload and form: median over {args.rounds} alternated rounds of the median of '
                  f'{len(bench.block_sizes(args.steps))} blocks of K={args.steps} steps (CUDA events, launches queued '
                  f'behind a spin kernel), rotating over resident prompt sets, {time.time() - t0:.1f} s',
    })


if __name__ == '__main__':
    main()
