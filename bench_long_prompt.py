#!/usr/bin/env python
"""Step time of the accumulate launch at 77-, 154- and 231-token contexts on one GPU, and the read cost.

    python bench_long_prompt.py [--steps K] [--warmup W] [--prompts P] [--rounds R]

A long context (two or three CLIP chunks, ``trace(pipe, long_prompts=True)``) is accumulated in full: every context row
of every key, so the accumulator and K grow with the context while Q does not. This script times the step of every
traced layer at the three lengths on resident Q/K, with the value leg of ``bench.py`` (whose workload shapes and byte
counts it imports): the same rotation over resident prompt sets larger than L2, blocks, spin kernel and medians. The
16-bit workloads are SD-2.1-base in bf16 and SDXL (60 layers) in fp16, on the wgmma kernel's long-context instances;
SD-2.1-base in fp32 times the long-context SIMT kernel. The lengths are alternated ``--rounds`` times in one process.
The read leg times ``compute_global_heat_map`` of a 150-token prompt (finalize of the prefix through the EOS row, then
the device gather) against a 75-token prompt's 77-token read, on the SD-2.1 slabs. One JSON line goes to stdout, with
the card's name, power limit and maximum SM clock; nothing is written anywhere.
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
from bench_negative import card         # noqa: E402

WORKLOADS = [('sd21', torch.bfloat16, 'bf16'), ('sdxl', torch.float16, 'fp16'), ('sd21', torch.float32, 'fp32')]
CONTEXTS = (77, 154, 231)


def long_sets(layers, n_prompts, dtype, n_sets, tokens, seed):
    """``bench.build_sets`` with K and the accumulators ``tokens`` rows tall."""
    from daam_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(seed)
    sets = []
    for _ in range(n_sets):
        descs, keep = [], []
        for hw, heads, d in layers:
            q = torch.randn(2 * n_prompts, hw, heads * d, generator=g, device='cuda', dtype=torch.float32).to(dtype)
            k = torch.randn(2 * n_prompts, tokens, heads * d, generator=g, device='cuda', dtype=torch.float32).to(dtype)
            acc = ops.new_accumulator(n_prompts, heads, hw, 'cuda', tokens)
            descs.append(ops.make_layer_desc(q, k, acc, heads, d ** -0.5))
            keep.append((q, k, acc))
        sets.append((ops.pack(descs), keep))
    return sets


def step_bytes(layers, n_prompts, esize, tokens):
    """Q + K in the input dtype and the fp32 accumulator read and written, every context row (conditional half)."""
    return n_prompts * sum(h * hw * d * esize + h * tokens * d * esize + h * tokens * hw * 4 * 2 for hw, h, d in layers)


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
        esize = torch.finfo(dtype).bits // 8
        with torch.no_grad():
            sets = {}
            for tokens in CONTEXTS:
                set_bytes = step_bytes(layers, args.prompts, esize, tokens)
                sets[tokens] = long_sets(layers, args.prompts, dtype, max(2, -(-int(320e6) // set_bytes)), tokens,
                                         1234 + tokens)
            rounds = [[timed(sets[t]) for t in CONTEXTS] for _ in range(args.rounds)]
        for i, tokens in enumerate(CONTEXTS):
            us = sorted(r[i] for r in rounds)[len(rounds) // 2]
            nbytes = step_bytes(layers, args.prompts, esize, tokens)
            results.append({
                'workload': f'{workload} ({len(layers)} traced layers, {args.prompts} prompt(s)), {dname}',
                'tokens': tokens, 'us': round(us, 2), 'rounds_us': [round(r[i], 2) for r in rounds],
                'bytes': nbytes, 'gbs': round(nbytes / (us * 1e-6) / 1e9, 1),
                'of_3350_gbs': round(nbytes / (us * 1e-6) / 3.35e12, 3), 'prompt_sets': len(sets[tokens]),
            })
        del sets
        torch.cuda.empty_cache()
    bench.emit({
        'device': torch.cuda.get_device_name(0), 'card': card(), 'results': results, 'reads': read_leg(args),
        'timing': f'per workload and context: median over {args.rounds} alternated rounds of the median of '
                  f'{len(bench.block_sizes(args.steps))} blocks of K={args.steps} steps (CUDA events, launches queued '
                  f'behind a spin kernel), rotating over resident prompt sets, {time.time() - t0:.1f} s',
    })


def read_leg(args):
    """Median device time of compute_global_heat_map (all layers, normalize=True) on the SD-2.1-base layer shapes:
    a 75-token prompt on 77-token slabs, and a 150-token prompt on 154- and 231-token slabs (finalize through the EOS
    row, gather, normalise)."""
    from daam_b200.testing.synthetic import SD21_SPEC, make_pipeline
    from daam_b200 import trace
    out = []
    for tokens, n_words in ((77, 75), (154, 150), (231, 150)):
        pipe = make_pipeline(SD21_SPEC, dtype=torch.bfloat16, device='cuda', seed=0, init_on_device=True)
        text = ' '.join(f'w{i}' for i in range(n_words))
        with trace(pipe, long_prompts=True) as tc:
            g = torch.Generator().manual_seed(0)
            emb = torch.randn(1, tokens, SD21_SPEC.cross_attention_dim, generator=g)
            pipe(prompt_embeds=emb, num_inference_steps=2, generator=torch.Generator().manual_seed(1))
            for _ in range(3):
                tc.compute_global_heat_map(prompt=text, normalize=True)
            times = []
            for _ in range(max(5, args.rounds * 5)):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                tc.compute_global_heat_map(prompt=text, normalize=True)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3)
        out.append({'tokens': tokens, 'prompt_tokens': n_words, 'read_us': round(sorted(times)[len(times) // 2], 1)})
        del pipe
        torch.cuda.empty_cache()
    return out


if __name__ == '__main__':
    main()
