#!/usr/bin/env python
"""Benchmark of per-image heat maps (``num_images_per_prompt``) and of the one-launch time-resolved step finalize.

    python bench_images.py [--workload sd21|sdxl] [--images N] [--rows R] [--iters K] [--warmup W]

The finalize reads fp32 slabs whatever the pipeline dtype, so the legs run on seeded fp32 key stacks shaped like the
workload's traced layers (``bench.traced_layers``), laid out as the tracer lays them out ([prompts][images * heads]
per layer), through the same ``_native`` calls the tracer makes. Per leg, the median over 5 rounds of K timed calls
(CUDA events, after W warm-up calls), in µs:

  (a) every image's map of a prompt: ``compute_image_heat_maps`` (one ``daam_finalize_maps``, one map per image)
      against a loop of ``compute_global_heat_map(image_idx=i)`` (one ``daam_finalize`` per image);
  (b) the time-resolved step finalize with one prompt and one image: one ``daam_finalize`` per prompt and half (what
      the tracer issued before) against one ``daam_finalize_maps`` for the step;
  (c) the same with 4 prompts and the negative half (8 maps): 8 ``daam_finalize`` calls against one call;
  (d) the step finalize with ``--images`` images per prompt: the blended map alone against the blended map plus every
      image's map in the same call (what a multi-image time-resolved trace now does per step).

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

GRID = {'sd21': 64, 'sdxl': 64}         # the heat-map grid: SD-2.1 512 px and SDXL 1024 px both map to 64 x 64


def _slabs(workload, blocks, seed=0):
    """One fp32 slab [blocks, heads, 77, h * w] per traced layer (blocks = prompts x images, image-major in a prompt)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    return [(torch.rand(blocks, h, 77, hw, generator=g, device='cuda'), h, int(round(hw ** 0.5)))
            for hw, h, _ in bench.traced_layers(workload)]


def _groups(slabs, block=None, count=1):
    """``block`` None: the maps call's groups over whole slabs; else the expanded daam_finalize groups of blocks
    [block, block + count) (head_sel -1: one group per layer with heads * count heads)."""
    if block is None:
        return [_native.DaamKeyGroup(acc=t.data_ptr(), heads=h, h=s, w=s, tokens=77, head_sel=-1, n_blocks=t.shape[0])
                for t, h, s in slabs]
    return [_native.DaamKeyGroup(acc=t[block].data_ptr(), heads=h * count, h=s, w=s, tokens=77, head_sel=-1,
                                 n_blocks=0) for t, h, s in slabs]


def _time(fn, iters, warmup):
    stream = torch.cuda.current_stream()
    for _ in range(warmup):
        fn()
    rounds = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(iters):
            fn()
        b.record(stream)
        b.synchronize()
        rounds.append(a.elapsed_time(b) * 1000.0 / iters)
    return round(statistics.median(rounds), 2)


def _card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except Exception:       # nvidia-smi absent: the name alone
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='sd21', choices=sorted(GRID))
    ap.add_argument('--images', type=int, default=4)
    ap.add_argument('--rows', type=int, default=12)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_images.py needs a CUDA device')
    x, n, rows, stream = GRID[args.workload], args.images, args.rows, torch.cuda.current_stream().cuda_stream
    res = {'workload': args.workload, 'images': n, 'rows': rows, 'card': _card()}

    # every argument array is built before timing, so the legs time the launches, not Python
    lib = _native.load()

    def packed(groups):
        return (_native.DaamKeyGroup * len(groups))(*groups), len(groups)

    def finalize(groups, out):
        arr, ng = groups
        lib.daam_finalize(arr, ng, x, x, rows, 0, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(stream))

    def maps_args(slabs, sels):
        return packed(_groups(slabs)) + ((_native.DaamMapSel * len(sels))(*sels), len(sels))

    def maps_call(args):
        arr, ng, sel, nm = args
        lib.daam_finalize_maps(arr, ng, sel, nm, x, x, 0, ctypes.c_void_p(stream))

    def sel(block, count, out):
        return _native.DaamMapSel(block_begin=block, block_count=count, n_rows=rows, out=out.data_ptr())

    # (a) one prompt, n images
    slabs = _slabs(args.workload, n)
    out = torch.empty(n, rows, x, x, device='cuda')
    per_image = [packed(_groups(slabs, i)) for i in range(n)]
    sels = [sel(i, 1, out[i]) for i in range(n)]
    res['a_loop_us'] = _time(lambda: [finalize(per_image[i], out[i]) for i in range(n)], args.iters, args.warmup)
    a_args = maps_args(slabs, sels)
    res['a_maps_us'] = _time(lambda: maps_call(a_args), args.iters, args.warmup)
    # (d) the step finalize with n images: blended alone, then blended + every image in one call
    blend = torch.empty(rows, x, x, device='cuda')
    alone, with_images = maps_args(slabs, [sel(0, n, blend)]), maps_args(slabs, [sel(0, n, blend)] + sels)
    res['d_blended_us'] = _time(lambda: maps_call(alone), args.iters, args.warmup)
    res['d_blended_and_images_us'] = _time(lambda: maps_call(with_images), args.iters, args.warmup)
    torch.cuda.synchronize()
    del slabs
    # (b) one prompt, one image: one daam_finalize vs one daam_finalize_maps
    slabs = _slabs(args.workload, 1)
    one = packed(_groups(slabs, 0))
    res['b_finalize_us'] = _time(lambda: finalize(one, blend), args.iters, args.warmup)
    single = maps_args(slabs, [sel(0, 1, blend)])
    res['b_maps_us'] = _time(lambda: maps_call(single), args.iters, args.warmup)
    torch.cuda.synchronize()
    del slabs
    # (c) 4 prompts, negative half too: storage [2 x 4] blocks, 8 maps
    slabs = _slabs(args.workload, 8)
    outs = torch.empty(8, rows, x, x, device='cuda')
    groups = [packed(_groups(slabs, b)) for b in range(8)]
    eight = maps_args(slabs, [sel(b, 1, outs[b]) for b in range(8)])
    res['c_finalize_x8_us'] = _time(lambda: [finalize(groups[b], outs[b]) for b in range(8)], args.iters, args.warmup)
    res['c_maps_us'] = _time(lambda: maps_call(eight), args.iters, args.warmup)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
