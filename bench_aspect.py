#!/usr/bin/env python
"""Benchmark of the heat-map reads at square and non-square image sizes on one GPU.

    python bench_aspect.py [--steps K] [--warmup W] [--rows R]

For each geometry -- SD-2.1 at 512x512, 512x768 and 768x512; SDXL at 1024x1024, 1216x832, 1344x768 and 1152x896 --
this script builds one prompt's fp32 key slabs for every traced layer of ``bench.py``'s ``sd21`` / ``sdxl`` workloads,
with each layer's key size taken from the geometry rule (``daam_b200.geometry``), and times:

* ``daam_finalize`` over all keys at 77 rows and at ``--rows`` rows (a 10-word prompt: 12);
* ``daam_expand_words`` for 8 words from a ``[rows, xh, xw]`` map to the image size.

Timing as in ``bench_time_resolved.py``: warm-up, then the median over blocks of K launches (CUDA events, launches
queued behind a spin kernel). Bytes are algorithmic: key bytes read plus map bytes written (finalize), map rows read
plus images written (expand). ``finalize_kernel`` names the kernel the library's dispatch rule picks (restated here:
``fast`` when every key has one integer factor 1 / 2 / 4 on both axes, 16-byte-aligned bases, and the grid is at most
256 wide; see DESIGN.md section 4.3). The card name and power limit are read in the same run. One JSON line per
geometry goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import math
import os
import subprocess
import sys

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench import TOKENS                # noqa: E402

# workload, sample_size (latent side of the model's own square size), image (height, width)
GEOMETRIES = [('sd21', 64, (512, 512)), ('sd21', 64, (512, 768)), ('sd21', 64, (768, 512)),
              ('sdxl', 128, (1024, 1024)), ('sdxl', 128, (1216, 832)), ('sdxl', 128, (1344, 768)),
              ('sdxl', 128, (1152, 896))]


def card():
    """``(name, power limit)`` of GPU 0, read-only query."""
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ''
    return name, out or 'not measured'


def layer_keys(workload, sample_size, image):
    """``[(h, w, heads)]`` of every traced layer at ``image`` and the grid ``(xh, xw)``."""
    from daam_b200.geometry import LatentGeometry
    H, W = image[0] // 8, image[1] // 8
    geo = LatentGeometry(4096, sample_size, (H, W))
    out = []
    for hw, heads, _ in bench.traced_layers(workload):
        s = int(round(math.log2(sample_size / math.isqrt(hw))))     # the layer's level in the model's own square size
        n = -(-H // (1 << s)) * -(-W // (1 << s))
        h, w, _ = geo.level(n)
        out.append((h, w, heads))
    return out, geo.grid


def fast_rule(keys, grid):
    """The library's choice of finalize kernel (finalize.cu, ``daam_finalize``), restated for the report."""
    xh, xw = grid
    if (xh == xw and xh % 16) or xw > 256 or sum(k for _, _, k in keys) > 2048:
        return 'generic'
    for h, w, _ in keys:
        if xh % h or xw % w or xh // h != xw // w or xh // h not in (1, 2, 4) or (h * w) % 4:
            return 'generic'
    return 'fast'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rows', type=int, default=12)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    torch.cuda.set_device(0)
    _native.load()
    name, power = card()
    stream = torch.cuda.current_stream()

    def timed(fn):
        for i in range(max(3, args.warmup)):
            fn()
        torch.cuda.synchronize()
        block_us = []
        for size in bench.block_sizes(args.steps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(int(max(2.0, size * 0.08) * 1.9e6))
            e0.record(stream)
            for _k in range(size):
                fn()
            e1.record(stream)
            torch.cuda.synchronize()
            block_us.append(e0.elapsed_time(e1) / size * 1e3)
        return sorted(block_us)[len(block_us) // 2]

    g = torch.Generator(device='cuda').manual_seed(0)
    for workload, sample_size, image in GEOMETRIES:
        keys, grid = layer_keys(workload, sample_size, image)
        slabs = [torch.exp(torch.randn(heads, TOKENS, h, w, generator=g, device='cuda')) for h, w, heads in keys]
        groups = [_native.DaamKeyGroup(acc=t.data_ptr(), heads=t.shape[0], h=t.shape[2], w=t.shape[3], tokens=TOKENS,
                                       head_sel=-1, reserved=0) for t in slabs]
        line = {'workload': workload, 'image': f'{image[0]}x{image[1]}', 'grid': list(grid),
                'keys': sum(k for _, _, k in keys), 'finalize_kernel': fast_rule(keys, grid),
                'device': name, 'power_limit': power}
        for rows in (TOKENS, args.rows):
            out = torch.empty((rows,) + grid, device='cuda')
            us = timed(lambda: _native.finalize(groups, grid, rows, False, out.data_ptr(), stream.cuda_stream))
            nbytes = sum(k * rows * h * w * 4 for h, w, k in keys) + rows * grid[0] * grid[1] * 4
            line.update({f'finalize_{rows}_us': round(us, 2), f'finalize_{rows}_bytes': nbytes,
                         f'finalize_{rows}_gbs': round(nbytes / (us * 1e-6) / 1e9, 1)})
        rows = args.rows
        maps = torch.rand((rows,) + grid, generator=g, device='cuda')
        words = [[1 + i % (rows - 2)] for i in range(8)]
        word_maps = torch.empty((8,) + grid, device='cuda')
        images = torch.empty((8,) + image, device='cuda')
        scratch = torch.empty(8 * _native.EXPAND_SCRATCH_FLOATS, device='cuda')
        us = timed(lambda: _native.expand_words(maps.data_ptr(), rows, grid, words, image[0], image[1], False, None,
                                                word_maps.data_ptr(), images.data_ptr(), scratch.data_ptr(),
                                                stream.cuda_stream))
        nbytes = 8 * grid[0] * grid[1] * 4 * 2 + 8 * image[0] * image[1] * 4     # rows read, word maps + images written
        line.update({'expand_words_8_us': round(us, 2), 'expand_words_8_bytes': nbytes,
                     'expand_words_8_gbs': round(nbytes / (us * 1e-6) / 1e9, 1),
                     'timing': f'median of {len(bench.block_sizes(args.steps))} blocks of K={args.steps} launches'})
        bench.emit(line)
        del slabs, groups


if __name__ == '__main__':
    main()
