#!/usr/bin/env python
"""Benchmark of edge-aware word maps on one GPU: ``GlobalHeatMap.refine_words`` / ``GlobalHeatMapStack.refine_words``
(``daam_refine_words``: the image statistics from exact integer window sums, then per round of planes the word maps
and two separable passes of direct window sums) against what a user writes today in torch on the device:

* ``expand_words(..., to_cpu=False)``;
* He's guided filter with box means by ``cumsum`` differences in fp32: 9 for the guide (3 means, 6 second moments) and
  8 per word (``m``, ``I m``, then ``a`` and ``b``), batched over the words;
* ``torch.linalg.inv`` on the ``[H W, 3, 3]`` regularised covariances;
* for a history, all of it once per step (``torch_loop``).

    python bench_refine.py [--steps K] [--warmup W] [--rounds R]

Workloads, each at radius 8 and 32 with eps 1e-3: SD-2.1 at 512x512 with 8 and 24 words; SDXL at 1024x1024 with 8 and
24 words; SDXL at 1216x832 with 8 words (grids as the tracer makes them: 64x64, 128x128, 76x52); a 50-step history at
512x512 with 8 words. Maps are uniform random rows; the image is flat random-coloured blocks with a little noise, so
that it has edges.

Before timing, the fused call is checked against the float64 reference of ``tests/refine64.py`` within its error bound
``refine_bound`` (every plane of a single map; the first and last maps of the history), and the torch composition
against the fused call within ``TORCH_TOLERANCE``: fp32 cumulative sums lose precision on ``mean(I I^T) - mu mu^T``,
so the composition is the less accurate of the two. Both errors are reported. Timing: warm-up, then blocks of K calls
queued behind a spin kernel and timed with CUDA events; the fused call and the torch composition alternate, R rounds
each, and the median is reported. The card name and power limit are read in the same run. One JSON line per workload
goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench_aspect import card           # noqa: E402
from tests.refine64 import refine64, refine_bound   # noqa: E402

# name, grid, image (h, w), words, maps (0: one global map)
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 0), ('sd21', (64, 64), (512, 512), 24, 0),
             ('sdxl', (128, 128), (1024, 1024), 8, 0), ('sdxl', (128, 128), (1024, 1024), 24, 0),
             ('sdxl', (76, 52), (1216, 832), 8, 0), ('sd21-history', (64, 64), (512, 512), 8, 50)]
RADII = (8, 32)
EPS = 1e-3
N_PROMPT_WORDS = 30
TORCH_TOLERANCE = 0.05   # max |torch composition - fused| accepted, in units of m (normalised maps: [0, 1])


def make_image(h, w, g):
    by, bx = 24, 17
    blocks = torch.randint(0, 256, (h // by + 1, w // bx + 1, 3), generator=g, device='cuda').float()
    img = blocks.repeat_interleave(by, 0).repeat_interleave(bx, 1)[:h, :w]
    img = img + torch.randint(-6, 7, (h, w, 3), generator=g, device='cuda')
    return img.clamp(0, 255).to(torch.uint8)


def box_mean(x, r):
    """The mean of ``x`` ``[..., h, w]`` (fp32) over each (2r+1)^2 window clipped to the image, by cumsum differences."""
    h, w = x.shape[-2:]
    dev = x.device
    xs, ys = torch.arange(w, device=dev), torch.arange(h, device=dev)
    xlo, xhi = (xs - r).clamp(min=0), (xs + r + 1).clamp(max=w)
    ylo, yhi = (ys - r).clamp(min=0), (ys + r + 1).clamp(max=h)
    c = torch.nn.functional.pad(x.cumsum(-1), (1, 0))
    g = c[..., xhi] - c[..., xlo]
    c = torch.nn.functional.pad(g.cumsum(-2), (0, 0, 1, 0))
    n = ((yhi - ylo)[:, None] * (xhi - xlo)[None, :]).float()
    return (c[..., yhi, :] - c[..., ylo, :]) / n


def torch_guided(m, image, r, eps):
    """He's guided filter of ``m`` ``[W, h, w]`` with ``image`` uint8 ``[h, w, 3]`` as guide, in fp32 torch."""
    h, w = m.shape[-2:]
    img = image.permute(2, 0, 1).float() / 255                          # [3, h, w]
    mu = box_mean(img, r)                                               # 3 filters
    iu = torch.triu_indices(3, 3, device=m.device)
    second = box_mean(img[iu[0]] * img[iu[1]], r)                       # 6 filters
    cov = torch.empty((3, 3, h, w), device=m.device)
    cov[iu[0], iu[1]] = second - mu[iu[0]] * mu[iu[1]]
    cov[iu[1], iu[0]] = cov[iu[0], iu[1]]
    cov = cov.permute(2, 3, 0, 1).reshape(h * w, 3, 3) + eps * torch.eye(3, device=m.device)
    inv = torch.linalg.inv(cov)                                         # [h w, 3, 3]
    p = box_mean(m, r)                                                  # [W, h, w]
    mi = box_mean(img[None] * m[:, None], r)                            # [W, 3, h, w]
    c = (mi - mu[None] * p[:, None]).flatten(2).transpose(1, 2)         # [W, h w, 3]
    a = torch.einsum('pcd,wpd->wpc', inv, c).transpose(1, 2).reshape(-1, 3, h, w)
    b = p - (a * mu[None]).sum(1)
    return (box_mean(a, r) * img[None]).sum(1) + box_mean(b, r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    bench.capture_stdout()

    from daam_b200 import _native
    from daam_b200.heatmap import GlobalHeatMap, TimeHeatMaps
    from daam_b200.testing.synthetic import WhitespaceTokenizer
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
    for workload, grid, hw, n_words, stack in WORKLOADS:
        out_hw = (hw[1], hw[0]) if grid[0] == grid[1] else hw
        image = make_image(*out_hw, g)
        words = [f'w{i}' for i in range(n_words)]
        n_maps = max(1, stack)
        maps = torch.rand((n_maps, N_PROMPT_WORDS + 2) + grid, generator=g, device='cuda')
        target = TimeHeatMaps(tok, prompt, maps) if stack else GlobalHeatMap(tok, prompt, maps[0])
        singles = [target[i] for i in range(n_maps)] if stack else [target]
        for radius in RADII:
            fused = lambda: target.refine_words(words, image, radius=radius, eps=EPS, to_cpu=False)

            def composition():
                return [torch_guided(ghm.expand_words(words, _size(image), to_cpu=False)[1], image, radius, EPS)
                        for ghm in singles]

            # the answers before timing: fused against float64 within its bound, torch against fused
            _, q = fused()
            q = q.reshape(n_maps, n_words, *out_hw)
            worst, ratio = 0.0, 0.0
            for i in sorted({0, n_maps - 1}):
                m = singles[i].expand_words(words, _size(image), to_cpu=False)[1].cpu().numpy().astype(np.float64)
                ref, parts = refine64(m, image.cpu().numpy(), radius, float(np.float32(EPS)), parts=True)
                err = np.abs(q[i].cpu().numpy() - ref)
                bound = refine_bound(m, parts, radius, float(np.float32(EPS)))
                assert bool((err <= bound).all()), (workload, radius, i, float(err.max()))
                worst, ratio = max(worst, float(err.max())), max(ratio, float((err / bound).max()))
            comp = torch.stack(composition())
            torch_err = float((comp - q).abs().max())
            assert torch_err <= TORCH_TOLERANCE, (workload, radius, torch_err)
            before = _native.launch_count()
            fused()
            launches = _native.launch_count() - before

            size = max(1, args.steps // max(1, n_maps // 5))
            loop_size = max(1, size // 4)
            for _ in range(max(1, args.warmup)):
                fused(); composition()
            torch.cuda.synchronize()
            a, b = [], []
            for _ in range(args.rounds):                     # alternated rounds
                a.append(block_us(fused, size, 5.0 + 0.2 * size * n_maps * n_words))
                b.append(block_us(composition, loop_size, 5.0 + 1.0 * loop_size * n_maps * n_words))
            fused_us, torch_us = med(a), med(b)
            bench.emit({'workload': workload, 'image': f'{out_hw[0]}x{out_hw[1]}', 'grid': list(grid),
                        'words': n_words, 'maps': n_maps, 'radius': radius, 'eps': EPS,
                        'fused_us': round(fused_us, 1), 'torch_us': round(torch_us, 1),
                        'speedup_vs_torch': round(torch_us / fused_us, 2), 'fused_launches': launches,
                        'fused_max_err_vs_float64': float(f'{worst:.3g}'), 'fused_err_over_bound': float(f'{ratio:.3g}'),
                        'torch_max_diff_vs_fused': float(f'{torch_err:.3g}'),
                        'timing': f'median of {args.rounds} alternated rounds of {size} calls ({loop_size} torch)',
                        'device': name, 'power_limit': power})


def _size(image):
    """A PIL-like size stand-in for expand_words, for an image array [H, W, 3]."""
    from types import SimpleNamespace
    h, w = int(image.shape[0]), int(image.shape[1])
    return SimpleNamespace(size=(w, h), height=h, width=w)


if __name__ == '__main__':
    main()
