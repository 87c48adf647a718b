#!/usr/bin/env python
"""Benchmark of CRF-refined word segmentation on one GPU: ``GlobalHeatMap.segment_crf`` /
``GlobalHeatMapStack.segment_crf`` (``daam_segment_crf``: the word maps, ``Q_0``, then one fused launch per mean-field
update) against what a user writes today in torch on the device:

* ``expand_words(..., to_cpu=False)`` for the word maps, the threshold plane stacked in front;
* the same mean field over shifted slices of a zero-padded ``Q``: the ``(2r+1)^2 - 1`` pairwise weights
  ``A exp(-|I_x - I_y|^2 coef) + S`` computed once per call and kept, then per update one ``addcmul_`` per window
  offset over every label and a softmax;
* for a history, all of it once per step (``torch_loop``).

    python bench_segment_crf.py [--steps K] [--warmup W] [--rounds R]

Workloads, all with a threshold of 0.4 and the defaults (5 updates, scale 16, appearance 10, sigma_xy 8, sigma_rgb 13,
smoothness 1, sigma_smooth 3): SD-2.1 at 512x512 with 8 and 24 words at r = 8; SDXL at 1024x1024 and 1216x832 with 8
words at r = 8 (grids as the tracer makes them: 64x64, 128x128, 76x52); a 50-step history at 512x512 with 8 words at
r = 8; SD-2.1 at 512x512 with 8 words at r = 4 and 16. Maps are uniform random rows; the image is flat random-coloured
blocks with a little noise, so that it has edges.

Before timing, the two forms are checked against each other: final ``Q`` within ``TORCH_TOLERANCE`` and labels equal
on all but ``LABEL_MISMATCH`` of the pixels (different fp32 summation orders can flip a pixel whose two best logits
tie to within rounding). Timing: warm-up, then blocks of K calls queued behind a spin kernel and timed with CUDA
events; the fused call and the torch form alternate, R rounds each, and the median is reported. Achieved FP32 rate:
``2 L (2r+1)^2 H W`` FLOP per map and update (the window's FMAs over every label, the issue's count; the weights'
``expf`` are not counted), over the fused call's time, against the data sheet's 67 TFLOP/s. The card name and power
limit are read in the same run. One JSON line per workload goes to stdout; nothing is written anywhere.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.dont_write_bytecode = True          # importing bench.py must not write a .pyc into the tree
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                            # noqa: E402
from bench_aspect import card           # noqa: E402

# name, grid, image (h, w), words, maps (0: one global map), radius
WORKLOADS = [('sd21', (64, 64), (512, 512), 8, 0, 8), ('sd21', (64, 64), (512, 512), 24, 0, 8),
             ('sdxl', (128, 128), (1024, 1024), 8, 0, 8), ('sdxl', (76, 52), (1216, 832), 8, 0, 8),
             ('sd21-history', (64, 64), (512, 512), 8, 50, 8),
             ('sd21', (64, 64), (512, 512), 8, 0, 4), ('sd21', (64, 64), (512, 512), 8, 0, 16)]
CRF = dict(threshold=0.4, iterations=5, scale=16.0, appearance=10.0, sigma_xy=8.0, sigma_rgb=13.0, smoothness=1.0,
           sigma_smooth=3.0)
N_PROMPT_WORDS = 30
TORCH_TOLERANCE = 1e-3   # max |Q_torch - Q_fused| accepted
LABEL_MISMATCH = 1e-3    # largest share of pixels whose labels may differ
PEAK_FP32 = 67e12        # H100 SXM data sheet, dense FP32


def make_image(h, w, g):
    by, bx = 24, 17
    blocks = torch.randint(0, 256, (h // by + 1, w // bx + 1, 3), generator=g, device='cuda').float()
    img = blocks.repeat_interleave(by, 0).repeat_interleave(bx, 1)[:h, :w]
    img = img + torch.randint(-6, 7, (h, w, 3), generator=g, device='cuda')
    return img.clamp(0, 255).to(torch.uint8)


def tables(r):
    """The fp32 appearance and smoothness tables ``[2r+1, 2r+1]`` and ``coef``, as daam_segment_crf forms them."""
    o = torch.arange(-r, r + 1, dtype=torch.float64)
    d2 = o[:, None] ** 2 + o[None, :] ** 2

    def table(weight, sigma):
        g = torch.exp(-d2 / (2 * sigma ** 2))
        g[r, r] = 0
        return (weight * g / g.sum()).float()

    return (table(CRF['appearance'], CRF['sigma_xy']), table(CRF['smoothness'], CRF['sigma_smooth']),
            float(1 / (2 * CRF['sigma_rgb'] ** 2)))


def torch_crf(m, image, r):
    """The mean field of ``m`` ``[W, h, w]`` with ``image`` uint8 ``[h, w, 3]`` in fp32 torch: ``(labels, Q)``."""
    h, w = m.shape[-2:]
    a, s, coef = tables(r)
    z = CRF['scale'] * torch.cat([torch.full((1, h, w), CRF['threshold'], device=m.device), m])
    img = torch.nn.functional.pad(image.permute(2, 0, 1).float(), (r, r, r, r))
    weights = []
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            if dy or dx:
                d2 = ((img[:, r:r + h, r:r + w] - img[:, r + dy:r + dy + h, r + dx:r + dx + w]) ** 2).sum(0)
                weights.append((dy, dx, a[dy + r, dx + r] * torch.exp(-d2 * coef) + s[dy + r, dx + r]))
    q = torch.softmax(z, 0)
    for _ in range(CRF['iterations']):
        qp = torch.nn.functional.pad(q, (r, r, r, r))          # zeros outside the image: the clipped window
        t = z.clone()
        for dy, dx, k in weights:
            t.addcmul_(k, qp[:, r + dy:r + dy + h, r + dx:r + dx + w])
        q = torch.softmax(t, 0)
    return t.argmax(0).to(torch.uint8), q


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
    for workload, grid, hw, n_words, stack, radius in WORKLOADS:
        out_hw = (hw[1], hw[0]) if grid[0] == grid[1] else hw
        image = make_image(*out_hw, g)
        words = [f'w{i}' for i in range(n_words)]
        n_maps = max(1, stack)
        maps = torch.rand((n_maps, N_PROMPT_WORDS + 2) + grid, generator=g, device='cuda')
        target = TimeHeatMaps(tok, prompt, maps) if stack else GlobalHeatMap(tok, prompt, maps[0])
        singles = [target[i] for i in range(n_maps)] if stack else [target]
        fused = lambda: target.segment_crf(words, image, radius=radius, to_cpu=False, **CRF)

        def composition():
            return [torch_crf(ghm.expand_words(words, _size(image), to_cpu=False)[1], image, radius) for ghm in singles]

        # the answers before timing: the torch form against the fused call
        _, labels, _, q = target.segment_crf(words, image, radius=radius, probs=True, to_cpu=False, **CRF)
        labels, q = labels.reshape(n_maps, *out_hw), q.reshape(n_maps, n_words + 1, *out_hw)
        comp = composition()
        q_diff = max(float((cq - q[i]).abs().max()) for i, (_, cq) in enumerate(comp))
        mismatch = max(float((cl != labels[i]).float().mean()) for i, (cl, _) in enumerate(comp))
        assert q_diff <= TORCH_TOLERANCE and mismatch <= LABEL_MISMATCH, (workload, radius, q_diff, mismatch)
        del comp
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
            a.append(block_us(fused, size, 5.0 + 0.5 * size * n_maps * radius))
            b.append(block_us(composition, loop_size, 5.0 + 20.0 * loop_size * n_maps * radius))
        fused_us, torch_us = med(a), med(b)
        flop = 2.0 * (n_words + 1) * (2 * radius + 1) ** 2 * out_hw[0] * out_hw[1] * n_maps * CRF['iterations']
        bench.emit({'workload': workload, 'image': f'{out_hw[0]}x{out_hw[1]}', 'grid': list(grid),
                    'words': n_words, 'maps': n_maps, 'radius': radius, 'iterations': CRF['iterations'],
                    'fused_us': round(fused_us, 1), 'torch_us': round(torch_us, 1),
                    'speedup_vs_torch': round(torch_us / fused_us, 2), 'fused_launches': launches,
                    'gflop': round(flop / 1e9, 2), 'fused_tflops': round(flop / fused_us / 1e6, 2),
                    'share_of_fp32_peak': round(flop / fused_us / 1e6 / (PEAK_FP32 / 1e12), 3),
                    'torch_max_q_diff': float(f'{q_diff:.3g}'), 'label_mismatch': float(f'{mismatch:.3g}'),
                    'timing': f'median of {args.rounds} alternated rounds of {size} calls ({loop_size} torch)',
                    'device': name, 'power_limit': power})


def _size(image):
    """A PIL-like size stand-in for expand_words, for an image array [H, W, 3]."""
    from types import SimpleNamespace
    h, w = int(image.shape[0]), int(image.shape[1])
    return SimpleNamespace(size=(w, h), height=h, width=w)


if __name__ == '__main__':
    main()
