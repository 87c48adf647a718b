"""Shared helpers of the test-suite (oracle access, fixture loading, CPU-side recomputation of GPU inputs, profiler
traces of the launches)."""
import json
import os
import re
import subprocess
import sys
from typing import List, Optional, Tuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
LAYER_FIXTURES = ['layer_hw256_h2_d64', 'layer_hw1024_h1_d64_peaky', 'layer_hw64_h2_d40', 'layer_hw576_h1_d64']


def golden(name):
    return np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)


def digest(t, n=64):
    """Exact fingerprint of a tensor for the golden files: [float64 sum, then a fixed seeded sample of n elements]."""
    a = np.ascontiguousarray(torch.as_tensor(t).detach().cpu().numpy()).reshape(-1)
    idx = np.sort(np.random.default_rng(0).choice(a.size, size=min(n, a.size), replace=False))
    return np.concatenate([[a.astype(np.float64).sum()], a[idx].astype(np.float64)])


def oracle_layer_maps(q, k, heads, scale, steps=1):
    """Oracle rows a3+a4 (+a6 summed over `steps` identical calls) for q [B, hw, C], k [B, 77, C]: [N*H, 77, hw] fp32.

    The inputs are moved to CPU fp32 first: products of fp16/bf16 values are exact in fp32, so the oracle sees exactly
    the values the kernel reads (SURVEY.md section 8c: parity is against the fp32 oracle fed identical Q/K)."""
    from oracle import daam_oracle as O
    maps = O.port_layer_step(q.detach().float().cpu(), k.detach().float().cpu(), heads, scale)
    maps = maps.reshape(maps.shape[0], maps.shape[1], -1)
    return maps * steps if steps != 1 else maps


def rel_err(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def assert_elementwise(got, ref, rtol, atol, what=''):
    """SURVEY.md section 8c's form: |got - ref| <= atol + rtol * |ref| for EVERY element (small probabilities included),
    reporting the worst element when it fails."""
    got, ref = torch.as_tensor(got).double().cpu(), torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, f'{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    excess = (got - ref).abs() / (atol + rtol * ref.abs())
    worst = float(excess.max())
    if not worst <= 1.0:
        i = int(excess.argmax())
        raise AssertionError(f'{what}: element {i}: got {got.flatten()[i]:.9e} ref {ref.flatten()[i]:.9e} '
                             f'= {worst:.2f} x (atol {atol:.1e} + rtol {rtol:.1e} * |ref|)')
    return worst


def kernel_events(prof, tmp_dir: str) -> List[Tuple[str, Optional[int]]]:
    """``(instance, grid.x)`` of every accumulate / attention_probs kernel of a trace, in launch order."""
    path = os.path.join(tmp_dir, 'launches.pt.trace.json')
    prof.export_chrome_trace(path)
    events = []
    with open(path) as f:
        trace = json.load(f)
    for e in trace['traceEvents']:
        if e.get('cat') != 'kernel':
            continue
        m = re.search(r'(accumulate_\w+_kernel|attention_probs_kernel)(<[^<>]*>)?', e['name'])
        if not m or m.group(1) == 'accumulate_probs_kernel':
            continue
        args = e.get('args', {})
        grid = args.get('grid')
        events.append((args.get('correlation', e['ts']), e['ts'], m.group(0).replace(' ', ''),
                       grid[0] if grid else None))
    return [(inst, grid) for _, _, inst, grid in sorted(events)]


def traced(module: str, request: dict) -> List[Tuple[str, Optional[int]]]:
    """``module._trace_main(json request)`` in a fresh Python process; it prints the traced ``(instance, grid.x)``
    list as JSON on its last line. A CUDA activity trace taken in a process that has already run
    tests/test_accumulate_steps_gpu.py (which does not profile) holds no kernel event at all, while the same trace
    taken before it does (H100, torch 2.11): some CUPTI / Kineto state left by the earlier work is the likely cause,
    not found yet. A process of its own gives the trace the state a lone run of the module has."""
    code = f'import {module} as m; m._trace_main({json.dumps(request)!r})'
    flags = ['-s'] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable] + flags + ['-c', code], cwd=ROOT, capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    return [tuple(e) for e in json.loads(out.stdout.strip().splitlines()[-1])]


class HookRecorder:
    """Wraps DiffusionHeatMapHooker._enqueue to keep CPU copies of every (layer, q, k) the hook handed to the kernel, and
    replays them through the oracle (rows a3+a4+a6) -- parity on the IDENTICAL Q/K the kernel read."""

    def __init__(self, tc):
        self.calls = []
        inner = tc._enqueue

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.calls.append((layer_idx, factor, q.detach().float().cpu(), k.detach().float().cpu(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def oracle_store(self, prompt_idx=0):
        from oracle import daam_oracle as O
        store = O.OracleHeatMaps()
        for layer_idx, factor, q, k, heads, scale in self.calls:
            n = q.shape[0] // 2
            pair = [prompt_idx, n + prompt_idx]
            maps = O.port_layer_step(q[pair], k[pair], heads, scale)
            for head, m in enumerate(maps):
                store.update(factor, layer_idx, head, m)
        return store
