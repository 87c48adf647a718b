"""Joint-attention (SD3) heat maps on one GPU: the per-step daam_accumulate_joint launch at SD3-medium and SD3.5-large
sizes against the HBM floor of its algorithmic bytes and against the torch composition a user would write, the hooked
against the un-hooked joint forward of the synthetic transformer, and the CLIP and T5 reads.

    python bench_joint.py [--steps 20] [--warmup 3]

Prints one JSON line; the card's name and power limit are read in the same run."""
import argparse
import json
import math
import subprocess

import torch

from daam_b200 import ops, trace
from daam_b200.testing.synthetic import SD3_MEDIUM_SPEC, SD35_LARGE_SPEC, make_sd3_pipeline

HBM = 3.35e12   # H100 SXM data sheet, bytes/s


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                      text=True).strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def step_bench(spec, tokens, steps, warmup):
    """One denoising step of every layer, 1 prompt, 1024 px (64 x 64 image tokens), bf16."""
    heads, d, hw, layers = spec.heads, spec.dim_head, 4096, spec.blocks
    g = torch.Generator(device='cuda').manual_seed(0)
    L = hw + tokens
    qs = [torch.randn(2, heads, L, d, generator=g, device='cuda', dtype=torch.bfloat16) for _ in range(layers)]
    ks = [torch.randn(2, heads, L, d, generator=g, device='cuda', dtype=torch.bfloat16) for _ in range(layers)]
    scale = 1.0 / math.sqrt(d)
    lses = [torch.logsumexp((q[:, :, :hw].float() @ k.float().transpose(-1, -2)) * scale, -1) for q, k in zip(qs, ks)]
    accs = [torch.zeros(1, heads, tokens, hw, device='cuda') for _ in range(layers)]
    descs = [ops.make_joint_desc(q, k, l, hw, a, heads, scale) for q, k, l, a in zip(qs, ks, lses, accs)]
    ms = timed(lambda: ops.accumulate_joint(descs, 'cuda'), steps, warmup)

    def composed():
        for q, k, l, a in zip(qs, ks, lses, accs):
            s = q[1:, :, :hw] @ k[1:, :, hw:].transpose(-1, -2)            # [1, H, hw, T]
            a += torch.exp(s.float() * scale - l[1:, :, :, None]).transpose(-1, -2)
    torch_ms = timed(composed, max(2, steps // 4), 1)
    algo = layers * (heads * hw * d * 2 + heads * tokens * d * 2 + heads * hw * 4 + 2 * heads * tokens * hw * 4)
    return dict(model=spec.name, tokens=tokens, layers=layers, kernel_ms=ms, bytes=algo, floor_ms=algo / HBM * 1e3,
                fraction_of_hbm=algo / HBM / (ms * 1e-3), torch_ms=torch_ms, speedup_vs_torch=torch_ms / ms)


def forward_bench(steps, warmup):
    """Hooked vs un-hooked joint forward of the SD3-medium-shaped synthetic transformer, bf16, CFG batch of 2."""
    pipe = make_sd3_pipeline(SD3_MEDIUM_SPEC, dtype=torch.bfloat16, device='cuda', init_on_device=True)
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.randn(2, 16, 128, 128, generator=g, device='cuda', dtype=torch.bfloat16)
    ctx = torch.randn(2, 333, 4096, generator=g, device='cuda', dtype=torch.bfloat16)
    t = torch.full((2,), 500.0, device='cuda')
    f = lambda: pipe.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)
    with torch.no_grad():
        plain = timed(f, steps, warmup)
        with trace(pipe) as tc:
            pipe.check_inputs('a photo of a red fox in the snow', None, None, 1024, 1024)
            tc.last_prompts_3 = [None]
            hooked = timed(f, steps, warmup)
            clip = timed(lambda: tc.compute_global_heat_map(), steps, warmup)
            t5 = timed(lambda: tc.compute_global_heat_map(encoder='t5'), steps, warmup)
    return dict(unhooked_ms=plain, hooked_ms=hooked, overhead=hooked / plain - 1, read_clip_ms=clip, read_t5_ms=t5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    res = dict(gpu=name, power_limit=power, step=[])
    for spec in (SD3_MEDIUM_SPEC, SD35_LARGE_SPEC):
        for tokens in (333, 589):
            res['step'].append(step_bench(spec, tokens, args.steps, args.warmup))
            torch.cuda.empty_cache()
    res['forward'] = forward_bench(args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
