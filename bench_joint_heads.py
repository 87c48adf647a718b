"""Head-reduced joint-attention heat maps (trace(pipe, reduce_heads=True)) on one GPU: the per-step
daam_accumulate_joint_heads launch against the per-head daam_accumulate_joint launch at SD3-medium, SD3.5-large,
FLUX.1-dev and FLUX.1-schnell sizes (1024 px, bf16, one prompt), the slab bytes of each, the head-reduced kernel's
tensor-core and ex2 rates as shares of the card's peaks, the hooked against the un-hooked forward of the synthetic
SD3-medium and FLUX.1-dev transformers with the option, and the cost of a compute_global_heat_map() read.

    python bench_joint_heads.py [--steps 10] [--warmup 2] [--rounds 5]

The two kernels are timed in alternated rounds (the card is shared) and each time is the median of the rounds. Prints
one JSON line per row, then one for the forwards; the card's name, power limit and maximum SM clock are read in the
same run."""
import argparse
import json
import math
import statistics
import subprocess

import torch

from daam_b200 import ops, trace
from daam_b200.testing.synthetic import (FLUX_DEV_SPEC, FLUX_SCHNELL_SPEC, SD3_MEDIUM_SPEC, SD35_LARGE_SPEC,
                                         flux_image_ids, make_flux_pipeline, make_sd3_pipeline)

MMA_PEAK = 989e12   # H100 SXM data sheet, dense BF16 FLOP/s (700 W card)
EX2_PER_SM_CLOCK = 16   # MUFU ex2 results per SM per clock


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                       '--format=csv,noheader,nounits'], text=True).strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(',')]
        return name, f'{power} W', float(clock) * 1e6
    except Exception:
        return torch.cuda.get_device_name(0), 'unknown', None


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


def alternated(fns, steps, warmup, rounds):
    """The median over ``rounds`` of each function's mean step time, the functions alternating within every round."""
    times = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            times[i].append(timed(fn, steps, warmup))
    return [statistics.median(t) for t in times]


def rows():
    """(name, heads, head_dim, layers, tokens, text_first): the layer calls of one denoising step."""
    out = []
    for spec in (SD3_MEDIUM_SPEC, SD35_LARGE_SPEC):
        for tokens in (333, 589):
            out.append((spec.name, spec.heads, spec.dim_head, spec.blocks, tokens, False))
    for spec in (FLUX_DEV_SPEC, FLUX_SCHNELL_SPEC):
        out.append((spec.name, spec.heads, spec.dim_head, spec.double + spec.single, spec.t5_rows, True))
    return out


def step_bench(name, heads, d, layers, tokens, text_first, steps, warmup, rounds, clock):
    """One step of every layer at 1024 px (4096 image tokens), bf16, one prompt: SD3 a CFG batch of 2 (the
    conditional sample kept), FLUX a batch of one, text-first. Both kernels read the same operands."""
    hw = 4096
    bsz = 1 if text_first else 2
    g = torch.Generator(device='cuda').manual_seed(0)
    L = hw + tokens
    scale = 1.0 / math.sqrt(d)
    qs = [torch.randn(bsz, heads, L, d, generator=g, device='cuda', dtype=torch.bfloat16) for _ in range(layers)]
    ks = [torch.randn(bsz, heads, L, d, generator=g, device='cuda', dtype=torch.bfloat16) for _ in range(layers)]
    img = slice(tokens, L) if text_first else slice(0, hw)
    lses = []
    for q, k in zip(qs, ks):
        lse = torch.zeros(bsz, heads, L, device='cuda')
        lse[:, :, img] = torch.logsumexp((q[:, :, img].float() @ k.float().transpose(-1, -2)) * scale, -1)
        lses.append(lse)
    kw = dict(text_first=text_first, whole_batch=text_first)
    per_head = [torch.zeros(1, heads, tokens, hw, device='cuda') for _ in range(layers)]
    reduced = [torch.zeros(1, tokens, hw, device='cuda') for _ in range(layers)]
    d_head = [ops.make_joint_desc(q, k, l, hw, a, heads, scale, **kw) for q, k, l, a in zip(qs, ks, lses, per_head)]
    d_mean = [ops.make_joint_desc(q, k, l, hw, a, heads, scale, reduce_heads=True, **kw)
              for q, k, l, a in zip(qs, ks, lses, reduced)]
    head_ms, mean_ms = alternated([lambda: ops.accumulate_joint(d_head, 'cuda'),
                                   lambda: ops.accumulate_joint_heads(d_mean, 'cuda')], steps, warmup, rounds)
    exps = layers * heads * tokens * hw
    flop = 2 * exps * d
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = dict(model=name, tokens=tokens, layers=layers, heads=heads, head_dim=d,
               per_head_ms=head_ms, head_mean_ms=mean_ms, speedup=head_ms / mean_ms,
               slab_bytes_per_head=layers * heads * tokens * hw * 4, slab_bytes_head_mean=layers * tokens * hw * 4,
               tflops=flop / (mean_ms * 1e-3) / 1e12, mma_share_of_peak=flop / (mean_ms * 1e-3) / MMA_PEAK,
               ex2_per_s=exps / (mean_ms * 1e-3))
    if clock:
        ex2_peak = EX2_PER_SM_CLOCK * sms * clock
        res.update(ex2_peak_per_s=ex2_peak, ex2_share_of_peak=exps / (mean_ms * 1e-3) / ex2_peak)
    return res


def sd3_forward(steps, warmup, rounds):
    pipe = make_sd3_pipeline(SD3_MEDIUM_SPEC, dtype=torch.bfloat16, device='cuda', init_on_device=True)
    g = torch.Generator(device='cuda').manual_seed(1)
    x = torch.randn(2, 16, 128, 128, generator=g, device='cuda', dtype=torch.bfloat16)
    ctx = torch.randn(2, 333, 4096, generator=g, device='cuda', dtype=torch.bfloat16)
    t = torch.full((2,), 500.0, device='cuda')
    f = lambda: pipe.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)

    def check():
        pipe.check_inputs('a photo of a red fox in the snow', None, None, 1024, 1024)
    return _forward('sd3-medium', pipe, f, check, steps, warmup, rounds)


def flux_forward(steps, warmup, rounds):
    pipe = make_flux_pipeline(FLUX_DEV_SPEC, dtype=torch.bfloat16, device='cuda', init_on_device=True)
    g = torch.Generator(device='cuda').manual_seed(1)
    kw = dict(hidden_states=torch.randn(1, 4096, 64, generator=g, device='cuda', dtype=torch.bfloat16),
              encoder_hidden_states=torch.randn(1, 512, 4096, generator=g, device='cuda', dtype=torch.bfloat16),
              pooled_projections=torch.randn(1, 768, generator=g, device='cuda', dtype=torch.bfloat16),
              timestep=torch.full((1,), 0.5, device='cuda', dtype=torch.bfloat16),
              img_ids=flux_image_ids(64, 64, 'cuda').bfloat16(),
              txt_ids=torch.zeros(512, 3, device='cuda', dtype=torch.bfloat16),
              guidance=torch.full((1,), 3.5, device='cuda'))
    f = lambda: pipe.transformer(**kw)

    def check():
        pipe.check_inputs('a photo of a red fox in the snow', None, 1024, 1024)
    return _forward('flux.1-dev', pipe, f, check, steps, warmup, rounds)


def _forward(name, pipe, f, check, steps, warmup, rounds):
    """Un-hooked, per-head-traced and head-reduced-traced forwards in alternated rounds, and one read of each trace."""
    plain, per_head, mean, read_head, read_mean = [], [], [], [], []
    with torch.no_grad():
        for _ in range(rounds):
            plain.append(timed(f, steps, warmup))
            for reduce_heads, out, read in ((False, per_head, read_head), (True, mean, read_mean)):
                with trace(pipe, reduce_heads=reduce_heads) as tc:
                    check()
                    out.append(timed(f, steps, warmup))
                    read.append(timed(lambda: tc.compute_global_heat_map(), steps, warmup))
                del tc
                torch.cuda.empty_cache()
    med = statistics.median
    return dict(model=name, unhooked_ms=med(plain), hooked_per_head_ms=med(per_head), hooked_head_mean_ms=med(mean),
                overhead_per_head=med(per_head) / med(plain) - 1, overhead_head_mean=med(mean) / med(plain) - 1,
                read_per_head_ms=med(read_head), read_head_mean_ms=med(read_mean))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    name, power, clock = card()
    for row in rows():
        res = step_bench(*row, args.steps, args.warmup, args.rounds, clock)
        print(json.dumps(dict(gpu=name, power_limit=power, max_sm_clock_hz=clock, **res)), flush=True)
        torch.cuda.empty_cache()
    for fwd in (sd3_forward, flux_forward):
        print(json.dumps(dict(gpu=name, power_limit=power, forward=fwd(args.steps, args.warmup, args.rounds))),
              flush=True)
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
