"""FLUX.1 heat maps on one GPU: the per-step daam_accumulate_joint launch over all 57 layers at FLUX.1-dev and
FLUX.1-schnell sizes against the HBM floor of its algorithmic bytes and against the per-layer torch composition, the
hooked against the un-hooked forward of the synthetic FLUX.1-dev transformer, and a compute_global_heat_map() read.

    python bench_flux.py [--steps 20] [--warmup 3]

Prints one JSON line; the card's name and power limit are read in the same run."""
import argparse
import json
import math

import torch

from bench_joint import HBM, card, timed
from daam_b200 import ops, trace
from daam_b200.testing.synthetic import FLUX_DEV_SPEC, FLUX_SCHNELL_SPEC, flux_image_ids, make_flux_pipeline


def step_bench(spec, steps, warmup):
    """One denoising step of every layer, a batch of one, 1024 px (64 x 64 image tokens), bf16, text-first operands."""
    heads, d, hw, tokens, layers = spec.heads, spec.dim_head, 4096, spec.t5_rows, spec.double + spec.single
    g = torch.Generator(device='cuda').manual_seed(0)
    L = tokens + hw
    qs = [torch.randn(1, heads, L, d, generator=g, device='cuda', dtype=torch.bfloat16) for _ in range(layers)]
    ks = [torch.randn(1, heads, L, d, generator=g, device='cuda', dtype=torch.bfloat16) for _ in range(layers)]
    scale = 1.0 / math.sqrt(d)
    lses = [torch.logsumexp((q.float() @ k.float().transpose(-1, -2)) * scale, -1) for q, k in zip(qs, ks)]
    accs = [torch.zeros(1, heads, tokens, hw, device='cuda') for _ in range(layers)]
    descs = [ops.make_joint_desc(q, k, l, hw, a, heads, scale, text_first=True, whole_batch=True)
             for q, k, l, a in zip(qs, ks, lses, accs)]
    ms = timed(lambda: ops.accumulate_joint(descs, 'cuda'), steps, warmup)

    def composed():
        for q, k, l, a in zip(qs, ks, lses, accs):
            s = q[:, :, tokens:] @ k[:, :, :tokens].transpose(-1, -2)         # [1, H, hw, T]
            a += torch.exp(s.float() * scale - l[:, :, tokens:, None]).transpose(-1, -2)
    torch_ms = timed(composed, max(2, steps // 4), 1)
    algo = layers * (heads * hw * d * 2 + heads * tokens * d * 2 + heads * hw * 4 + 2 * heads * tokens * hw * 4)
    return dict(model=spec.name, tokens=tokens, layers=layers, kernel_ms=ms, bytes=algo, floor_ms=algo / HBM * 1e3,
                fraction_of_hbm=algo / HBM / (ms * 1e-3), torch_ms=torch_ms, speedup_vs_torch=torch_ms / ms)


def forward_bench(steps, warmup):
    """Hooked vs un-hooked forward of the FLUX.1-dev-shaped synthetic transformer, bf16, a batch of one at 1024 px
    with 512 T5 rows, and the cost of a compute_global_heat_map() read of the trace."""
    spec = FLUX_DEV_SPEC
    pipe = make_flux_pipeline(spec, dtype=torch.bfloat16, device='cuda', init_on_device=True)
    g = torch.Generator(device='cuda').manual_seed(1)
    kw = dict(hidden_states=torch.randn(1, 4096, 64, generator=g, device='cuda', dtype=torch.bfloat16),
              encoder_hidden_states=torch.randn(1, 512, 4096, generator=g, device='cuda', dtype=torch.bfloat16),
              pooled_projections=torch.randn(1, 768, generator=g, device='cuda', dtype=torch.bfloat16),
              timestep=torch.full((1,), 0.5, device='cuda', dtype=torch.bfloat16),
              img_ids=flux_image_ids(64, 64, 'cuda').bfloat16(),
              txt_ids=torch.zeros(512, 3, device='cuda', dtype=torch.bfloat16),
              guidance=torch.full((1,), 3.5, device='cuda'))
    f = lambda: pipe.transformer(**kw)
    with torch.no_grad():
        plain = timed(f, steps, warmup)
        with trace(pipe) as tc:
            pipe.check_inputs('a photo of a red fox in the snow', None, 1024, 1024)
            hooked = timed(f, steps, warmup)
            read = timed(lambda: tc.compute_global_heat_map(), steps, warmup)
    return dict(unhooked_ms=plain, hooked_ms=hooked, overhead=hooked / plain - 1, read_ms=read)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    res = dict(gpu=name, power_limit=power, step=[])
    for spec in (FLUX_DEV_SPEC, FLUX_SCHNELL_SPEC):
        res['step'].append(step_bench(spec, args.steps, args.warmup))
        torch.cuda.empty_cache()
    res['forward'] = forward_bench(args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
