"""Every kernel at the sizes users run (SD-2.1, SD-2.1-768, SD-1.5, SDXL), element by element against float64.

At these sizes the persistent accumulate kernels reach steady state: a CTA walks about 11 tiles per SD-2.1 launch and
dozens per SDXL launch, so the 3-slot accumulator ring and the 2-stage Q/K ring wrap many times, and the finalize
kernel streams several cp.async chunks per key class. The older full-size tests check properties that a swapped head,
tile or prompt would still satisfy (tests/test_reference64.py shows that); these compare every element.

Shapes come from ``bench.traced_layers``; inputs are seeded on the device. The float64 reference
(tests/reference64.py) is computed one layer at a time, so a workload is never held in float64 as a whole.

Tolerances:

* per-key accumulators: the contract's (SURVEY.md section 8c; ``RTOL`` / ``ATOL`` of test_parity_elementwise_gpu.py),
  ``|got - ref| <= ATOL * steps + RTOL * |ref|``; the reference reads the same 16-bit-rounded Q/K as the kernel;
* finalize: derived in ``reference64.finalize_tolerance`` (mean of n fp32 terms, 16-tap fp32 stencil) and
  ``reference64.normalized_tolerance``;
* traced generations: the contract's global-map tolerance, ``1e-5 * steps + 1e-4 * |ref|``, x 10 for 16-bit inputs.
"""
import math
import zlib

import pytest
import torch

import bench
from daam_b200 import _native, ops, trace
from daam_b200.testing.synthetic import SD21_SPEC, SDXL_SPEC, make_pipeline
from oracle import daam_oracle as O
from tests.reference64 import (ACC_DIMS, MAP_DIMS, assert_close64, finalize_tolerance, global_map64, layer_maps64,
                               normalized_tolerance, per_key_maps64, upsample64)
from tests.test_accumulate_steps_gpu import GuardedSlab, bits
from tests.test_parity_elementwise_gpu import ATOL, RTOL

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MAX_PEAK_BYTES = 10 * 2 ** 30
TRACER_FLAGS = _native.ACC_AUTO | _native.ACC_EARLY_LOADS        # what trace() issues every step
bf16, fp16, fp32 = torch.bfloat16, torch.float16, torch.float32


@pytest.fixture(autouse=True)
def _peak_memory():
    """Each case holds one workload's accumulators and projections on the device and its reference one layer at a time:
    keep it within 10 GiB of device memory."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    print(f'\npeak device memory {peak / 2 ** 30:.2f} GiB')
    assert peak < MAX_PEAK_BYTES


def _latent_x(workload):
    return 96 if workload == 'sd21_768' else 64


def _projections(layers, prompts, dtype, steps, g):
    """Per step, per layer: q [2P, hw, heads*d], k [2P, 77, heads*d] (a CFG batch, as to_q / to_k emit them)."""
    return [[(torch.randn(2 * prompts, hw, h * d, generator=g, device=DEV).to(dtype),
              torch.randn(2 * prompts, 77, h * d, generator=g, device=DEV).to(dtype)) for hw, h, d in layers]
            for _ in range(steps)]


def _descs(layers, qk, accs):
    return [ops.make_layer_desc(q, k, a, h, d ** -0.5) for (q, k), a, (hw, h, d) in zip(qk, accs, layers)]


# --------------------------------------------------------------------------------------------------------------------
# 1. accumulate: 3 steps of distinct Q/K onto seeded accumulators, every element against float64
# --------------------------------------------------------------------------------------------------------------------
ACC_CASES = [  # id, workload, dtype, prompts, flags
    ('sd21-bf16', 'sd21', bf16, 1, TRACER_FLAGS),
    ('sd21-fp32', 'sd21', fp32, 1, TRACER_FLAGS),
    ('sd21-8prompts-bf16', 'sd21', bf16, 8, TRACER_FLAGS),
    ('sd21_768-fp16', 'sd21_768', fp16, 1, TRACER_FLAGS),
    ('sd15-fp16', 'sd15', fp16, 1, TRACER_FLAGS),
    ('sd15-fp32', 'sd15', fp32, 1, TRACER_FLAGS),
    ('sdxl70-2prompts-fp16', 'sdxl70', fp16, 2, TRACER_FLAGS),
    ('sd21-simt-fp32', 'sd21', fp32, 1, _native.ACC_FORCE_SIMT | _native.ACC_EARLY_LOADS),
    ('sd21-simt-bf16', 'sd21', bf16, 1, _native.ACC_FORCE_SIMT | _native.ACC_EARLY_LOADS),
    ('sd21-split-ldst-fp32', 'sd21', fp32, 1, _native.ACC_FORCE_MMA | _native.ACC_RMW_LDST | _native.ACC_EARLY_LOADS),
]


@pytest.mark.parametrize('case,workload,dtype,prompts,flags', ACC_CASES, ids=[c[0] for c in ACC_CASES])
def test_accumulate_at_production_sizes(case, workload, dtype, prompts, flags):
    """Non-zero seeded accumulators (a skipped load or a tile stored to the wrong place is not masked by zeros), then
    one call per step, each step with its own Q/K (a stale ring slot adds the wrong step's values)."""
    steps = 3
    layers = bench.traced_layers(workload)
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(case.encode()))
    qk = _projections(layers, prompts, dtype, steps, g)
    init = [torch.rand(prompts, h, 77, hw, generator=g, device=DEV) / 77 for hw, h, d in layers]
    accs = [a.clone() for a in init]
    descs = [ops.pack(_descs(layers, qk[s], accs)) for s in range(steps)]
    torch.cuda.synchronize()                     # every input is complete before the first launch (EARLY_LOADS)
    for s in range(steps):
        ops.accumulate(descs[s], DEV, flags=flags)
    torch.cuda.synchronize()
    for i, (hw, h, d) in enumerate(layers):
        ref = init[i].double()
        for s in range(steps):
            ref += layer_maps64(*qk[s][i], h, d ** -0.5)
        assert_close64(accs[i], ref, RTOL[dtype], ATOL[dtype] * steps, f'{case} layer {i} ({hw}, {h}, {d})', ACC_DIMS)
        del ref


# --------------------------------------------------------------------------------------------------------------------
# 2. step slabs at the same sizes
# --------------------------------------------------------------------------------------------------------------------
STEP_CASES = [
    ('sd21-bf16', 'sd21', bf16, 1),
    ('sd15-fp16', 'sd15', fp16, 1),
    ('sdxl70-2prompts-fp16', 'sdxl70', fp16, 2),
    ('sd21-split-fp32', 'sd21', fp32, 1),
]


@pytest.mark.parametrize('case,workload,dtype,prompts', STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_step_slabs_at_production_sizes(case, workload, dtype, prompts):
    """daam_accumulate_steps over two steps into the same step slabs: after each step every slab holds exactly that
    step (against float64), nothing around a slab changes, and the accumulators stay bit-equal to daam_accumulate's."""
    steps = 2
    layers = bench.traced_layers(workload)
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(case.encode()))
    qk = _projections(layers, prompts, dtype, steps, g)
    plain = [torch.rand(prompts, h, 77, hw, generator=g, device=DEV) for hw, h, d in layers]
    stepped = [a.clone() for a in plain]
    guarded = [GuardedSlab(a.shape) for a in stepped]
    torch.cuda.synchronize()
    for s in range(steps):
        ops.accumulate(_descs(layers, qk[s], plain), DEV, flags=TRACER_FLAGS)
        ops.accumulate_steps(_descs(layers, qk[s], stepped), [gs.slab for gs in guarded], DEV, flags=TRACER_FLAGS)
        torch.cuda.synchronize()
        for i, (hw, h, d) in enumerate(layers):
            what = f'{case} step {s} layer {i} ({hw}, {h}, {d})'
            guarded[i].check(what)
            assert_close64(guarded[i].slab, layer_maps64(*qk[s][i], h, d ** -0.5), RTOL[dtype], ATOL[dtype], what,
                           ACC_DIMS)
    for i, (a, b) in enumerate(zip(plain, stepped)):
        assert torch.equal(bits(a), bits(b)), f'{case} layer {i}: accumulator differs from daam_accumulate'


# --------------------------------------------------------------------------------------------------------------------
# 3. finalize at production key counts
# --------------------------------------------------------------------------------------------------------------------
def _key_stacks(workload, images, seed):
    """One fp32 key stack [images * heads, 77, side, side] of seeded exp(randn) maps per traced layer (a prompt's slice
    of the tracer's slabs), with the layer's spatial factor."""
    x = _latent_x(workload)
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for hw, h, d in bench.traced_layers(workload):
        side = math.isqrt(hw)
        out.append((x // side, torch.exp(torch.randn(images * h, 77, side, side, generator=g, device=DEV))))
    return out, x


def _groups(stacks, head_sel=None):
    return [_native.DaamKeyGroup(acc=t.data_ptr(), heads=t.shape[0], h=t.shape[2], w=t.shape[3], tokens=t.shape[1],
                                 head_sel=-1 if head_sel is None else head_sel, reserved=0) for t in stacks]


def _finalize(monkeypatch, groups, x, n_rows, normalize, generic, per_key=False, n_keys=0):
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1' if generic else '0')
    out = torch.empty(((n_keys,) if per_key else ()) + (n_rows, x, x), device=DEV)
    fn = _native.finalize_per_key if per_key else _native.finalize
    fn(groups, x, n_rows, normalize, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


def _reference_and_bounds(stacks, x, n_rows, normalize, head_sel):
    ref = global_map64(stacks, x, n_rows, False, head_sel)
    n = sum(t.shape[0] if head_sel is None else 1 for t in stacks)
    rtol, atol = finalize_tolerance(stacks, n, x)
    if normalize:
        atol = normalized_tolerance(ref, rtol, atol)
        ref, rtol = ref / (ref[1:-1].sum(dim=0, keepdim=True) + 1e-6), 0.0
    return ref, rtol, atol, n


FIN_CASES = [(w, n) for w in ('sd21', 'sd21_768', 'sd15', 'sdxl', 'sdxl70') for n in (12, 40, 77)]


@pytest.mark.parametrize('workload,n_rows', FIN_CASES)
def test_finalize_at_production_key_counts(monkeypatch, workload, n_rows):
    """The fast kernel (several chunks per factor-2 / factor-4 class, chunk tails, both band heights: 4-row bands at 12
    rows, 8-row bands at 40 and 77 on a 132-SM H100) and the generic kernel against float64; two fast runs bit-equal
    (its sums are deterministic). At 40 rows also normalize, one head, and the factor-2 class alone."""
    keyed, x = _key_stacks(workload, 1, n_rows)
    options = [{}]
    if n_rows == 40:
        options += [{'normalize': True}, {'head_sel': 1}, {'factors': {2}}]
    for opt in options:
        stacks = [t for f, t in keyed if f in opt.get('factors', {1, 2, 4})]
        normalize, head_sel = opt.get('normalize', False), opt.get('head_sel')
        ref, rtol, atol, n = _reference_and_bounds(stacks, x, n_rows, normalize, head_sel)
        assert n <= 2048                                  # all on the fast kernel
        groups = _groups(stacks, head_sel)
        what = f'{workload} n_rows {n_rows} {opt} ({n} keys)'
        fast = _finalize(monkeypatch, groups, x, n_rows, normalize, generic=False)
        again = _finalize(monkeypatch, groups, x, n_rows, normalize, generic=False)
        generic = _finalize(monkeypatch, groups, x, n_rows, normalize, generic=True)
        assert torch.equal(bits(fast), bits(again)), f'{what}: two runs of the fast kernel differ'
        assert_close64(fast, ref, rtol, atol, f'fast {what}', MAP_DIMS)
        assert_close64(generic, ref, rtol, atol, f'generic {what}', MAP_DIMS)


@pytest.mark.parametrize('n_rows', [12, 77])
def test_finalize_sdxl_two_images_per_prompt(monkeypatch, n_rows):
    """SDXL with 2 images per prompt: 2200 keys, more than one class can stage (2048), so the generic kernel runs."""
    keyed, x = _key_stacks('sdxl', 2, 100 + n_rows)
    stacks = [t for _, t in keyed]
    ref, rtol, atol, n = _reference_and_bounds(stacks, x, n_rows, False, None)
    assert n == 2200
    out = _finalize(monkeypatch, _groups(stacks), x, n_rows, False, generic=False)
    assert_close64(out, ref, rtol, atol, f'sdxl 2 images n_rows {n_rows}', MAP_DIMS)


@pytest.mark.parametrize('normalize', [False, True])
def test_finalize_per_key_sd21(monkeypatch, normalize):
    """daam_finalize_per_key over the 175 SD-2.1 keys: every key's own map against float64."""
    keyed, x = _key_stacks('sd21', 1, 7)
    stacks = [t for _, t in keyed]
    n_rows = 77
    out = _finalize(monkeypatch, _groups(stacks), x, n_rows, normalize, generic=False, per_key=True, n_keys=175)
    first = 0
    for i, t in enumerate(stacks):
        raw = per_key_maps64(t, x, n_rows, False)
        for h in range(t.shape[0]):
            rtol, atol = finalize_tolerance([t[h:h + 1]], 1, x)
            ref = raw[h]
            if normalize:
                atol = normalized_tolerance(ref, rtol, atol)
                ref, rtol = ref / (ref[1:-1].sum(dim=0, keepdim=True) + 1e-6), 0.0
            assert_close64(out[first + h], ref, rtol, atol, f'layer {i} head {h} normalize={normalize}', MAP_DIMS)
        first += t.shape[0]
    assert first == 175


# --------------------------------------------------------------------------------------------------------------------
# 4. traced generations end to end
# --------------------------------------------------------------------------------------------------------------------
PROMPT = 'a dog chasing a red ball on the beach'


class DeviceStepRecorder:
    """Keeps device copies of every (layer, q, k) the hooks hand to the kernel, grouped by UNet forward."""

    def __init__(self, tc, unet):
        self.steps = []
        inner = tc._enqueue
        unet.register_forward_pre_hook(lambda *_: self.steps.append([]))

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.steps[-1].append((layer_idx, q.detach().clone(), k.detach().clone(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue


def _traced_reference(rec, x, n_rows):
    """Float64 global map of the time sum, and one per step, from the recorded Q/K, one layer at a time."""
    steps = len(rec.steps)
    total = torch.zeros(n_rows, x, x, dtype=torch.float64, device=DEV)
    per_step = torch.zeros(steps, n_rows, x, x, dtype=torch.float64, device=DEV)
    n_keys = 0
    for j in range(len(rec.steps[0])):
        time_sum = None
        for s in range(steps):
            layer_idx, q, k, heads, scale = rec.steps[s][j]
            assert layer_idx == rec.steps[0][j][0]
            m = layer_maps64(q, k, heads, scale)[0]                     # prompt 0: [heads, 77, hw]
            side = math.isqrt(m.shape[-1])
            m = m.reshape(m.shape[0], 77, side, side)
            per_step[s] += upsample64(m[:, :n_rows], x).clamp_(min=0.0).sum(dim=0)
            time_sum = m if time_sum is None else time_sum + m
        total += upsample64(time_sum[:, :n_rows], x).clamp_(min=0.0).sum(dim=0)
        n_keys += time_sum.shape[0]
    return total / n_keys, per_step / n_keys


@pytest.mark.parametrize('spec,dtype', [(SD21_SPEC, bf16), (SDXL_SPEC, fp16)], ids=['sd21-bf16', 'sdxl-fp16'])
def test_traced_generation_against_float64(spec, dtype):
    steps = 3
    pipe = make_pipeline(spec, 'skeleton', dtype=dtype, device=DEV, seed=1, init_on_device=True)
    with trace(pipe, time_resolved=True) as tc:
        rec = DeviceStepRecorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(7))
        full = tc.compute_global_heat_map().heat_maps
        norm = tc.compute_global_heat_map(normalize=True).heat_maps
        tm = tc.compute_time_heat_maps()
        ball = tm.word_heat_maps('ball')
    assert len(rec.steps) == len(tm) == steps
    n_rows, x = full.shape[0], full.shape[-1]
    assert n_rows == len(PROMPT.split()) + 2
    ref, ref_steps = _traced_reference(rec, x, n_rows)
    rtol, atol = 1e-3, 1e-4                              # the contract's global-map tolerance for 16-bit inputs
    what = f'{spec.name} {dtype}'
    assert_close64(full, ref, rtol, atol * steps, f'{what} global map', MAP_DIMS)
    assert_close64(norm, ref / (ref[1:-1].sum(dim=0, keepdim=True) + 1e-6), rtol, atol * steps,
                   f'{what} normalized global map', MAP_DIMS)
    for t in range(steps):
        assert_close64(tm.heat_maps[t], ref_steps[t], rtol, atol, f'{what} step {t}', MAP_DIMS)
    rows, _ = O.port_token_merge_indices(pipe.tokenizer, PROMPT, 'ball')
    assert_close64(ball, ref_steps[:, rows].mean(dim=1), rtol, atol, f'{what} word map "ball"', ('step', 'y', 'x'))
