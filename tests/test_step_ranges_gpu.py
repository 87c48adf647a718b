"""trace(pipe, step_ranges=[...]): the exact DAAM map over chosen spans of denoising steps, next to the unchanged time sum.

* Turning the mode on changes nothing the time sum exposes: per-key slabs and global maps are bit-identical.
* A range's slabs are the accumulators a trace of only its steps would hold: bit-equal to a replay of the recorded Q/K
  of those steps through daam_accumulate, so a range over every step gives the full maps, a one-step range gives the
  time-resolved map of that step, and a range map matches the oracle of those steps within the global-map tolerances
  of DESIGN.md section 3 (steps = b - a).
"""
import pytest
import torch

from daam_b200 import _native, ops, trace
from daam_b200.testing.synthetic import TINY15_SPEC, TINY96_SPEC, TINY_SPEC, make_pipeline
from oracle import daam_oracle as O
from tests.util import assert_elementwise

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'
FILTERS = [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bits(t):
    return t.contiguous().view(torch.int32)


class ForwardRecorder:
    """Keeps device copies of every (layer, factor, q, k, heads, scale) the hooks handed to the kernel, grouped by UNet
    forward."""

    def __init__(self, tc, unet):
        self.steps = []
        inner = tc._enqueue
        unet.register_forward_pre_hook(lambda *_: self.steps.append([]))

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.steps[-1].append((layer_idx, factor, q.detach().clone(), k.detach().clone(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def oracle_store(self, steps):
        store = O.OracleHeatMaps()
        for t in steps:
            for layer_idx, factor, q, k, heads, scale in self.steps[t]:
                maps = O.port_layer_step(q.float().cpu(), k.float().cpu(), heads, scale)
                for head, m in enumerate(maps):
                    store.update(factor, layer_idx, head, m)
        return store


def _generate(pipe, prompt, steps, seed=11, **kw):
    with trace(pipe, **kw) as tc:
        pipe(prompt, num_inference_steps=steps, generator=torch.Generator().manual_seed(seed))
        keys = {k: v.clone() for k, v in tc.all_heat_maps}
        maps = [tc.compute_global_heat_map(**f).heat_maps.clone() for f in FILTERS]
        per_prompt = [tc.compute_global_heat_map(prompt_idx=i).heat_maps.clone()
                      for i in range(1, len(tc.last_prompts))]
    return keys, maps, per_prompt


@pytest.mark.parametrize('spec', [TINY_SPEC, TINY96_SPEC, TINY15_SPEC], ids=lambda s: s.name)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_time_sum_is_unchanged_by_the_mode(spec, dtype):
    pipe = make_pipeline(spec, dtype=dtype, device=DEV, seed=3)
    keys0, maps0, _ = _generate(pipe, PROMPT, 3)
    keys1, maps1, _ = _generate(pipe, PROMPT, 3, step_ranges=[(0, 1), (2, 3)])
    assert set(keys0) == set(keys1) and len(keys0) > 0
    for k in keys0:
        assert torch.equal(bits(keys0[k]), bits(keys1[k])), k
    for f, a, b in zip(FILTERS, maps0, maps1):
        assert torch.equal(bits(a), bits(b)), f


def test_time_sum_is_unchanged_with_batched_prompts():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=2)
    prompts = ['a red ball', 'two dogs on the beach', 'a cat']
    keys0, maps0, per0 = _generate(pipe, prompts, 2, batch_prompts=True)
    keys1, maps1, per1 = _generate(pipe, prompts, 2, batch_prompts=True, step_ranges=[(1, 2)])
    for k in keys0:
        assert torch.equal(bits(keys0[k]), bits(keys1[k])), k
    for a, b in zip(maps0 + per0, maps1 + per1):
        assert torch.equal(bits(a), bits(b))


@pytest.mark.parametrize('spec,dtype', [(TINY_SPEC, torch.float16), (TINY15_SPEC, torch.float32),
                                        (TINY96_SPEC, torch.bfloat16)], ids=['tiny-fp16', 'tiny15-fp32', 'tiny96-bf16'])
def test_a_range_over_every_step_gives_the_full_maps(spec, dtype):
    pipe = make_pipeline(spec, dtype=dtype, device=DEV, seed=5)
    with trace(pipe, step_ranges=[range(0, 3)]) as tc:
        pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(4))
        assert tc.step_range_counts == [3]
        for f in FILTERS:
            full = tc.compute_global_heat_map(**f).heat_maps
            assert torch.equal(bits(tc.compute_global_heat_map(**f, step_range=0).heat_maps), bits(full)), f
        keys, maps = tc.compute_per_head_heat_maps()
        rkeys, rmaps = tc.compute_per_head_heat_maps(step_range=0)
        assert keys == rkeys and torch.equal(bits(maps), bits(rmaps))
        full_raw = dict(tc.all_heat_maps.items())
        range_raw = dict(tc.all_heat_maps.items(step_range=0))
        assert set(full_raw) == set(range_raw)
        for k in full_raw:
            assert torch.equal(bits(full_raw[k]), bits(range_raw[k])), k


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_a_range_equals_a_replay_of_its_steps(dtype):
    pipe = make_pipeline(TINY15_SPEC, dtype=dtype, device=DEV, seed=7)
    ranges = [(1, 3), (4, 6)]
    with trace(pipe, step_ranges=ranges) as tc:
        rec = ForwardRecorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=6, generator=torch.Generator().manual_seed(3))
        assert tc.step_range_counts == [2, 2] and len(rec.steps) == 6
        slabs = {s.layer_idx: s for s in tc.all_heat_maps.live_slabs()}
        for i, (a, b) in enumerate(ranges):
            replay = {idx: torch.zeros_like(s.acc) for idx, s in slabs.items()}
            for t in range(a, b):
                descs = [ops.make_layer_desc(q, k, replay[idx], heads, scale)
                         for idx, _, q, k, heads, scale in rec.steps[t]]
                ops.accumulate(descs, DEV, flags=tc.kernel_flags | _native.ACC_EARLY_LOADS)
            torch.cuda.synchronize()
            for idx, s in slabs.items():
                assert torch.equal(bits(s.ranges[i]), bits(replay[idx])), (i, idx)
            for (key, got), (_, want) in zip(tc.all_heat_maps.items(step_range=i), tc.all_heat_maps.items()):
                assert got.shape == want.shape, key


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_a_one_step_range_equals_the_time_resolved_step(dtype):
    steps, t = 4, 2
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=9)
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(8))
        step_map = tc.compute_time_heat_maps().heat_maps[t].clone()
    with trace(pipe, step_ranges=[(t, t + 1)]) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(8))
        range_map = tc.compute_global_heat_map(step_range=0).heat_maps
    assert torch.equal(bits(range_map), bits(step_map))


def _peaky(pipe, factor):
    with torch.no_grad():
        for name, m in pipe.unet.named_modules():
            if name.endswith('attn2'):
                m.to_q.weight.mul_(factor)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('peaky', [False, True])
def test_range_maps_match_the_oracle_of_their_steps(dtype, peaky):
    steps, ranges = 5, [(0, 2), (2, 5)]
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=3)
    if peaky:                          # sharp attention: the bicubic upsample overshoots below zero and the clamp fires
        _peaky(pipe, 8.0)
    n_tok = len(pipe.tokenizer.tokenize(PROMPT))
    scale = 1.0 if dtype == torch.float32 else 10.0
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(11))
        per_step = tc.compute_time_heat_maps().heat_maps.clone()
    with trace(pipe, step_ranges=ranges) as tc:
        rec = ForwardRecorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(11))
        assert len(rec.steps) == steps and tc.step_range_counts == [2, 3]
        gaps = []
        for i, (a, b) in enumerate(ranges):
            got = tc.compute_global_heat_map(step_range=i).heat_maps
            ref = O.port_global_heat_map(rec.oracle_store(range(a, b)), 4096, n_tok)
            assert_elementwise(got, ref, 1e-4 * scale, 1e-5 * (b - a) * scale, f'range {i} [{a}, {b})')
            gaps.append(per_step[a:b].sum(0) - got)
        # per step the clamp only ever raises a map, so the steps sum to at least the range map; where the clamp fires
        # they sum to more: the range map is not a combination of per-step maps
        top = max(float(g.max()) for g in gaps)
        ref_max = float(per_step.abs().max())
        assert all(float(g.min()) > -1e-4 * steps * ref_max for g in gaps)
        if peaky:
            assert top > 1e-3 * ref_max


def test_a_new_generation_restarts_the_count_and_zeroes_the_ranges():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    with trace(pipe, step_ranges=[(0, 2), (3, 10)]) as tc:
        pipe('a cat', num_inference_steps=5, generator=torch.Generator().manual_seed(1))
        assert tc.step_range_counts == [2, 2]           # the second range runs past the generation's end
        first = [tc.compute_global_heat_map(step_range=i).heat_maps.clone() for i in range(2)]
        pipe('a cat', num_inference_steps=5, generator=torch.Generator().manual_seed(1))
        assert tc.step_range_counts == [2, 2]
        for i in range(2):
            assert torch.equal(bits(tc.compute_global_heat_map(step_range=i).heat_maps), bits(first[i])), i
        pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(1))
        assert tc.step_range_counts == [2, 0]
        assert torch.equal(bits(tc.compute_global_heat_map(step_range=0).heat_maps), bits(
            tc.compute_global_heat_map().heat_maps))
        with pytest.raises(RuntimeError, match='No heat maps found for the given parameters'):
            tc.compute_global_heat_map(step_range=1)
        with pytest.raises(RuntimeError, match='No heat maps found for the given parameters'):
            tc.compute_per_head_heat_maps(step_range=1)
        with pytest.raises(RuntimeError, match='No heat maps found for the given parameters'):
            list(tc.all_heat_maps.items(step_range=1))
        for s in tc.all_heat_maps.live_slabs():
            assert not s.ranges[1].any()


def test_step_range_passes_through_to_experiment(tmp_path):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    with trace(pipe, step_ranges=[(1, 2)]) as tc:
        pipe('a cat', num_inference_steps=3, generator=torch.Generator().manual_seed(1))
        exp = tc.to_experiment(tmp_path, step_range=0)
        assert torch.equal(bits(exp.global_heat_map), bits(tc.compute_global_heat_map(step_range=0).heat_maps))
        assert not torch.equal(exp.global_heat_map, tc.compute_global_heat_map().heat_maps)


def test_cuda_graph_capture_in_the_mode_is_refused():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4, cuda_graph=True)
    with trace(pipe, step_ranges=[(0, 3)]) as tc:
        with pytest.raises(RuntimeError, match='CUDA graph'):
            pipe('a cat', num_inference_steps=3)             # step 0 runs eagerly, step 1 is captured
        tc.synchronize()
    torch.cuda.synchronize()


def test_step_range_needs_the_mode():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    with trace(pipe) as tc:
        pipe('a cat', num_inference_steps=1)
        with pytest.raises(RuntimeError, match='step_ranges'):
            tc.compute_global_heat_map(step_range=0)
