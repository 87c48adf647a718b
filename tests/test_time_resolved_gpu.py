"""trace(pipe, time_resolved=True): one global heat map per denoising step, next to the unchanged time sum.

* Turning the mode on changes nothing the time sum exposes: per-key slabs and global maps are bit-identical.
* Step t's map is what compute_global_heat_map would give had only step t been traced: bit-identical to it for a
  one-step generation, and within the global-map tolerances of DESIGN.md section 3 (steps = 1) of the oracle fed the
  Q/K the hooks saw in that step.
"""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import TimeHeatMaps, trace
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


class StepRecorder:
    """Keeps CPU copies of every (layer, q, k) the hooks handed to the kernel, grouped by UNet forward."""

    def __init__(self, tc, unet):
        self.steps = []
        inner = tc._enqueue
        unet.register_forward_pre_hook(lambda *_: self.steps.append([]))

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.steps[-1].append((layer_idx, factor, q.detach().float().cpu(), k.detach().float().cpu(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def oracle_store(self, step, prompt_idx=0):
        store = O.OracleHeatMaps()
        for layer_idx, factor, q, k, heads, scale in self.steps[step]:
            n = q.shape[0] // 2
            maps = O.port_layer_step(q[[prompt_idx, n + prompt_idx]], k[[prompt_idx, n + prompt_idx]], heads, scale)
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
        time_maps = [tc.compute_time_heat_maps(prompt_idx=i) for i in range(len(tc.last_prompts))] \
            if kw.get('time_resolved') else None
    return keys, maps, per_prompt, time_maps


@pytest.mark.parametrize('spec', [TINY_SPEC, TINY96_SPEC, TINY15_SPEC], ids=lambda s: s.name)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_time_sum_is_unchanged_by_the_mode(spec, dtype):
    pipe = make_pipeline(spec, dtype=dtype, device=DEV, seed=3)
    keys0, maps0, _, _ = _generate(pipe, PROMPT, 3)
    keys1, maps1, _, tm = _generate(pipe, PROMPT, 3, time_resolved=True)
    assert set(keys0) == set(keys1) and len(keys0) > 0
    for k in keys0:
        assert torch.equal(bits(keys0[k]), bits(keys1[k])), k
    for f, a, b in zip(FILTERS, maps0, maps1):
        assert torch.equal(bits(a), bits(b)), f
    assert len(tm[0]) == 3


def test_time_sum_is_unchanged_with_batched_prompts():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=2)
    prompts = ['a red ball', 'two dogs on the beach', 'a cat']
    keys0, maps0, per0, _ = _generate(pipe, prompts, 2, batch_prompts=True)
    keys1, maps1, per1, tms = _generate(pipe, prompts, 2, batch_prompts=True, time_resolved=True)
    for k in keys0:
        assert torch.equal(bits(keys0[k]), bits(keys1[k])), k
    for a, b in zip(maps0 + per0, maps1 + per1):
        assert torch.equal(bits(a), bits(b))
    assert [len(t) for t in tms] == [2, 2, 2]
    assert [t.heat_maps.shape[1] for t in tms] == [len(pipe.tokenizer.tokenize(p)) + 2 for p in prompts]


def test_images_per_prompt_time_sum_unchanged_and_one_step_equal():
    """num_images_per_prompt = 2: one prompt, images x heads keys per layer (a direct UNet call with a 2 x 2 CFG batch)."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    spec = pipe.unet.spec
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(4, spec.in_channels, 64, 64, generator=g).half().to(DEV)
    emb = torch.randn(4, 77, spec.cross_attention_dim, generator=g).half().to(DEV)
    out = []
    for tr in (False, True):
        with torch.no_grad(), trace(pipe, time_resolved=tr) as tc:
            tc.last_prompts, tc.last_prompt = ['a cat'], 'a cat'
            pipe.unet(lat, torch.full((1,), 500.0, device=DEV), emb)
            keys = {k: v.clone() for k, v in tc.all_heat_maps}
            full = tc.compute_global_heat_map().heat_maps.clone()
            out.append((keys, full, tc.compute_time_heat_maps() if tr else None))
    (k0, m0, _), (k1, m1, tm) = out
    assert len(k0) == 2 * 25 and all(torch.equal(bits(k0[k]), bits(k1[k])) for k in k0)
    assert torch.equal(bits(m0), bits(m1))
    assert len(tm) == 1 and torch.equal(bits(tm.heat_maps[0]), bits(m1))


@pytest.mark.parametrize('spec', [TINY_SPEC, TINY96_SPEC, TINY15_SPEC], ids=lambda s: s.name)
@pytest.mark.parametrize('normalize', [False, True])
def test_one_step_generation_equals_the_global_map(spec, normalize):
    pipe = make_pipeline(spec, dtype=torch.bfloat16, device=DEV, seed=4)
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=1, generator=torch.Generator().manual_seed(2))
        tm = tc.compute_time_heat_maps(normalize=normalize)
        full = tc.compute_global_heat_map(normalize=normalize).heat_maps
        assert isinstance(tm, TimeHeatMaps) and len(tm) == 1
        assert tm.heat_maps.shape == (1,) + tuple(full.shape)
        assert torch.equal(bits(tm.heat_maps[0]), bits(full))


def _peaky(pipe, factor):
    with torch.no_grad():
        for name, m in pipe.unet.named_modules():
            if name.endswith('attn2'):
                m.to_q.weight.mul_(factor)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('peaky', [False, True])
def test_each_step_matches_a_one_step_oracle(dtype, peaky):
    steps = 4
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=3)
    if peaky:                          # sharp attention: the bicubic upsample overshoots below zero and the clamp fires
        _peaky(pipe, 8.0)
    n_tok = len(pipe.tokenizer.tokenize(PROMPT))
    scale = 1.0 if dtype == torch.float32 else 10.0
    with trace(pipe, time_resolved=True) as tc:
        rec = StepRecorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(11))
        tm = tc.compute_time_heat_maps()
        full = tc.compute_global_heat_map().heat_maps
        assert len(tm) == len(rec.steps) == steps and all(len(s) == 15 for s in rec.steps)
        clamped = False
        for t in range(steps):
            store = rec.oracle_store(t)
            ref = O.port_global_heat_map(store, 4096, n_tok)
            assert_elementwise(tm.heat_maps[t], ref, 1e-4 * scale, 1e-5 * scale, f'step {t}')
            unclamped = torch.stack([torch.nn.functional.interpolate(m.unsqueeze(1), size=(64, 64), mode='bicubic')
                                     for _, m in store]).min()
            clamped = clamped or float(unclamped) < 0
        # per step the clamp only ever raises a map, so the steps sum to at least the all-steps map; where the clamp
        # fires they sum to more (it follows the time sum there)
        gap = tm.heat_maps.sum(0) - full
        assert float(gap.min()) > -1e-4 * float(full.abs().max())
        if peaky:
            assert clamped and float(gap.max()) > 1e-4 * float(full.abs().max())


def test_len_counts_unet_forwards_and_a_new_generation_restarts():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    forwards = []
    pipe.unet.register_forward_hook(lambda *_: forwards.append(1))
    with trace(pipe, time_resolved=True) as tc:
        pipe('a cat', num_inference_steps=5, generator=torch.Generator().manual_seed(1))
        first = tc.compute_time_heat_maps()
        kept = first.heat_maps.clone()
        assert len(first) == len(forwards) == 5 and first.heat_maps.shape[1] == 4
        pipe('two small dogs on a red carpet', num_inference_steps=3, generator=torch.Generator().manual_seed(2))
        second = tc.compute_time_heat_maps()
        assert len(second) == 3 and second.heat_maps.shape[1] == len(pipe.tokenizer.tokenize('two small dogs on a red carpet')) + 2
        assert torch.equal(first.heat_maps, kept)            # maps handed out earlier are not overwritten
        # more steps than the history's first capacity: it grows between steps and keeps the early ones
        snaps = []
        pipe('a cat', num_inference_steps=40, generator=torch.Generator().manual_seed(1),
             callback=lambda i, t, lat: snaps.append(tc.compute_time_heat_maps().heat_maps[i].clone()))
        third = tc.compute_time_heat_maps()
        assert len(third) == 40 == len(snaps)
        assert torch.equal(bits(third.heat_maps), bits(torch.stack(snaps)))


def test_word_maps_and_expand_words_per_step():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=8)
    image = SimpleNamespace(size=(96, 80))
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(1))
        tm = tc.compute_time_heat_maps()
        for word in ('ball', 'dog'):
            per_step = tm.word_heat_maps(word)
            assert per_step.shape == (3, 64, 64)
            for t in range(3):
                assert torch.equal(bits(per_step[t]), bits(tm[t].compute_word_heat_map(word).heatmap))
        by_idx = tm.word_heat_maps('ignored', word_idx=2)
        assert torch.equal(bits(by_idx[1]), bits(tm[1].compute_word_heat_map('ignored', word_idx=2).heatmap))
        whms, expanded = tm[2].expand_words(['dog', 'ball'], image)
        assert expanded.shape == (2, 96, 80)
        for i, w in enumerate(['dog', 'ball']):
            assert torch.allclose(whms[i].heatmap, tm[2].compute_word_heat_map(w).heatmap, rtol=1e-6, atol=0)
            assert torch.allclose(expanded[i], tm[2].compute_word_heat_map(w).expand_as(image), atol=1e-6)
        with pytest.raises(ValueError, match='not found'):
            tm.word_heat_maps('zebra')
        assert torch.equal(tm[-1].heat_maps, tm.heat_maps[2])


def test_cuda_graph_capture_of_a_time_resolved_step_is_refused():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4, cuda_graph=True)
    with trace(pipe, time_resolved=True) as tc:
        with pytest.raises(RuntimeError, match='CUDA graph'):
            pipe('a cat', num_inference_steps=3)             # step 0 runs eagerly, step 1 is captured
        tc.synchronize()
    torch.cuda.synchronize()


def test_time_maps_need_the_mode():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    with trace(pipe) as tc:
        pipe('a cat', num_inference_steps=1)
        with pytest.raises(RuntimeError, match='time_resolved=True'):
            tc.compute_time_heat_maps()
    with trace(pipe, time_resolved=True) as tc:
        with pytest.raises(RuntimeError, match='No heat maps found'):
            tc.compute_time_heat_maps()
