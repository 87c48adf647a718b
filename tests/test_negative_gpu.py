"""trace(pipe, negative=True): the DAAM map of the unconditional half of the guidance batch, next to the unchanged one.

* Turning the mode on changes nothing the positive maps expose: accumulator slabs and every read are bit-identical.
* Through the C ABI, one whole-batch descriptor (n_prompts = 2N from sample 0) gives bit for bit what two half-batch
  descriptors give, on every accumulate class and in the step and range second-slab forms.
* The negative slabs and maps match the oracle fed the unconditional rows the hooks saw, within DESIGN.md section 3's
  tolerances; each prompt's negative map is reduced against its own negative text.
* The mode combines with batches, images per prompt, every launch mode, CUDA graphs, save_heads / load_heads,
  non-square sizes, time_resolved and step_ranges.
"""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, ops, trace
from daam_b200.testing.synthetic import TINY15_SPEC, TINY96_SPEC, TINY_SPEC, make_pipeline
from oracle import daam_oracle as O
from tests.test_accumulate_steps_gpu import PATHS
from tests.util import assert_elementwise, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'
NEGATIVE = 'blurry dark grainy photo'
FILTERS = [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bits(t):
    return t.contiguous().view(torch.int32)


def n_rows(pipe, text):
    return len(pipe.tokenizer.tokenize(text)) + 2


class StepRecorder:
    """Keeps device copies of every (layer, factor, q, k, heads, scale) the hooks handed to the kernel, grouped by UNet
    forward."""

    def __init__(self, tc, unet):
        self.steps = []
        inner = tc._enqueue
        self.handle = unet.register_forward_pre_hook(lambda *_: self.steps.append([]))

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.steps[-1].append((layer_idx, factor, q.detach().clone(), k.detach().clone(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def oracle_store(self, steps, prompt_idx=0, negative=True):
        """The oracle's per-key sums over ``steps`` of prompt ``prompt_idx``'s unconditional (or conditional) rows:
        ``port_layer_step`` keeps the second sample of the pair it is given, so the pair is ``(u, u)`` or ``(u, c)``."""
        store = O.OracleHeatMaps()
        for t in steps:
            for layer_idx, factor, q, k, heads, scale in self.steps[t]:
                n = q.shape[0] // 2
                pair = [prompt_idx, prompt_idx if negative else n + prompt_idx]
                maps = O.port_layer_step(q[pair].float().cpu(), k[pair].float().cpu(), heads, scale)
                for head, m in enumerate(maps):
                    store.update(factor, layer_idx, head, m)
        return store


def _reads(tc, negative=False, prompts=1):
    """Every read of the last generation: the per-key maps, the filtered global maps, the per-head maps."""
    kw = {'negative': True} if negative else {}
    return {
        'keys': {k: v.clone() for k, v in tc.all_heat_maps.items(**kw)},
        'maps': [tc.compute_global_heat_map(**f, **kw).heat_maps.clone() for f in FILTERS],
        'per_prompt': [tc.compute_global_heat_map(prompt_idx=i, **kw).heat_maps.clone() for i in range(1, prompts)],
        'heads': tc.compute_per_head_heat_maps(**kw)[1].clone(),
    }


def _generate(pipe, prompt, steps, seed=11, size=None, negative_prompt=NEGATIVE, **kw):
    h, w = size if size is not None else (None, None)
    prompts = 1 if isinstance(prompt, str) else len(prompt)
    with trace(pipe, **kw) as tc:
        pipe(prompt, num_inference_steps=steps, generator=torch.Generator().manual_seed(seed), height=h, width=w,
             negative_prompt=negative_prompt)
        out = _reads(tc, prompts=prompts)
        out['acc'] = {s.layer_idx: s.acc.clone() for s in tc.all_heat_maps.live_slabs()}
        if kw.get('negative'):
            out['neg'] = _reads(tc, negative=True, prompts=prompts)
            out['slabs'] = {s.layer_idx: s.neg.clone() for s in tc.all_heat_maps.live_slabs()}
    return out


def _assert_same(a, b, what=''):
    assert set(a['keys']) == set(b['keys']) and len(a['keys']) > 0, what
    for k in a['keys']:
        assert torch.equal(bits(a['keys'][k]), bits(b['keys'][k])), (what, k)
    for f, x, y in zip(FILTERS, a['maps'], b['maps']):
        assert torch.equal(bits(x), bits(y)), (what, f)
    for x, y in zip(a['per_prompt'], b['per_prompt']):
        assert torch.equal(bits(x), bits(y)), what
    assert torch.equal(bits(a['heads']), bits(b['heads'])), what


# -- 1. the positive maps do not change ---------------------------------------------------------------------------------
CASES = [  # id, spec, dtype, (height, width) or None for the model's own size
    ('tiny-fp16', TINY_SPEC, torch.float16, None),
    ('tiny-bf16', TINY_SPEC, torch.bfloat16, None),
    ('tiny-fp32', TINY_SPEC, torch.float32, None),
    ('tiny15-fp16', TINY15_SPEC, torch.float16, None),
    ('tiny96-bf16', TINY96_SPEC, torch.bfloat16, None),
    ('tiny-bf16-512x768', TINY_SPEC, torch.bfloat16, (512, 768)),
    ('tiny-fp16-600x600', TINY_SPEC, torch.float16, (600, 600)),    # 75^2 and 19^2 pixels: the SIMT kernel
]


@pytest.mark.parametrize('case,spec,dtype,size', CASES, ids=[c[0] for c in CASES])
def test_positive_maps_are_unchanged_by_the_mode(case, spec, dtype, size):
    pipe = make_pipeline(spec, dtype=dtype, device=DEV, seed=3)
    plain = _generate(pipe, PROMPT, 3, size=size)
    neg = _generate(pipe, PROMPT, 3, size=size, negative=True)
    _assert_same(plain, neg, case)
    assert set(plain['acc']) == set(neg['acc'])
    for idx in plain['acc']:
        assert torch.equal(bits(plain['acc'][idx]), bits(neg['acc'][idx])), idx
    # the negative half is a real, different map: every key sums to steps * pixels, and it is not the positive one
    assert set(neg['neg']['keys']) == set(neg['keys'])
    for k, v in neg['neg']['keys'].items():
        s = float(v.double().sum())
        assert abs(s - 3 * v.shape[-1] * v.shape[-2]) < 1e-3 * s, k
        assert not torch.equal(v, neg['keys'][k]), k


def test_positive_maps_are_unchanged_with_batched_prompts():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=2)
    prompts = ['a red ball', 'two dogs on the beach', 'a cat']
    plain = _generate(pipe, prompts, 2, batch_prompts=True, negative_prompt=None)
    neg = _generate(pipe, prompts, 2, batch_prompts=True, negative=True, negative_prompt=None)
    _assert_same(plain, neg)
    for idx in plain['acc']:
        assert torch.equal(bits(plain['acc'][idx]), bits(neg['acc'][idx])), idx


# -- 2. the C ABI contract: one whole-batch descriptor == two half-batch descriptors --------------------------------------
ABI_SHAPES = [  # hw, heads, head_dim: single-chunk 16-bit, K-chunked SD-1.x head dims, partial tiles, an odd pixel count
    (1024, 10, 64), (576, 4, 64), (256, 8, 160), (4096, 2, 40), (475, 4, 64),
]
ABI_CASES = [(p, f, s) for p, f in PATHS for s in ABI_SHAPES if s[0] % 4 == 0 or not f & _native.ACC_FORCE_MMA]


def _batch_qk(n, hw, heads, d, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(2 * n, hw, heads * d, generator=g) * 1.5).to(dtype).to(DEV)
    k = torch.randn(2 * n, 77, heads * d, generator=g).to(dtype).to(DEV)
    return q, k


@pytest.mark.parametrize('n', [1, 2])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('path,flags,shape', ABI_CASES, ids=[f'{p}-hw{s[0]}-h{s[1]}-d{s[2]}' for p, _, s in ABI_CASES])
def test_whole_batch_descriptor_equals_two_half_batch_descriptors(path, flags, shape, dtype, n):
    """The unconditional half through a whole-batch descriptor of its own samples, the conditional half through the
    plain (cond-half) descriptor, both in one launch, against one whole-batch descriptor over all 2n samples: the
    accumulators, the step slabs and the range slabs must be bit-identical."""
    hw, heads, d = shape
    q, k = _batch_qk(n, hw, heads, d, dtype, hw * 31 + heads * 7 + d + n)
    scale = d ** -0.5
    shape4 = (2 * n, heads, 77, hw)
    g = torch.Generator(DEV).manual_seed(5)
    acc0, seed = torch.rand(shape4, generator=g, device=DEV), torch.randn(shape4, generator=g, device=DEV) * 3

    def whole(acc):
        return [ops.make_layer_desc(q, k, acc, heads, scale, whole_batch=True)]

    def halves(acc):
        return [ops.make_layer_desc(q[:n], k[:n], acc[:n], heads, scale, whole_batch=True),
                ops.make_layer_desc(q, k, acc[n:], heads, scale)]

    what = f'{path} hw{hw} H{heads} d{d} {dtype} n{n}'
    a_w, a_h = acc0.clone(), acc0.clone()
    ops.accumulate(whole(a_w), DEV, flags=flags)
    ops.accumulate(halves(a_h), DEV, flags=flags)
    # step form: the step slabs start as NaN (every element must be written)
    s_w, s_h = acc0.clone(), acc0.clone()
    st_w, st_h = torch.full(shape4, float('nan'), device=DEV), torch.full(shape4, float('nan'), device=DEV)
    ops.accumulate_steps(whole(s_w), [st_w], DEV, flags=flags)
    ops.accumulate_steps(halves(s_h), [st_h[:n], st_h[n:]], DEV, flags=flags)
    # range form: the range slabs start from an arbitrary seed
    r_w, r_h = acc0.clone(), acc0.clone()
    rg_w, rg_h = seed.clone(), seed.clone()
    ops.accumulate_range(whole(r_w), [rg_w], DEV, flags=flags)
    ops.accumulate_range(halves(r_h), [rg_h[:n], rg_h[n:]], DEV, flags=flags)
    torch.cuda.synchronize()
    assert torch.equal(bits(a_w), bits(a_h)), f'{what}: accumulator'
    assert torch.equal(bits(s_w), bits(a_w)) and torch.equal(bits(r_w), bits(a_w)), f'{what}: second-slab forms'
    assert torch.equal(bits(s_h), bits(a_h)) and torch.equal(bits(r_h), bits(a_h)), f'{what}: second-slab forms'
    assert not torch.isnan(st_w).any(), f'{what}: step slab elements left unwritten'
    assert torch.equal(bits(st_w), bits(st_h)), f'{what}: step slab'
    assert torch.equal(bits(rg_w), bits(rg_h)), f'{what}: range slab'
    assert not torch.equal(a_w[:n], acc0[:n]) and not torch.equal(a_w[n:], acc0[n:])    # both halves were added to


def test_whole_batch_probabilities_equal_the_two_halves():
    """daam_accumulate_probs from row 0 over a [2N] slab == the conditional rows into the upper half plus the
    unconditional rows into the lower one."""
    for dtype, hw in ((torch.float16, 1024), (torch.float32, 361)):
        q, k = _batch_qk(2, hw, 3, 64, dtype, hw)
        probs = ops.attention_probs(q, k, 3)
        whole = torch.rand(4, 3, 77, hw, generator=torch.Generator(DEV).manual_seed(1), device=DEV)
        split = whole.clone()
        ops.accumulate_probs(probs, whole, whole_batch=True)
        ops.accumulate_probs(probs, split[2:])                        # rows [6, 12): the conditional half
        ops.accumulate_probs(probs[:6].repeat(2, 1, 1), split[:2])     # rows [0, 6), as the upper half of a copy
        torch.cuda.synchronize()
        assert torch.equal(bits(whole), bits(split)), dtype


# -- 3. against the oracle -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('steps', [1, 3])
def test_negative_maps_match_the_oracle(dtype, steps):
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=3)
    s = 1.0 if dtype == torch.float32 else 10.0
    n_tok = len(pipe.tokenizer.tokenize(NEGATIVE))
    with trace(pipe, negative=True) as tc:
        rec = StepRecorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(11), negative_prompt=NEGATIVE)
        assert len(rec.steps) == steps and all(len(st) == 15 for st in rec.steps)
        store = rec.oracle_store(range(steps))
        got = dict(tc.all_heat_maps.items(negative=True))
        assert set(got) == {key for key, _ in store} and len(got) == 25
        for key, ref in store:
            assert_elementwise(got[key], ref, 1e-5 * s, 1e-6 * steps * s, f'key {key}')
        for f in FILTERS:
            ghm = tc.compute_global_heat_map(negative=True, **f)
            ref = O.port_global_heat_map(store, 4096, n_tok, **f)
            assert ghm.prompt == NEGATIVE and ghm.heat_maps.shape == (n_tok + 2, 64, 64)
            assert_elementwise(ghm.heat_maps, ref, 1e-4 * s, 1e-5 * steps * s, f'global {f}')
        # the positive side against its own oracle, in the same trace
        pos = rec.oracle_store(range(steps), negative=False)
        ref = O.port_global_heat_map(pos, 4096, len(pipe.tokenizer.tokenize(PROMPT)))
        assert_elementwise(tc.compute_global_heat_map().heat_maps, ref, 1e-4 * s, 1e-5 * steps * s, 'positive')


def test_images_per_prompt_negative_keys_enumerate_images_x_heads():
    """num_images_per_prompt = 2: a direct UNet call with a [uncond x 2, cond x 2] batch for one prompt."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=6)
    spec = pipe.unet.spec
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(4, spec.in_channels, 64, 64, generator=g).to(DEV)
    emb = torch.randn(4, 77, spec.cross_attention_dim, generator=g).to(DEV)
    with torch.no_grad(), trace(pipe, negative=True) as tc:
        tc.last_prompts, tc.last_prompt, tc.last_negative_prompts = ['a cat'], 'a cat', ['']
        rec = StepRecorder(tc, pipe.unet)
        pipe.unet(lat, torch.full((1,), 500.0, device=DEV), emb)
        got = dict(tc.all_heat_maps.items(negative=True))
        assert len(got) == 2 * 25
        for layer_idx, factor, q, k, heads, scale in rec.steps[0]:
            for image in range(2):
                maps = O.port_layer_step(q[[image, image]].float().cpu(), k[[image, image]].float().cpu(), heads, scale)
                for head, m in enumerate(maps):
                    assert_elementwise(got[(factor, layer_idx, image * heads + head)], m, 1e-5, 1e-6,
                                       f'{layer_idx}/{image}/{head}')
        assert tc.compute_global_heat_map(negative=True).heat_maps.shape == (2, 64, 64)


# -- 4. batches and texts ------------------------------------------------------------------------------------------------
def test_each_prompt_reads_against_its_own_negative_text():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=2)
    prompts = ['a red ball', 'two dogs on the beach', 'a cat']
    negatives = ['blurry', 'dark grainy photo of a cat', '']
    with trace(pipe, negative=True, batch_prompts=True) as tc:
        rec = StepRecorder(tc, pipe.unet)
        pipe(prompts, num_inference_steps=2, generator=torch.Generator().manual_seed(4), negative_prompt=negatives)
        assert tc.last_negative_prompts == negatives
        for p, text in enumerate(negatives):
            ghm = tc.compute_global_heat_map(prompt_idx=p, negative=True)
            assert ghm.prompt == text and ghm.heat_maps.shape[0] == n_rows(pipe, text)
            ref = O.port_global_heat_map(rec.oracle_store(range(2), prompt_idx=p), 4096, n_rows(pipe, text) - 2)
            assert_elementwise(ghm.heat_maps, ref, 1e-4, 2e-5, f'prompt {p}')
            keys, maps = tc.compute_per_head_heat_maps(prompt_idx=p, negative=True)
            assert maps.shape[:2] == (len(keys), n_rows(pipe, text))
        # a str applies to every prompt
        pipe(prompts, num_inference_steps=1, negative_prompt='blurry')
        assert tc.last_negative_prompts == ['blurry'] * 3
        assert [tc.compute_global_heat_map(prompt_idx=p, negative=True).heat_maps.shape[0] for p in range(3)] == [3] * 3


def test_default_negative_prompt_is_the_empty_text_and_word_lookup():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=8)
    image = SimpleNamespace(size=(96, 80))
    with trace(pipe, negative=True) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(1))
        assert tc.last_negative_prompts == ['']
        ghm = tc.compute_global_heat_map(negative=True)
        assert ghm.prompt == '' and ghm.heat_maps.shape == (2, 64, 64)
        with pytest.raises(ValueError, match='not found'):
            ghm.compute_word_heat_map('dog')
        # prompt= still overrides the text (callers that passed negative_prompt_embeds)
        over = tc.compute_global_heat_map(prompt='ugly hands', negative=True)
        assert over.prompt == 'ugly hands' and over.heat_maps.shape == (4, 64, 64)
        assert torch.equal(bits(over.heat_maps[:2]), bits(ghm.heat_maps))
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(1), negative_prompt=NEGATIVE)
        ghm = tc.compute_global_heat_map(negative=True)
        assert ghm.prompt == NEGATIVE and ghm.heat_maps.shape[0] == n_rows(pipe, NEGATIVE)
        word = ghm.compute_word_heat_map('dark')
        assert torch.equal(bits(word.heatmap), bits(ghm.heat_maps[2].contiguous()))
        with pytest.raises(ValueError, match='not found'):
            ghm.compute_word_heat_map('dog')
        whms, expanded = ghm.expand_words(['grainy', 'blurry'], image)
        assert expanded.shape == (2, 96, 80)
        for i, w in enumerate(['grainy', 'blurry']):
            assert torch.allclose(whms[i].heatmap, ghm.compute_word_heat_map(w).heatmap, rtol=1e-6, atol=0)
            assert torch.allclose(expanded[i], ghm.compute_word_heat_map(w).expand_as(image), atol=1e-6)
        with pytest.raises(ValueError, match='not found'):
            ghm.expand_words(['ball'], image)


def test_to_experiment_records_the_negative_text(tmp_path):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=8)
    with trace(pipe, negative=True) as tc:
        pipe(PROMPT, num_inference_steps=1, negative_prompt=NEGATIVE)
        exp = tc.to_experiment(str(tmp_path), negative=True)
        assert exp.prompt == NEGATIVE
        assert torch.equal(exp.global_heat_map, tc.compute_global_heat_map(negative=True).heat_maps)
        plain = tc.to_experiment(str(tmp_path))
        assert plain.prompt == PROMPT
        assert torch.equal(plain.global_heat_map, tc.compute_global_heat_map().heat_maps)


# -- 5. combined modes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('normalize', [False, True])
def test_time_resolved_one_step_equals_the_negative_global_map(normalize):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.bfloat16, device=DEV, seed=4)
    with trace(pipe, time_resolved=True, negative=True) as tc:
        pipe(PROMPT, num_inference_steps=1, generator=torch.Generator().manual_seed(2), negative_prompt=NEGATIVE)
        tm = tc.compute_time_heat_maps(normalize=normalize, negative=True)
        full = tc.compute_global_heat_map(normalize=normalize, negative=True).heat_maps
        assert len(tm) == 1 and tm.prompt == NEGATIVE and tm.heat_maps.shape == (1,) + tuple(full.shape)
        assert torch.equal(bits(tm.heat_maps[0]), bits(full))
        pos = tc.compute_time_heat_maps(normalize=normalize)
        assert torch.equal(bits(pos.heat_maps[0]), bits(tc.compute_global_heat_map(normalize=normalize).heat_maps))


def test_time_resolved_positive_maps_unchanged_and_batched_negative_histories():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=2)
    prompts = ['a red ball', 'two dogs on the beach']
    negatives = ['blurry', 'dark grainy photo']
    out = []
    for negative in (False, True):
        with trace(pipe, time_resolved=True, batch_prompts=True, negative=negative) as tc:
            pipe(prompts, num_inference_steps=3, generator=torch.Generator().manual_seed(1), negative_prompt=negatives)
            out.append([tc.compute_time_heat_maps(prompt_idx=p).heat_maps.clone() for p in range(2)])
            if negative:
                for p, text in enumerate(negatives):
                    tm = tc.compute_time_heat_maps(prompt_idx=p, negative=True)
                    assert len(tm) == 3 and tm.heat_maps.shape[1] == n_rows(pipe, text) and tm.prompt == text
    for a, b in zip(*out):
        assert torch.equal(bits(a), bits(b))


def test_a_negative_range_equals_a_trace_of_only_its_steps():
    """The range's maps against a second negative trace fed the identical recorded Q/K of those steps only."""
    pipe = make_pipeline(TINY15_SPEC, dtype=torch.float16, device=DEV, seed=7)
    with trace(pipe, step_ranges=[(1, 3)], negative=True) as tc:
        rec = StepRecorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3), negative_prompt=NEGATIVE)
        rec.handle.remove()
        got = {neg: _range_reads(tc, neg, step_range=0) for neg in (False, True)}
    with trace(pipe, negative=True) as only:
        only.last_prompts, only.last_prompt, only.last_negative_prompts = [PROMPT], PROMPT, [NEGATIVE]
        for t in (1, 2):
            for call in rec.steps[t]:
                only._enqueue(*call)
            only.flush()
        want = {neg: _range_reads(only, neg) for neg in (False, True)}
    for neg in (False, True):
        a, b = got[neg], want[neg]
        assert set(a['keys']) == set(b['keys']) and len(a['keys']) > 0
        for k in a['keys']:
            assert torch.equal(bits(a['keys'][k]), bits(b['keys'][k])), (neg, k)
        for f, x, y in zip(FILTERS, a['maps'], b['maps']):
            assert torch.equal(bits(x), bits(y)), (neg, f)
        assert torch.equal(bits(a['heads']), bits(b['heads'])), neg


def _range_reads(tc, negative, **kw):
    kw = dict(kw, negative=negative)
    return {'keys': {k: v.clone() for k, v in tc.all_heat_maps.items(**kw)},
            'maps': [tc.compute_global_heat_map(**f, **kw).heat_maps.clone() for f in FILTERS],
            'heads': tc.compute_per_head_heat_maps(**kw)[1].clone()}


@pytest.mark.parametrize('launch', ['overlap', 'layer'])
def test_launch_modes_are_bit_equal_to_the_step_launch(launch):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    eager = _generate(pipe, PROMPT, 3, negative=True)
    other = _generate(pipe, PROMPT, 3, negative=True, launch=launch)
    _assert_same(eager, other, 'positive')
    _assert_same(eager['neg'], other['neg'], 'negative')
    for idx in eager['slabs']:
        assert torch.equal(bits(eager['slabs'][idx]), bits(other['slabs'][idx])), idx


@pytest.mark.parametrize('launch', ['step', 'overlap', 'layer'])
def test_cuda_graph_replay_traces_the_negative_half(launch):
    """The whole-batch descriptors become nodes of the captured UNet step. Eager vs graph differ only as far as cuBLAS
    picks other algorithms under capture (as for the positive maps). The second and third generations replay the same
    graph from step 0 on the same inputs (the first ran step 0 eagerly): they are bit-equal."""
    eager_pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    graph_pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4, cuda_graph=True)
    ref = _generate(eager_pipe, PROMPT, 5, seed=9, negative=True, launch=launch)
    with trace(graph_pipe, launch=launch, negative=True) as tc:
        runs = []
        for _ in range(3):
            graph_pipe(PROMPT, num_inference_steps=5, generator=torch.Generator().manual_seed(9),
                       negative_prompt=NEGATIVE)
            runs.append({'pos': _reads(tc), 'neg': _reads(tc, negative=True)})
            for k, v in tc.all_heat_maps.items(negative=True):
                s = float(v.double().sum())
                assert abs(s - 5 * v.shape[-1] * v.shape[-2]) < 1e-3 * s, k     # exactly 5 steps were accumulated
        assert any(st['graph'] is not None for st in graph_pipe._graphs.values())
    _assert_same(runs[1]['pos'], runs[2]['pos'], 'positive replay')
    _assert_same(runs[1]['neg'], runs[2]['neg'], 'negative replay')
    assert rel_err(runs[0]['neg']['maps'][0], ref['neg']['maps'][0]) < 2e-3
    assert rel_err(runs[0]['pos']['maps'][0], ref['maps'][0]) < 2e-3


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 2e-5), (torch.float16, 2e-3)])
def test_save_heads_and_load_heads(tmp_path, dtype, tol):
    steps = 2
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=5)
    with trace(pipe, save_heads=True, data_dir=str(tmp_path / 'plain')) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2), negative_prompt=NEGATIVE)
        plain = _reads(tc)
    with trace(pipe, save_heads=True, negative=True, data_dir=str(tmp_path / 'neg')) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2), negative_prompt=NEGATIVE)
        saved = {'pos': _reads(tc), 'neg': _reads(tc, negative=True)}
    _assert_same(plain, saved['pos'], 'positive save_heads')
    other = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=6)       # other weights: the maps come from the files
    with trace(other, load_heads=True, negative=True, data_dir=str(tmp_path / 'neg')) as tc:
        other(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2), negative_prompt=NEGATIVE)
        loaded = {'pos': _reads(tc), 'neg': _reads(tc, negative=True)}
    _assert_same(saved['pos'], loaded['pos'], 'positive load_heads')
    _assert_same(saved['neg'], loaded['neg'], 'negative load_heads')
    fused = _generate(pipe, PROMPT, steps, seed=2, negative=True)
    for f, a, b in zip(FILTERS, saved['neg']['maps'], fused['neg']['maps']):
        assert rel_err(a, b) < tol, f
    assert set(saved['neg']['keys']) == set(fused['neg']['keys'])


# -- 6. errors -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('launch', ['step', 'layer'])
def test_a_batch_without_guidance_is_refused(launch):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    spec = pipe.unet.spec
    lat = torch.randn(1, spec.in_channels, 64, 64, device=DEV).half()
    emb = torch.randn(1, 77, spec.cross_attention_dim, device=DEV).half()
    with torch.no_grad(), trace(pipe, negative=True, launch=launch) as tc:
        tc.last_prompts, tc.last_prompt = ['a cat'], 'a cat'
        with pytest.raises(RuntimeError, match='negative=True needs classifier-free guidance'):
            pipe.unet(lat, torch.full((1,), 500.0, device=DEV), emb)
    with torch.no_grad(), trace(pipe, launch=launch) as tc:                 # the plain mode keeps the B = 1 quirk
        tc.last_prompts, tc.last_prompt = ['a cat'], 'a cat'
        pipe.unet(lat, torch.full((1,), 500.0, device=DEV), emb)
        assert len(tc.all_heat_maps) > 0
    torch.cuda.synchronize()


def test_reads_need_the_mode_and_lists_must_match():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    with trace(pipe) as tc:
        pipe('a cat', num_inference_steps=1, negative_prompt='blurry')
        for read in (lambda: tc.compute_global_heat_map(negative=True),
                     lambda: tc.compute_per_head_heat_maps(negative=True),
                     lambda: dict(tc.all_heat_maps.items(negative=True))):
            with pytest.raises(RuntimeError, match=r'trace\(pipe, negative=True\)'):
                read()
    with trace(pipe, negative=True, batch_prompts=True) as tc:
        with pytest.raises(ValueError, match='1 entries for 2 prompts'):
            pipe(['a cat', 'a dog'], num_inference_steps=1, negative_prompt=['blurry'])
